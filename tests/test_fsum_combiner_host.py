"""The number-sum combiner on the CPU: the greedy split of an exact sum (acc_split and two_split in
csrc/mrhbm_numsum.cuh), host-compiled from tests/native/fsum_split_check.cu, against exact rational arithmetic
(Fraction); the ledger's replace_open (tests/native/pool_ledger_replace_check.cu); and server.configure's check of the
declaration hbm_combinerfn = "fsum" with a stand-in ctx."""
import math
import os
import random
import shutil
import subprocess
import sys
import types
from fractions import Fraction

import pytest

import mrhbm_loader

mrhbm_loader.load()
from lua_mapreduce_b200.mapreduce import server  # noqa: E402

from test_fsum_host import MAXF, StandIn, bits, cases, from_bits  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WWC_PKG = "lua_mapreduce_b200.mapreduce.examples.WeightedWordCount"
INF_BITS = 0x7FF0000000000000


def rne(x):
    """a nonzero Fraction of magnitude below MAXF rounded to the nearest double, ties to even"""
    return float(x)


def expected(values):
    """MRHBM_COMBINE_FSUM's rule for one key's values: a list of doubles, "keep" or None (the commit fails)"""
    pinf = any(v == math.inf for v in values)
    ninf = any(v == -math.inf for v in values)
    if pinf and ninf:
        return None
    if pinf or ninf:
        return [math.inf if pinf else -math.inf]
    s = sum(Fraction(v) for v in values)
    if s == 0:
        return [-0.0 if all(math.copysign(1, v) < 0 for v in values) else 0.0]
    if abs(s) >= MAXF:
        return "keep"
    terms, r = [], s
    while r != 0:
        c = rne(r)
        terms.append(c)
        r -= Fraction(c)
        if len(terms) > len(values):
            return "keep"
    return terms


def split_cases():
    rng = random.Random(11)
    tiny, big = 5e-324, 1.7976931348623157e308
    out = [vals for vals in cases() if len(vals) <= 250]
    out += [
        [big, big], [big, -big], [big, 2.0 ** 970], [big, 2.0 ** 969], [-big, -2.0 ** 970],  # both sides of 2^1024 - 2^970
        [big, 2.0 ** 970, -2.0 ** 971], [1e308, 1e308, -1e308], [1e308, 1e308],
        [1.0, 2.0 ** -53], [1.0 + 2.0 ** -52, 2.0 ** -53], [1.0, -2.0 ** -54], [1.0, 2.0 ** -53, 2.0 ** -200],  # ties
        [1.0, 2.0 ** -60, 2.0 ** -120], [2.0 ** 1000, 1.0, 2.0 ** -1000, tiny],  # long expansions of few values
        [tiny, -tiny], [-0.0], [-0.0, -0.0], [0.0, -0.0], [-0.0, 0.0, -0.0], [1.0, -1.0], [-1.0, 1.0],
        [math.inf], [-math.inf], [math.inf, math.inf], [math.inf, 1.0], [-math.inf, -big, -big], [math.inf, -math.inf],
        [math.inf, 5.0, -math.inf], [2.2250738585072014e-308, -tiny], [3 * tiny, 2.0 ** -1022],
    ]
    for _ in range(600):  # pairs: finite, near the edges, tied
        kind = rng.randrange(3)
        if kind == 0:
            vals = [from_bits(rng.getrandbits(64)) for _ in range(2)]
            vals = [v if math.isfinite(v) else 1.0 for v in vals]
        elif kind == 1:
            e = rng.randrange(-1074, 971)
            vals = [rng.choice((-1, 1)) * rng.random() * 2.0 ** e, rng.choice((-1, 1)) * rng.random() * 2.0 ** (e - rng.randrange(0, 80))]
        else:
            a = rng.choice((-1, 1)) * (1 + rng.getrandbits(52) * 2.0 ** -52) * 2.0 ** rng.randrange(-1000, 1000)
            vals = [a, math.copysign(math.ulp(a) / 2, rng.choice((-1, 1)))]
        out.append(vals)
    for n in (3, 5, 17):  # cancellation across the exponent range
        for _ in range(60):
            vals = [rng.choice((-1, 1)) * rng.random() * 2.0 ** rng.randrange(-1074, 1020) for _ in range(n)]
            vals += [-v for v in vals[: rng.randrange(n)]]
            rng.shuffle(vals)
            out.append(vals)
    return out


def run_native(tmp_path, src, name, lines=None):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / name)
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "lua-mapreduce_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", src)])
    out = subprocess.run([exe], input="\n".join(lines or []) + "\n", capture_output=True, text=True, timeout=300)
    res = out.stdout.splitlines()
    assert out.returncode == 0 and res and res[-1] == "ok", out.stdout[-2000:] + out.stderr[-2000:]
    return res[:-1]


def test_split_matches_fractions(tmp_path):
    cs = split_cases()
    got = run_native(tmp_path, "fsum_split_check.cu", "fsum_split_check",
                     ["%d %s" % (len(v), " ".join("%x" % bits(x) for x in v)) for v in cs])
    assert len(got) == len(cs)
    seen = {"keep": 0, "nan": 0, "long": 0}
    for vals, g in zip(cs, got):
        want = expected(vals)
        if want is None:
            assert g == "nan", vals
            seen["nan"] += 1
        elif want == "keep":
            assert g == "keep", vals
            seen["keep"] += 1
        else:
            terms = [from_bits(int(t, 16)) for t in g.split()]
            assert [bits(t) for t in terms] == [bits(t) for t in want], (vals, terms, want)
            if all(math.isfinite(v) for v in vals):
                assert sum(Fraction(t) for t in terms) == sum(Fraction(v) for v in vals), vals
            assert len(terms) <= len(vals), vals
            seen["long"] += len(terms) > 2
    assert seen["keep"] >= 5 and seen["nan"] >= 2 and seen["long"] >= 2, seen


def test_two_values_never_need_more_than_two_terms(tmp_path):
    rng = random.Random(3)
    cs = []
    for _ in range(3000):
        vals = [from_bits(rng.getrandbits(64)) for _ in range(2)]
        if all(math.isfinite(v) for v in vals):
            cs.append(vals)
    got = run_native(tmp_path, "fsum_split_check.cu", "fsum_split_check",
                     ["2 %x %x" % (bits(a), bits(b)) for a, b in cs])
    for vals, g in zip(cs, got):
        assert g == "keep" or len(g.split()) <= 2, (vals, g)
        assert (g == "keep") == (expected(vals) == "keep"), vals


def test_ledger_replace_open(tmp_path):
    run_native(tmp_path, "pool_ledger_replace_check.cu", "pool_ledger_replace_check")


def configure(reducefn, combinerfn, value_kind="bytes"):
    S = WWC_PKG + ".init"
    s = server.new("hbm://local", "fsum-combiner-configure")
    s.ctx_factory = StandIn
    s.configure(dict(taskfn=S, mapfn=S, partitionfn=S, reducefn=reducefn, finalfn=S, combinerfn=combinerfn,
                     storage="hbm", hbm={"value_kind": value_kind}))
    return s


def combiner_plugin(monkeypatch, name, fn, decl="fsum"):
    mod = types.ModuleType(name)
    mod.init = lambda arg=None: None
    mod.combinerfn = fn
    mod.hbm_combinerfn = decl
    monkeypatch.setitem(sys.modules, name, mod)
    return name


def test_configure_selects_the_fsum_combiner():
    s = configure(WWC_PKG + ".reducefn_device", WWC_PKG + ".combinerfn")
    assert s.config["hbm"]["reducer"] == 3 and s.config["hbm"]["combiner"] == "fsum"


def test_configure_accepts_a_plain_sum(monkeypatch):
    def plain(key, values, emit):
        count = 0
        for v in values:
            count = count + v
        emit(count)
    for name, fn in (("plain", plain), ("builtin", lambda k, vs, emit: emit(sum(vs))),
                     ("fsum", lambda k, vs, emit: emit(math.fsum(vs)))):
        s = configure(WWC_PKG + ".reducefn_device", combiner_plugin(monkeypatch, "fsum_comb_" + name, fn))
        assert s.config["hbm"]["combiner"] == "fsum"


@pytest.mark.parametrize("name,fn", [
    ("average", lambda k, vs, emit: emit(sum(vs) / len(vs))),
    ("drops_first", lambda k, vs, emit: emit(sum(vs[1:]))),
    ("absolute", lambda k, vs, emit: emit(sum(abs(v) for v in vs))),
    ("identity", lambda k, vs, emit: [emit(v) for v in vs]),
    ("count", lambda k, vs, emit: emit(len(vs))),
])
def test_configure_refuses_a_combinerfn_that_does_not_sum(monkeypatch, name, fn):
    with pytest.raises(ValueError, match="hbm_combinerfn"):
        configure(WWC_PKG + ".reducefn_device", combiner_plugin(monkeypatch, "fsum_comb_" + name, fn))


def test_configure_refuses_fsum_combiner_without_the_fsum_reducer():
    with pytest.raises(ValueError, match="hbm_combinerfn"):
        configure(WWC_PKG + ".init", WWC_PKG + ".combinerfn")
    with pytest.raises(ValueError, match="hbm_combinerfn"):
        configure("lua_mapreduce_b200.mapreduce.examples.InvertedIndex.reducefn_device", WWC_PKG + ".combinerfn")


def test_configure_refuses_fsum_combiner_without_byte_values():
    with pytest.raises(ValueError, match="hbm_combinerfn"):
        configure(WWC_PKG + ".init", WWC_PKG + ".combinerfn", value_kind="int")


def test_unknown_combiner_lists_both_builtins(monkeypatch):
    name = combiner_plugin(monkeypatch, "fsum_comb_unknown", lambda k, vs, emit: emit(sum(vs)), decl="max")
    with pytest.raises(ValueError, match="hbm_combinerfn.*distinct.*fsum"):
        configure(WWC_PKG + ".init", name)
