"""The number-sum reducer on the CPU: the shared decoding and superaccumulator (csrc/mrhbm_numsum.cuh), host-compiled
from tests/native/num_sum_check.cu, against exact rational sums (Fraction) on random and adversarial doubles, and
server.configure's check of the declaration hbm_reducefn = "fsum" with a stand-in ctx."""
import math
import os
import random
import shutil
import struct
import subprocess
import sys
import types
from fractions import Fraction

import pytest

import mrhbm_loader

mrhbm_loader.load()
from lua_mapreduce_b200.mapreduce import server  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WWC_PKG = "lua_mapreduce_b200.mapreduce.examples.WeightedWordCount"
MAXF = Fraction(2) ** 1024 - Fraction(2) ** 970  # where rounding to nearest starts to give inf


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def from_bits(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def oracle(values):
    """float(sum(Fraction(v))), overflow to +-inf, the inf and -0 rules of MRHBM_RED_FSUM; None for a NaN sum."""
    pinf = any(v == math.inf for v in values)
    ninf = any(v == -math.inf for v in values)
    if pinf and ninf:
        return None
    if pinf or ninf:
        return math.inf if pinf else -math.inf
    s = sum(Fraction(v) for v in values)
    if s == 0:
        return -0.0 if all(math.copysign(1, v) < 0 for v in values) else 0.0
    if abs(s) >= MAXF:
        return math.inf if s > 0 else -math.inf
    return float(s)


def cases():
    rng = random.Random(5)
    tiny, big = 5e-324, 1.7976931348623157e308
    out = [
        [1e308, -1e308, 5e-324], [tiny], [tiny, tiny], [tiny, -tiny], [2.2250738585072014e-308, -tiny],
        [1.0, 2.0 ** -53], [1.0, 2.0 ** -53, 2.0 ** -105], [1.0 + 2.0 ** -52, 2.0 ** -53],  # ties: even down, up
        [1.0, 2.0 ** -53, -2.0 ** -106], [big, big], [big, 2.0 ** 970], [big, 2.0 ** 970, -tiny], [big, 2.0 ** 969],
        [-big, -2.0 ** 970], [math.inf, 1.0], [-math.inf, -math.inf, 3.0], [math.inf, -math.inf], [-0.0],
        [-0.0, -0.0, -0.0], [-0.0, 0.0], [0.0], [1.0, -1.0], [-1.0, 1.0, -0.0], [2.0 ** 60, 1.0, -2.0 ** 60],
        [0.1] * 10, [1e16, 1.0, -1e16], [3.0, 5.0, 7.0], [float(2 ** 53 - 1), 1.0, 1.0],
        [2.0 ** 1023, 2.0 ** 1023, -2.0 ** 1023], [tiny] * 1000, [big] * 3 + [-big] * 3 + [1.5],
    ]
    for n in (1, 2, 3, 7, 33, 200):
        for _ in range(40):
            kind = rng.randrange(4)
            if kind == 0:    # anything finite
                vals = []
                while len(vals) < n:
                    x = from_bits(rng.getrandbits(64))
                    if math.isfinite(x):
                        vals.append(x)
            elif kind == 1:  # one scale, both signs: heavy cancellation
                e = rng.randrange(-1074, 1000)
                vals = [rng.choice((-1, 1)) * rng.random() * 2.0 ** e for _ in range(n)]
            elif kind == 2:  # weights as a word count gives them
                vals = [1 / rng.randrange(1, 40) for _ in range(n)]
            else:            # near the edges of the range
                vals = [rng.choice((-1, 1)) * from_bits(rng.choice((rng.randrange(1, 1 << 20),
                                                                    0x7fe0000000000000 + rng.getrandbits(52))))
                        for _ in range(n)]
            out.append(vals)
    return out


def run_check(tmp_path, lines):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "num_sum_check")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "lua-mapreduce_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "num_sum_check.cu")])
    out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    res = out.stdout.splitlines()
    assert out.returncode == 0 and res[-1] == "ok", out.stdout[-2000:]
    return res[:-1]


def test_exact_sum_matches_fractions(tmp_path):
    cs = cases()
    lines = []
    for vals in cs:
        body = " ".join("%x" % bits(v) for v in vals)
        lines.append("%d %s" % (len(vals), body))
        lines.append("%d %s split" % (len(vals), body))
    got = run_check(tmp_path, lines)
    assert len(got) == 2 * len(cs)
    for i, vals in enumerate(cs):
        want = oracle(vals)
        for g in got[2 * i:2 * i + 2]:
            if want is None:
                assert g == "nan", vals
            else:
                assert g != "nan" and int(g, 16) == bits(want), (vals, from_bits(int(g, 16)), want)


class StandIn:
    def __init__(self, h):
        self.h = dict(h)


def configure(reducefn, value_kind="bytes", combinerfn=None):
    S = WWC_PKG + ".init"
    s = server.new("hbm://local", "fsum-configure")
    s.ctx_factory = StandIn
    s.configure(dict(taskfn=S, mapfn=S, partitionfn=S, reducefn=reducefn, finalfn=S, combinerfn=combinerfn,
                     storage="hbm", hbm={"value_kind": value_kind}))
    return s


def plugin(monkeypatch, name, reducefn, decl="fsum"):
    mod = types.ModuleType(name)
    mod.init = lambda arg=None: None
    mod.reducefn = reducefn
    mod.hbm_reducefn = decl
    monkeypatch.setitem(sys.modules, name, mod)
    return name


def test_configure_selects_the_fsum_reducer():
    assert configure(WWC_PKG + ".reducefn_device").config["hbm"]["reducer"] == 3
    assert configure(WWC_PKG + ".init").config["hbm"]["reducer"] == 1


def test_configure_accepts_a_plain_sum(monkeypatch):
    def plain(key, values, emit):
        count = 0
        for v in values:
            count = count + v
        emit(count)
    assert configure(plugin(monkeypatch, "fsum_plain", plain)).config["hbm"]["reducer"] == 3
    assert configure(plugin(monkeypatch, "fsum_builtin", lambda k, vs, emit: emit(sum(vs)))).config["hbm"]["reducer"] == 3
    assert configure(plugin(monkeypatch, "fsum_fsum", lambda k, vs, emit: emit(math.fsum(vs)))).config["hbm"]["reducer"] == 3


@pytest.mark.parametrize("name,fn", [
    ("average", lambda k, vs, emit: emit(sum(vs) / len(vs))),
    ("drops_first", lambda k, vs, emit: emit(sum(vs[1:]))),
    ("absolute", lambda k, vs, emit: emit(sum(abs(v) for v in vs))),
    ("count", lambda k, vs, emit: emit(len(vs))),
    ("every_value", lambda k, vs, emit: [emit(v) for v in vs]),
    ("max", lambda k, vs, emit: emit(max(vs))),
])
def test_configure_refuses_a_reducefn_that_does_not_sum(monkeypatch, name, fn):
    with pytest.raises(ValueError, match="hbm_reducefn"):
        configure(plugin(monkeypatch, "fsum_" + name, fn))


def test_configure_refuses_fsum_without_byte_values():
    with pytest.raises(ValueError, match="value_kind"):
        configure(WWC_PKG + ".reducefn_device", value_kind="int")


def test_sum_with_byte_values_stays_refused(monkeypatch):
    with pytest.raises(ValueError, match="hbm_reducefn"):
        configure(plugin(monkeypatch, "fsum_declares_sum", lambda k, vs, emit: emit(sum(vs)), decl="sum"))


def test_configure_refuses_fsum_with_a_device_combiner():
    with pytest.raises(ValueError, match="hbm_combinerfn"):
        configure(WWC_PKG + ".reducefn_device", combinerfn="lua_mapreduce_b200.mapreduce.examples.InvertedIndex.combinerfn")
