"""Byte values on the host side, without a GPU: the value codec (Python and hbm.lua), the mirror's value_kind = "bytes"
flow and refusals over a stand-in ctx, and the value kernels' sm_90a build (no register spills)."""
import math
import os
import re
import shutil
import struct
import subprocess

import pytest
from hypothesis import given, settings, strategies as st

import mrhbm_loader
from conftest import ROOT, expand_tokens

mrhbm_loader.load()
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce import tuple as T  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.InvertedIndex import init as II  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WordCount import init as WordCount  # noqa: E402

PKG = os.path.join(ROOT, "lua-mapreduce_b200")
HBM = os.path.join(PKG, "lua", "mapreduce", "hbm.lua")
II_MOD = "lua_mapreduce_b200.mapreduce.examples.InvertedIndex.init"


def same(a, b):
    """same Lua type and value (-0.0 is not 0)"""
    if isinstance(a, float) and isinstance(b, float) and a == 0 == b:
        return math.copysign(1, a) == math.copysign(1, b)
    return type(a) is type(b) and a == b


@pytest.mark.parametrize("v", [-3, 0.5, 2 ** 53, -(2 ** 53), 0, -0.0, 1e308, -1e-300, 5e-324, math.inf, -math.inf, 7.0])
def test_numbers_round_trip_with_their_type(v):
    want = int(v) if isinstance(v, float) and v.is_integer() and 0 < abs(v) <= 2 ** 53 else v
    assert same(T.decode_value(T.encode_value(v)), want)


def test_strings_round_trip_as_bytes():
    for s in (b"", b"\x00", bytes(range(256)) * 3, "file1.txt"):
        enc = T.encode_value(s)
        assert enc[0] == 0x20 and T.decode_value(enc) == (s.encode() if isinstance(s, str) else s)


def test_values_that_are_refused():
    for v, exc in ((math.nan, ValueError), (2 ** 53 + 1, OverflowError), (True, TypeError), ({}, TypeError)):
        with pytest.raises(exc):
            T.encode_value(v)
    with pytest.raises(ValueError):
        T.decode_value(b"\x10\x80")  # truncated number


def test_keys_still_fold_negative_zero():
    assert T.encode(-0.0) == T.encode(0) and T.decode(T.encode(-0.0)) == 0


@settings(max_examples=300, deadline=None)
@given(st.floats(allow_nan=False))
def test_every_double_round_trips(x):
    enc = T.encode_value(x)
    assert len(enc) == 11 and enc[0] == 0x10
    got = T.decode_value(enc)
    assert struct.pack(">d", float(got)) == struct.pack(">d", x)


def test_lua_value_codec_matches_the_mirror():
    """hbm.lua is not runnable here: pin its value codec to the same tags, the same number encoding and -0 rule"""
    src = open(HBM).read()
    assert T._NUM == 16 and T._STR == 32
    for frag in ('if type(v) == "string" then return "\\32" .. v end',
                 "enc_num(v, out, true)",
                 "if value and x == 0 and 1 / x < 0 then",
                 "hi, lo = 0x80000000, 0 -- a value keeps -0",
                 'assert(tag == 16 and #s == 11, "bad value encoding")',
                 "if tag == 32 then return s:sub(2) end",
                 "if byte_values then value = hbm.encode_value(value) end",
                 "for i = 1, #v do v[i] = hbm.decode_value(v[i]) end",
                 'values = byte_values and "bytes" or "int"'):
        assert frag in src, frag
    # the Lua number path of a value is the key path (enc_num) except for -0: same words as struct.pack
    neg0 = struct.unpack(">Q", struct.pack(">d", -0.0))[0]
    assert (neg0 >> 32, neg0 & 0xFFFFFFFF) == (0x80000000, 0)


class ByteStandInCtx:
    """Dict-based stand-in for a byte-values mrhbm.Ctx (tests only; the product has no CPU path): it takes bytes
    values only, as the library does."""

    class _Map:
        def __init__(self, ctx, job):
            self.ctx, self.job, self.buf = ctx, job, []

        def emit(self, k, v):
            assert isinstance(k, bytes) and isinstance(v, bytes), (k, v)
            self.buf.append((k, v))

        def commit(self):
            self.ctx.jobs[self.job] = self.buf

        def abort(self):
            self.buf = None

    made = []

    def __init__(self, h):
        type(self).made.append(dict(h))
        self.P, self.jobs, self.parts = h["num_partitions"], {}, {}

    def map_begin(self, job):
        return self._Map(self, str(job))

    def reset(self):
        self.jobs, self.parts = {}, {}

    def shuffle(self):
        self.parts = {}
        for buf in self.jobs.values():
            for k, v in buf:
                self.parts.setdefault(WordCount.partitionfn(k), {}).setdefault(k, []).append(v)

    def partitions(self):
        return sorted(self.parts)

    def groups(self, p):
        for k in sorted(self.parts.get(p, {})):
            yield k, list(self.parts[p][k])

    def stats(self):
        return {}


def test_inverted_index_over_a_stand_in(tmp_path, golden_wordcount):
    files = []
    for job in range(4):
        toks = expand_tokens(golden_wordcount, job)
        p = tmp_path / ("file%d.txt" % job)
        p.write_bytes(b"\n".join(b" ".join(toks[i:i + 7]) for i in range(0, len(toks), 7)) + b"\n")
        files.append(str(p))
    WordCount.FILES[:] = files
    II.RESULT.clear()
    ByteStandInCtx.made.clear()
    s = server.new("hbm://local", "ii-host")
    s.ctx_factory = ByteStandInCtx
    s.configure(dict(taskfn=II_MOD, mapfn=II_MOD, partitionfn=II_MOD, reducefn=II_MOD, finalfn=II_MOD, storage="hbm",
                     hbm={"value_kind": "bytes"}))
    assert s.config["hbm"]["reducer"] == 1 and not s.config["hbm"]["combiner"]
    s.loop()
    assert ByteStandInCtx.made[0]["value_kind"] == "bytes"
    assert II.RESULT == {k: sorted(files[j].encode() for j in range(4) if c[j] > 0) for k, _, c in golden_wordcount}


def test_mixed_values_reach_the_reducefn_with_their_type(tmp_path, monkeypatch):
    import types
    import sys
    seen = []
    mod = types.ModuleType("byte_values_plugin")
    vals = [-3, 0.5, 2 ** 53, -0.0, 1e308, "s", b"\x00b"]
    mod.NUM_REDUCERS, mod.hbm_partitionfn = 15, "fnv_lua"
    mod.init = lambda arg: None
    mod.taskfn = lambda emit: emit(1, "x")
    mod.mapfn = lambda key, value, emit: [emit(b"k", v) for v in vals]
    mod.partitionfn = WordCount.partitionfn
    mod.reducefn = lambda key, values, emit: seen.extend(values) or emit(len(values))
    mod.finalfn = lambda it: list(it) and True
    monkeypatch.setitem(sys.modules, "byte_values_plugin", mod)
    s = server.new("hbm://local", "bv-types")
    s.ctx_factory = ByteStandInCtx
    s.configure(dict(taskfn=mod.__name__, mapfn=mod.__name__, partitionfn=mod.__name__, reducefn=mod.__name__,
                     finalfn=mod.__name__, storage="hbm", hbm={"value_kind": "bytes"}))
    s.loop()
    want = [v.encode() if isinstance(v, str) else v for v in vals]
    assert len(seen) == len(want) and all(same(a, b) for a, b in zip(seen, want))
    mod.mapfn = lambda key, value, emit: emit(b"k", math.nan)  # NaN is refused at emit: the map job breaks
    s2 = server.new("hbm://local", "bv-nan")
    s2.ctx_factory = ByteStandInCtx
    s2.configure(dict(taskfn=mod.__name__, mapfn=mod.__name__, partitionfn=mod.__name__, reducefn=mod.__name__,
                      finalfn=mod.__name__, storage="hbm", hbm={"value_kind": "bytes"}))
    s2.loop()
    assert s2.stats["failed_maps"] == 1


def test_value_kind_refusals():
    WC = "lua_mapreduce_b200.mapreduce.examples.WordCount"
    base = dict(taskfn=WC + ".taskfn", mapfn=WC + ".mapfn", partitionfn=WC + ".partitionfn", finalfn=WC + ".finalfn",
                storage="hbm")
    s = server.new("hbm://local", "bv-refuse")
    with pytest.raises(ValueError, match="hbm_reducefn"):  # the built-in sum cannot take byte values
        s.configure(dict(base, reducefn=WC + ".reducefn", hbm={"value_kind": "bytes"}))
    with pytest.raises(ValueError, match="value_kind"):
        s.configure(dict(base, reducefn=WC + ".reducefn2", hbm={"value_kind": "strings"}))
    s.configure(dict(base, reducefn=WC + ".reducefn2"))
    assert s.config["hbm"]["value_kind"] == "int"  # the default is unchanged: integer values


@pytest.mark.skipif(not (shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc")), reason="needs nvcc")
def test_value_kernels_build_for_sm90a_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(PKG, "csrc", "mrhbm_values.cu"), "-o", str(tmp_path / "v.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    kernels = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    assert {k for k in kernels if "k_value_" in k} and len(kernels) == 5, kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) == len(kernels) and all(a == "0" and b == "0" for a, b in spills), r.stderr
