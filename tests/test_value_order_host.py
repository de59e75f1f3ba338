"""The distinct reducer on the CPU: the shared byte-value compare (csrc/mrhbm_valbytes.cuh) against memcmp at all four
arena alignments, host-compiled from tests/native/value_order_check.cu, and server.configure's check of the
declaration hbm_reducefn = "distinct" with a stand-in ctx."""
import os
import shutil
import subprocess
import sys
import types

import pytest

import mrhbm_loader

mrhbm_loader.load()
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.InvertedIndex import init as II  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
II_PKG = "lua_mapreduce_b200.mapreduce.examples.InvertedIndex"


def test_value_compare_matches_memcmp(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "value_order_check")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "lua-mapreduce_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "value_order_check.cu")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.splitlines()[-1] == "ok", out.stdout


class StandIn:
    def __init__(self, h):
        self.h = dict(h)


def configure(reducefn, value_kind="bytes", combinerfn=None):
    S = II_PKG + ".init"
    s = server.new("hbm://local", "dr-configure")
    s.ctx_factory = StandIn
    s.configure(dict(taskfn=S, mapfn=S, partitionfn=S, reducefn=reducefn, finalfn=S, combinerfn=combinerfn,
                     storage="hbm", hbm={"value_kind": value_kind}))
    return s


def plugin(monkeypatch, name, reducefn, decl="distinct"):
    mod = types.ModuleType(name)
    mod.init = lambda arg=None: None
    mod.reducefn = reducefn
    mod.hbm_reducefn = decl
    monkeypatch.setitem(sys.modules, name, mod)
    return name


def test_configure_selects_the_distinct_reducer():
    assert configure(II_PKG + ".reducefn_device").config["hbm"]["reducer"] == 2
    s = configure(II_PKG + ".reducefn_device", combinerfn=II_PKG + ".combinerfn")
    assert s.config["hbm"]["reducer"] == 2 and s.config["hbm"]["combiner"] == "distinct"
    assert configure(II_PKG + ".init").config["hbm"]["reducer"] == 1


def test_configure_refuses_a_reducefn_the_declaration_does_not_describe(monkeypatch):
    def unsorted(key, values, emit):  # dedupes, keeps the order of first occurrence
        for v in dict.fromkeys(values):
            emit(v)

    def duplicates(key, values, emit):  # sorts, keeps every copy
        for v in sorted(values):
            emit(v)

    def descending(key, values, emit):
        for v in sorted(set(values), reverse=True):
            emit(v)

    def dropping(key, values, emit):
        for v in sorted(set(values))[1:]:
            emit(v)
    for fn in (unsorted, duplicates, descending, dropping):
        with pytest.raises(ValueError, match="the declaration must describe"):
            configure(plugin(monkeypatch, "dr_plugin_" + fn.__name__, fn))
    with pytest.raises(NotImplementedError, match="hbm_reducefn"):
        configure(plugin(monkeypatch, "dr_plugin_unknown", II.reducefn, decl="unique"))


def test_configure_refuses_distinct_on_integer_values():
    with pytest.raises(ValueError, match="value_kind"):
        configure(II_PKG + ".reducefn_device", value_kind="int")


def test_configure_still_refuses_sum_on_byte_values(monkeypatch):
    with pytest.raises(ValueError, match="hbm_reducefn"):
        configure(plugin(monkeypatch, "dr_plugin_sum", II.reducefn, decl="sum"))
