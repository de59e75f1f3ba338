"""The count-distinct reducer on the CPU: server.configure's check of the declaration hbm_reducefn = "count_distinct"
(with a stand-in ctx), the combiners it takes and refuses, the Lua binding's constant, and the bulk path that decodes
the device's one encoded count per key."""
import os
import re
import sys
import types

import numpy as np
import pytest

import mrhbm_loader

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402
from lua_mapreduce_b200.mapreduce import job as job_mod  # noqa: E402
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce import tuple as T  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DF_PKG = "lua_mapreduce_b200.mapreduce.examples.DocumentFrequency"
II_PKG = "lua_mapreduce_b200.mapreduce.examples.InvertedIndex"
KNS_PKG = "lua_mapreduce_b200.mapreduce.examples.KeyNumberSum"


class StandIn:
    def __init__(self, h):
        self.h = dict(h)


def configure(reducefn, value_kind="bytes", combinerfn=None):
    S = DF_PKG + ".init"
    s = server.new("hbm://local", "count-distinct-configure")
    s.ctx_factory = StandIn
    s.configure(dict(taskfn=S, mapfn=S, partitionfn=S, reducefn=reducefn, finalfn=S, combinerfn=combinerfn,
                     storage="hbm", hbm={"value_kind": value_kind}))
    return s


def plugin(monkeypatch, name, reducefn, decl="count_distinct"):
    mod = types.ModuleType(name)
    mod.init = lambda arg=None: None
    mod.reducefn = reducefn
    mod.hbm_reducefn = decl
    monkeypatch.setitem(sys.modules, name, mod)
    return name


def test_the_constant_matches_the_header():
    with open(os.path.join(ROOT, "include", "mrhbm.h")) as fh:
        assert re.search(r"MRHBM_RED_COUNT_DISTINCT = (\d+)", fh.read()).group(1) == str(mrhbm.RED_COUNT_DISTINCT) == "4"
    with open(os.path.join(ROOT, "lua-mapreduce_b200", "lua", "mrhbm_lua.c")) as fh:
        assert '"count_distinct") == 0 ? MRHBM_RED_COUNT_DISTINCT' in fh.read()
    with open(os.path.join(ROOT, "lua-mapreduce_b200", "lua", "mapreduce", "hbm.lua")) as fh:
        assert 'count_red and "count_distinct"' in fh.read()


def test_configure_selects_the_count_distinct_reducer():
    s = configure(DF_PKG + ".reducefn_device")
    assert s.config["hbm"]["reducer"] == 4 and s.config["hbm"]["combiner"] is False
    s = configure(DF_PKG + ".reducefn_device", combinerfn=DF_PKG + ".combinerfn")
    assert s.config["hbm"]["reducer"] == 4 and s.config["hbm"]["combiner"] == "distinct"
    assert configure(DF_PKG + ".init").config["hbm"]["reducer"] == 1  # no declaration: the reducefn on the host
    assert configure(DF_PKG + ".init", combinerfn=DF_PKG + ".combinerfn").config["hbm"]["combiner"] == "distinct"


@pytest.mark.parametrize("name,fn", [
    ("set_len", lambda k, vs, emit: emit(len(set(vs)))),
    ("float", lambda k, vs, emit: emit(float(len(set(vs))))),
    ("dict", lambda k, vs, emit: emit(len(dict.fromkeys(vs)))),
])
def test_configure_accepts_a_count_of_distinct_values(monkeypatch, name, fn):
    assert configure(plugin(monkeypatch, "cd_" + name, fn)).config["hbm"]["reducer"] == 4


@pytest.mark.parametrize("name,fn", [
    ("count_all", lambda k, vs, emit: emit(len(vs))),  # counts repeats
    ("distinct_values", lambda k, vs, emit: [emit(v) for v in sorted(set(vs))]),
    ("two_numbers", lambda k, vs, emit: (emit(len(set(vs))), emit(0))),
    ("nothing", lambda k, vs, emit: None),
    ("bool", lambda k, vs, emit: emit(True)),
    ("string", lambda k, vs, emit: emit(str(len(set(vs))))),
    ("raises", lambda k, vs, emit: 1 / 0),
])
def test_configure_refuses_a_reducefn_that_does_not_count_distinct_values(monkeypatch, name, fn):
    with pytest.raises(ValueError, match="count_distinct"):
        configure(plugin(monkeypatch, "cd_bad_" + name, fn))


def test_probes_tell_equal_bytes_from_equal_numbers():
    # 3 and 3.0 have one encoding (one value), b"" is a value: exactly the device's rule
    vals = [3, 3.0, 1.5, 0]
    assert len({T.encode_value(v) for v in vals}) == 3
    assert T.encode_value(-0.0) != T.encode_value(0.0)
    assert any(b"" in p for p in server._DISTINCT_PROBES)


def test_configure_refuses_count_distinct_without_byte_values():
    with pytest.raises(ValueError, match="value_kind"):
        configure(DF_PKG + ".reducefn_device", value_kind="int")


def test_configure_refuses_the_fsum_combiner():
    with pytest.raises(ValueError, match="fsum"):
        configure(DF_PKG + ".reducefn_device", combinerfn=KNS_PKG + ".combinerfn")


def test_unknown_builtins_name_count_distinct(monkeypatch):
    with pytest.raises(NotImplementedError, match="count_distinct"):
        configure(plugin(monkeypatch, "cd_unknown", lambda k, vs, emit: emit(1), decl="countdistinct"))


def test_the_distinct_combiner_still_takes_the_other_reducers():
    assert configure(II_PKG + ".reducefn_device", combinerfn=DF_PKG + ".combinerfn").config["hbm"]["reducer"] == 2


class BulkCtx:
    """result_copy / result_values / result_info of a byte-values ctx whose rows hold one encoded number each"""

    def __init__(self, keys, numbers, po, sorted_=1):
        self.keys, self.po, self.sorted = keys, po, sorted_
        self.blob = np.frombuffer(b"".join(T.encode_value(float(x)) for x in numbers), dtype=np.uint8)

    def result_copy(self):
        return self.keys, None, self.po

    def result_values(self):
        return self.blob, np.arange(len(self.keys) + 1, dtype=np.uint64) * 11

    def result_info(self):
        return types.SimpleNamespace(sorted=self.sorted)


def bulk(ctx, part, reducer=4):
    board = types.SimpleNamespace(ctx=ctx, iteration=0)
    j = job_mod.Job(board, "red_jobs", {"_id": part, "value": {}}, dict(hbm={"reducer": reducer}))
    return j._bulk_numbers(part)


def test_bulk_path_decodes_the_counts():
    counts = [1, 3, 2 ** 31 - 1, 7, 1, 2]
    keys = np.array([b"a", b"b\x01\x01c", b"zz", b"k", b"m", b"x"], dtype="S28")
    po = np.array([0, 3, 3, 6], dtype=np.uint64)
    ctx = BulkCtx(keys, counts, po)
    assert bulk(ctx, 0) == [(b"a", [1]), (b"b\x00c", [3]), (b"zz", [2 ** 31 - 1])]
    assert bulk(ctx, 1) == []
    got = bulk(ctx, 2)
    assert got == [(b"k", [7]), (b"m", [1]), (b"x", [2])]
    assert all(type(v[0]) is int for _, v in got)  # as tuple.decode_value gives an integral number


def test_bulk_path_merges_hash_runs_and_u64_keys():
    keys = np.array([9, 2, 5, 1], dtype=np.uint64)
    ctx = BulkCtx(keys, [4, 1, 6, 2], np.array([0, 4], dtype=np.uint64), sorted_=0)
    assert bulk(ctx, 0) == [((1).to_bytes(8, "big"), [2]), ((2).to_bytes(8, "big"), [1]),
                            ((5).to_bytes(8, "big"), [6]), ((9).to_bytes(8, "big"), [4])]


def test_bulk_path_still_decodes_sums():
    keys = np.array([b"a", b"b"], dtype="S28")
    ctx = BulkCtx(keys, [0.5, -0.0], np.array([0, 2], dtype=np.uint64))
    got = bulk(ctx, 0, reducer=3)
    assert got[0] == (b"a", [0.5]) and got[1][1][0] == 0 and str(got[1][1][0]) == "-0.0"
