"""Host side of the range partitioner (no GPU): the C ABI export list, the Python mirror's declaration check, the
SortedWordCount example's configuration and the Lua sources that declare it."""
import os
import re
import sys
import types

import pytest

import mrhbm_loader

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402
from lua_mapreduce_b200.mapreduce import server  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SWC = "lua_mapreduce_b200.mapreduce.examples.SortedWordCount"
WC = "lua_mapreduce_b200.mapreduce.examples.WordCount"


def test_exports_carry_the_splitter_calls():
    hdr = open(os.path.join(ROOT, "include", "mrhbm.h")).read()
    for name in ("mrhbm_set_splitters", "mrhbm_sample_splitters"):
        assert name in mrhbm.EXPORTS and re.search(r"\b%s\(" % name, hdr)
    assert "MRHBM_PART_RANGE = 3" in hdr and mrhbm.PART_RANGE == 3


def _module(name, nparts, splitters, fn):
    m = types.ModuleType(name)
    m.NUM_REDUCERS, m.hbm_partitionfn, m.hbm_splitters, m.partitionfn = nparts, "range", splitters, fn
    m.init = lambda arg=None: None
    sys.modules[name] = m
    return name


def _configure(part_name, key_kind="str"):
    s = server.new("hbm://local", "range-%s" % part_name)
    s.configure(dict(taskfn=WC + ".taskfn", mapfn=WC + ".mapfn", partitionfn=part_name, reducefn=WC + ".reducefn",
                     storage="hbm", hbm={"key_kind": key_kind}))
    return s


def test_sorted_wordcount_configures_as_a_range():
    s = _configure(SWC + ".partitionfn")
    h = s.config["hbm"]
    assert h["partitioner"] == 3 and h["num_partitions"] == 26
    assert h["splitters"] == [bytes([c]) for c in range(ord("b"), ord("z") + 1)]


def test_declaration_must_agree_with_the_function():
    good = _module("range_good", 3, ["g", "p"], lambda k: (k >= b"g") + (k >= b"p"))
    assert _configure(good).config["hbm"]["splitters"] == [b"g", b"p"]
    bad = _module("range_bad", 3, ["g", "p"], lambda k: (k > b"g") + (k >= b"p"))  # "g" itself on the lower side
    with pytest.raises(ValueError, match="partitionfn"):
        _configure(bad)
    # u64 keys: the key just below a splitter is checked too
    bad64 = _module("range_bad64", 2, [1000], lambda k: int(k >= 999))
    with pytest.raises(ValueError, match="partitionfn"):
        _configure(bad64, "u64")
    ok64 = _module("range_ok64", 2, [1000], lambda k: int(k >= 1000))
    assert _configure(ok64, "u64").config["hbm"]["splitters"] == [1000]


def test_num_reducers_must_match_the_splitters():
    name = _module("range_count", 4, ["g", "p"], lambda k: (k >= b"g") + (k >= b"p"))
    with pytest.raises(ValueError, match="NUM_REDUCERS"):
        _configure(name)
    dec = _module("range_decreasing", 3, ["p", "g"], lambda k: 0)
    with pytest.raises(ValueError, match="non-decreasing"):
        _configure(dec)


def test_sampled_splitters_are_declared_without_a_list():
    name = _module("range_sample", 16, "sample", lambda k: 0)
    assert _configure(name).config["hbm"]["splitters"] == "sample"


def test_lua_sources_declare_the_range_partitioner():
    lua = os.path.join(ROOT, "lua-mapreduce_b200", "lua")
    c = open(os.path.join(lua, "mrhbm_lua.c")).read()
    for name in ("mrhbm_set_splitters", "mrhbm_sample_splitters", '"set_splitters"', '"sample_splitters"', '"range"'):
        assert name in c
    h = open(os.path.join(lua, "mapreduce", "hbm.lua")).read()
    assert "hbm_splitters" in h and "ctx:sample_splitters()" in h and "ctx:set_splitters(" in h
    # the same declaration semantics as the mirror: non-decreasing, and u64 keys checked just below every splitter
    assert "must be non-decreasing" in h and "be_minus_one(spl[i])" in h
