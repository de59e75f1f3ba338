"""Document frequency over the WordCount files, as ONE module providing all six functions.

mapfn emits (word, file name) for every occurrence of a word; the general reducefn (no hbm_reducefn: it runs on the
host per group) collects the word's file names in a set and emits its size; finalfn keeps that number in RESULT.
String values need a byte-values shuffle: configure with hbm = {"value_kind": "bytes"}.  combinerfn (module
combinerfn.py) keeps one copy of each (word, file) pair of a map job on the device; reducefn_device.py declares the
reducefn as the device's "count_distinct" reducer."""
from ..WordCount.init import FILES, _TOKEN, partitionfn, taskfn  # noqa: F401

NUM_REDUCERS = 15
hbm_partitionfn = "fnv_lua"  # == partitionfn (examples/WordCount/partitionfn.lua)
RESULT = {}  # word -> number of distinct files it occurs in


def init(arg):
    pass


def mapfn(key, value, emit):
    with open(value, "rb") as fh:
        for line in fh:
            for w in _TOKEN.findall(line):
                emit(w, value)


def reducefn(key, values, emit):
    emit(len(set(values)))


# Keeping one copy of each distinct value of a key does not change how many distinct values it has, so the distinct
# values are a valid combinerfn for this reducefn.  Declared as the device's "distinct" combiner, it drops the repeated
# (word, file) pairs of each map job at its commit.
def combinerfn(key, values, emit):
    for f in sorted(set(values)):
        emit(f)


hbm_combinerfn = "distinct"


def finalfn(pairs_iterator):
    for key, values in pairs_iterator:
        RESULT[key] = values[0]
    return False  # keep the result partitions (export_results writes them)
