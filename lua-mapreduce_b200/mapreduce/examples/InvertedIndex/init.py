"""Inverted index over the WordCount files, as ONE module providing all six functions.

mapfn emits (word, file name) for every occurrence of a word; the general reducefn (no hbm_reducefn: it runs on the
host per group) emits the word's distinct file names in ascending order; finalfn keeps them in RESULT.  String values
need a byte-values shuffle: configure with hbm = {"value_kind": "bytes"}.  combinerfn (module combinerfn.py) keeps one
copy of each (word, file) pair of a map job on the device."""
from ..WordCount.init import FILES, _TOKEN, partitionfn, taskfn  # noqa: F401

NUM_REDUCERS = 15
hbm_partitionfn = "fnv_lua"  # == partitionfn (examples/WordCount/partitionfn.lua)
RESULT = {}  # word -> [file name, ...] (bytes, ascending)


def init(arg):
    pass


def mapfn(key, value, emit):
    with open(value, "rb") as fh:
        for line in fh:
            for w in _TOKEN.findall(line):
                emit(w, value)


def reducefn(key, values, emit):
    for f in sorted(set(values)):
        emit(f)


# The reducefn emits the distinct values of a key, so it is also a valid combinerfn: combining a map job's values first
# does not change what reducing them gives.  Declared as the device's "distinct" combiner, it drops the repeated
# (word, file) pairs of each map job at its commit; the reducefn still runs on the host.
combinerfn = reducefn
hbm_combinerfn = "distinct"


def finalfn(pairs_iterator):
    for key, values in pairs_iterator:
        RESULT[key] = list(values)
    return False  # keep the result partitions (export_results writes them)
