"""Weighted word count over the WordCount files, as ONE module providing all six functions.

mapfn gives every word of a line the weight 1 / (words in the line), so that each line counts once in total; the
general reducefn (no hbm_reducefn: it runs on the host per group) adds a word's weights left to right, as the Lua
`count = count + v` does; finalfn keeps the totals in RESULT.  Fractional values need a byte-values shuffle: configure
with hbm = {"value_kind": "bytes"}.  reducefn_device.py declares the same reducefn as the device's "fsum" reducer, which
sums each word's weights exactly and rounds once."""
from ..WordCount.init import FILES, _TOKEN, partitionfn, taskfn  # noqa: F401

NUM_REDUCERS = 15
hbm_partitionfn = "fnv_lua"  # == partitionfn (examples/WordCount/partitionfn.lua)
RESULT = {}  # word -> total weight


def init(arg):
    pass


def mapfn(key, value, emit):
    with open(value, "rb") as fh:
        for line in fh:
            words = _TOKEN.findall(line)
            for w in words:
                emit(w, 1 / len(words))


def reducefn(key, values, emit):
    count = 0
    for v in values:
        count = count + v
    emit(count)


def finalfn(pairs_iterator):
    for key, values in pairs_iterator:
        RESULT[key] = values[0]
    return False  # keep the result partitions (export_results writes them)
