"""Key-number sum over files of text lines "key number", as ONE module providing all six functions.

mapfn emits (key, float(number)) for every line that is not blank, and refuses any other line; the general reducefn (no
hbm_reducefn: it runs on the host per group) adds a key's numbers left to right, as the Lua `count = count + v` does;
finalfn keeps the totals in RESULT.  Number values need a byte-values shuffle: configure with
hbm = {"value_kind": "bytes"}.  mapfn_device.py declares the same mapfn as the device's line parser, reducefn_device.py
and combinerfn.py the device's exact "fsum" reducer and combiner."""
import re

from ..WordCount.init import partitionfn  # noqa: F401

NUM_REDUCERS = 15
hbm_partitionfn = "fnv_lua"  # == partitionfn (examples/WordCount/partitionfn.lua)
FILES = []  # the input files, one map job each
RESULT = {}  # key -> total
_FIELD = re.compile(rb"[^ \t\n\v\f\r]+")  # C-locale white space separates fields
_NUMBER = re.compile(rb"[+-]?([0-9]+(\.[0-9]*)?|\.[0-9]+)([eE][+-]?[0-9]+)?\Z")  # decimal, as mrhbm_map_key_numbers


def init(arg):
    pass


def taskfn(emit):
    for i, f in enumerate(FILES):
        emit(i + 1, f)


def mapfn(key, value, emit):
    with open(value, "rb") as fh:
        for off, line in enumerate(fh):
            fields = _FIELD.findall(line)
            if not fields:
                continue
            if len(fields) != 2 or not _NUMBER.match(fields[1]):
                raise ValueError("%s: line %d is not 'key number': %r" % (value, off + 1, line[:80]))
            emit(fields[0], float(fields[1]))


def reducefn(key, values, emit):
    count = 0
    for v in values:
        count = count + v
    emit(count)


def finalfn(pairs_iterator):
    for key, values in pairs_iterator:
        RESULT[key] = values[0]
    return False  # keep the result partitions (export_results writes them)
