"""The DocumentFrequency mapfn with the tokeniser declared as the device built-in: every word of the file paired with
the file name (needs hbm = {"value_kind": "bytes"})."""
from .init import mapfn  # noqa: F401  (host definition, used when the storage has no device tokeniser)

hbm_mapfn = "words_file"


def init(arg=None):
    pass
