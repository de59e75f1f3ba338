"""The KeyNumberSum mapfn declared as the device's line parser: every line "key number" of the file becomes
(key, float(number)) on the device (needs hbm = {"value_kind": "bytes"} and string keys)."""
from .init import mapfn  # noqa: F401  (host definition, used when the storage has no device parser)

hbm_mapfn = "key_numbers_file"


def init(arg=None):
    pass
