"""The KeyNumberSum reducefn declared as the device's "fsum" reducer: every key's numbers summed exactly on the device
and rounded once, so the reducefn is not called (needs hbm = {"value_kind": "bytes"})."""
from .init import reducefn  # noqa: F401  (host definition: what the declaration describes)

hbm_reducefn = "fsum"


def init(arg=None):
    pass
