"""The InvertedIndex reducefn declared as the device's "distinct" reducer: every word's distinct file names, ascending,
computed on the device, so the reducefn is not called (needs hbm = {"value_kind": "bytes"})."""
from .init import reducefn  # noqa: F401  (host definition: what the declaration describes)

hbm_reducefn = "distinct"


def init(arg=None):
    pass
