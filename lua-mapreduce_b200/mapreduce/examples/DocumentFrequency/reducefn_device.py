"""The DocumentFrequency reducefn declared as the device's "count_distinct" reducer: every word's number of distinct
file names, counted on the device, so the reducefn is not called (needs hbm = {"value_kind": "bytes"})."""
from .init import reducefn  # noqa: F401  (host definition: what the declaration describes)

hbm_reducefn = "count_distinct"


def init(arg=None):
    pass
