"""The WeightedWordCount combinerfn: its reducefn, which emits the sum of a word's weights, declared as the device's
"fsum" combiner.  At each map job's commit the device keeps every word's weights of that job as the exact expansion of
their sum (one or two numbers), so the "fsum" reducer gives bit for bit what it gives without the combiner (needs
reducefn_device.py and hbm = {"value_kind": "bytes"})."""
from .init import reducefn as combinerfn  # noqa: F401  (host definition: what the declaration describes)

hbm_combinerfn = "fsum"


def init(arg=None):
    pass
