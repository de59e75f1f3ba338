"""The KeyNumberSum combinerfn: its reducefn declared as the device's "fsum" combiner, so each map job's numbers per
key become the exact expansion of their sum at its commit (needs reducefn_device.py and hbm = {"value_kind": "bytes"})."""
from .init import reducefn as combinerfn  # noqa: F401  (host definition: what the declaration describes)

hbm_combinerfn = "fsum"


def init(arg=None):
    pass
