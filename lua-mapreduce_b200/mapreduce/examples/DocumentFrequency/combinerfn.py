"""The DocumentFrequency combinerfn: the distinct values of a key, declared as the device's "distinct" combiner (needs
hbm = {"value_kind": "bytes"})."""
from .init import combinerfn, hbm_combinerfn  # noqa: F401


def init(arg=None):
    pass
