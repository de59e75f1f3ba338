"""SortedWordCount's first-letter key-range partitionfn, declared as the device's range partitioner."""
from .init import NUM_REDUCERS, hbm_partitionfn, hbm_splitters, partitionfn  # noqa: F401


def init(arg=None):
    pass
