"""WordCount with a key-range partitionfn: partition k takes the words whose first byte is the k-th letter of
"a".."z" (bytes below "a" go to the first partition, bytes above "z" to the last).  Because the partitions are key
ranges, finalfn sees every word in one ascending key order, and result file k holds the k-th slice of the key space.

The partitionfn is a plain function; hbm_partitionfn = "range" with the 25 splitters "b".."z" declares the same key
ranges so that the shuffle evaluates it on the device (configure checks that the two agree)."""
from ..WordCount.init import FILES, mapfn, reducefn, taskfn  # noqa: F401

NUM_REDUCERS = 26
hbm_partitionfn = "range"
hbm_splitters = [chr(c) for c in range(ord("b"), ord("z") + 1)]
hbm_reducefn = "sum"
RESULT = []  # (word, count) in the order finalfn sees them


def init(arg):
    pass


def partitionfn(key):
    first = key[0] if key else 0
    return min(max(first - ord("a"), 0), NUM_REDUCERS - 1)


combinerfn = reducefn


def finalfn(pairs_iterator):
    for key, values in pairs_iterator:
        RESULT.append((key, values[0]))
    return False  # keep the result partitions: result.P<kk> holds the kk-th slice of the key space


associative_reducer = True
commutative_reducer = True
idempotent_reducer = True
