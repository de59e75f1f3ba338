"""k_combine splits its warps into stream warps (the pair stream and the shared-memory table) and table warps (the
global table and the long-key walks); every pair the stream warps cannot settle is handed over through a
shared-memory queue per table warp.  Streams that fill those queues faster than the table warps drain them, that
hand over nothing but long keys, launches whose slices are shorter than one trip, a global table that fills up and
is grown, and a checked sum that overflows must all give the oracle's result."""
import numpy as np
import pytest

import mrhbm_loader
import oracle as O
from test_gpu_combiner_and_wide_sums import kbytes, long_keys, records, shuffle_str, snapshot
from test_gpu_parity import check_vs_oracle_str, check_vs_oracle_u64, u64_records

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402

pytestmark = pytest.mark.gpu
N0 = 1 << 20  # the combiner runs from 2^20 pairs


def short_keys(idx, tag=b"s"):
    """distinct keys of 11 bytes (tag + 10 digits) from the numbers idx (< 10^10), vectorised"""
    a = np.zeros((idx.size, 11), dtype=np.uint8)
    a[:, 0] = tag[0]
    for d in range(10):
        a[:, 10 - d] = 48 + (idx // 10 ** d) % 10
    return a.view("S11").reshape(-1)


@pytest.mark.parametrize("kind", ["str27", "u64"])
def test_every_pair_misses(kind):
    """1.5 M keys drawn uniformly: past the first trips nearly every pair misses the shared table, so the stream
    warps hand over entries as fast as they read pairs and the queues stay full (the stream waits, nothing is lost)"""
    rng = np.random.default_rng(61)
    n, P, nk = 2 * N0 + 33, 15, 1_500_000
    idx = rng.integers(0, nk, n)
    vals = rng.integers(1, 1000, n)
    if kind == "u64":
        keys = O.gen_u64(17, 0, nk)[0][idx]
        with mrhbm.Ctx(mrhbm.KEY_U64, P, combiner=True) as ctx:
            m = ctx.map_begin(1)
            m.emit_batch(u64_records(keys, vals.astype(np.uint64)))
            m.commit()
            ctx.shuffle()
            assert ctx.stats()["ms_combine"] > 0 and ctx.result_info().pairs_recv < 0.8 * n
            check_vs_oracle_u64(ctx, keys, vals.astype(np.uint64), P)
        return
    recs = records(short_keys(rng.permutation(nk))[idx], vals.astype(np.uint32), 27)
    with shuffle_str([recs], 27, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        assert ctx.stats()["ms_combine"] > 0 and ctx.result_info().pairs_recv < 0.8 * n
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)


@pytest.mark.parametrize("mkb", [27, 59, 123])
def test_only_long_keys(mkb):
    """every key 13..mkb bytes: every pair is handed over by index and walked by a table warp"""
    rng = np.random.default_rng(62 + mkb)
    n, P, nk = N0 + 997, 15, 30_000
    kb = kbytes(mkb)
    keys = long_keys(np.arange(nk), rng.integers(13, mkb + 1, nk), kb)[rng.integers(0, nk, n)]
    recs = records(keys, rng.integers(1, 1000, n).astype(np.uint32), mkb)
    with shuffle_str([recs], mkb, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.pairs_recv < n // 4
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)


def test_slices_shorter_than_one_trip():
    """one launch per committed range: ranges of 1, 31, 500 and 20,000 pairs give every CTA a slice of at most one
    trip (most CTAs none at all), 130,000 pairs a slice just past one trip; with a range of 2^20 pairs they combine
    into one table"""
    rng = np.random.default_rng(63)
    P, vocab = 15, 4000
    words = np.concatenate([short_keys(np.arange(vocab // 2), b"w").astype("S28"),
                            long_keys(np.arange(vocab // 2), rng.integers(13, 28, vocab // 2), 28)])
    jobs = []
    for size in (N0, 1, 31, 500, 20_000, 130_000):
        jobs.append(records(words[rng.integers(0, vocab, size)], rng.integers(1, 100, size).astype(np.uint32), 27))
    with shuffle_str(jobs, 27, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        assert ctx.stats()["ms_combine"] > 0 and ctx.result_info().pairs_recv <= 6 * vocab
        check_vs_oracle_str(ctx, np.concatenate(jobs), P, O.PART_FNV_LUA)


def test_global_table_full_then_grown():
    """2^21 + 200,000 distinct short keys: more than the 2^21-entry global table takes.  The table warps raise the
    table-full flag and still end their drain; the shuffle grows the table and combines again"""
    rng = np.random.default_rng(64)
    P, nk = 15, (1 << 21) + 200_000
    idx = np.concatenate([np.arange(nk), rng.integers(0, nk, 300_000)])
    rng.shuffle(idx)
    recs = records(short_keys(rng.permutation(nk))[idx], rng.integers(1, 1000, idx.size).astype(np.uint32), 27)
    with shuffle_str([recs], 27, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.groups == nk and info.pairs_recv < 0.95 * idx.size
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)


def test_checked_sum_overflows():
    """values up to 2^26 (pairs x the largest value pass 2^32: checked adds), and a short and a long key whose sums
    pass 2^32 in the global table: the combine raises the overflow flag, every warp ends, and the raw pairs give the
    exact sums"""
    rng = np.random.default_rng(65)
    n, P, nk = N0 + 4093, 15, 200_000
    keys = short_keys(rng.integers(0, nk, n)).astype("S28")
    vals = rng.integers(1, 1000, n).astype(np.uint32)
    hot = {b"hot-short12": slice(0, None, 512), b"hot-long-key-14": slice(7, None, 512)}
    for k, sl in hot.items():
        keys[sl] = k
        vals[sl] = rng.integers(1 << 25, 1 << 26, vals[sl].size)
    recs = records(keys, vals, 27)
    with shuffle_str([recs], 27, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        assert ctx.stats()["ms_combine"] > 0 and ctx.result_info().pairs_recv == n  # the raw pairs went on
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)
        got = {k: v[0] for _, k, v in snapshot(ctx)}
    for k, sl in hot.items():
        assert got[k] == int(vals[sl].astype(np.uint64).sum()) > 0xFFFFFFFF
