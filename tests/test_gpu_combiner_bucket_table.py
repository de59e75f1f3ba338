"""The combiner's global table is made of 32-byte buckets of two entries, sized to the keys (a bucket count that is
not a power of two), with a long-entry area sized on its own.  A table filled to 0.78 load (long bucket chains that
wrap at the last bucket), more keys than it holds (the table grows and a later shuffle on the same ctx starts at the
grown size), u64 keys, more distinct long keys than the long area holds, and checked sums at the largest value a
combined record carries must all give the oracle's result."""
import numpy as np
import pytest

import mrhbm_loader
import oracle as O
from test_gpu_combiner_and_wide_sums import kbytes, long_keys, records, snapshot
from test_gpu_combiner_warp_roles import short_keys
from test_gpu_parity import check_vs_oracle_str, check_vs_oracle_u64, u64_records

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402

pytestmark = pytest.mark.gpu
P = 15
DEFAULT_ENTRIES = 2 * 819200  # GtabLayout::sized(rb, 0).nshort()
MAX_COMBINED_SUM = 0xFFFFFFEF  # kMaxCombinedSum


def every_key_once(rng, nk, extra):
    """indices 0..nk-1 each at least once, plus `extra` random repeats, shuffled"""
    idx = np.concatenate([np.arange(nk), rng.integers(0, nk, extra)])
    rng.shuffle(idx)
    return idx


def shuffle_twice(ctx, emit):
    """the same job shuffled twice on one ctx (reset in between): the launch counts of both shuffles"""
    launches = []
    for _ in range(2):
        ctx.reset()
        m = ctx.map_begin(1)
        emit(m)
        m.commit()
        ctx.shuffle()
        launches.append(ctx.stats()["launches"])
    return launches


def test_table_at_high_load():
    """0.78 of the default table's entries as distinct short keys: the table does not grow (both shuffles launch the
    same kernels) and its long bucket chains, some wrapping past the last bucket, lose nothing"""
    rng = np.random.default_rng(71)
    nk = int(0.78 * DEFAULT_ENTRIES)
    idx = every_key_once(rng, nk, 250_000)
    recs = records(short_keys(rng.permutation(nk))[idx], rng.integers(1, 1000, idx.size).astype(np.uint32), 27)
    with mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=27, combiner=True) as ctx:
        first, second = shuffle_twice(ctx, lambda m: m.emit_batch(recs))
        assert first == second
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.groups == nk and info.pairs_recv < idx.size
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)


def test_table_grows_and_stays_grown():
    """1.8 M distinct short keys, more than the default table takes: the first shuffle fills it, grows it and combines
    again; the next shuffle on the same ctx starts at the grown size (one combine and one compaction fewer)"""
    rng = np.random.default_rng(72)
    nk = 1_800_000
    idx = every_key_once(rng, nk, 200_000)
    recs = records(short_keys(rng.permutation(nk))[idx], rng.integers(1, 1000, idx.size).astype(np.uint32), 27)
    with mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=27, combiner=True) as ctx:
        first, second = shuffle_twice(ctx, lambda m: m.emit_batch(recs))
        assert second == first - 2
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.groups == nk and info.pairs_recv < idx.size
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)


@pytest.mark.parametrize("nk", [1_250_000, 1_800_000])
def test_u64_keys(nk):
    """u64 keys ({key, u64 state} entries) in the same buckets: at 0.76 load, and past the default table"""
    rng = np.random.default_rng(73)
    idx = every_key_once(rng, nk, 200_000)
    keys = O.gen_u64(29, 0, nk)[0][idx]
    vals = rng.integers(1, 1 << 40, idx.size).astype(np.uint64)
    with mrhbm.Ctx(mrhbm.KEY_U64, P, combiner=True) as ctx:
        m = ctx.map_begin(1)
        m.emit_batch(u64_records(keys, vals))
        m.commit()
        ctx.shuffle()
        assert ctx.stats()["ms_combine"] > 0 and ctx.result_info().pairs_recv < idx.size
        check_vs_oracle_u64(ctx, keys, vals, P)


@pytest.mark.parametrize("mkb", [27, 59, 123])
def test_many_distinct_long_keys(mkb):
    """60,000 distinct keys of 13..mkb bytes, more than the 2^15 long entries: the long area fills, grows, and a
    later shuffle starts at the grown size"""
    rng = np.random.default_rng(74 + mkb)
    nk = 60_000
    idx = every_key_once(rng, nk, (1 << 20) - nk + 1000)
    keys = long_keys(np.arange(nk), rng.integers(13, mkb + 1, nk), kbytes(mkb))[idx]
    recs = records(keys, rng.integers(1, 1000, idx.size).astype(np.uint32), mkb)
    with mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=mkb, combiner=True) as ctx:
        first, second = shuffle_twice(ctx, lambda m: m.emit_batch(recs))
        assert second < first
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.groups == nk and info.pairs_recv < idx.size
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)


@pytest.mark.parametrize("off", [-1, 1])
def test_checked_sums_at_the_limit(off):
    """a short and a long key whose 64 values of about 2^26 sum to kMaxCombinedSum + off: pairs x the largest value
    pass 2^32, so the adds are checked.  Just below the limit the combined records carry the sums; just above it the
    shuffle hands on the raw pairs.  Either way the sums are exact"""
    rng = np.random.default_rng(75)
    n, nk = (1 << 20) + 4093, 200_000
    keys = short_keys(rng.integers(0, nk, n)).astype("S28")
    vals = rng.integers(1, 1000, n).astype(np.uint32)
    target = MAX_COMBINED_SUM + off
    hot = {b"hot-short12": slice(3, 64 * 4099, 4099), b"hot-long-key-14": slice(11, 64 * 4099, 4099)}
    for k, sl in hot.items():
        keys[sl] = k
        v = np.full(64, 67_108_863, dtype=np.uint64)
        v[-1] = target - int(v[:-1].sum())
        vals[sl] = v.astype(np.uint32)
    recs = records(keys, vals, 27)
    with mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=27, combiner=True) as ctx:
        m = ctx.map_begin(1)
        m.emit_batch(recs)
        m.commit()
        ctx.shuffle()
        pairs_recv = ctx.result_info().pairs_recv
        assert ctx.stats()["ms_combine"] > 0 and (pairs_recv == n if off > 0 else pairs_recv < n // 2)
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)
        got = {k: v[0] for _, k, v in snapshot(ctx)}
    for k in hot:
        assert got[k] == target
