"""The map-side combiner streams trips of 1024 pairs per CTA, 32 consecutive pairs per warp, and walks long keys and
table probes in batches of 32 per warp.  Pair counts around those widths, streams in which every pair misses the
shared table or every key is long (the long-key queue fills within one trip), and values that force checked adds must
all give the oracle's result."""
import numpy as np
import pytest

import mrhbm_loader
import oracle as O
from test_gpu_combiner_and_wide_sums import long_keys, records, shuffle_str
from test_gpu_parity import check_vs_oracle_str, check_vs_oracle_u64, u64_records

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm, synth  # noqa: E402

pytestmark = pytest.mark.gpu
SEED = synth.SEED
N0 = 1 << 20  # the combiner runs from 2^20 pairs


@pytest.mark.parametrize("extra", [1, 31, 33, 63, 65, 1023])
def test_combiner_strings_around_warp_and_cta_trips(extra):
    n, P = N0 + extra, 15
    table = synth.zipf_table(1 << 16)
    recs = O.gen_zipf_rec32(SEED, 0, n, table).view(mrhbm.record_dtype(mrhbm.KEY_STR, 27)).reshape(-1)
    with shuffle_str([recs], 27, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.pairs_in == n and info.pairs_recv < n // 2
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)


@pytest.mark.parametrize("extra", [1, 31, 33, 63, 65, 1023])
def test_combiner_u64_around_warp_and_cta_trips(extra):
    n, P = N0 + extra, 15
    rng = np.random.default_rng(extra)
    keys = O.gen_u64(SEED, 0, 20_000)[0][rng.integers(0, 20_000, n)]
    vals = rng.integers(1, 1 << 40, n, dtype=np.uint64)
    with mrhbm.Ctx(mrhbm.KEY_U64, P, combiner=True) as ctx:
        m = ctx.map_begin(1)
        m.emit_batch(u64_records(keys, vals))
        m.commit()
        ctx.shuffle()
        assert ctx.stats()["ms_combine"] > 0 and ctx.result_info().pairs_recv < n // 2
        check_vs_oracle_u64(ctx, keys, vals, P)


def test_combiner_all_distinct_short_keys():
    """every key once: after the shared table has filled, every pair of every trip misses it"""
    n, P = N0 + 33, 15
    rng = np.random.default_rng(51)
    keys = np.array([b"d%010d" % i for i in rng.permutation(n)], dtype="S28")
    recs = records(keys, rng.integers(1, 1000, n).astype(np.uint32), 27)
    with shuffle_str([recs], 27, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        assert ctx.stats()["ms_combine"] > 0 and ctx.result_info().groups == n
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)


def test_combiner_only_long_keys():
    """every key 13..27 bytes: every pair of a trip goes to the long-key queue"""
    n, P, nk = N0 + 65, 15, 40_000
    rng = np.random.default_rng(52)
    keys = long_keys(np.arange(nk), rng.integers(13, 28, nk), 28)[rng.integers(0, nk, n)]
    recs = records(keys, rng.integers(1, 1000, n).astype(np.uint32), 27)
    with shuffle_str([recs], 27, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.pairs_recv < n // 4
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)


def test_combiner_checked_adds():
    """values up to 2^20 with short and long keys: pairs x the largest value pass 2^32, so the combine is re-run with
    checked adds (k_combine<32, true>); no sum of one key reaches 2^32, so the combined result stands"""
    n, P = N0 + 63, 15
    rng = np.random.default_rng(53)
    table = synth.zipf_table(1 << 16)
    recs = O.gen_zipf_rec32(SEED, 0, n, table).view(mrhbm.record_dtype(mrhbm.KEY_STR, 27)).reshape(-1)
    recs[::5]["key"] = long_keys(np.arange(3000), rng.integers(13, 28, 3000), 28)[rng.integers(0, 3000, recs[::5].size)]
    recs["val"] = rng.integers(0, 64, n)
    recs["val"][::101] = rng.integers(1 << 19, 1 << 20, recs[::101].size)
    with shuffle_str([recs], 27, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.pairs_recv < n // 4
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)
