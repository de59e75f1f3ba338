"""The split stage (k_split_tma, planned by plan_split) branch by branch, at the edges between its branches.

Which path a shuffle's records take through the split is decided by data sizes: full and partial 40 KB tiles, the
static first tiles and the ticket counter of level 1 (one counter shared by the launches of every pool range), one
level or two (B <= 1024 or not), a partial last coarse region, the region and fine-bin capacities of the optimistic
layout (an overflow abandons the attempt and switches the ctx to the exact layout), the exact layout's direct scatter
below 2048 and above 2^20 bins, and the hash and range partitioner instances.  The placement model of
tests/test_gpu_sort_paths.py and the plan model of tests/test_split_plan.py build inputs that land on a chosen branch
at a chosen edge; every construction asserts that the models put it where it is meant to go (the CPU tests at the end
check the constructions alone), every shuffle is compared in full with exact per-key sums, and the path it took is
read from stats(): attempts, bins, sub-bins, launches (level 2 is one more launch than one level)."""
import math

import numpy as np
import pytest

import oracle as O
from test_gpu_sort_paths import (GOLD, cap_of, mix64_np, mrhbm, mulhi_np, pick_sub_bins, rb_of, str_candidates,
                                 u64_sub_hash_np, word_hash_np)
from test_split_plan import l2_ctas, plan_split

gpu = pytest.mark.gpu
TILE_BYTES = 40 * 1024
MKB = {16: None, 32: 27, 64: 59, 128: 123}
NOMINAL_SMS = 132  # H100 SXM: what the CPU checks of the constructions assume; the GPU cases read the device


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tile_records(rb):
    return TILE_BYTES // rb


def target_of(cap):
    return int(max(1.0, cap - 6.0 * math.sqrt(cap)))


# ---- placement (numpy forms) -------------------------------------------------------------------------------------------

def mulhash_pid_np(keys, P):
    return mulhi_np(keys * np.uint64(GOLD), P)


def fnv_lua_pid_np(slots, P):
    """O.part_fnv_lua of every NUL-free key slot of an 'S<kb>' array: the Lua FNV in doubles (53-bit products)"""
    kb = slots.dtype.itemsize
    b = slots.view(np.uint8).reshape(slots.size, kb)
    n = np.argmin(np.concatenate([b, np.zeros((slots.size, 1), np.uint8)], axis=1) != 0, axis=1)
    h = np.full(slots.size, 2166136261.0)
    for i in range(kb):
        prod = h * 16777619.0
        g = prod - np.floor(prod / 4294967296.0) * 4294967296.0
        g = (g.astype(np.uint64).astype(np.uint32) ^ b[:, i].astype(np.uint32)).astype(np.float64)
        h = np.where(i < n, g, h)
    return (h - np.floor(h / float(P)) * float(P)).astype(np.uint64)


def range_pid_np(keys, spl):
    return np.searchsorted(spl, keys, side="right").astype(np.uint64)


def even_splitters(P):
    return np.array([(i << 64) // P for i in range(1, P)], dtype=np.uint64)


def random_u64(rng, n):
    """n random u64 keys, every 8th repeating the key before it"""
    k = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    k[7::8] = k[6::8][:k[7::8].size]
    return k


def str_vocab(rng, n, kb, tag="v"):
    """n distinct stored key slots, every 8th repeating the slot before it"""
    s = str_candidates(rng, n, kb, tag)
    s[7::8] = s[6::8][:s[7::8].size]
    return s


def keys_for_bins(cand, bins, counts, rng):
    """counts[b] records of bin b for every b, from candidate keys `cand` whose bins are `bins` (distinct candidates,
    every 4th record of a bin repeating the one before it), in random order"""
    order = np.argsort(bins, kind="stable")
    sb = bins[order]
    have = np.bincount(sb.astype(np.int64), minlength=counts.size)
    assert (have[:counts.size] >= counts).all()
    start = np.concatenate([[0], np.cumsum(have)])[:-1]
    rank = np.arange(sb.size) - start[sb.astype(np.int64)]
    keep = rank < counts[sb.astype(np.int64)]
    out, rk = cand[order][keep], rank[keep]
    dup = np.nonzero(rk % 4 == 3)[0]
    out[dup] = out[dup - 1]
    return out[rng.permutation(out.size)]


# ---- running a shuffle and checking it ----------------------------------------------------------------------------------

def records(ctx_kind, mkb, keys, vals):
    recs = np.zeros(keys.size, dtype=mrhbm.record_dtype(ctx_kind, mkb or 27))
    recs["key"] = keys
    recs["val"] = vals
    return recs


def open_ctx(P, mkb=None, flags=0, part=None):
    if mkb is None:
        return mrhbm.Ctx(mrhbm.KEY_U64, P, part if part is not None else mrhbm.PART_MULHASH, flags=flags)
    return mrhbm.Ctx(mrhbm.KEY_STR, P, part if part is not None else mrhbm.PART_FNV_LUA, max_key_bytes=mkb, flags=flags)


def emit_job(ctx, job, keys, vals, mkb=None):
    m = ctx.map_begin(job)
    if keys.size:
        m.emit_batch(records(ctx.key_kind, mkb, keys, vals))
    m.commit()


def check(ctx, keys, vals, P, pid_of):
    """result_copy (keys, sums, part_off) against per-key sums over the input, every row in its key's partition,
    ascending inside a partition when the result says it is sorted, checksum parity, pairs received"""
    uk, inv = np.unique(keys, return_inverse=True)
    us = np.zeros(uk.size, dtype=np.uint64)
    np.add.at(us, inv, vals.astype(np.uint64))  # exact: every sum < 2^64
    info = ctx.result_info()
    assert info.pairs_recv == keys.size and info.groups == uk.size
    gk, gs, po = ctx.result_copy()
    po = po.astype(np.int64)
    assert po[0] == 0 and po[-1] == uk.size and (np.diff(po) >= 0).all()
    part = np.repeat(np.arange(P, dtype=np.uint64), np.diff(po))
    assert (pid_of(gk) == part).all()
    order = np.argsort(gk, kind="stable")
    assert (gk[order] == uk).all() and (gs[order] == us).all()
    if info.sorted:
        same = part[1:] == part[:-1]
        assert (gk[1:][same] > gk[:-1][same]).all()
    cin, cout = ctx.checksum_input(), ctx.checksum_result()
    assert cin[:3] == cout[:3] and cin[3] == keys.size and cout[3] == uk.size


def ex_launches(n):
    """launch_exscan over n counters with scratch: two kernels from 4 to 4096 blocks of 1024"""
    nb = -(-n // 1024)
    return 2 if 4 <= nb <= 4096 else 1


def fast_launches(ranges, sampled, two_level, B):
    """shuffle_fast on one GPU: the key sample and level 1 per non-empty range, level 2, the sort, the group-offset
    scan, the region totals"""
    return ranges * (2 if sampled else 1) + int(two_level) + 1 + ex_launches(B) + 1


def exact_launches(ranges, B, two_level, nbig=0):
    """shuffle_single_exact on one GPU: histogram per range, the bin scan, level 1 per range + level 2 or the
    scatter per range, the sort, k_big_bins, the group-offset scan"""
    return ranges + ex_launches(B) + ranges + int(two_level) + 1 + int(nbig > 0) + ex_launches(B)


def expect_stats(ctx, **want):
    st = ctx.stats()
    st["sorted"] = ctx.result_info().sorted
    assert {k: st[k] for k in want} == want, st


# ---- A. tile geometry, every record class ---------------------------------------------------------------------------

A_SIZES = ["1", "T-1", "T", "T+1", "GT-1", "GT", "GT+1", "3GT+17"]


def a_n(rb, size, sms):
    T, G = tile_records(rb), 2 * sms
    return {"1": 1, "T-1": T - 1, "T": T, "T+1": T + 1, "GT-1": G * T - 1, "GT": G * T, "GT+1": G * T + 1,
            "3GT+17": 3 * G * T + 17}[size]


def a_case(rb, size, layout, sms):
    """(n, P, S, plan): one range of n records, P = 256 (one level) or 1100 (two levels)"""
    n = a_n(rb, size, sms)
    cap = cap_of(rb)
    P = 256 if layout == "one" else 1100
    S = pick_sub_bins(n, cap, P)
    return n, P, S, plan_split([P * S], 0, cap, n, False)


def check_a_model(rb, size, layout, sms):
    n, P, S, pl = a_case(rb, size, layout, sms)
    T, U = tile_records(rb), -(-tile_records(rb) // 512)
    assert pl["levels"] == (1 if layout == "one" else 2)
    assert (rb == 16) == (T == 512 * U)  # only the 16-byte class fills its last record slot per thread
    full, part = divmod(n, T)
    tiles = full + (part > 0)
    assert {"1": tiles == 1 and part == 1, "T-1": tiles == 1 and part == T - 1, "T": (full, part) == (1, 0),
            "T+1": (full, part) == (1, 1), "GT-1": tiles == 2 * sms and part == T - 1,
            "GT": (full, part) == (2 * sms, 0), "GT+1": tiles == 2 * sms + 1 and part == 1,
            "3GT+17": tiles == 6 * sms + 1 and part == 17}[size]
    return n, P, S, pl


A_CASES = [(rb, size, layout) for rb in (16, 32, 64, 128) for size in A_SIZES for layout in ("one", "two")
           if not (layout == "one" and size == "3GT+17")]  # (more records than 1024 bins take at one level)


@gpu
@pytest.mark.parametrize("rb,size,layout", A_CASES)
def test_a_tile_geometry(rb, size, layout):
    """One range of 1, T - 1, T, T + 1, 2 SMs T - 1, 2 SMs T, 2 SMs T + 1 and 3 * 2 SMs T + 17 records: a lone
    partial tile, fewer tiles than CTAs, exactly one static tile per CTA, the first tile from the ticket counter, and
    many of them, through one level and through two."""
    sms = sm_count()
    n, P, S, pl = check_a_model(rb, size, layout, sms)
    rng = np.random.default_rng(n + rb)
    mkb = MKB[rb]
    if mkb is None:
        keys, pid_of = random_u64(rng, n), lambda k: mulhash_pid_np(k, P)
    else:
        keys, pid_of = str_vocab(rng, n, rb - 4), lambda k: fnv_lua_pid_np(k, P)
    vals = rng.integers(0, 1 << 32, n, dtype=np.uint64)
    with open_ctx(P, mkb) as ctx:
        emit_job(ctx, "a", keys, vals, mkb)
        ctx.shuffle()
        sampled = mkb is None and n >= 4096
        expect_stats(ctx, attempts=1, bins=P * S, sub_bins=S,
                     launches=fast_launches(1, sampled, pl["levels"] == 2, P * S))
        check(ctx, keys, vals, P, pid_of)


# ---- B. several ranges sharing one ticket counter -----------------------------------------------------------------------

def b_jobs(sms, rng):
    """(job, keys) in emit order: a job id seen before replaces that job, "aborted" is aborted"""
    T, G = tile_records(16), 2 * sms
    sizes = [("t-1", T - 1), ("big", 2 * G * T + 5 * T + 3), ("one", 1), ("empty", 0), ("r1", 3 * T + 11),
             ("aborted", 5 * T + 9), ("mid", G * T + 7), ("r2", T + 5), ("tail", 2 * T - 3), ("r1", T + 1),
             ("r2", 2 * T + 9)]
    return [(job, random_u64(rng, n)) for job, n in sizes]


def b_pool(jobs):
    """the committed ranges in pool order as (job, records, live): a replaced job's records stay in the pool, dead,
    until reset; the aborted job lies between two ranges that die, so it is part of a hole whether its room is
    given back or not"""
    pool = []
    for job, keys in jobs:
        if job == "aborted":
            continue
        pool = [(j, n, live and j != job) for j, n, live in pool] + [(job, keys.size, True)]
    return pool


def b_launch_ranges(pool):
    """live() merges adjacent committed ranges: the launches per stage are the runs of live records between dead
    ones"""
    runs, open_run = 0, False
    for _, n, live in pool:
        if n and live and not open_run:
            runs += 1
        if n:
            open_run = live
    return runs


@gpu
def test_b_ranges_share_the_ticket_counter():
    """Several committed jobs of mixed sizes (one record, T - 1, more than 2 SMs tiles, an empty job, a job that is
    replaced, an aborted job in the middle): the two replaced jobs leave dead holes in the pool, so level 1 runs
    three launches over the live runs between them, each after the first starting at a pool offset that is not tile
    aligned, all on one ticket counter that the last CTA of each launch resets.  A second shuffle of the
    same ctx gives the same result."""
    sms = sm_count()
    rng = np.random.default_rng(21)
    P = 1100
    final = {}
    jobs = b_jobs(sms, rng)
    ranges = b_launch_ranges(b_pool(jobs))
    with open_ctx(P) as ctx:
        for job, keys in jobs:
            vals = rng.integers(0, 1 << 32, keys.size, dtype=np.uint64)
            if job == "aborted":
                m = ctx.map_begin(job)
                m.emit_batch(records(ctx.key_kind, None, keys, vals))
                m.abort()
                continue
            emit_job(ctx, job, keys, vals)
            final[job] = (keys, vals)
        keys = np.concatenate([k for k, _ in final.values()])
        vals = np.concatenate([v for _, v in final.values()])
        S = pick_sub_bins(keys.size, 2048, P)
        assert ranges == 3 and P * S > 1024
        for _ in range(2):
            ctx.shuffle()
            expect_stats(ctx, attempts=1, bins=P * S, sub_bins=S, launches=fast_launches(ranges, True, True, P * S))
            check(ctx, keys, vals, P, lambda k: mulhash_pid_np(k, P))


# ---- C. one level / two levels -----------------------------------------------------------------------------------------

C_CASES = {  # name: (P, n): S = 1 at 1024 / 1025 partitions (level 2 at x = 1 and x > 1), S = 2 / 3 at 512
    "P1024": (1024, 1_000_000), "P1025_x1": (1025, 200_000), "P1025_xbig": (1025, 1_000_000),
    "S2_P512": (512, 1_500_000), "S3_P512_xbig": (512, 2_700_000)}


def check_c_model(name, sms):
    P, n = C_CASES[name]
    S = pick_sub_bins(n, 2048, P)
    pl = plan_split([P * S], 0, 2048, n, False)
    x = l2_ctas(pl["C1_local"], pl["sub_stride"], 1, 16, 2 * sms) if pl["levels"] == 2 else None
    if name.startswith("P1025"):
        assert (S, pl["levels"], pl["F"], pl["C1"], P - (pl["C1"] - 1) * pl["F"]) == (1, 2, 64, 17, 1)
    elif name == "P1024":
        assert (S, pl["levels"]) == (1, 1)
    elif name == "S2_P512":
        assert (S, pl["levels"]) == (2, 1)
    else:
        assert (S, pl["levels"], pl["F"], pl["C1"]) == (3, 2, 64, 24)
    if x is not None:
        assert (x == 1) == name.endswith("x1"), x
    return P, n, S, pl


@gpu
@pytest.mark.parametrize("name", list(C_CASES))
def test_c_one_level_or_two(name):
    """S = 1 with 1024 partitions (one level) against 1025 (two levels, F = 64, 17 regions, the last of one bin; level
    2 with one CTA per region and with several), and 1024 bins against 1536 at S > 1 (S = 3 takes more than 1.8 M
    records: regions of 16 or more tiles, always several CTAs each)."""
    P, n, S, pl = check_c_model(name, sm_count())
    rng = np.random.default_rng(n + P)
    keys, vals = random_u64(rng, n), rng.integers(0, 1 << 32, n, dtype=np.uint64)
    with open_ctx(P) as ctx:
        emit_job(ctx, "c", keys, vals)
        ctx.shuffle()
        expect_stats(ctx, attempts=1, bins=P * S, sub_bins=S, sorted=1,
                     launches=fast_launches(1, True, pl["levels"] == 2, P * S))
        check(ctx, keys, vals, P, lambda k: mulhash_pid_np(k, P))


# ---- D. capacity of the two-level optimistic layout ----------------------------------------------------------------------

D_S = 1148  # one partition, 1148 hash sub-bins: F = 64, 18 regions, the last of 60 bins
D_CASES = [(what, where) for what in ("region", "bin") for where in ("first", "last")]


def d_counts(rb, what, where, over):
    """records per fine bin: one region at exactly sub_stride (+ over) records with every bin <= cap, or one bin at
    exactly cap (+ over) inside a region under sub_stride; the first region / bin or the last (partial) ones.  The
    total stays N: the records come from a region in the middle."""
    cap = cap_of(rb)
    N = D_S * target_of(cap) - 50
    pl = plan_split([D_S], 0, cap, N, False)
    F, C1, ss = pl["F"], pl["C1"], pl["sub_stride"]
    counts = np.full(D_S, N // D_S, dtype=np.int64)
    counts[:N % D_S] += 1
    r = 0 if where == "first" else C1 - 1
    rbins = np.arange(r * F, min(D_S, (r + 1) * F))
    if what == "region":
        want = ss + over
        counts[rbins] = want // rbins.size
        counts[rbins[:want % rbins.size]] += 1
    else:
        counts[rbins[0] if where == "first" else D_S - 1] = cap + over
    donors = np.arange((C1 // 2) * F, (C1 // 2 + 1) * F)
    extra = int(counts.sum()) - N
    counts[donors] -= extra // donors.size
    counts[donors[:extra % donors.size]] -= 1
    assert counts.sum() == N
    return counts, N, pl


def check_d_model(rb, what, where, over):
    counts, N, pl = d_counts(rb, what, where, over)
    cap, F, C1, ss = cap_of(rb), pl["F"], pl["C1"], pl["sub_stride"]
    assert pick_sub_bins(N, cap) == D_S and (pl["levels"], F, C1, D_S - (C1 - 1) * F) == (2, 64, 18, 60)
    region = np.add.reduceat(counts, np.arange(0, D_S, F))
    r = 0 if where == "first" else C1 - 1
    others = np.delete(region, r)
    assert others.max() < ss and counts.min() > 0
    if what == "region":
        assert region[r] == ss + over and counts.max() <= cap  # a level-1 overflow alone
    else:
        b = r * F if where == "first" else D_S - 1
        assert counts[b] == cap + over and np.delete(counts, b).max() < cap and region[r] < ss  # level 2 alone
    return counts, N, pl


def d_keys(rb, counts, N, seed):
    rng = np.random.default_rng(seed)
    m = int(1.7 * N)
    if rb == 16:
        cand = np.unique(rng.integers(0, 1 << 64, m, dtype=np.uint64))
        bins = u64_sub_hash_np(cand, D_S)
    else:
        cand = str_candidates(rng, m, rb - 4, "d")
        bins = mulhi_np(word_hash_np(cand), D_S)
    keys = keys_for_bins(cand, bins, counts, rng)
    return keys, rng.integers(0, 1 << 32, N, dtype=np.uint64)


@gpu
@pytest.mark.parametrize("over", [0, 1])
@pytest.mark.parametrize("what,where", D_CASES)
@pytest.mark.parametrize("rb", [16, 32])
def test_d_capacity_at_the_limit_and_one_over(rb, what, where, over):
    """Hash sub-bins (u64 keys with F_FORCE_RUNS; 32-byte strings), one partition, two levels.  A region of exactly
    sub_stride records, or a fine bin of exactly cap, in the first region / bin or the last (partial) ones: one
    attempt.  One record more: the attempt is abandoned (ERRF_CAPACITY), the exact layout gives the same result, and
    the next shuffle of the ctx goes there directly."""
    counts, N, pl = check_d_model(rb, what, where, over)
    keys, vals = d_keys(rb, counts, N, 100 * rb + 10 * D_CASES.index((what, where)) + over)
    mkb = MKB[rb]
    nbig = int((counts > cap_of(rb)).sum())
    fast = fast_launches(1, False, True, D_S)
    exact = exact_launches(1, D_S, False, nbig)
    with open_ctx(1, mkb, mrhbm.F_FORCE_RUNS) as ctx:
        emit_job(ctx, "d", keys, vals, mkb)
        ctx.shuffle()
        if over:
            expect_stats(ctx, attempts=2, bins=D_S, sub_bins=D_S, big_bins=nbig, sorted=0, launches=fast + exact)
        else:
            expect_stats(ctx, attempts=1, bins=D_S, sub_bins=D_S, big_bins=0, sorted=0, launches=fast)
        check(ctx, keys, vals, 1, lambda k: np.zeros(k.size, dtype=np.uint64))
        ctx.shuffle()
        expect_stats(ctx, attempts=1, sub_bins=D_S, launches=exact if over else fast)
        check(ctx, keys, vals, 1, lambda k: np.zeros(k.size, dtype=np.uint64))


def d_ordered_keys(seed=5):
    """u64 keys spread evenly over [0, 2^64) (a flat sample), except key-ordered sub-bin 5 of D_S, which holds cap + 1"""
    rng = np.random.default_rng(seed)
    N = D_S * target_of(2048) - 50
    step = (1 << 64) // N
    keys = np.arange(N, dtype=np.uint64) * np.uint64(step) + rng.integers(0, step, N, dtype=np.uint64)
    lo, hi = -(-(5 << 64) // D_S), -(-(6 << 64) // D_S)
    keys = keys[(keys < np.uint64(lo)) | (keys >= np.uint64(hi))]
    keys = rng.permutation(keys)[:N - 2049]
    w = (hi - lo) // 2049
    hot = np.array([lo + i * w for i in range(2049)], dtype=np.uint64)
    keys = np.concatenate([keys, hot])
    return keys[rng.permutation(keys.size)]


def check_d_ordered_model(keys):
    S = pick_sub_bins(keys.size, 2048)
    sub = mulhi_np(keys, S)
    h = np.bincount((keys >> np.uint64(56)).astype(np.int64), minlength=256)
    mean = keys.size / 256.0
    assert S == D_S and h.max() <= mean * 1.08 + 5.0 * math.sqrt(mean) + 2.0  # the sample asks for key order
    c = np.bincount(sub.astype(np.int64), minlength=S)
    assert c[5] == 2049 and np.delete(c, 5).max() <= 2048
    assert np.bincount(u64_sub_hash_np(keys, S).astype(np.int64)).max() <= 2048  # hash sub-bins: nothing over
    return S


@gpu
def test_d_key_ordered_overflow_gives_up_key_order():
    """A key-ordered u64 sub-bin of cap + 1 records: the optimistic attempt overflows, the exact layout takes hash
    sub-bins, and later shuffles of the ctx stay unordered."""
    keys = d_ordered_keys()
    S = check_d_ordered_model(keys)
    vals = np.random.default_rng(6).integers(0, 1 << 32, keys.size, dtype=np.uint64)
    with open_ctx(1) as ctx:
        emit_job(ctx, "o", keys, vals)
        ctx.shuffle()
        expect_stats(ctx, attempts=2, sub_bins=S, big_bins=0, sorted=0,
                     launches=fast_launches(1, True, True, S) + exact_launches(1, S, False))
        check(ctx, keys, vals, 1, lambda k: np.zeros(k.size, dtype=np.uint64))
        ctx.shuffle()
        expect_stats(ctx, attempts=1, sub_bins=S, sorted=0, launches=exact_launches(1, S, False))
        check(ctx, keys, vals, 1, lambda k: np.zeros(k.size, dtype=np.uint64))


# ---- E. the exact layout ------------------------------------------------------------------------------------------------

E_CASES = {  # name: (P, n, shape)
    "B2047": (2047, 1_000_000, "hole"), "B2048": (2048, 1_000_000, "hole"), "B2049": (2049, 1_000_000, "hole"),
    "B3000": (3000, 2_000_000, "hole"), "B3000_ends": (3000, 150_000, "ends")}


def e_keys(P, n, shape, seed):
    """n u64 keys over P partitions (S = 1); "hole": partition 1 (inside the first region) gets none; "ends": only
    the first and the last coarse region get keys"""
    rng = np.random.default_rng(seed)
    F = plan_split([P], 0, 2048, 0, True)["F"] if P >= 2048 else 1
    keys = np.zeros(0, dtype=np.uint64)
    while keys.size < n:
        c = random_u64(rng, 2 * n)
        pid = mulhash_pid_np(c, P)
        ok = pid != 1 if shape == "hole" else (pid < F) | (pid >= np.uint64((P - 1) // F * F))
        keys = np.concatenate([keys, c[ok]])
    return keys[:n]


def check_e_model(name, keys):
    P, n, shape = E_CASES[name]
    assert keys.size == n and pick_sub_bins(n, 2048, P) == 1
    pl = plan_split([P], 0, 2048, 0, True)
    pid = mulhash_pid_np(keys, P).astype(np.int64)
    c = np.bincount(pid, minlength=P)
    assert c.max() <= 2048
    if pl is None:
        assert P == 2047
        return None
    F, C1 = pl["F"], pl["C1"]
    assert (P - (C1 - 1) * F < F) == (name != "B2048")  # a partial last region, except at 2048 = 32 x 64 bins
    region = np.add.reduceat(c, np.arange(0, P, F))
    if shape == "hole":
        assert c[1] == 0 and region.min() > 0
    else:
        assert region[0] > 0 and region[-1] > 0 and (region[1:-1] == 0).all() and C1 > 40
    return pl


@gpu
@pytest.mark.parametrize("name", list(E_CASES))
def test_e_exact_layout_at_2048_bins(name):
    """F_NO_OPTIMISTIC: 2047 bins (the direct scatter), 2048, 2049 and 3000 (the two-level split, regions read from
    the bin offsets, a partial last region), an empty fine bin inside a non-empty region, and only the first and the
    last of 47 regions holding records."""
    P, n, shape = E_CASES[name]
    keys = e_keys(P, n, shape, P + n)
    pl = check_e_model(name, keys)
    vals = np.random.default_rng(P).integers(0, 1 << 32, n, dtype=np.uint64)
    with open_ctx(P, flags=mrhbm.F_NO_OPTIMISTIC) as ctx:
        emit_job(ctx, "e", keys, vals)
        ctx.shuffle()
        expect_stats(ctx, attempts=1, bins=P, sub_bins=1, big_bins=0,
                     launches=exact_launches(1, P, pl is not None))
        check(ctx, keys, vals, P, lambda k: mulhash_pid_np(k, P))


E_BIG = [(1 << 20, 0), (1 << 20, 1), ((1 << 20) + 1, 0), ((1 << 20) + 1, 1)]


@gpu
@pytest.mark.parametrize("P,no_opt", E_BIG)
def test_e_small_bins_at_2_pow_20_bins(P, no_opt):
    """F_SMALL_BINS (96 slots per bin), S = 1: 2^20 bins is the largest plan two levels reach (F = C1 = 1024), in
    both layouts; at 2^20 + 1 the optimistic planner refuses before counting an attempt and the exact layout
    scatters."""
    n = 3_000_000
    assert pick_sub_bins(n, 96, P) == 1
    opt = plan_split([P], 0, 96, n, False)
    ex = plan_split([P], 0, 96, 0, True)
    if P == 1 << 20:
        assert (opt["F"], opt["C1"], ex["F"], ex["C1"]) == (1024, 1024, 1024, 1024)
    else:
        assert opt is None and ex is None
    rng = np.random.default_rng(P + no_opt)
    keys, vals = random_u64(rng, n), rng.integers(0, 1 << 32, n, dtype=np.uint64)
    flags = mrhbm.F_SMALL_BINS | (mrhbm.F_NO_OPTIMISTIC if no_opt else 0)
    with open_ctx(P, flags=flags) as ctx:
        emit_job(ctx, "e", keys, vals)
        ctx.shuffle()
        if opt is not None and not no_opt:
            launches = fast_launches(1, True, True, P)
        else:  # (the optimistic layout samples the keys before its planner refuses)
            launches = exact_launches(1, P, ex is not None) + int(not no_opt)
        expect_stats(ctx, attempts=1, bins=P, sub_bins=1, big_bins=0, launches=launches)
        check(ctx, keys, vals, P, lambda k: mulhash_pid_np(k, P))


# ---- F. range partitioner instances -------------------------------------------------------------------------------------

F_CASES = {"one": (600, 500_000, 0), "two": (1100, 1_500_000, 0), "exact_two": (2100, 1_500_000, 1)}


@gpu
@pytest.mark.parametrize("name", list(F_CASES))
def test_f_range_partitioner(name):
    """PART_RANGE with caller-given splitters through one level, two levels and the exact two-level split: every
    key in partition bisect_right(splitters, key), one global key order."""
    P, n, no_opt = F_CASES[name]
    S = pick_sub_bins(n, 2048, P)
    pl = plan_split([P * S], 0, 2048, n, bool(no_opt))
    assert pl["levels"] == (1 if name == "one" else 2)
    spl = even_splitters(P)
    rng = np.random.default_rng(P)
    keys, vals = random_u64(rng, n), rng.integers(0, 1 << 32, n, dtype=np.uint64)
    with open_ctx(P, flags=mrhbm.F_NO_OPTIMISTIC if no_opt else 0, part=mrhbm.PART_RANGE) as ctx:
        ctx.set_splitters([int(s) for s in spl])
        emit_job(ctx, "f", keys, vals)
        ctx.shuffle()
        launches = exact_launches(1, P * S, True) if no_opt else fast_launches(1, True, pl["levels"] == 2, P * S)
        expect_stats(ctx, attempts=1, bins=P * S, sub_bins=S, sorted=1, launches=launches)
        check(ctx, keys, vals, P, lambda k: range_pid_np(k, spl))
        gk = ctx.result_copy()[0]
        assert (gk[1:] > gk[:-1]).all()  # the partitions in order: one global key order


# ---- the constructions (no GPU) ----------------------------------------------------------------------------------------

def test_model_fnv_lua_pid_matches_the_oracle():
    rng = np.random.default_rng(8)
    for kb in (28, 60, 124):
        slots = str_candidates(rng, 300, kb, "q")
        for P in (1, 15, 1100, (1 << 20) + 1):
            got = fnv_lua_pid_np(slots, P)
            assert [int(g) for g in got] == [O.part_fnv_lua(bytes(s), P) for s in slots.tolist()]


def test_model_mulhash_and_range_pids():
    rng = np.random.default_rng(9)
    keys = rng.integers(0, 1 << 64, 300, dtype=np.uint64)
    for P in (1, 1025, 1 << 20):
        assert [int(p) for p in mulhash_pid_np(keys, P)] == [O.part_mulhash(int(k), P) for k in keys.tolist()]
    import bisect
    spl = even_splitters(600)
    probe = np.concatenate([keys, spl, spl - np.uint64(1)])
    want = [bisect.bisect_right([int(s) for s in spl], int(k)) for k in probe.tolist()]
    assert [int(p) for p in range_pid_np(probe, spl)] == want


def test_model_places_every_construction():
    """the constructions the GPU cases run land where they are meant to (the GPU cases repeat these checks)"""
    for rb, size, layout in A_CASES:
        check_a_model(rb, size, layout, NOMINAL_SMS)
    for name in C_CASES:
        check_c_model(name, NOMINAL_SMS)
    for rb in (16, 32):
        for what, where in D_CASES:
            for over in (0, 1):
                counts, N, pl = check_d_model(rb, what, where, over)
        counts, N, _ = check_d_model(rb, "bin", "last", 1)
        keys, _ = d_keys(rb, counts, N, 1)
        bins = u64_sub_hash_np(keys, D_S) if rb == 16 else mulhi_np(word_hash_np(keys), D_S)
        assert (np.bincount(bins.astype(np.int64), minlength=D_S) == counts).all()
    check_d_ordered_model(d_ordered_keys())
    for name, (P, n, shape) in E_CASES.items():
        check_e_model(name, e_keys(P, n, shape, P + n))
    pool = b_pool(b_jobs(NOMINAL_SMS, np.random.default_rng(0)))
    T = tile_records(16)
    assert pool[1][1] > 2 * NOMINAL_SMS * T and b_launch_ranges(pool) == 3
    starts = np.cumsum([0] + [n for _, n, _ in pool])[:-1]
    assert (starts[1:] % T != 0).all()  # no range after the first starts on a tile edge
    assert [j for j, n, live in pool if n and not live] == ["r1", "r2"]
