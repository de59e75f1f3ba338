"""The distinct reducer (MRHBM_RED_DISTINCT) branch by branch, at the edges between its branches.

Before the shuffle, collect_sources runs the distinct set (mrhbm_distinct.cu) over all committed pairs: every live
ledger range is cut into tiles of 256 records, each record joins a linear-probing table of max(1024, pow2 >= 2n) entries
at the home slot fingerprint & (T - 1), and only when some pair repeats are the first copies scattered to one scratch
source (one more launch); otherwise the pool ranges stay the sources.  After the group-only sort, k_value_order orders
each bin of at most cap rows in one CTA (thread t holds rows [t kPer, (t + 1) kPer), a group head needs the previous
thread's last row, a bin whose keys all have one row skips the sort, else a bitonic sort over np = pow2 >= m slots by
(group, 8-byte big-endian prefix), the arena bytes compared only on a prefix tie).  An oversized bin (exact layout only)
has its cap-row chunks ordered the same way by a (nbig, 64) grid, CTA y taking chunks y, y + 64, ...; then k_value_merge
merges them in passes of width cap, 2 cap, ... below the bin's own row count, alternating between the output rows and
the scratch, with a copy-back when the bin's pass count is odd.

A model (pure Python, P = 1 so that bin = sub-bin and the exact layout's bin offset is the scan of the bin counts)
restates the thread rows, heads, skip and np of a bin, the chunks and their CTAs, the merge passes, parity and run
pairs of each thread, the set's size, tiles and home slots, and the pair fingerprint (tied to the header's by a host
driver).  The constructions below place key groups on chosen rows of chosen bins; the CPU tests check that each lands
where it claims, and the GPU tests compare every shuffle in full with sorted(set(values)) per key."""
import itertools
import math

import numpy as np
import pytest

import mrhbm_loader
from test_fsum_combiner_host import run_native
from test_gpu_distinct_reducer import check, want_groups
from test_gpu_fsum_combiner_paths import fp_step, key_words, place, slot_words
from test_gpu_fsum_reducer_paths import Kind as FsumKind
from test_gpu_fsum_reducer_paths import Layout, check_keys, groups_with, merge_runs
from test_gpu_sort_paths import cap_of, expect_stats, mix64, mulhi_np, pick_sub_bins, str_candidates, word_hash_np

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402

gpu = pytest.mark.gpu
M64 = (1 << 64) - 1
ORDER_THREADS = 256    # kOrderThreads
CHUNK_CTAS = 64        # kChunkCtas: chunks of one oversized bin ordered at a time
MERGE_THREADS = 1024   # kMergeThreads: one CTA per oversized bin
TILE = 256             # kDistinctTile
STAGE = 4 << 20        # value bytes staged next to the records
NO_OPT = mrhbm.F_NO_OPTIMISTIC
KINDS = ["u64", "str27", "str59", "str123", "u64-small"]
BIG_KINDS = ["u64", "str27", "str59", "str123"]


# ---- the placement model ---------------------------------------------------------------------------------------------

class Kind(FsumKind):
    """FsumKind's key classes and key placement (kPer is the same 32 KB / RB / 256) on a distinct-reducer ctx"""

    def keys(self, lay, seed):
        """FsumKind.keys; string keys drawn in batches of candidates (the bins of E hold thousands of keys at S > 200)"""
        if self.mkb is None:
            return super().keys(lay, seed)
        out = {}
        for s, g in lay.bins.items():
            rng = np.random.default_rng([seed, s])
            got = {}
            while len(got) < len(g):
                c = str_candidates(rng, 1 << 15, self.rb - 4, "r")
                for k in c[mulhi_np(word_hash_np(c), lay.S) == np.uint64(s)].tolist():
                    got.setdefault(k, None)
            out[s] = sorted(list(got)[:len(g)])
        return out

    def ctx(self, flags=NO_OPT, combiner=mrhbm.COMBINE_NONE):
        kind = mrhbm.KEY_U64 if self.mkb is None else mrhbm.KEY_STR
        return mrhbm.Ctx(kind, 1, max_key_bytes=self.mkb or 27, device=0, reducer=mrhbm.RED_DISTINCT,
                         flags=mrhbm.F_BYTE_VALUES | self.flags | flags, combiner=combiner)


def next_pow2(m):
    return 1 << (m - 1).bit_length() if m > 1 else 1


def order_model(sizes, per):
    """k_value_order on a bin (or chunk) whose key groups have `sizes` rows: the first row of every thread past 0 (its
    head needs prev), the heads, whether the sort is skipped, np"""
    m = sum(sizes)
    starts = [0] + list(itertools.accumulate(sizes))[:-1]
    return dict(edges=list(range(per, m, per)), heads=starts, skip=len(sizes) == m, np=next_pow2(m))


def crossed(sizes, per):
    """per group: (first row, rows, thread edges strictly inside it)"""
    out, a = [], 0
    for L in sizes:
        out.append((a, L, (a + L - 1) // per - a // per))
        a += L
    return out


def sorted_by_chance(a, L, per):
    """the chance that a group of L random values at row a, sorted as separate pieces cut at each thread edge, still
    comes out in order: prod(piece!) / L!"""
    cuts = [a] + [e for e in range((a // per + 1) * per, a + L, per)] + [a + L]
    p = 1.0
    for x, y in zip(cuts, cuts[1:]):
        p *= math.factorial(y - x)
    return p / math.factorial(L)


def chunk_ctas(n, cap):
    """CTA y (and round) of every cap-row chunk of an oversized bin of n rows"""
    return [(c % CHUNK_CTAS, c // CHUNK_CTAS) for c in range(-(-n // cap))]


def merge_model(n, cap):
    """k_value_merge on a bin of n rows: the pass widths, whether the copy-back runs, the output rows per thread"""
    ws, w = [], cap
    while w < n:
        ws.append(w)
        w <<= 1
    return ws, len(ws) % 2 == 1, -(-n // MERGE_THREADS)


def thread_pairs(n, w, per, t):
    """the run pairs (p0, la, lb) thread t's output positions fall in during the pass of width w"""
    out = []
    for p0 in sorted({k // (2 * w) * 2 * w for k in range(t * per, min(n, (t + 1) * per))}):
        la = min(w, n - p0)
        out.append((p0, la, min(w, n - p0 - la)))
    return out


def table_entries(n):
    T = 1024
    while T < 2 * n:
        T <<= 1
    return T


def set_tiles(lengths):
    """(range, first record of the tile in its range, records) of every tile of the live ranges"""
    return [(k, j, min(TILE, ln - j)) for k, ln in enumerate(lengths) for j in range(0, ln, TILE)]


def pair_fingerprint(key, rb, val):
    """pair_fingerprint<RB> of mrhbm_job_tiles.cuh: fp_step over the key slot's word pairs, then the value's little-endian
    word pairs, seeded with the value length; mix64; ~0 taken to 0"""
    return fingerprint_words(slot_words(key, rb), rb, val)


def fingerprint_words(words, rb, val):
    kw = key_words(rb)
    h = fp_step(0x5851F42D4C957F2D, len(val))
    for i in range(0, kw, 2):
        h = fp_step(h, words[i] | (words[i + 1] << 32 if i + 1 < kw else 0))
    b = bytes(val) + b"\0" * (-len(val) % 8)
    for i in range(0, len(b), 8):
        h = fp_step(h, int.from_bytes(b[i:i + 8], "little"))
    h = mix64(h)
    return 0 if h == M64 else h


# ---- values, emission, one shuffle -----------------------------------------------------------------------------------

def rand_values(rng, n, lo=6, hi=20):
    lens = rng.integers(lo, hi + 1, n)
    raw = rng.integers(0, 256, (n, hi), dtype=np.uint8)
    return [raw[i, :lens[i]].tobytes() for i in range(n)]


def layout_pairs(kind, lay, seed):
    """the layout's rows in order, each group's rows with distinct random values"""
    keys = kind.keys(lay, seed)
    vals = rand_values(np.random.default_rng([seed, 1]), lay.N)
    pairs, i = [], 0
    for s in lay.bins:
        for k, c in zip(keys[s], lay.bins[s]):
            pairs += [(k, v) for v in vals[i:i + c]]
            i += c
    return pairs


def batch(ctx, m, pairs):
    recs = np.zeros(len(pairs), dtype=mrhbm.record_dtype(ctx.key_kind, ctx.cfg.max_key_bytes))
    ks = [k for k, _ in pairs]
    recs["key"] = np.array(ks, dtype=np.uint64) if ctx.key_kind == mrhbm.KEY_U64 else ks
    off = np.zeros(len(pairs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(v) for _, v in pairs])
    m.emit_batch_values(recs, b"".join(v for _, v in pairs), off)


def emit_job(ctx, pairs, job="job0", seed=None):
    """the pairs as one batch (in a random order when seed is given)"""
    if seed is not None:
        pairs = [pairs[i] for i in np.random.default_rng(seed).permutation(len(pairs))]
    m = ctx.map_begin(job)
    batch(ctx, m, pairs)
    m.commit()


def bins_of(kind, pairs, cap):
    """the sub-bin counts of the distinct pairs (P = 1): S and the oversized bins"""
    d = set(pairs)
    S = pick_sub_bins(len(d), cap)
    cnt = [0] * S
    for k, _ in d:
        cnt[kind.sub(k, S)] += 1
    return S, sum(1 for c in cnt if c > cap)


def run_layout(kind, lay, seed, flags=NO_OPT, attempts=1):
    """one shuffle of the layout, checked in full; its rows and stats"""
    pairs = layout_pairs(kind, lay, seed)
    with kind.ctx(flags) as ctx:
        emit_job(ctx, pairs, seed=seed)
        rows, _ = check(ctx, want_groups([pairs]))
        expect_stats(ctx, attempts=attempts, bins=lay.S, sub_bins=lay.S, big_bins=len(lay.big()))
        return rows, ctx.stats()


def check_layout(kind, lay, seed):
    check_keys(kind, lay, kind.keys(lay, seed))
    pairs = layout_pairs(kind, lay, seed)
    assert len(set(pairs)) == lay.N  # every row survives the set


# ---- A. whole bins ---------------------------------------------------------------------------------------------------

def fill(n, sizes):
    out = []
    for c in itertools.cycle(sizes):
        if sum(out) >= n:
            return out
        out.append(min(c, n - sum(out)))


def a_layout(kind, plus=0):
    """bins of exactly cap rows (cap + 1 with plus): cap distinct keys, one key, pairs, groups on every thread edge and
    the same shifted by a row; bins of 2^k and 2^k + 1 rows (the largest 2^k below cap: np doubles)"""
    cap, per = kind.cap, kind.per
    half = next_pow2(cap) // 2
    rng = np.random.default_rng(21)
    g = {0: [1] * cap, 1: [cap], 2: [2] * (cap // 2), 3: fill(cap, [per]), 4: [1] + fill(cap - 1, [per])}
    bins = {s: gs[:-1] + [gs[-1] + plus] for s, gs in g.items()}
    bins[5] = groups_with(half, [], rng)
    bins[6] = groups_with(half + 1, [], rng)
    return Layout(cap, bins)


def check_a_model(kind, plus):
    lay = a_layout(kind, plus)
    cap, per = kind.cap, kind.per
    assert lay.S > 6 and [lay.count[s] for s in range(5)] == [cap + plus] * 5
    half = lay.count[5]
    assert half < cap <= 2 * half and half & (half - 1) == 0 and lay.count[6] == half + 1
    o5, o6 = order_model(lay.bins[5], per), order_model(lay.bins[6], per)
    assert o6["np"] == 2 * o5["np"] == 2 * half
    if not plus:
        assert lay.big() == [] and order_model(lay.bins[0], per)["skip"]
        assert not any(order_model(lay.bins[s], per)["skip"] for s in (1, 2))
        assert all(a % per == 0 for a in lay.starts(3))
        assert per == 1 or all(a % per == 1 for a in lay.starts(4)[1:])
    else:
        assert lay.big() == [0, 1, 2, 3, 4]
        assert merge_model(cap + 1, cap)[:2] == ([cap], True)
    return lay


def one_row_layout(kind):
    return Layout(kind.cap, {0: [1]})


@gpu
@pytest.mark.parametrize("plus", [0, 1], ids=["cap", "cap+1"])
@pytest.mark.parametrize("flags", [0, NO_OPT], ids=["fast", "exact"])
@pytest.mark.parametrize("name", KINDS)
def test_a_whole_bins(name, flags, plus):
    """at cap + 1 each former cap bin is oversized: the optimistic attempt overflows first"""
    kind = Kind(name)
    run_layout(kind, check_a_model(kind, plus), 31, flags, attempts=2 if plus and not flags else 1)


@gpu
@pytest.mark.parametrize("flags", [0, NO_OPT], ids=["fast", "exact"])
@pytest.mark.parametrize("name", KINDS)
def test_a_one_row_bin(name, flags):
    kind = Kind(name)
    lay = one_row_layout(kind)
    assert order_model(lay.bins[0], kind.per) == dict(edges=[], heads=[0], skip=True, np=1)
    run_layout(kind, lay, 32, flags)


# ---- B. thread edges -------------------------------------------------------------------------------------------------

def b_layout(kind, seed=22):
    """bin 0: groups from a thread's first row to the row before the next-but-one thread (one edge inside); bin 1:
    groups of kPer + 2 rows from the row before an edge (two edges inside); bin 2: groups over 20 edges (as many as the
    bin has at cap 96)"""
    cap, per = kind.cap, kind.per
    nt = cap // per
    rng = np.random.default_rng(seed)
    e = min(20, nt - 2)
    f0 = [(t * per, 2 * per) for t in range(1, nt - 2, 3)]
    f1 = [(t * per - 1, per + 2) for t in range(1, nt - 1, 2 if per > 1 else 3)]
    f2 = [(t * per - 1, (e - 1) * per + 2) for t in range(1, nt - e, e + 1)]
    lay = Layout(cap, {0: groups_with(cap, f0, rng), 1: groups_with(cap, f1, rng), 2: groups_with(cap, f2, rng)})
    return lay, e, (f0, f1, f2)


def check_b_model(kind):
    lay, e, fixed = b_layout(kind)
    per = kind.per
    assert lay.big() == [] and lay.S > 2 and cap_of(kind.rb, kind.flags) == kind.cap
    for s, want in ((0, 1), (1, 2), (2, e)):
        groups = {(a, L): x for a, L, x in crossed(lay.bins[s], per)}
        assert fixed[s] and all(groups[g] == want for g in fixed[s])
        if s == 0:  # starts on an edge, ends on the row before one
            assert all(a % per == 0 and (a + L) % per == 0 for a, L in fixed[s])
        else:  # starts on the row before an edge
            assert all((a + 1) % per == 0 for a, _ in fixed[s])
        chance = 1.0
        for a, L, x in crossed(lay.bins[s], per):
            if x:
                chance *= sorted_by_chance(a, L, per)
        assert chance < 1e-6, (s, chance)
    assert e == 20 or kind.cap == 96
    return lay


@gpu
@pytest.mark.parametrize("name", KINDS)
def test_b_groups_over_thread_edges(name):
    kind = Kind(name)
    run_layout(kind, check_b_model(kind), 33)


# ---- C. the skip -----------------------------------------------------------------------------------------------------

def c_layout(cap):
    """cap unique keys; the same with a 2-row group at the first row and at the last; oversized bins of unique keys
    and of one key"""
    return Layout(cap, {0: [1] * cap, 1: [2] + [1] * (cap - 2), 2: [1] * (cap - 2) + [2], 3: [1] * (3 * cap + 5),
                        4: [3 * cap + 5]})


def check_c_model(kind):
    cap = kind.cap
    lay = c_layout(cap)
    assert [order_model(lay.bins[s], kind.per)["skip"] for s in range(3)] == [True, False, False]
    assert lay.big() == [3, 4]
    for s, skip in ((3, True), (4, False)):  # fixed by the construction, whatever rows each chunk gets
        sizes = [min(cap, lay.count[s] - c0) for c0 in range(0, lay.count[s], cap)]
        assert len(sizes) == 4
        assert all(order_model([1] * m if skip else [m], kind.per)["skip"] == skip for m in sizes)
    return lay


@gpu
@pytest.mark.parametrize("name", KINDS)
def test_c_skip(name):
    kind = Kind(name)
    run_layout(kind, check_c_model(kind), 34)


# ---- D. prefix ties --------------------------------------------------------------------------------------------------

def tie_values():
    rng = np.random.default_rng(7)
    p8 = bytes(rng.integers(0, 256, 8, dtype=np.uint8))
    tail = bytes(rng.integers(0, 256, 9, dtype=np.uint8))
    base = p8 + tail
    out = [base]
    for i in (8, 9, 11, 12):  # equal in bytes 0 .. 7, different at byte i
        out.append(base[:i] + bytes([base[i] ^ 0x40]) + base[i + 1:])
        out.append(base[:i + 1])
    long = p8 + bytes(rng.integers(0, 256, 6000 - 8, dtype=np.uint8))
    out += [long, long[:-1] + bytes([long[-1] ^ 1]), long[:-1]]
    out += [b"\0" * i for i in range(13)]  # prefix 0, ordered by length alone
    out += [b"abcdefgh", b"abcdefgh\0", b"abcdefgh\0\0\0\0\x01"]
    big = p8 + bytes(rng.integers(0, 256, STAGE + 100, dtype=np.uint8))
    out += [big, big[:-1] + bytes([big[-1] ^ 0x80])]
    assert len(set(out)) == len(out)
    return out


def d_pairs(kind, seed, hot=0):
    """four keys that each hold every tie value, key j's value i at arena alignment (i + j) % 4 (fillers of another
    key in between); hot > 0: the first key also holds hot values with a shared 20-byte prefix (an oversized group)"""
    ties = tie_values()
    rng = np.random.default_rng(seed)
    if kind.mkb is None:
        keys = [int(k) for k in rng.integers(1, 1 << 63, 5, dtype=np.uint64)]
    else:
        keys = [b"tie-key-%d" % j for j in range(5)]
    pairs, aligns, off, nfill = [], [], 0, 0
    for j in range(4):
        for i, v in enumerate(ties):
            want = (i + j) % 4
            if off % 4 != want:
                f = b"%08d" % nfill + b"f" * ((want - off) % 4)
                nfill += 1
                pairs.append((keys[4], f))
                off += len(f)
            aligns.append((j, i, off % 4))
            pairs.append((keys[j], v))
            off += len(v)
    pairs += [(keys[0], b"/data/corpus/file-name-%07d" % i) for i in range(hot)]
    return pairs, aligns, keys


def check_d_model(kind, hot):
    pairs, aligns, keys = d_pairs(kind, 35, hot)
    ties = tie_values()
    assert len(set(pairs)) == len(pairs)
    for i, v in enumerate(ties):
        assert sorted(a for _, ii, a in aligns if ii == i) == [0, 1, 2, 3]
    assert sum(1 for v in ties if v[:8] == ties[0][:8]) >= 13 and max(len(v) for v in ties) > STAGE
    S, big = bins_of(kind, pairs, kind.cap)
    assert big == (1 if hot else 0)
    return pairs, S, big


@gpu
@pytest.mark.parametrize("where", ["bin", "oversized"])
@pytest.mark.parametrize("name", BIG_KINDS)
def test_d_prefix_ties(name, where):
    """one batch in a fresh ctx: the arena is packed byte for byte, so the filler lengths fix each value's alignment"""
    kind = Kind(name)
    pairs, S, big = check_d_model(kind, 3 * kind.cap if where == "oversized" else 0)
    with kind.ctx() as ctx:
        emit_job(ctx, pairs)
        check(ctx, want_groups([pairs]))
        expect_stats(ctx, attempts=1, bins=S, sub_bins=S, big_bins=big)


# ---- E. chunks -------------------------------------------------------------------------------------------------------

E_CHUNKS = [2, 64, 65, 129]


def e_layout(cap, nch, seed=24):
    """an oversized bin of nch full chunks, all but cap / 2 of its rows one key, and a small bin.  k_big_bins cuts an
    oversized bin into cap-row chunks in the order its rows arrived (each chunk then ascending by key), so which keys
    share a chunk is not fixed; the hot key is: every chunk holds at least cap / 2 of its values, whatever rows it gets"""
    rng = np.random.default_rng([seed, nch])
    n = nch * cap
    return Layout(cap, {0: groups_with(n, [(cap // 4, n - cap // 2)], rng), 1: groups_with(cap // 3, [], rng)})


def check_e_model(cap, nch):
    lay = e_layout(cap, nch)
    n, hot = lay.count[0], max(lay.bins[0])
    ctas = chunk_ctas(n, cap)
    assert len(ctas) == nch and n == nch * cap and lay.big() == [0]
    # the hot values of any chunk, left unordered, come out ascending by chance at most 1 / (cap / 2)! of the time
    assert cap - (n - hot) == cap // 2 and 1 / math.factorial(cap // 2) < 1e-6
    rounds = max(r for _, r in ctas) + 1
    assert rounds == {2: 1, 64: 1, 65: 2, 129: 3}[nch]
    if nch > CHUNK_CTAS:  # CTA 0 orders chunk 64 (and 128) too
        assert [c for c, (y, _) in enumerate(ctas) if y == 0] == list(range(0, nch, CHUNK_CTAS))
    return lay


@gpu
@pytest.mark.parametrize("nch", E_CHUNKS)
@pytest.mark.parametrize("name", ["u64-small", "str123", "u64"], ids=["cap96", "str123", "u64"])
def test_e_chunks(name, nch):
    kind = Kind(name)
    run_layout(kind, check_e_model(kind.cap, nch), 36)


# ---- F. merge passes -------------------------------------------------------------------------------------------------

SPAN_N = 5 * MERGE_THREADS - 7  # per = 5 rows per thread, which divides no 2 w = 2 cap 2^i
# case: (rows as (a, b) for a cap + b, or SPAN_N), (passes, copy-back)
F_CASES = {"cap+1": ((1, 1), (1, True)), "2cap": ((2, 0), (1, True)), "2cap+1": ((2, 1), (2, False)),
           "4cap": ((4, 0), (2, False)), "4cap+1": ((4, 1), (3, True)), "span": (SPAN_N, None)}


def f_rows(case, cap):
    r = F_CASES[case][0]
    return r if case == "span" else r[0] * cap + r[1]


def f_bin(n, rng):
    """n rows, half of them one key: a chunk holds half of its rows on average, so the merges compare its values
    across runs"""
    return groups_with(n, [(n // 4, n // 2)], rng)


def f_layout(cap, case, seed=25):
    rng = np.random.default_rng([seed, len(case)])
    if case == "mixed":  # every parity in one launch
        return Layout(cap, {i: f_bin(f_rows(c, cap), rng) for i, c in enumerate(F_CASES)})
    return Layout(cap, {0: f_bin(f_rows(case, cap), rng), 1: groups_with(cap // 4, [], rng)})


def check_f_model(cap, case):
    lay = f_layout(cap, case)
    cases = list(F_CASES) if case == "mixed" else [case]
    assert lay.big() == list(range(len(cases)))
    for s, c in enumerate(cases):
        n = lay.count[s]
        ws, back, per = merge_model(n, cap)
        if c != "span":
            assert (len(ws), back) == F_CASES[c][1]
        for w in ws:
            runs = merge_runs(n, w)
            for t in range(min(MERGE_THREADS, -(-n // per))):
                assert set(thread_pairs(n, w, per, t)) <= set(runs)
        if c == "span":
            assert per == 5 and all((2 * w) % per for w in ws)
            assert any(len(thread_pairs(n, cap, per, t)) == 2 for t in range(MERGE_THREADS))
        if c == "2cap+1":
            assert merge_runs(n, cap)[-1] == (2 * cap, 1, 0) and merge_runs(n, 2 * cap) == [(0, 2 * cap, 1)]
    if case == "mixed":
        assert {merge_model(lay.count[s], cap)[1] for s in lay.big()} == {True, False}
        # a pass whose last run pair has no run B, and one whose run B is short
        last = [(merge_runs(lay.count[s], w)[-1][2], w) for s in lay.big() for w in merge_model(lay.count[s], cap)[0]]
        assert any(lb == 0 for lb, _ in last) and any(0 < lb < w for lb, w in last)
    return lay


@gpu
@pytest.mark.parametrize("case", list(F_CASES) + ["mixed"])
@pytest.mark.parametrize("name", KINDS)
def test_f_merge_passes(name, case):
    kind = Kind(name)
    run_layout(kind, check_f_model(kind.cap, case), 37)


# ---- G. scratch reuse ------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("name", KINDS)
def test_g_same_job_after_a_larger_one(name):
    """the same job in a fresh ctx and in one whose out_cap and vo_cap an earlier, larger job raised"""
    kind = Kind(name)
    small, large = check_f_model(kind.cap, "2cap+1"), check_f_model(kind.cap, "mixed")
    rows_fresh, _ = run_layout(kind, small, 38)
    ps, pl = layout_pairs(kind, small, 38), layout_pairs(kind, large, 39)
    with kind.ctx() as ctx:
        emit_job(ctx, pl, seed=39)
        check(ctx, want_groups([pl]))
        ctx.reset()
        emit_job(ctx, ps, seed=38)
        rows, _ = check(ctx, want_groups([ps]))
        expect_stats(ctx, attempts=1, bins=small.S, sub_bins=small.S, big_bins=1)
    assert rows == rows_fresh


# ---- H. the set before the sort --------------------------------------------------------------------------------------

def plain_keys(kind, n, rng):
    if kind.mkb is None:
        return [int(k) for k in rng.integers(1, 1 << 63, n, dtype=np.uint64)]
    return [b"h%05d" % i for i in range(n)]


def h_jobs(kind, seed=40):
    """distinct pairs for the ranges A1, B1, A2, B2 of two interleaved handles and A's replacement"""
    rng = np.random.default_rng(seed)
    keys = plain_keys(kind, 50, rng)
    out = {}
    for tag, n in (("A1", 300), ("B1", 200), ("A2", 100), ("B2", 150), ("Ar", 250)):
        out[tag] = [(keys[int(rng.integers(50))], tag.encode() + b"-%d" % i) for i in range(n)]
    return out


def h_interleaved(ctx, jobs, extra=()):
    """live ranges B1, B2 (+ extra), Ar; the holes of A1 and A2 between them"""
    a, b = ctx.map_begin("A"), ctx.map_begin("B")
    batch(ctx, a, jobs["A1"])
    batch(ctx, b, jobs["B1"])
    batch(ctx, a, jobs["A2"])
    batch(ctx, b, jobs["B2"] + list(extra))
    a.commit()
    b.commit()
    emit_job(ctx, jobs["Ar"], "A")


@gpu
@pytest.mark.parametrize("name", ["u64", "str27"])
def test_h_pool_ranges_are_the_sources_until_a_pair_repeats(name):
    """no repeated pair: the three live ranges are the shuffle's sources (more per-source launches than one range);
    one repeated pair: one source and exactly one more launch (the scatter) than the same distinct pairs as one range"""
    kind = Kind(name)
    jobs = h_jobs(kind)
    live = jobs["B1"] + jobs["B2"] + jobs["Ar"]
    want = want_groups([live])
    launches, rows = {}, {}
    for case in ("ranges", "repeat", "one"):
        with kind.ctx() as ctx:
            if case == "one":
                emit_job(ctx, live)
            else:
                h_interleaved(ctx, jobs, [jobs["Ar"][5]] if case == "repeat" else [])
            rows[case], _ = check(ctx, want)
            launches[case] = ctx.stats()["launches"]
            assert ctx.result_info().pairs_in == len(live) + (case == "repeat")  # (pairs_in: before the set)
            S, big = bins_of(kind, live, kind.cap)
            expect_stats(ctx, attempts=1, bins=S, sub_bins=S, big_bins=big)
    assert rows["ranges"] == rows["repeat"] == rows["one"]
    assert launches["repeat"] == launches["one"] + 1
    d = launches["ranges"] - launches["one"]
    assert d > 0 and d % 2 == 0  # the per-source launches of two more sources


H_LENGTHS = [1, 255, 256, 257, 511]


def h_tile_jobs(kind, seed=41):
    """one job per length; copies of a record at the other side of a tile edge, and of other jobs' records"""
    rng = np.random.default_rng(seed)
    keys = plain_keys(kind, 40, rng)
    jobs = []
    for j, L in enumerate(H_LENGTHS):
        jobs.append([(keys[int(rng.integers(40))], b"t%d-%d" % (j, i)) for i in range(L)])
    jobs[3][256] = jobs[3][255]      # tile 1's first record repeats tile 0's last
    jobs[4][256] = jobs[4][0]
    jobs[4][510] = jobs[4][300]
    jobs[2][255] = jobs[1][254]      # the last record of a full tile repeats another job's
    jobs[3][0] = jobs[0][0]          # a one-record range's pair again
    jobs[4][255] = jobs[3][256]      # a copy of a copy
    return jobs


def test_h_tile_model():
    tl = set_tiles(H_LENGTHS)
    assert len(tl) == 7 and [t[2] for t in tl] == [1, 255, 256, 256, 1, 256, 255]
    assert table_entries(sum(H_LENGTHS)) == 4096 and table_entries(512) == 1024 and table_entries(513) == 2048
    jobs = h_tile_jobs(Kind("str27"))
    assert [len(j) for j in jobs] == H_LENGTHS
    n = sum(H_LENGTHS)
    assert len(set(x for j in jobs for x in j)) == n - 6


@gpu
@pytest.mark.parametrize("name", ["u64", "str27", "str123"])
def test_h_ranges_across_tile_edges(name):
    kind = Kind(name)
    jobs = h_tile_jobs(kind)
    with kind.ctx() as ctx:
        for j, p in enumerate(jobs):
            emit_job(ctx, p, "job%d" % j)
        check(ctx, want_groups(jobs))
        assert ctx.result_info().pairs_in == sum(H_LENGTHS)
        S, big = bins_of(kind, [x for j in jobs for x in j], kind.cap)
        expect_stats(ctx, attempts=1, bins=S, sub_bins=S, big_bins=big)


@gpu
@pytest.mark.parametrize("name", ["u64", "str27"])
def test_h_bins_come_from_the_distinct_count(name):
    """every distinct pair three times, over three jobs: the sub-bins are those of the distinct count"""
    kind = Kind(name)
    n = 3000 if kind.cap == 2048 else 1500
    rng = np.random.default_rng(42)
    keys = plain_keys(kind, 700, rng)
    pairs = [(keys[int(rng.integers(700))], b"x%d" % i) for i in range(n)]
    S, big = bins_of(kind, pairs, kind.cap)
    assert S == pick_sub_bins(n, kind.cap) != pick_sub_bins(3 * n, kind.cap) and big == 0
    jobs = [pairs[i::3] + pairs[(i + 1) % 3::3] + pairs[(i + 2) % 3::3] for i in range(3)]
    with kind.ctx() as ctx:
        for j, p in enumerate(jobs):
            emit_job(ctx, p, "job%d" % j, seed=j)
        check(ctx, want_groups(jobs))
        expect_stats(ctx, attempts=1, bins=S, sub_bins=S, big_bins=0)


def chain_pairs(kind, homes, T):
    """pairs whose fingerprint's home slot at T entries is given: homes = {slot: how many}"""
    need = dict(homes)
    keys = [1 << 40, 5, 77 << 33] if kind.mkb is None else [b"ck0", b"ck1", b"chain-key"]
    out = []
    for c in itertools.count():
        k, v = keys[c % 3], b"v%d" % c
        h = pair_fingerprint(k, kind.rb, v) & (T - 1)
        if need.get(h, 0):
            need[h] -= 1
            out.append((k, v))
            if not any(need.values()):
                return out


def h_chain_jobs(kind, case):
    """(jobs, T, home slot of the cluster, its pairs): 64 pairs on one home slot, or 8 on slot T - 1 wrapping to slot 0;
    their copies in later jobs, filler pairs to bring the live records to the set size"""
    n, home, cnt = {"home": (400, 100, 64), "wrap": (400, None, 8), "wrap8k": (3000, None, 8)}[case]
    T = table_entries(n)
    home = T - 1 if home is None else home
    cl = chain_pairs(kind, {home: cnt}, T)
    rng = np.random.default_rng(43)
    fill = [(k, b"fill%d" % i) for i, k in enumerate(plain_keys(kind, n - 2 * cnt, rng))]
    jobs = [fill[: len(fill) // 2] + cl, fill[len(fill) // 2:] + cl[::2], cl[1::2]]
    return jobs, T, home, cl


@pytest.mark.parametrize("case", ["home", "wrap", "wrap8k"])
@pytest.mark.parametrize("name", ["u64", "str27"])
def test_h_chain_constructions(name, case):
    kind = Kind(name)
    jobs, T, home, cl = h_chain_jobs(kind, case)
    n = sum(len(j) for j in jobs)
    assert table_entries(n) == T and T == (8192 if case == "wrap8k" else 1024)
    fps = [pair_fingerprint(k, kind.rb, v) for k, v in cl]
    assert len(set(fps)) == len(cl) and all(f & (T - 1) == home for f in fps)
    slots = sorted(place(fps, T - 1).values())
    if case == "home":
        assert slots == list(range(100, 164))
    else:
        assert slots == list(range(0, 7)) + [T - 1]
    assert len(set(x for j in jobs for x in j)) == n - len(cl)


@gpu
@pytest.mark.parametrize("case", ["home", "wrap", "wrap8k"])
@pytest.mark.parametrize("name", ["u64", "str27"])
def test_h_probe_chains(name, case):
    kind = Kind(name)
    jobs, T, home, cl = h_chain_jobs(kind, case)
    with kind.ctx() as ctx:
        for j, p in enumerate(jobs):
            emit_job(ctx, p, "job%d" % j, seed=j)
        check(ctx, want_groups(jobs))
        assert ctx.result_info().pairs_in == sum(len(j) for j in jobs)
        S, big = bins_of(kind, [x for j in jobs for x in j], kind.cap)
        expect_stats(ctx, attempts=1, bins=S, sub_bins=S, big_bins=big)


# ---- the distinct combiner's empty kept range ------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("name", ["u64", "str27"])
def test_combiner_range_that_keeps_nothing(name):
    """job A's second range repeats only pairs of its first range, with job B's range between them: the second range
    keeps 0 pairs; the ledger, pool_read, a shuffle, and the job replaced"""
    kind = Kind(name)
    rng = np.random.default_rng(44)
    keys = plain_keys(kind, 30, rng)
    a1 = [(keys[int(rng.integers(30))], b"a%d" % int(rng.integers(120))) for _ in range(400)]
    b1 = [(keys[int(rng.integers(30))], b"b%d" % i) for i in range(100)]
    a2 = [a1[int(i)] for i in rng.integers(0, 400, 300)]
    first = {}
    for i, x in enumerate(a1):
        first.setdefault(x, i)
    d1 = len(first)
    assert d1 < len(a1) and set(a2) <= set(a1)
    with kind.ctx(combiner=mrhbm.COMBINE_DISTINCT) as ctx:
        a, b = ctx.map_begin("A"), ctx.map_begin("B")
        batch(ctx, a, a1)
        batch(ctx, b, b1)
        batch(ctx, a, a2)
        a.commit()
        b.commit()
        recs = ctx.pool_read(0, d1 + len(b1))  # (the committed pairs, live range after live range)
        u64 = kind.mkb is None
        got_keys = [int(k) for k in recs["key"]] if u64 else [bytes(k) for k in recs["key"]]
        assert got_keys == [k for k, _ in first] + [k for k, _ in b1]
        assert [int(v) for v in recs["val"]] == list(first.values()) + list(range(len(a1), len(a1) + len(b1)))
        assert ctx.checksum_input()[3] == d1 + len(b1)
        check(ctx, want_groups([a1, b1]))
        S, big = bins_of(kind, a1 + b1, kind.cap)
        expect_stats(ctx, attempts=1, bins=S, sub_bins=S, big_bins=big)
        a3 = a2[:50] + a2[:50] + [(keys[0], b"new")]
        emit_job(ctx, a3, "A")
        assert ctx.checksum_input()[3] == len(set(a3)) + len(b1)
        check(ctx, want_groups([a3, b1]))
        S, big = bins_of(kind, a3 + b1, kind.cap)
        expect_stats(ctx, attempts=1, bins=S, sub_bins=S, big_bins=big)


# ---- the model itself and the constructions (no GPU) -----------------------------------------------------------------

def test_fingerprint_model_is_the_header(tmp_path):
    """every record class, value lengths 0 .. 40 (the driver places each at all four alignments)"""
    rng = np.random.default_rng(45)
    lines, want = [], []
    for rb in (16, 32, 64, 128):
        for L in range(41):
            for t in range(3):
                w = [int(x) for x in rng.integers(0, 1 << 32, key_words(rb), dtype=np.uint64)]
                v = bytes(rng.integers(0, 256, L, dtype=np.uint8)) if t else b"\0" * L
                lines.append("%d %s %s" % (rb, v.hex() or "-", " ".join("%x" % x for x in w)))
                want.append(fingerprint_words(w, rb, v))
    got = run_native(tmp_path, "distinct_fingerprint_check.cu", "distinct_fingerprint_check", lines)
    assert [int(g, 16) for g in got] == want


def test_order_and_merge_models():
    assert order_model([1, 3, 4], 4) == dict(edges=[4], heads=[0, 1, 4], skip=False, np=8)
    assert order_model([1] * 5, 2)["skip"] and order_model([1] * 5, 2)["np"] == 8
    assert crossed([3, 6, 1], 4) == [(0, 3, 0), (3, 6, 2), (9, 1, 0)]
    assert sorted_by_chance(3, 6, 4) == 1 * 24 * 1 / 720
    assert chunk_ctas(65 * 96, 96)[64] == (0, 1) and chunk_ctas(96 * 2 + 1, 96) == [(0, 0), (1, 0), (2, 0)]
    assert merge_model(96, 96)[:2] == ([], False) and merge_model(97, 96)[:2] == ([96], True)
    assert merge_model(4 * 96 + 1, 96) == ([96, 192, 384], True, 1)
    assert merge_model(SPAN_N, 2048) == ([2048, 4096], False, 5)
    assert thread_pairs(SPAN_N, 96, 5, 38) == [(0, 96, 96), (192, 96, 96)]  # rows 190 .. 194
    assert thread_pairs(2 * 96 + 1, 96, 1, 192) == [(192, 1, 0)]


@pytest.mark.parametrize("name", KINDS)
def test_constructions_land_where_they_claim(name):
    kind = Kind(name)
    cap = kind.cap
    # (layout, the seed its GPU test uses)
    lays = [(check_a_model(kind, 0), 31), (check_a_model(kind, 1), 31), (one_row_layout(kind), 32),
            (check_b_model(kind), 33), (check_c_model(kind), 34)]
    lays += [(check_f_model(cap, c), 37) for c in list(F_CASES) + ["mixed"]]
    lays += [(check_f_model(cap, "2cap+1"), 38), (check_f_model(cap, "mixed"), 39)]
    if name in ("u64-small", "str123", "u64"):
        lays += [(check_e_model(cap, n), 36) for n in E_CHUNKS]
    if name in BIG_KINDS:
        check_d_model(kind, 0)
        check_d_model(kind, 3 * cap)
    for lay, seed in lays:
        check_layout(kind, lay, seed)
