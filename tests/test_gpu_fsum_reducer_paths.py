"""The number-sum reducer (MRHBM_RED_FSUM) branch by branch, at the edges between its branches.

A bin of at most cap rows is summed by one CTA of k_num_sum (list == nullptr): the key groups are numbered with one
CTA scan over kPer rows per thread, a group of one or two values is added by one thread, a longer one by a warp.  A
larger bin (exact layout only) has its cap-row chunks merged into one key-ordered run by k_num_key_merge, in passes of
doubling width from cap up to the ctx's out_cap (plus a copy-back pass when their count is odd); then k_num_sum sums
each chunk, leaving the parts of groups that cross a chunk edge as partial accumulators in the scratch slot num_slot()
of the chunk, flagged LEAD / TAIL / THROUGH; k_num_merge adds a group's partials chunk after chunk and k_num_compact
moves each group's first row to the front.  At the end k_num_encode writes every row's 11-byte number.

A model (pure Python, P = 1 so that bin = sub-bin and the exact layout's bin offset is the scan of the bin counts)
restates the chunk flags, the slots, the merge passes and their runs.  The constructions below place key groups on
chosen rows of chosen bins; the CPU tests check that each lands where it claims, and the GPU tests compare every
shuffle in full with the exact oracle: the rational sum of each key's values rounded once."""
import itertools
import math
from bisect import bisect_left
from collections import Counter
from fractions import Fraction

import numpy as np
import pytest

import mrhbm_loader
from test_fsum_combiner_host import run_native
from test_gpu_fsum_combiner_paths import emit_np, enc_np
from test_gpu_fsum_reducer import INVAL, MAXF, bits, check, enc, fs_ctx, oracle, want_sums
from test_gpu_sort_paths import (cap_of, distinct_u64, expect_stats, pick_sub_bins, rb_of, str_keys_in_sub, str_sub,
                                 u64_keys_in_sub, u64_sub)

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402

gpu = pytest.mark.gpu
SUM_THREADS = 256            # kSumThreads
CHUNK_CTAS = 128             # kSumChunkCtas: chunks of one oversized bin summed (merged) at a time
MERGE_THREADS = 32 * 256     # kMergeCtas x kMergeThreads: the threads of one oversized bin in a merge pass
ENCODE_ROWS = 4096 * 256     # launch_num_encode: at most 4096 CTAs of 256 threads
LEAD, TAIL, THROUGH = 1, 2, 4
SCALE = 1 << 1074            # every finite double is a multiple of 2^-1074
NO_OPT = mrhbm.F_NO_OPTIMISTIC
KINDS = ["u64", "str27", "str59", "str123", "u64-small"]
BIG_KINDS = ["u64", "str27", "str59", "str123"]


# ---- the placement model ---------------------------------------------------------------------------------------------

class Kind:
    """a key class: u64 keys (F_FORCE_RUNS: hash sub-bins) or string keys of up to mkb bytes; "-small": F_SMALL_BINS"""

    def __init__(self, name):
        base, _, small = name.partition("-")
        self.name = name
        self.mkb = None if base == "u64" else int(base[3:])
        self.rb = rb_of(self.mkb)
        self.flags = (mrhbm.F_SMALL_BINS if small else 0) | (mrhbm.F_FORCE_RUNS if self.mkb is None else 0)
        self.cap = cap_of(self.rb, self.flags)
        self.per = 32 * 1024 // self.rb // SUM_THREADS  # kPer: rows per thread of k_num_sum (kCapBytes / RB / 256)

    def sub(self, key, S):
        return u64_sub(key, S, False) if self.mkb is None else str_sub(key, S)

    def keys(self, lay, seed):
        """for every bin of the layout as many distinct keys of its hash sub-bin as it has groups, ascending"""
        out = {}
        for s, g in lay.bins.items():
            rng = np.random.default_rng([seed, s])
            if self.mkb is None:
                out[s] = sorted(int(k) for k in u64_keys_in_sub(rng, len(g), lay.S, [s]))
            else:
                out[s] = sorted(bytes(k) for k in str_keys_in_sub(rng, len(g), self.rb - 4, lay.S, [s], "r"))
        return out

    def ctx(self, flags=NO_OPT):
        kind = mrhbm.KEY_U64 if self.mkb is None else mrhbm.KEY_STR
        return fs_ctx(kind, self.mkb or 27, flags=self.flags | flags, parts=1)


def num_slot(first_row, cap, first_chunk):
    return 2 * (first_row // cap) + (1 if first_chunk else 0)


def num_slots(N, cap):
    return 2 * (-(-N // cap)) + 2


def chunk_model(starts, n, o, cap):
    """k_num_sum's view of each cap-row chunk of an oversized bin of n key-ordered rows at row o whose groups start at
    the local rows `starts`: (c0, m, lead, G, s_tail, tail_part, flags, head_row, slot)"""
    out = []
    for c0 in range(0, n, cap):
        m = min(cap, n - c0)
        i, j = bisect_left(starts, c0), bisect_left(starts, c0 + m)
        lead = c0 > 0 and (i == len(starts) or starts[i] != c0)
        G = (j - i) + lead
        s_tail = c0 + m < n and (j == len(starts) or starts[j] != c0 + m)
        tail_part = s_tail and not (G == 1 and lead)
        flags = (LEAD if lead else 0) | (TAIL if tail_part else 0) | (THROUGH if s_tail and G == 1 and lead else 0)
        out.append(dict(c0=c0, m=m, lead=lead, G=G, s_tail=s_tail, tail_part=tail_part, flags=flags,
                        head_row=o + starts[j - 1] if tail_part else None, slot=num_slot(o + c0, cap, c0 == 0)))
    return out


def merge_widths(out_cap, cap):
    """k_num_key_merge's passes: the widths w = cap 2^i below out_cap, and whether a copy-back pass follows"""
    ws, w = [], cap
    while w < out_cap:
        ws.append(w)
        w <<= 1
    return ws, len(ws) % 2 == 1


def merge_launches(out_cap, cap):
    ws, back = merge_widths(out_cap, cap)
    return len(ws) + back


def merge_runs(n, w):
    """the run pairs (p0, la, lb) of a pass of width w over a bin of n rows ((0, n, 0): the bin is only copied)"""
    if w >= n:
        return [(0, n, 0)]
    return [(p0, min(w, n - p0), min(w, max(0, n - p0 - w))) for p0 in range(0, n, 2 * w)]


def merge_per(n):
    """rows per thread of a merge pass over a bin of n rows"""
    return -(-n // MERGE_THREADS)


def out_cap_of(N, S, cap, optimistic, prev=0):
    """the ctx's output rows after a shuffle of N pairs at S sub-bins (P = 1): ensure_buffers takes N, an optimistic
    attempt S cap; grow() never shrinks"""
    return max(prev, N, 1, S * cap if optimistic else 0)


class Layout:
    """a P = 1 shuffle given as bins: bins[s] = the row counts of bin s's groups in ascending key order"""

    def __init__(self, cap, bins, S=None):
        self.cap = cap
        self.bins = {s: list(g) for s, g in sorted(bins.items())}
        self.N = sum(sum(g) for g in self.bins.values())
        self.S = pick_sub_bins(self.N, cap) if S is None else S
        assert max(self.bins) < self.S
        self.count = [sum(self.bins.get(s, ())) for s in range(self.S)]
        self.off = [0] + list(itertools.accumulate(self.count))

    def starts(self, s):
        return [0] + list(itertools.accumulate(self.bins[s]))[:-1]

    def big(self):
        return [s for s in range(self.S) if self.count[s] > self.cap]

    def chunks(self, s):
        return chunk_model(self.starts(s), self.count[s], self.off[s], self.cap)

    def flags(self, s):
        return [c["flags"] for c in self.chunks(s)]

    def window(self, s, last):
        """the cap window of bin s's first or last chunk"""
        c0 = 0 if not last else (self.count[s] - 1) // self.cap * self.cap
        return (self.off[s] + c0) // self.cap

    def parts(self, s, g):
        """rows of group g of bin s in each chunk"""
        a = self.starts(s)[g]
        out = Counter()
        for r in range(a, a + self.bins[s][g]):
            out[r // self.cap] += 1
        return out

    def row(self, s, g):
        """the group's first row in layout order (bin after bin, each in key order)"""
        return self.off[s] + self.starts(s)[g]

    def group_of(self, s, local_row):
        return bisect_left(self.starts(s), local_row + 1) - 1


def groups_with(n, fixed, rng, hi=7, mix=False):
    """group sizes of an n-row bin: the fixed (first row, rows) groups, random groups of 1 .. hi rows between them
    (mix: 40 % of one row, 20 % of two, the others 3 .. hi)"""
    out, pos = [], 0
    for start, length in sorted(fixed) + [(n, 0)]:
        assert start >= pos
        while pos < start:
            if mix:
                r = rng.random()
                c = 1 if r < 0.4 else 2 if r < 0.6 else int(rng.integers(3, hi + 1))
            else:
                c = int(rng.integers(1, hi + 1))
            c = min(c, start - pos)
            out.append(c)
            pos += c
        if length:
            out.append(length)
            pos += length
    assert pos == n
    return out


def check_keys(kind, lay, keys):
    every = [k for s in lay.bins for k in keys[s]]
    assert len(set(every)) == len(every)
    for s, g in lay.bins.items():
        assert len(keys[s]) == len(g) and keys[s] == sorted(keys[s])
        assert all(kind.sub(k, lay.S) == s for k in keys[s])


# ---- values and the exact oracle -------------------------------------------------------------------------------------

def values(rng, n):
    """doubles of both signs from 2^-60 to 2^61: most sums round"""
    return rng.choice([-1.0, 1.0], n) * (1 + rng.random(n)) * np.exp2(rng.integers(-60, 61, n)).astype(np.float64)


def exact_bits(vals):
    """bits(oracle(vals)) by exact integers scaled by 2^1074 (finite values), rounded once by float(Fraction)"""
    vals = np.asarray(vals, dtype=np.float64)
    if len(vals) <= 64 or not np.isfinite(vals).all():
        return bits(oracle(vals.tolist()))
    m, e = np.frexp(vals)
    mi = (m * 2.0 ** 53).astype(np.int64)
    sh = e.astype(np.int64) + (1074 - 53)
    t = 0
    for x in np.unique(sh).tolist():
        s = sum(mi[sh == x].tolist())
        t += s << x if x >= 0 else s >> -x  # (mantissas of subnormals carry the low zero bits the shift drops)
    if t == 0:
        return bits(-0.0 if np.signbit(vals).all() else 0.0)
    f = Fraction(t, SCALE)
    if abs(f) >= MAXF:
        return bits(math.inf if t > 0 else -math.inf)
    return bits(float(f))


def row_keys(lay, keys):
    """every row's key in layout order"""
    ks = [k for s in lay.bins for k in keys[s]]
    cs = [c for s in lay.bins for c in lay.bins[s]]
    arr = np.array(ks, dtype=np.uint64) if isinstance(ks[0], int) else np.array(ks, dtype=object)
    return np.repeat(arr, cs)


def want_of(lay, keys, vals):
    want, i = {}, 0
    for s in lay.bins:
        for k, c in zip(keys[s], lay.bins[s]):
            want[k] = exact_bits(vals[i:i + c])
            i += c
    return want


def emit_layout(ctx, lay, keys, vals, seed, blob=None, job="job0"):
    """the layout's rows as one map job, in a random order"""
    kr = row_keys(lay, keys)
    perm = np.random.default_rng(seed).permutation(lay.N)
    blob = enc_np(vals) if blob is None else blob
    kr = kr[perm]
    m = ctx.map_begin(job)
    emit_np(m, ctx, kr if kr.dtype == np.uint64 else list(kr), vals[perm], blob[perm])
    m.commit()


def run_layout(kind, lay, seed, flags=NO_OPT, vals=None, attempts=1):
    """one shuffle of the layout checked in full against the oracle, and its stats"""
    keys = kind.keys(lay, seed)
    vals = values(np.random.default_rng(seed), lay.N) if vals is None else vals
    with kind.ctx(flags) as ctx:
        emit_layout(ctx, lay, keys, vals, seed)
        rows = check(ctx, want_of(lay, keys, vals), pairs=lay.N)
        expect_stats(ctx, attempts=attempts, bins=lay.S, sub_bins=lay.S, big_bins=len(lay.big()))
        return rows, ctx.stats()


# ---- A. whole bins ---------------------------------------------------------------------------------------------------

A_SUBS = {"distinct": 0, "one": 2, "pairs": 3, "lanes": 4, "kper": 5, "shifted": 6}


def fill(n, sizes):
    """groups of the sizes, cycled, until n rows (the last one cut short)"""
    out = []
    for c in itertools.cycle(sizes):
        if sum(out) >= n:
            return out
        out.append(min(c, n - sum(out)))


def a_layout(kind, plus=0):
    """bins of exactly cap rows (cap + 1 with plus: the last group one value longer), empty bins between them"""
    cap, per = kind.cap, kind.per
    lanes = [3, 32, 3, 33, 3, 64, 3, 65] if cap >= 256 else [3, 3, 32, 3, 3, 33]
    g = {"distinct": [1] * cap, "one": [cap], "pairs": [2] * (cap // 2), "lanes": fill(cap, lanes),
         "kper": fill(cap, [per]), "shifted": [1] + fill(cap - 1, [per])}
    bins = {A_SUBS[name]: gs[:-1] + [gs[-1] + plus] for name, gs in g.items()}
    return Layout(cap, bins)


def check_a_model(kind):
    lay, big = a_layout(kind), a_layout(kind, 1)
    cap, per = kind.cap, kind.per
    assert lay.S == big.S and lay.S > max(A_SUBS.values()) and lay.count[1] == 0
    assert all(lay.count[s] == cap for s in A_SUBS.values()) and lay.big() == []
    assert len(lay.bins[A_SUBS["distinct"]]) == cap and lay.bins[A_SUBS["one"]] == [cap]
    lanes = lay.bins[A_SUBS["lanes"]]
    assert sum(1 for c in lanes if c >= 3) > 8 and {32, 33} <= set(lanes)
    assert cap < 256 or {64, 65} <= set(lanes)
    assert all(a % per == 0 for a in lay.starts(A_SUBS["kper"]))
    assert per == 1 or all(a % per == 1 for a in lay.starts(A_SUBS["shifted"])[1:])
    assert big.big() == sorted(A_SUBS.values()) and all(big.count[s] == cap + 1 for s in A_SUBS.values())
    shared = 0
    for s in A_SUBS.values():
        assert big.flags(s) == [TAIL, LEAD]  # the last group's last value alone in chunk 1
        shared += s + 1 in big.bins and big.window(s, True) == big.window(s + 1, False)
    assert shared >= 1
    return lay, big


@gpu
@pytest.mark.parametrize("plus", [0, 1], ids=["cap", "cap+1"])
@pytest.mark.parametrize("flags", [0, NO_OPT], ids=["fast", "exact"])
@pytest.mark.parametrize("name", KINDS)
def test_a_whole_bins_at_cap(name, flags, plus):
    """bins of exactly cap rows: cap distinct keys, one group of cap values, cap / 2 pairs, lane-loop groups of 3, 32,
    33, 64, 65, groups on every kPer thread boundary and the same shifted by one row; at cap + 1 each bin goes to the
    oversized path (the optimistic attempt overflows first)"""
    kind = Kind(name)
    lay = check_a_model(kind)[plus]
    run_layout(kind, lay, 11, flags, attempts=2 if plus and not flags else 1)


# ---- B. chunk flags --------------------------------------------------------------------------------------------------

def b_layout(cap, seed=3):
    rng = np.random.default_rng(seed)
    return Layout(cap, {
        # a clean edge at cap; a 2-value group over 2 cap; a group from chunk 2's last row, one to chunk 4's first
        # row; chunk 5 one lead group
        0: groups_with(5 * cap + 7, [(cap - 5, 5), (cap, 4), (2 * cap - 1, 2), (3 * cap - 1, 40), (4 * cap - 40, 41),
                                     (5 * cap - 3, 10)], rng),
        1: groups_with(3 * cap, [(cap, cap)], rng),  # a group that fills chunk 1
        # groups that run THROUGH 1, 2 and 5 chunks
        2: groups_with(12 * cap + 7, [(cap - 3, cap + 6), (3 * cap - 1, 2 * cap + 2), (6 * cap + 5, 6 * cap)], rng),
        3: [3 * cap], 4: [3 * cap + 1],  # one group as the whole bin
        5: groups_with(cap + 1, [(cap - 2, 3)], rng),
        6: groups_with(2 * cap, [(cap - 2, 5)], rng),
        7: groups_with(2 * cap + 1, [(cap - 1, 2), (2 * cap - 3, 4)], rng),
    })


def check_b_model(cap):
    lay = b_layout(cap)
    f = {s: lay.flags(s) for s in lay.bins}
    ch0 = lay.chunks(0)
    assert not f[0][0] & TAIL and not f[0][1] & LEAD  # a group ends on the edge, the next starts on it
    assert f[0][1] & TAIL and f[0][2] & LEAD and lay.parts(0, lay.group_of(0, 2 * cap - 1)) == {1: 1, 2: 1}
    assert f[0][2] & TAIL and ch0[2]["head_row"] == lay.off[0] + 3 * cap - 1  # first row: chunk 2's last
    assert f[0][3] & TAIL and f[0][4] & LEAD and lay.parts(0, lay.group_of(0, 4 * cap)) == {3: 40, 4: 1}
    assert f[0][5] == LEAD and ch0[5]["G"] == 1 and not ch0[5]["s_tail"]  # chunk 5's only group: a lead
    c1 = lay.chunks(1)[1]
    assert c1["G"] == 1 and c1["flags"] == 0  # a group that fills the chunk: summed whole
    assert f[2][:5] == [TAIL, LEAD | THROUGH, LEAD | TAIL, LEAD | THROUGH, LEAD | THROUGH] and f[2][5] & LEAD
    assert f[2][6] & TAIL and f[2][7:12] == [LEAD | THROUGH] * 5 and f[2][12] & LEAD and not f[2][12] & THROUGH
    assert lay.chunks(2)[2]["G"] >= 2  # a leading and a trailing partial in one chunk
    assert f[3] == [TAIL, LEAD | THROUGH, LEAD] and f[4] == [TAIL, LEAD | THROUGH, LEAD | THROUGH, LEAD]
    assert [lay.count[s] for s in (3, 4, 5, 6, 7)] == [3 * cap, 3 * cap + 1, cap + 1, 2 * cap, 2 * cap + 1]
    assert f[5] == [TAIL, LEAD] and f[6] == [TAIL, LEAD] and f[7] == [TAIL, LEAD | TAIL, LEAD]
    assert lay.big() == list(range(8))
    return lay


@gpu
@pytest.mark.parametrize("name", KINDS)
def test_b_chunk_flags(name):
    kind = Kind(name)
    run_layout(kind, check_b_model(kind.cap), 12)


# ---- C. more than 128 chunks -----------------------------------------------------------------------------------------

def c_layout(cap, seed=4):
    """bins of 128 cap and 128 cap + 1 rows; two of about 300 cap rows, one with a group across chunks 127 -> 128,
    one with a group over chunks 126 .. 130 (k_num_merge's chain crosses the grid stride)"""
    rng = np.random.default_rng(seed)
    hi = 2 * cap
    return Layout(cap, {
        0: groups_with(128 * cap, [], rng, hi, True),
        1: groups_with(128 * cap + 1, [], rng, hi, True),
        2: groups_with(300 * cap, [(128 * cap - 5, 10)], rng, hi, True),
        3: groups_with(300 * cap + 17, [(126 * cap + 7, 4 * cap)], rng, hi, True),
    })


def check_c_model(cap):
    lay = c_layout(cap)
    assert [len(lay.chunks(s)) for s in range(4)] == [128, 129, 300, 301]
    f2, f3 = lay.flags(2), lay.flags(3)
    assert f2[127] & TAIL and f2[128] & LEAD and 128 // CHUNK_CTAS == 1  # chunk 128: CTA 0's second chunk
    assert f3[126] & TAIL and f3[127:130] == [LEAD | THROUGH] * 3 and f3[130] & LEAD and not f3[130] & THROUGH
    assert len(lay.chunks(3)) > 2 * CHUNK_CTAS  # a third round of the grid stride
    assert lay.big() == [0, 1, 2, 3]
    return lay


@gpu
@pytest.mark.parametrize("name", ["u64", "u64-small"], ids=["cap2048", "cap96"])
def test_c_more_chunks_than_ctas(name):
    kind = Kind(name)
    run_layout(kind, check_c_model(kind.cap), 13)


# ---- D. adjacent oversized bins --------------------------------------------------------------------------------------

def d_layout(cap, seed=5):
    rng = np.random.default_rng(seed)
    return Layout(cap, {
        0: groups_with(7, [], rng),
        1: groups_with(2 * cap + 10, [(2 * cap - 4, 6)], rng),
        2: groups_with(cap + 20, [(cap - 3, 6)], rng),
        3: groups_with(3 * cap - 40, [(cap - 2, 4), (2 * cap - 3, 5)], rng),
        4: groups_with(2, [], rng),
        5: groups_with(9 * cap + 7, [(cap - 1, 3)], rng),
        6: groups_with(cap - 3, [], rng),
    })


def check_d_model(cap):
    lay = d_layout(cap)
    assert lay.big() == [1, 2, 3, 5]
    for a, b in ((1, 2), (2, 3), (3, 5)):  # bin a's last chunk and bin b's first share a cap window ...
        last, first = lay.chunks(a)[-1], lay.chunks(b)[0]
        assert lay.window(a, True) == lay.window(b, False)
        assert last["flags"] & LEAD and first["flags"] & TAIL  # ... the former with a LEAD, the latter a TAIL partial
        assert last["slot"] == first["slot"] - 1  # only num_slot's first-chunk term tells them apart
    assert lay.count[4] and lay.count[0] and lay.count[6]  # normal bins before, between and after
    # passes in which one bin is only copied (n <= w) while another merges
    mixed = [w for w in merge_widths(lay.N, cap)[0] if {lay.count[s] <= w for s in lay.big()} == {True, False}]
    assert {2 * cap, 4 * cap} <= set(mixed)
    return lay


@gpu
@pytest.mark.parametrize("name", KINDS)
def test_d_adjacent_oversized_bins(name):
    kind = Kind(name)
    run_layout(kind, check_d_model(kind.cap), 14)


# ---- E. merge passes -------------------------------------------------------------------------------------------------

def e_layout(case, cap, seed=6):
    """fresh-ctx shuffles whose out_cap (= N) gives 1 pass + copy-back, 2 passes, 3 passes + copy-back; bin 0 holds a
    hot key with more than n - cap rows, so every full chunk of its scattered rows holds some"""
    rng = np.random.default_rng(seed)
    n, other = {"e1": (cap + cap // 2, {1: groups_with(cap // 4, [], rng)}),
                "e2": (3 * cap + 5, {1: groups_with(20, [], rng)}),
                "e3": (6 * cap + 5, {1: groups_with(cap + 3, [], rng)})}[case]
    hot = n - cap + 1 + cap // 8
    a = (n - hot) // 2
    bins = {0: groups_with(n, [(a, hot)], rng)}
    bins.update(other)
    return Layout(cap, bins)


E_PASSES = {"e1": (1, True), "e2": (2, False), "e3": (3, True)}


def check_e_model(case, cap):
    lay = e_layout(case, cap)
    ws, back = merge_widths(out_cap_of(lay.N, lay.S, cap, False), cap)
    assert (len(ws), back) == E_PASSES[case]
    n = lay.count[0]
    hot = max(lay.bins[0])
    assert hot > n - cap  # a hot key in every full chunk: equal keys meet across run boundaries
    assert lay.flags(0).count(LEAD | THROUGH) >= (n // cap) - 2
    runs = merge_runs(n, cap)
    if case == "e2":
        assert runs[-1][2] == 5  # the last run of pass 1 is partial
    if case == "e3":
        assert runs[-1] == (6 * cap, 5, 0)  # ... empty
        assert merge_runs(n, 2 * cap)[-1][2] == 5
        assert merge_runs(lay.count[1], 2 * cap) == [(0, cap + 3, 0)]  # bin 1 only copied while bin 0 merges
    return lay


@gpu
@pytest.mark.parametrize("case", list(E_PASSES))
@pytest.mark.parametrize("name", KINDS)
def test_e_merge_passes(name, case):
    kind = Kind(name)
    lay = check_e_model(case, kind.cap)
    assert (merge_per(lay.count[0]) > 1) == (lay.count[0] > MERGE_THREADS)
    run_layout(kind, lay, 15)


@gpu
@pytest.mark.parametrize("name", KINDS)
def test_e_same_job_after_a_larger_one(name):
    """the same job in a fresh ctx and in one whose out_cap an earlier, larger job raised: identical results, and the
    launch counts differ by the merge passes the model gives for the two out_caps"""
    kind = Kind(name)
    small, large = check_e_model("e1", kind.cap), check_e_model("e3", kind.cap)
    rows_fresh, st_fresh = run_layout(kind, small, 16)
    keys_l, keys_s = kind.keys(large, 17), kind.keys(small, 16)
    vl = values(np.random.default_rng(17), large.N)
    vs = values(np.random.default_rng(16), small.N)
    with kind.ctx() as ctx:
        emit_layout(ctx, large, keys_l, vl, 17)
        check(ctx, want_of(large, keys_l, vl), pairs=large.N)
        ctx.reset()
        emit_layout(ctx, small, keys_s, vs, 16)
        rows = check(ctx, want_of(small, keys_s, vs), pairs=small.N)
        expect_stats(ctx, attempts=1, bins=small.S, big_bins=1)
        launches = ctx.stats()["launches"]
    assert sorted(rows) == sorted(rows_fresh)
    raised = out_cap_of(large.N, large.S, kind.cap, False, out_cap_of(small.N, small.S, kind.cap, False))
    want = merge_launches(raised, kind.cap) - merge_launches(small.N, kind.cap)
    assert want == 2 and launches - st_fresh["launches"] == want


# ---- F. deferred carries ---------------------------------------------------------------------------------------------

V_MAX = 2.0 - 2.0 ** -52  # the largest mantissa at exponent 0
F_N1, F_K = (1 << 24) + 12345, 1 << 21


def f_layout():
    """one key of about 2^24 copies of V_MAX (every addend lands in the same few digits), one of 2^21 copies of +V_MAX,
    2^21 - 1 of -V_MAX and one -(V_MAX - 2^-52), whose sum is one ulp, and a few small keys"""
    return Layout(2048, {0: [F_N1], 1: [2 * F_K], 2: [1, 2, 3, 40, 5]})


def f_values(lay):
    v = np.empty(lay.N)
    v[:F_N1] = V_MAX
    v[F_N1:F_N1 + F_K] = V_MAX
    v[F_N1 + F_K:F_N1 + 2 * F_K - 1] = -V_MAX
    v[F_N1 + 2 * F_K - 1] = -(V_MAX - 2.0 ** -52)
    v[F_N1 + 2 * F_K:] = values(np.random.default_rng(7), lay.N - F_N1 - 2 * F_K)
    return v


def check_f_model():
    lay = f_layout()
    ch = lay.chunks(0)
    assert len(ch) > 8000 and all(c["flags"] == LEAD | THROUGH for c in ch[1:-1])
    assert len(lay.chunks(1)) == 2 * F_K // 2048 and lay.big() == [0, 1]
    assert merge_widths(lay.N, 2048)[0][-1] >= F_N1 // 2
    return lay


@gpu
def test_f_deferred_carries():
    kind = Kind("u64")
    lay = check_f_model()
    keys = kind.keys(lay, 18)
    vals = f_values(lay)
    small = np.cumsum([F_N1 + 2 * F_K] + lay.bins[2])
    want = {k: exact_bits(vals[a:e]) for k, a, e in zip(keys[2], small[:-1], small[1:])}
    want[keys[0][0]] = bits(float(F_N1 * Fraction(V_MAX)))
    want[keys[1][0]] = bits(2.0 ** -52)
    with kind.ctx() as ctx:
        emit_layout(ctx, lay, keys, vals, 18)
        check(ctx, want, pairs=lay.N)
        expect_stats(ctx, attempts=1, bins=lay.S, big_bins=2)


# ---- G. errors on each path ------------------------------------------------------------------------------------------

def g_case(case, cap, seed=8):
    """(layout, (bin, group) of the bad values, how many, what they are, shuffle flags)"""
    rng = np.random.default_rng(seed)
    if case in ("notnum-1", "notnum-2", "nan-2", "notnum-warp"):
        lay = Layout(cap, {0: [3, 1, 2, 5, 40, 1]})
        g = {"notnum-1": 1, "notnum-2": 2, "nan-2": 2, "notnum-warp": 4}[case]
        return lay, (0, g), 2 if case == "nan-2" else 1, case.split("-")[0], NO_OPT
    if case == "notnum-fast":  # the optimistic attempt overflows: its k_num_sum returns early
        lay = Layout(cap, {0: [1] + groups_with(cap, [], rng)})
        return lay, (0, 0), 1, "notnum", 0
    fixed = {"notnum-lead": (cap - 1, cap // 2), "notnum-through": (cap - 1, cap + 2),
             "notnum-tail": (cap - cap // 2, cap // 2 + 1), "nan-cross3": (cap - 5, cap + 10)}[case]
    lay = Layout(cap, {0: groups_with(3 * cap, [fixed], rng)})
    g = lay.group_of(0, fixed[0])
    parts = lay.parts(0, g)
    if case == "nan-cross3":
        return lay, (0, g), 2, "nan", NO_OPT
    named = {"lead": max(parts), "through": min(parts) + 1, "tail": min(parts)}[case.split("-")[1]]
    # bad values in every row of the group outside the named chunk and one more: at least one lands there
    return lay, (0, g), fixed[1] - parts[named] + 1, "notnum", NO_OPT


G_CASES = ["notnum-1", "notnum-2", "notnum-warp", "notnum-lead", "notnum-through", "notnum-tail", "nan-2",
           "nan-cross3", "notnum-fast"]


def check_g_model(case, cap):
    lay, (s, g), nbad, what, flags = g_case(case, cap)
    size = lay.bins[s][g]
    assert nbad <= size
    if case in ("notnum-1", "notnum-2", "nan-2"):
        assert size == int(case[-1]) and lay.big() == []
    elif case == "notnum-warp":
        assert size > 2 and lay.big() == []
    elif case == "notnum-fast":
        assert lay.count[0] == cap + 1 and size == 1
    else:
        parts = lay.parts(s, g)
        f = lay.flags(s)
        c = sorted(parts)
        assert len(c) == (3 if case in ("notnum-through", "nan-cross3") else 2)
        assert f[c[0]] & TAIL and f[c[-1]] & LEAD and all(f[x] == LEAD | THROUGH for x in c[1:-1])
        if what == "notnum":
            named = {"lead": c[-1], "through": c[1] if len(c) == 3 else None, "tail": c[0]}[case.split("-")[1]]
            assert size - parts[named] < nbad  # at least one bad value in the named chunk
    return lay, (s, g), nbad, what, flags


@gpu
@pytest.mark.parametrize("case", G_CASES)
@pytest.mark.parametrize("name", BIG_KINDS)
def test_g_errors_on_each_path(name, case):
    """a value that is not a number, or +inf with -inf, on each path: MRHBM_E_INVAL and no result; the job replaced
    with numbers, the same ctx's next shuffle succeeds"""
    kind = Kind(name)
    lay, (s, g), nbad, what, flags = check_g_model(case, kind.cap)
    keys = kind.keys(lay, 19)
    vals = values(np.random.default_rng(19), lay.N)
    r = lay.row(s, g)
    blob = enc_np(vals)
    if what == "nan":
        blob[r] = enc_np([math.inf])[0]
        blob[r + 1] = enc_np([-math.inf])[0]
    else:
        blob[r:r + nbad, 0] = 0x11  # not the number tag
    with kind.ctx(flags) as ctx:
        emit_layout(ctx, lay, keys, vals, 19, blob)
        with pytest.raises(mrhbm.MrhbmError) as e:
            ctx.shuffle()
        assert e.value.code == INVAL and ("NaN" if what == "nan" else "not a number") in str(e.value)
        with pytest.raises(mrhbm.MrhbmError):
            ctx.result_info()
        emit_layout(ctx, lay, keys, vals, 20)  # (job0 replaced)
        check(ctx, want_of(lay, keys, vals), pairs=lay.N)
        expect_stats(ctx, attempts=1, bins=lay.S, big_bins=len(lay.big()))  # (an overflow ends optimism for good)


# ---- H. the encode grid ----------------------------------------------------------------------------------------------

def dec_np(blob, n):
    assert len(blob) == 11 * n
    r = blob.reshape(n, 11)
    assert (r[:, 0] == 0x10).all() and (r[:, 1:] & 0x80 == 0x80).all()
    u = np.zeros(n, np.uint64)
    for k in range(10):  # (the first byte carries the top bit only)
        u |= (r[:, 1 + k] & 0x7F).astype(np.uint64) << np.uint64(63 - 7 * k)
    return np.where(u >> np.uint64(63) != 0, u & np.uint64((1 << 63) - 1), ~u)


def h_job(n, seed):
    """n distinct u64 keys, the first half with two values (one IEEE addition is their exact sum rounded once)"""
    rng = np.random.default_rng(seed)
    keys = distinct_u64(rng, n)
    two = n // 2
    a, b = values(rng, n), values(rng, two)
    want = a.copy()
    want[:two] = a[:two] + b
    return np.concatenate([keys, keys[:two]]), np.concatenate([a, b]), keys, want


def test_h_model():
    # launch_num_encode: min((n + 256) / 256, 4096) CTAs over the n + 1 entries of row_off
    grid = [min((n + 256) // 256, 4096) * 256 for n in (ENCODE_ROWS - 1, ENCODE_ROWS, ENCODE_ROWS + 1)]
    assert grid == [ENCODE_ROWS] * 3  # n + 1 = 2^20 entries fill the grid; past it the grid-stride loop takes the rest
    keys, vals, k, want = h_job(1000, 1)
    assert len(set(k.tolist())) == 1000 and len(keys) == 1500
    pairs = list(zip(keys.tolist(), vals.tolist()))
    assert want_sums([pairs]) == dict(zip(k.tolist(), want.view(np.uint64).tolist()))
    blob = enc_np(want)
    assert dec_np(blob.ravel(), 1000).tolist() == want.view(np.uint64).tolist()
    assert bytes(blob[3]) == enc(float(want[3]))


@gpu
@pytest.mark.parametrize("n", [ENCODE_ROWS - 1, ENCODE_ROWS, ENCODE_ROWS + 1], ids=["below", "at", "above"])
def test_h_encode_grid(n):
    """results of 4096 x 256 - 1 .. + 1 rows: k_num_encode's capped grid covers the last rows and row_off[n] through
    its grid-stride loop"""
    keys, vals, k, want = h_job(n, n)
    with fs_ctx(mrhbm.KEY_U64, parts=1) as ctx:
        m = ctx.map_begin("job0")
        emit_np(m, ctx, keys, vals)
        m.commit()
        ctx.shuffle()
        info = ctx.result_info()
        assert info.groups == n and info.pairs_recv == len(keys) and ctx.checksum_input()[3] == len(keys)
        gk, _, po = ctx.result_copy()
        blob, roff = ctx.result_values()
        assert [int(po[0]), int(po[-1])] == [0, n]
        assert np.array_equal(roff, np.arange(n + 1, dtype=np.uint64) * np.uint64(11))
        got = dec_np(blob, n)
    order, wo = np.argsort(gk), np.argsort(k)
    assert np.array_equal(gk[order], k[wo])
    assert np.array_equal(got[order], want.view(np.uint64)[wo])


# ---- the model itself and the constructions (no GPU) -----------------------------------------------------------------

def test_num_slot_model_is_the_header(tmp_path):
    rng = np.random.default_rng(1)
    lines, want = [], []
    for _ in range(400):
        cap = int(rng.choice([96, 256, 512, 1024, 2048]))
        r, first = int(rng.integers(0, 1 << 33)), int(rng.integers(0, 2))
        lines.append("slot %d %d %d" % (r, cap, first))
        want.append(num_slot(r, cap, first))
        N = int(rng.integers(1, 1 << 33))
        lines.append("slots %d %d" % (N, cap))
        want.append(num_slots(N, cap))
    got = run_native(tmp_path, "num_slot_check.cu", "num_slot_check", lines)
    assert [int(x) for x in got] == want


def test_no_two_chunks_of_oversized_bins_share_a_slot():
    """the header's claim: over layouts of oversized and normal bins, every chunk of an oversized bin has its own slot,
    below num_slots(N, cap)"""
    rng = np.random.default_rng(2)
    for t in range(300):
        cap = int(rng.choice([4, 96, 256, 2048]))
        counts = [int(rng.integers(cap + 1, 5 * cap)) if rng.random() < 0.5 else int(rng.integers(0, cap + 1))
                  for _ in range(int(rng.integers(1, 30)))]
        off = [0] + list(itertools.accumulate(counts))
        N = off[-1]
        seen = set()
        for b, n in enumerate(counts):
            if n <= cap:
                continue
            for c0 in range(0, n, cap):
                s = num_slot(off[b] + c0, cap, c0 == 0)
                assert s not in seen and s < num_slots(N, cap)
                seen.add(s)
    # without the first-chunk term a bin's first chunk takes the slot of the previous bin's last chunk
    lay = d_layout(96)
    assert num_slot(lay.off[2], 96, False) == lay.chunks(1)[-1]["slot"]


def test_chunk_model_on_small_bins():
    # cap 4, at row 100, rows (key): a a a b | b b c c | c c c c | c d  -> groups start at 0, 3, 6, 13
    ch = chunk_model([0, 3, 6, 13], 14, 100, 4)
    assert [c["flags"] for c in ch] == [TAIL, LEAD | TAIL, LEAD | THROUGH, LEAD]
    assert [c["G"] for c in ch] == [2, 2, 1, 2]
    assert [c["head_row"] for c in ch] == [103, 106, None, None]
    assert [c["slot"] for c in ch] == [51, 52, 54, 56]
    assert [c["flags"] for c in chunk_model([0, 4], 8, 0, 4)] == [0, 0]  # an edge between groups
    assert [c["flags"] for c in chunk_model([0], 9, 0, 4)] == [TAIL, LEAD | THROUGH, LEAD]


def test_merge_model():
    cap = 96
    assert merge_widths(cap, cap) == ([], False)
    assert merge_widths(cap + 1, cap) == ([96], True)
    assert merge_widths(4 * cap, cap) == ([96, 192], False)
    assert merge_widths(4 * cap + 1, cap) == ([96, 192, 384], True)
    assert merge_launches(8 * cap, cap) == 4 and merge_launches(8 * cap + 1, cap) == 4
    assert merge_runs(2 * cap + 5, cap) == [(0, cap, cap), (2 * cap, 5, 0)]
    assert merge_runs(3 * cap + 5, cap) == [(0, cap, cap), (2 * cap, cap, 5)]
    assert merge_runs(50, cap) == [(0, 50, 0)]
    assert merge_per(8192) == 1 and merge_per(8193) == 2 and merge_per(6 * 2048 + 5) == 2
    assert out_cap_of(500, 14, 96, True) == 14 * 96 and out_cap_of(500, 14, 96, False, 9000) == 9000


def test_exact_oracle_matches_fractions():
    rng = np.random.default_rng(3)
    for n in (65, 100, 400):
        for t in range(20):
            v = values(rng, n)
            if t % 4 == 1:
                v[: n // 2] = -v[n - n // 2:][::-1][: n // 2]  # pairs that cancel
            if t % 4 == 2:
                v = v * 2.0 ** -1060  # subnormal sums
            if t % 4 == 3:
                v[0], v[1] = 1.7976931348623157e308, 1.7976931348623157e308  # overflow
            assert exact_bits(v) == bits(oracle(v.tolist()))
    assert exact_bits(np.array([-0.0] * 70)) == bits(-0.0) and exact_bits(np.array([-0.0] * 69 + [0.0])) == bits(0.0)
    # the closed forms of F
    n = 1000
    assert exact_bits(np.full(n, V_MAX)) == bits(float(n * Fraction(V_MAX)))
    k = 100
    assert exact_bits(np.array([V_MAX] * k + [-V_MAX] * (k - 1) + [-(V_MAX - 2.0 ** -52)])) == bits(2.0 ** -52)


@pytest.mark.parametrize("name", KINDS)
def test_constructions_land_where_they_claim(name):
    kind = Kind(name)
    cap = kind.cap
    lays = list(check_a_model(kind)) + [check_b_model(cap), check_d_model(cap)]
    lays += [check_e_model(c, cap) for c in E_PASSES]
    if name == "u64" or name == "u64-small":
        lays.append(check_c_model(cap))
    for case in G_CASES:
        lays.append(check_g_model(case, cap)[0])
    for i, lay in enumerate(lays):
        check_keys(kind, lay, kind.keys(lay, 100 + i))
    check_f_model()
