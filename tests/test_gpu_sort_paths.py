"""The sort stage branch by branch, at the edges between its branches.

Which algorithm sorts a bin is decided by the data: the pipelined u64 kernel (k_sort_reduce_u64, in its hint form for
key-ordered sub-bins and its MINMAX form), the counting path and the general bitonic + LSD path of process_loaded, and
the merge rounds of k_big_bins with the skew retry behind them.  A placement model (pure Python, the device's
partitioner and bucket arithmetic restated) builds inputs that land on a chosen branch, at a chosen edge: bins of
exactly cap and cap + 1 records, buckets of exactly 4 / 5 and 8 / 9 records, keys at the ends of key-ordered sub-bins,
string keys that differ in one bit beside a 52-bit chunk or 32-bit word boundary, bins that need two or more merge
rounds and bins that no number of sub-bins splits.  Every construction asserts that the model puts it where it is
meant to go (the CPU tests below check the constructions alone), and every shuffle is compared in full with an exact
reference: Python-int sums in a dict, sorted() over ints or key bytes."""
import math
from collections import Counter

import numpy as np
import pytest

import mrhbm_loader
import oracle as O

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402

gpu = pytest.mark.gpu
M64 = (1 << 64) - 1
GOLD = 0x9E3779B97F4A7C15
HASH_SUB_SALT = 0x632BE59BD9B4E019
NB_U64 = 4096  # buckets of the u64 kernel: 2 * its 2048-record capacity
KFIX_MAX = 8  # bucket mates the rank-among-mates step accepts
MKBS = [27, 59, 123]
REDUCERS = [mrhbm.RED_SUM, mrhbm.RED_NONE]


# ---- the placement model ---------------------------------------------------------------------------------------------

def mix64(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def mulhi(x, m):
    """floor(x * m / 2^64): the device's mulhi_u64_u32 is exact for a 32-bit m"""
    return (x * m) >> 64


def word_hash(slot):
    """64-bit hash over the little-endian u32 words of a stored key slot while they are non-zero"""
    slot = bytes(slot)
    slot += b"\0" * (-len(slot) % 4)
    h = GOLD
    for i in range(0, len(slot), 4):
        w = int.from_bytes(slot[i:i + 4], "little")
        if w == 0:
            break
        h = ((h ^ w) * 0xBF58476D1CE4E5B9) & M64
        h ^= h >> 29
    h ^= h >> 32
    return (h * 0x94D049BB133111EB) & M64


def mulhash_pid(key, P):
    return mulhi((key * GOLD) & M64, P)


def u64_hash_src(key, P=1):
    """source of the hash sub-bin of a u64 key under MULHASH (independent of the partition)"""
    return mix64((((key * GOLD) & M64) * P + HASH_SUB_SALT) & M64)


def u64_sub(key, S, ordered):
    return mulhi(key, S) if ordered else mulhi(u64_hash_src(key), S)


def str_sub(slot, S):
    """FNV_LUA partitioner: the sub-bin of a string key comes from word_hash"""
    return mulhi(word_hash(slot), S)


def rb_of(mkb):
    return 16 if mkb is None else mrhbm.record_dtype(mrhbm.KEY_STR, mkb).itemsize


def cap_of(rb, flags=0):
    return 96 if flags & mrhbm.F_SMALL_BINS else 32 * 1024 // rb


def pick_sub_bins(n, cap, P=1):
    target = int(max(1.0, cap - 6.0 * math.sqrt(cap)))
    return max(1, -(-n // (P * target)))


def bitlen(x):
    return x.bit_length()


def minmax_shifts(lo, hi):
    """the MINMAX form: (sh0, sh1) of a bin whose keys span [lo, hi]"""
    bits = bitlen(hi - lo)
    sh0 = max(bits - 32, 0)
    return sh0, max(bits - 12, 0) - sh0


def minmax_buckets(keys):
    """32-bit sort key and bucket of every key of one bin sorted in the MINMAX form"""
    lo, hi = min(keys), max(keys)
    sh0, sh1 = minmax_shifts(lo, hi)
    kk = [((k - lo) >> sh0) & 0xFFFFFFFF for k in keys]
    return kk, [(x >> sh1) & (NB_U64 - 1) for x in kk]


def hint_bucket(key, S):
    """the hint form: bucket of a key of sub-bin mulhi(key, S) BEFORE the & (NB - 1) mask (must be < NB)"""
    q = (1 << 64) // S
    bits = bitlen(q + S)
    sh0 = max(bits - 32, 0)
    sh1 = max(bits - 12, 0) - sh0
    return ((key - mulhi(key, S) * q) >> sh0) >> sh1


def prefix64(slot):
    return int.from_bytes(bytes(slot)[:8].ljust(8, b"\0"), "big")


def counting_buckets(slots, cap):
    """counting_path: bucket of every key (NB = 2 * cap interpolated buckets of the 64-bit prefix) and the
    general path's `drop` (low prefix bits its 52-bit digit loses)"""
    p = [prefix64(s) for s in slots]
    lo, hi = min(p), max(p)
    bits = bitlen(hi - lo)
    sh = max(bits - bitlen(2 * cap - 1), 0)
    return [(x - lo) >> sh for x in p], max(bits - 52, 0)


def big_bin_rounds(keys, cap):
    """k_big_bins on one bin (records in bin order): the record count after every merge round, None when a round
    merges nothing (ERRF_SKEW).  Chunks of cap records, each sorted and reduced to one record per key."""
    sizes, cur = [], list(keys)
    while len(cur) > cap:
        nxt = []
        for c in range(0, len(cur), cap):
            nxt += sorted(set(cur[c:c + cap]))
        if len(nxt) == len(cur):
            return None
        sizes.append(len(nxt))
        cur = nxt
    return sizes


def sample_is_uniform(keys):
    """the optimistic layout's test for key-ordered sub-bins: a histogram of the top 8 key bits (n < 2^18: every
    key is sampled) must have no bucket above mean * 1.08 + 5 sigma + 2"""
    h = Counter(k >> 56 for k in keys)
    mean = len(keys) / 256.0
    return max(h.values()) <= mean * 1.08 + 5.0 * math.sqrt(mean) + 2.0


# vectorised forms for filtering many candidates (numpy uint64 arithmetic wraps mod 2^64)
def mix64_np(z):
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def mulhi_np(x, m):
    lo = (x & np.uint64(0xFFFFFFFF)) * np.uint64(m)
    hi = (x >> np.uint64(32)) * np.uint64(m)
    return (hi + (lo >> np.uint64(32))) >> np.uint64(32)


def u64_sub_hash_np(keys, S):
    return mulhi_np(mix64_np(keys * np.uint64(GOLD) + np.uint64(HASH_SUB_SALT)), S)


def word_hash_np(slots):
    """word_hash of every slot of an 'S<kb>' array"""
    kb = slots.dtype.itemsize
    w = np.zeros((slots.size, -(-kb // 4) * 4), dtype=np.uint8)
    w[:, :kb] = slots.view(np.uint8).reshape(slots.size, kb)
    w = w.view("<u4").astype(np.uint64)
    h = np.full(slots.size, GOLD, dtype=np.uint64)
    live = np.ones(slots.size, dtype=bool)
    for i in range(w.shape[1]):
        live &= w[:, i] != 0
        g = (h ^ w[:, i]) * np.uint64(0xBF58476D1CE4E5B9)
        h = np.where(live, g ^ (g >> np.uint64(29)), h)
    h ^= h >> np.uint64(32)
    return h * np.uint64(0x94D049BB133111EB)


def distinct_u64(rng, n):
    k = np.unique(rng.integers(0, 1 << 64, int(n * 1.1) + 16, dtype=np.uint64))
    return rng.permutation(k)[:n]


def u64_keys_in_sub(rng, count, S, subs, src_below=None):
    """`count` distinct random u64 keys whose hash sub-bin at S is one of `subs` (and whose hash source is below
    src_below when given), in input order"""
    out = np.zeros(0, dtype=np.uint64)
    while out.size < count:
        c = distinct_u64(rng, 1 << 16)
        ok = np.isin(u64_sub_hash_np(c, S), np.array(subs, dtype=np.uint64))
        if src_below is not None:
            ok &= mix64_np(c * np.uint64(GOLD) + np.uint64(HASH_SUB_SALT)) < np.uint64(src_below)
        out = np.unique(np.concatenate([out, c[ok]]))
    return rng.permutation(out)[:count]


def str_candidates(rng, count, kb, tag):
    """`count` distinct stored key slots (NUL-free, 9..kb-1 bytes) as an 'S<kb>' array"""
    lens = rng.integers(9, kb, count)
    a = rng.integers(97, 123, (count, kb), dtype=np.uint8)
    idx = np.arange(count)
    a[:, 0] = ord(tag)
    for d in range(7):
        a[:, 1 + d] = 48 + (idx // 10 ** d) % 10
    a[np.arange(kb)[None, :] >= lens[:, None]] = 0
    return a.view("S%d" % kb).reshape(-1)


def str_keys_in_sub(rng, count, kb, S, subs, tag="k", src_below=None):
    """`count` distinct stored key slots whose sub-bin at S is one of `subs` (word hash below src_below if given)"""
    n = max(4 * count * S, 1024)
    if src_below is not None:
        n = max(n, int(4 * count * ((1 << 64) / src_below)))
    c = str_candidates(rng, n, kb, tag)
    h = word_hash_np(c)
    ok = np.isin(mulhi_np(h, S), np.array(subs, dtype=np.uint64))
    if src_below is not None:
        ok &= h < np.uint64(src_below)
    c = c[ok]
    assert c.size >= count
    return list(rng.permutation(c)[:count])


def escape(k):
    return b"".join(b"\x01" + bytes([c + 1]) if c <= 1 else bytes([c]) for c in k)


def unescape(e):
    out, i = bytearray(), 0
    while i < len(e):
        if e[i] == 1 and i + 1 < len(e):
            out.append(e[i + 1] - 1)
            i += 2
        else:
            out.append(e[i])
            i += 1
    return bytes(out)


# ---- running a shuffle and checking it ----------------------------------------------------------------------------------

def shuffle(keys, vals, mkb=None, flags=0, reducer=mrhbm.RED_SUM):
    """one map job with the records (keys: u64 ints or stored key slots), one shuffle on P = 1"""
    if mkb is None:
        ctx = mrhbm.Ctx(mrhbm.KEY_U64, 1, flags=flags, reducer=reducer)
        recs = np.zeros(len(keys), dtype=mrhbm.record_dtype(mrhbm.KEY_U64))
        recs["key"] = np.array([int(k) for k in keys], dtype=np.uint64)
        recs["val"] = np.array([int(v) for v in vals], dtype=np.uint64)
    else:
        ctx = mrhbm.Ctx(mrhbm.KEY_STR, 1, mrhbm.PART_FNV_LUA, max_key_bytes=mkb, flags=flags, reducer=reducer)
        recs = np.zeros(len(keys), dtype=mrhbm.record_dtype(mrhbm.KEY_STR, mkb))
        recs["key"] = [bytes(k) for k in keys]
        recs["val"] = np.array([int(v) for v in vals], dtype=np.uint32)
    try:
        m = ctx.map_begin("sort-paths")
        m.emit_batch(recs)
        m.commit()
        ctx.shuffle()
    except Exception:
        ctx.close()
        raise
    return ctx


def check(ctx, keys, vals, reducer, u64=True):
    """the whole result against dict / sorted() references: result_copy (keys, sums, part_off), groups(0) in
    ascending key order, checksum parity with no key out of order or out of its bin"""
    keys = [int(k) if u64 else bytes(k) for k in keys]
    vals = [int(v) for v in vals]
    want = {}
    for k, v in zip(keys, vals):
        want.setdefault(k, []).append(v)
    order = sorted(want)
    info, st = ctx.result_info(), ctx.stats()
    gk, gs, po = ctx.result_copy()
    gk = [int(k) for k in gk.tolist()] if u64 else gk.tolist()
    gs = gs.tolist()
    n_rows = len(order) if reducer == mrhbm.RED_SUM else len(keys)
    assert info.groups == n_rows and po.tolist() == [0, n_rows]
    if reducer == mrhbm.RED_SUM:
        rows = [(k, sum(want[k])) for k in order]
    else:
        rows = sorted(zip(keys, vals))
    if info.sorted and reducer == mrhbm.RED_SUM:
        assert list(zip(gk, gs)) == rows
    else:
        assert sorted(zip(gk, gs)) == rows
        if info.sorted:
            assert gk == sorted(gk)
    got = list(ctx.groups(0))
    want_keys = [k.to_bytes(8, "big") if u64 else unescape(k) for k in order]
    assert [k for k, _ in got] == want_keys
    if reducer == mrhbm.RED_SUM:
        assert [v for _, v in got] == [[sum(want[k])] for k in order]
    else:
        assert [sorted(v) for _, v in got] == [sorted(want[k]) for k in order]
    cin, cout = ctx.checksum_input(), ctx.checksum_result()
    assert cin[:3] == cout[:3] and cin[3] == len(keys) and cout[3] == n_rows and cout[5] == 0
    if not (reducer == mrhbm.RED_NONE and st["big_bins"]):  # (group-only big bins are runs of cap rows)
        assert cout[4] == 0


def expect_stats(ctx, **want):
    st = ctx.stats()
    st["sorted"] = ctx.result_info().sorted
    assert {k: st[k] for k in want} == want, st


# ---- A. bucket crowding, u64, MINMAX form ------------------------------------------------------------------------------

def crowded_bucket(rng, base, m, flavour, width):
    """m keys in [base, base + 2^width) of one bucket: distinct 32-bit sort keys, pairs that tie on the sort key
    (same key >> (width - 20) ... differing in the low bits the sort key drops), or real duplicates"""
    drop = width - 20  # bits of the bucket's offset below the 32-bit sort key (sh0, with sh1 = 20)
    if flavour == "distinct":
        hi = rng.choice(1 << 20, m, replace=False)
        return [base + (int(h) << drop) + int(rng.integers(0, 1 << drop)) for h in hi]
    hi = rng.choice(1 << 20, (m + 1) // 2, replace=False)
    out = []
    for h in hi:
        a = base + (int(h) << drop)
        if flavour == "tie32":
            lo = rng.choice(1 << drop, 2, replace=False)
            out += [a + int(lo[0]), a + int(lo[1])]
        else:
            k = a + int(rng.integers(0, 1 << drop))
            out += [k, k]
    return out[:m]


SIZES_A = (4, 5, 8, 9)
FLAVOURS_A = ("distinct", "tie32", "dup")
A_VARIANTS = ["crowded", "crowded9", "full_range", "full_range9", "single"]


def build_a(variant, seed=1):
    """u64 keys of one bin (P = 1, n <= target: S = 1, the MINMAX form) and the bucket sizes the model expects.
    One bucket of 9 sends the whole bin to process_loaded, so the four-slot window and the exact walk are tested
    by bins whose buckets stop at 8, the fall-back by the "...9" variants."""
    rng = np.random.default_rng(seed + len(variant))
    if variant == "single":
        return [int(rng.integers(0, 1 << 64, dtype=np.uint64))], Counter({1: 1})
    sizes = SIZES_A if variant.endswith("9") else SIZES_A[:-1]
    if variant.startswith("crowded"):  # keys in [lo, lo + 2^44): sh0 = 12, sh1 = 20, bucket = (key - lo) >> 32
        lo = int(rng.integers(1 << 40, 1 << 62))
        width = 32
        free = rng.permutation(np.arange(1, NB_U64 - 1))
        keys = [lo, lo + 5 * (1 << 12) + 7, lo + 9 * (1 << 12), lo + 9 * (1 << 12)]  # bucket 0: the min, a duplicate
        top = lo + ((NB_U64 - 1) << 32)
        hi = lo + (1 << 44) - 1  # the max: its sort key is 0xFFFFFFFF, the sentinel value
        keys += [hi, hi - 1, top, top + 77 * (1 << 12), hi - (1 << 12)]  # bucket 4095: five, one tie with the max
        want = Counter({4: 1, 5: 1})
        nb = 0
        for m in sizes:
            for fl in FLAVOURS_A:
                for _ in range(5):
                    keys += crowded_bucket(rng, lo + (int(free[nb]) << width), m, fl, width)
                    want[m] += 1
                    nb += 1
        for b in free[nb:nb + 900]:  # one record per bucket
            keys.append(lo + (int(b) << width) + int(rng.integers(0, 1 << width)))
            want[1] += 1
    else:  # "full_range": keys 0 and 2^64 - 1, range 2^64 - 1: sh0 = 32, sh1 = 20, bucket = key >> 52
        width = 52
        free = rng.permutation(np.arange(1, NB_U64 - 1))
        keys = [0, 1, 1 << 32, (1 << 32) + 5]  # bucket 0
        # bucket 4095: three sort keys equal to the sentinels behind the bin, inside the four-slot window
        keys += [M64, M64 - 1, M64 - (1 << 32) + 1, M64 ^ (1 << 40)]
        want = Counter({4: 2})
        nb = 0
        for m in sizes:
            for fl in FLAVOURS_A:
                for _ in range(3):
                    keys += crowded_bucket(rng, int(free[nb]) << width, m, fl, width)
                    want[m] += 1
                    nb += 1
        for b in free[nb:nb + 300]:
            keys.append((int(b) << width) + int(rng.integers(0, 1 << width)))
            want[1] += 1
    keys = [keys[i] for i in rng.permutation(len(keys))]
    return keys, want


def check_a_model(variant, keys, want):
    assert pick_sub_bins(len(keys), 2048) == 1
    kk, bk = minmax_buckets(keys)
    assert Counter(Counter(bk).values()) == want
    assert (max(want) > KFIX_MAX) == variant.endswith("9")  # the pipelined kernel keeps the bin / falls back
    if variant != "single":
        assert kk[keys.index(max(keys))] == 0xFFFFFFFF
        ties = Counter(kk)
        assert any(ties[x] == 2 and len({k for k, y in zip(keys, kk) if y == x}) == 2 for x in ties)  # tie, not dup


@gpu
@pytest.mark.parametrize("flags", [0, mrhbm.F_NO_OPTIMISTIC])
@pytest.mark.parametrize("reducer", REDUCERS)
@pytest.mark.parametrize("variant", A_VARIANTS)
def test_a_bucket_crowding_minmax_form(variant, reducer, flags):
    """One bin (S = 1: the MINMAX form of the u64 kernel).  Buckets of exactly 1, 4 (the four-slot window), 5 (one
    past it: the exact walk), 8 (kFixMax) and, in a bin of its own, 9 (the whole bin falls back to process_loaded),
    built from distinct sort keys, from keys that tie on the 32-bit sort key and from real duplicates; the bin's min
    and max keys inside crowded buckets; keys 0 and 2^64 - 1 in one bin, whose top keys' sort keys equal the
    sentinel; a bin of one record."""
    keys, want = build_a(variant)
    check_a_model(variant, keys, want)
    vals = np.random.default_rng(2).integers(0, 1 << 40, len(keys)).tolist()
    with shuffle(keys, vals, flags=flags, reducer=reducer) as ctx:
        expect_stats(ctx, attempts=1, big_bins=0, sub_bins=1, sorted=1)
        check(ctx, keys, vals, reducer)


# ---- B. the hint form at the ends of key-ordered sub-bins ---------------------------------------------------------------

N_FOR_S = {3: 4700, 5: 8000, 7: 11500}  # n in ((S-1) * 1776, S * 1776], above the 4096 the sampled layout needs


def build_b(S, seed=3):
    """uniform keys (stratified: the sampled histogram stays flat) plus, for every k, floor(k 2^64 / S) and its
    neighbours, and 0 / 2^64 - 1"""
    rng = np.random.default_rng(seed + S)
    edges = [0, M64, 1, M64 - 1]
    for k in range(1, S):
        t = (k << 64) // S
        edges += [t - 1, t, t + 1, t + 2, t, t + 1]  # (t and t + 1 twice: sums across the sub-bin end)
    m = N_FOR_S[S] - len(edges)
    u = rng.random(m)
    fill = [((i << 64) + int(u[i] * (1 << 64))) // m for i in range(m)]
    keys = edges + fill
    return [keys[i] for i in rng.permutation(len(keys))]


def check_b_model(S, keys):
    assert pick_sub_bins(len(keys), 2048) == S and sample_is_uniform(keys)
    for k in range(1, S):
        t = (k << 64) // S
        assert mulhi(t, S) == k - 1 and mulhi(t + 1, S) == k  # floor(k 2^64 / S) is the LAST key of sub-bin k - 1
    assert max(Counter(mulhi(k, S) for k in keys).values()) <= 2048
    assert max(hint_bucket(k, S) for k in keys) < NB_U64  # the & (NB - 1) mask never wraps


@gpu
@pytest.mark.parametrize("reducer", REDUCERS)
@pytest.mark.parametrize("S", [3, 5, 7])
def test_b_hint_form_at_sub_bin_ends(S, reducer):
    """Key-ordered sub-bins of a sub-bin count that is not a power of two: the hint form takes bin k's keys to lie
    in [k q, k q + q + S), q = floor(2^64 / S).  Keys at both sides of every sub-bin end, and 0 and 2^64 - 1, must
    come out in one global order."""
    keys = build_b(S)
    check_b_model(S, keys)
    vals = np.random.default_rng(S).integers(0, 1 << 33, len(keys)).tolist()
    with shuffle(keys, vals, reducer=reducer) as ctx:
        expect_stats(ctx, attempts=1, big_bins=0, sub_bins=S, sorted=1)
        check(ctx, keys, vals, reducer)


# ---- C. bins of exactly cap and cap + 1 records ---------------------------------------------------------------------------

def spread(lo, hi, m, rng):
    """m keys spread evenly over [lo, hi)"""
    u = rng.random(m)
    return [lo + ((hi - lo) * i + int((hi - lo) * u[i])) // m for i in range(m)]


def build_c_u64(form, extra, seed=5):
    """S = 3 (n = 4648 + extra); sub-bin 0 holds cap + extra records: key-ordered ("hint": evenly spread keys below
    2^64 / 3) or hash-crafted ("minmax", F_FORCE_RUNS).  With extra = 1 the first two records are one duplicate
    pair, so that the merge round of k_big_bins leaves exactly cap records."""
    rng = np.random.default_rng(seed + extra)
    S, cap, rest = 3, 2048, 1300
    if form == "hint":
        ends = [-(-(k << 64) // S) for k in range(S + 1)]
        k0 = spread(ends[0], ends[1], cap + extra - 1 if extra else cap, rng)
        others = spread(ends[1], ends[2], rest, rng) + spread(ends[2], ends[3], rest, rng)
    else:
        k0 = [int(k) for k in u64_keys_in_sub(rng, cap + extra - 1 if extra else cap, S, [0])]
        others = [int(k) for k in u64_keys_in_sub(rng, 2 * rest, S, [1, 2])]
    keys = k0 + others
    keys = [keys[i] for i in rng.permutation(len(keys))]
    if extra:
        dup = k0[0]
        keys.remove(dup)
        keys = [dup, dup] + keys
    return keys


def build_c_str(mkb, extra, seed=7):
    """strings: S = 4, word-hash sub-bin 0 holds cap + extra records (a duplicate pair first when extra = 1)"""
    rng = np.random.default_rng(seed + mkb + extra)
    kb, cap = rb_of(mkb) - 4, cap_of(rb_of(mkb))
    target = int(cap - 6 * math.sqrt(cap))
    r = int((3.5 * target - cap) / 3)
    k0 = str_keys_in_sub(rng, cap + extra - 1 if extra else cap, kb, 4, [0], "a")
    others = str_keys_in_sub(rng, 3 * r, kb, 4, [1, 2, 3], "b")
    keys = k0 + others
    keys = [keys[i] for i in rng.permutation(len(keys))]
    if extra:
        keys.remove(k0[0])
        keys = [k0[0], k0[0]] + keys
    return keys


def check_c_model(keys, sub_of, cap, extra, big):
    """sub-bin 0 holds cap + extra records, no other more than cap; a big bin (cap + 1, its duplicate pair inside
    the first chunk) takes one merge round down to exactly cap"""
    cnt = Counter(sub_of(k) for k in keys)
    assert cnt[0] == cap + extra and max(c for s, c in cnt.items() if s) <= cap
    if extra and big:
        assert keys[0] == keys[1] and big_bin_rounds([k for k in keys if sub_of(k) == 0], cap) == [cap]


def c_expectations(form, extra, flags, reducer):
    """what shuffle_fast / shuffle_single_exact must do with the bin"""
    fast = not flags & mrhbm.F_NO_OPTIMISTIC
    if not extra:
        return dict(attempts=1, big_bins=0, sorted=int(form == "hint"))
    if form == "hint":  # the key-ordered bin overflows: hash sub-bins for good, the crafted bin spreads out
        return dict(attempts=2, big_bins=0, sorted=0)
    return dict(attempts=2 if fast else 1, big_bins=1, sorted=0)  # (optimistic overflow ->) exact layout, k_big_bins


@gpu
@pytest.mark.parametrize("flags", [0, mrhbm.F_NO_OPTIMISTIC])
@pytest.mark.parametrize("reducer", REDUCERS)
@pytest.mark.parametrize("extra", [0, 1])
@pytest.mark.parametrize("form", ["hint", "minmax"])
def test_c_u64_bin_at_cap_and_cap_plus_one(form, extra, reducer, flags):
    """A u64 bin of exactly cap records (every register slot of the pipelined kernel and the four sentinels at
    kk2[cap..cap+3]) and of cap + 1 (the optimistic layout overflows; the exact layout sorts it in k_big_bins, or,
    key-ordered, gives up ordered sub-bins)."""
    keys = build_c_u64(form, extra)
    S, cap = 3, 2048
    assert pick_sub_bins(len(keys), cap) == S
    check_c_model(keys, lambda k: u64_sub(k, S, form == "hint"), cap, extra, form == "minmax")
    if form == "hint":
        assert sample_is_uniform(keys)
        # after the overflow the exact layout uses hash sub-bins: no bin too large there
        assert max(Counter(u64_sub(k, S, False) for k in keys).values()) <= cap
    vals = np.random.default_rng(extra).integers(0, 1 << 36, len(keys)).tolist()
    f = flags | (mrhbm.F_FORCE_RUNS if form == "minmax" else 0)
    with shuffle(keys, vals, flags=f, reducer=reducer) as ctx:
        expect_stats(ctx, sub_bins=S, **c_expectations(form, extra, flags, reducer))
        check(ctx, keys, vals, reducer)


@gpu
@pytest.mark.parametrize("flags", [0, mrhbm.F_NO_OPTIMISTIC])
@pytest.mark.parametrize("extra", [0, 1])
@pytest.mark.parametrize("mkb", MKBS)
def test_c_string_bin_at_cap_and_cap_plus_one(mkb, extra, flags):
    """The same for string keys, 1024 / 512 / 256 records per bin: at cap the one-CTA sort, at cap + 1 k_big_bins
    with a final round of exactly cap records (u64 partial sums beside the records)."""
    keys = build_c_str(mkb, extra)
    cap, S = cap_of(rb_of(mkb)), 4
    assert pick_sub_bins(len(keys), cap) == S
    check_c_model(keys, lambda k: str_sub(k, S), cap, extra, True)
    vals = np.random.default_rng(mkb).integers(0xF0000000, 1 << 32, len(keys)).tolist()
    with shuffle(keys, vals, mkb=mkb, flags=flags) as ctx:
        expect_stats(ctx, sub_bins=S, **c_expectations("minmax", extra, flags, mrhbm.RED_SUM))
        check(ctx, keys, vals, mrhbm.RED_SUM, u64=False)


# ---- D. LSD boundaries, string keys ----------------------------------------------------------------------------------------

def flip(slot, bit):
    b = bytearray(slot)
    b[bit // 8] ^= 0x80 >> (bit % 8)
    return bytes(b)


def lsd_bits(kb):
    """bits (from the slot's most significant bit) on both sides of every 52-bit chunk boundary and every 32-bit
    word boundary, and the bits of the last byte a key can use (the slot's last byte is always its zero end)"""
    last = kb - 2
    bits = set()
    for step in (52, 32):
        for b in range(step, 8 * last + 8, step):
            bits |= {b - 1, b}
    bits |= set(range(8 * last, 8 * last + 8))
    return sorted(b for b in bits if b // 8 <= last)


def lsd_family(kb, first=b"p"):
    """a full-length key of lower-case letters (a single bit flip keeps every byte above 0x01), its one-bit
    neighbours, and keys with an escaped 0x00 / 0x01 at the byte of a 52-bit chunk boundary"""
    base = (first + bytes(97 + (7 * i) % 26 for i in range(1, kb - 1)))
    keys = [base] + [flip(base, b) for b in lsd_bits(kb)]
    for b in range(52, 8 * (kb - 2), 52):
        j = b // 8
        if 2 <= j and j + 1 <= kb - 2:
            keys += [base[:j] + escape(bytes([c])) + base[j + 2:] for c in (0, 1)]
    return keys


def build_d(mkb, kind, seed=9):
    rng = np.random.default_rng(seed + mkb)
    kb = rb_of(mkb) - 4
    fam = lsd_family(kb)
    if kind in ("mates8", "mates9"):
        keys = [fam[0]] + [k for k in fam if k[:8] == fam[0][:8]][1:int(kind[-1])]
    else:
        keys = list(fam)
        if kind == "wide":  # other prefixes far away: the general path's digit drops prefix bits
            keys += [bytes([c]) + k[1:] for c, k in zip(b"bgkmuz", (fam[3], fam[-1], fam[-2], fam[10], fam[0], fam[5]))]
        keys += [keys[int(i)] for i in rng.integers(0, len(keys), 8)]  # duplicates: sums
    assert all(0 not in k and len(k) < kb for k in keys)  # stored slots: NUL-free, the slot's last byte zero
    return [keys[i] for i in rng.permutation(len(keys))]


def check_d_model(mkb, kind, keys):
    cap = cap_of(rb_of(mkb))
    assert pick_sub_bins(len(keys), cap) == 1
    distinct = sorted(set(keys))
    bk, drop = counting_buckets(distinct, cap)
    mates = max(Counter(bk).values())  # distinct keys in the fullest counting bucket
    if kind in ("mates8", "mates9"):  # the counting path at its limit / one past it (the general path)
        assert len(keys) == len(distinct) == mates == int(kind[-1]) and len({k[:8] for k in keys}) == 1
    else:
        assert mates > KFIX_MAX and (drop == 0) == (kind == "near")


@gpu
@pytest.mark.parametrize("kind", ["near", "wide", "mates8", "mates9"])
@pytest.mark.parametrize("mkb", MKBS)
def test_d_lsd_passes_at_chunk_and_word_boundaries(mkb, kind):
    """String keys that share their first bytes and differ in one bit, beside every 52-bit chunk boundary and
    every 32-bit word boundary of the slot and in its last usable byte, plus escaped 0x00 / 0x01 bytes at the
    chunk boundaries.  "near": all prefixes within 2^52 (drop = 0, only the tie test sends the bin to the LSD
    passes); "wide": other prefixes too (drop > 0, the passes also reorder by chunk 0); 8 and 9 keys with one
    8-byte prefix: the counting path's mate limit and one past it."""
    keys = build_d(mkb, kind)
    check_d_model(mkb, kind, keys)
    vals = np.random.default_rng(len(keys)).integers(0, 1 << 32, len(keys)).tolist()
    with shuffle(keys, vals, mkb=mkb) as ctx:
        expect_stats(ctx, attempts=1, big_bins=0, sub_bins=1, sorted=1)
        check(ctx, keys, vals, mrhbm.RED_SUM, u64=False)


# ---- E. k_big_bins over several merge rounds ----------------------------------------------------------------------------

def build_e(mkb, flags, seed=11):
    """one bin of 5 cap records over 0.9 cap distinct keys, shuffled, all in hash sub-bin 0 at the S the shuffle
    picks; returns (keys, S, cap)"""
    rng = np.random.default_rng(seed + (mkb or 0) + flags)
    cap = cap_of(rb_of(mkb), flags)
    n, d = 5 * cap, int(0.9 * cap)
    S = pick_sub_bins(n, cap)
    if mkb is None:
        dk = [int(k) for k in u64_keys_in_sub(rng, d, S, [0])]
    else:
        dk = str_keys_in_sub(rng, d, rb_of(mkb) - 4, S, [0], "e")
    idx = np.concatenate([np.arange(d), rng.integers(0, d, n - d)])
    return [dk[i] for i in rng.permutation(idx)], S, cap


def check_e_model(keys, S, cap, sub_of):
    assert all(sub_of(k) == 0 for k in keys) and len(keys) > cap
    rng = np.random.default_rng(0)
    for order in [keys] + [[keys[i] for i in rng.permutation(len(keys))] for _ in range(20)]:
        rounds = big_bin_rounds(order, cap)
        assert rounds is not None and len(rounds) >= 2 and rounds[0] > cap, rounds  # every round merges; >= 2 rounds
    return big_bin_rounds(keys, cap)


@gpu
@pytest.mark.parametrize("reducer", REDUCERS)
@pytest.mark.parametrize("flags", [0, mrhbm.F_SMALL_BINS])
@pytest.mark.parametrize("mkb", [None] + MKBS)
def test_e_big_bin_merges_over_several_rounds(mkb, flags, reducer):
    """5 cap records over 0.9 cap keys in one bin: the first merge round leaves more than cap records, so later
    rounds read the partial sums the earlier ones wrote (string keys: u64 sums beside the records, at
    `side + chunk`).  String values are 0xFFFFFFFF: the partial sums pass 2^32 in the first round."""
    keys, S, cap = build_e(mkb, flags)
    u64 = mkb is None
    check_e_model(keys, S, cap, (lambda k: u64_sub(k, S, False)) if u64 else (lambda k: str_sub(k, S)))
    if u64:
        vals = np.random.default_rng(cap).integers(0, 1 << 40, len(keys)).tolist()
    else:
        vals = [0xFFFFFFFF] * len(keys)
    with shuffle(keys, vals, mkb=mkb, flags=flags | mrhbm.F_FORCE_RUNS, reducer=reducer) as ctx:
        expect_stats(ctx, attempts=2, big_bins=1, sub_bins=S, sorted=0)
        check(ctx, keys, vals, reducer, u64=u64)


# ---- F. the skew retry and MRHBM_E_SKEW --------------------------------------------------------------------------------

F_N = 150  # distinct keys; F_SMALL_BINS: cap 96, S = ceil(150 / 37) = 5


def build_f(mkb, widen_ok, seed=13):
    """F_N distinct keys in hash sub-bin 0 at S = 5: split evenly over sub-bins 0 and 1 at 2S (the retry succeeds),
    or with a hash source below 2^64 / 16S (in sub-bin 0 at S, 2S, 4S, 8S and 16S: the host gives up)"""
    rng = np.random.default_rng(seed + (mkb or 0) + widen_ok)
    S = 5
    if mkb is None:
        if widen_ok:
            keys = [int(k) for k in np.concatenate([u64_keys_in_sub(rng, F_N // 2, 2 * S, [s]) for s in (0, 1)])]
        else:
            keys = [int(k) for k in u64_keys_in_sub(rng, F_N, 1, [0], src_below=(1 << 64) // (16 * S))]
    else:
        kb = rb_of(mkb) - 4
        if widen_ok:
            keys = str_keys_in_sub(rng, F_N // 2, kb, 2 * S, [0], "f") + str_keys_in_sub(rng, F_N // 2, kb, 2 * S, [1], "g")
        else:
            keys = str_keys_in_sub(rng, F_N, kb, 1, [0], "h", src_below=(1 << 64) // (16 * S))
    return [keys[i] for i in rng.permutation(len(keys))], S


def check_f_model(keys, S, sub_of, widen_ok):
    assert pick_sub_bins(len(keys), 96) == S and len(set(keys)) == len(keys)
    for s in [S, 2 * S] if widen_ok else [S, 2 * S, 4 * S, 8 * S, 16 * S]:
        c = Counter(sub_of(k, s) for k in keys)
        if s == S or not widen_ok:
            assert c == {0: len(keys)} and big_bin_rounds(keys, 96) is None  # one bin, nothing to merge: skew
        else:
            assert max(c.values()) <= 96


@gpu
@pytest.mark.parametrize("mkb", [None] + MKBS)
def test_f_skew_retry_widens_the_sub_bins(mkb):
    """More distinct keys in one bin than one CTA sorts: the merge round merges nothing (ERRF_SKEW) and the exact
    layout is retried with twice the sub-bins, which splits them."""
    keys, S = build_f(mkb, True)
    u64 = mkb is None
    sub_of = (lambda k, s: u64_sub(k, s, False)) if u64 else str_sub
    check_f_model(keys, S, sub_of, True)
    vals = np.random.default_rng(3).integers(0, 1 << 32, len(keys)).tolist()
    with shuffle(keys, vals, mkb=mkb, flags=mrhbm.F_SMALL_BINS | mrhbm.F_FORCE_RUNS) as ctx:
        expect_stats(ctx, attempts=3, big_bins=0, sub_bins=2 * S, sorted=0)  # optimistic, exact at S, exact at 2S
        check(ctx, keys, vals, mrhbm.RED_SUM, u64=u64)


@gpu
@pytest.mark.parametrize("mkb", [None] + MKBS)
def test_f_skew_gives_up_and_the_ctx_stays_usable(mkb):
    """Keys that stay in one bin at every sub-bin count the host tries (S .. 16S): MRHBM_E_SKEW.  The ctx is still
    usable: reset() and a normal shuffle give the right result."""
    keys, S = build_f(mkb, False)
    u64 = mkb is None
    sub_of = (lambda k, s: u64_sub(k, s, False)) if u64 else str_sub
    check_f_model(keys, S, sub_of, False)
    flags = mrhbm.F_SMALL_BINS | mrhbm.F_FORCE_RUNS
    if u64:
        ctx = mrhbm.Ctx(mrhbm.KEY_U64, 1, flags=flags)
    else:
        ctx = mrhbm.Ctx(mrhbm.KEY_STR, 1, mrhbm.PART_FNV_LUA, max_key_bytes=mkb, flags=flags)
    rng = np.random.default_rng(17)

    def emit(ks, vs):
        recs = np.zeros(len(ks), dtype=mrhbm.record_dtype(ctx.key_kind, mkb or 27))
        recs["key"] = [int(k) for k in ks] if u64 else [bytes(k) for k in ks]
        recs["val"] = vs
        m = ctx.map_begin("f")
        m.emit_batch(recs)
        m.commit()

    with ctx:
        emit(keys, [1] * len(keys))
        with pytest.raises(mrhbm.MrhbmError) as e:
            ctx.shuffle()
        assert e.value.code == -5
        ctx.reset()
        if u64:
            keys2 = [int(k) for k in rng.integers(0, 1 << 64, 3000, dtype=np.uint64)]
        else:
            keys2 = str_candidates(rng, 3000, rb_of(mkb) - 4, "n").tolist()
        keys2 += keys2[:500]
        vals2 = rng.integers(0, 1 << 31, len(keys2)).tolist()
        emit(keys2, vals2)
        ctx.shuffle()
        check(ctx, keys2, vals2, mrhbm.RED_SUM, u64=u64)


# ---- the model itself (no GPU) --------------------------------------------------------------------------------------------

def test_model_mix64_matches_the_oracle_splitmix64():
    rng = np.random.default_rng(1)
    for x in [0, 1, GOLD, M64, 1 << 63] + [int(v) for v in rng.integers(0, 1 << 64, 200, dtype=np.uint64)]:
        assert mix64(x) == O.splitmix64((x - GOLD) & M64)
        assert int(mix64_np(np.array([x], dtype=np.uint64))[0]) == mix64(x)


def test_model_mulhi_is_the_exact_high_word():
    rng = np.random.default_rng(2)
    xs = [0, 1, M64, 1 << 63, (1 << 64) // 3] + [int(v) for v in rng.integers(0, 1 << 64, 300, dtype=np.uint64)]
    ms = [1, 2, 3, 5, 7, 0xFFFFFFFF] + [int(v) for v in rng.integers(1, 1 << 32, 20)]
    for x in xs:
        for m in ms:
            assert mulhi(x, m) == (x * m) // (1 << 64)
            assert int(mulhi_np(np.array([x], dtype=np.uint64), m)[0]) == mulhi(x, m)


def test_model_hashes_match_the_oracle_partitioners():
    """MULHASH and the word hash against the oracle's partitioners (mulhi of the same hashes)"""
    rng = np.random.default_rng(3)
    for k in [int(v) for v in rng.integers(0, 1 << 64, 200, dtype=np.uint64)]:
        for P in (1, 7, 1024):
            assert mulhash_pid(k, P) == O.part_mulhash(k, P)
    slots = str_candidates(rng, 300, 60, "w")
    hv = word_hash_np(slots)
    for s, h in zip(slots.tolist(), hv.tolist()):
        assert word_hash(s) == h
        for P in (3, 15, 4096):
            assert mulhi(word_hash(s), P) == O.part_fnv64(s, P)


def test_model_places_every_construction():
    """the constructions the GPU cases run land where they are meant to (the GPU cases repeat these checks)"""
    for variant in A_VARIANTS:
        check_a_model(variant, *build_a(variant))
    for S in N_FOR_S:
        check_b_model(S, build_b(S))
    for form in ("hint", "minmax"):
        for extra in (0, 1):
            keys = build_c_u64(form, extra)
            assert pick_sub_bins(len(keys), 2048) == 3
            check_c_model(keys, lambda k: u64_sub(k, 3, form == "hint"), 2048, extra, form == "minmax")
    for mkb in MKBS:
        for extra in (0, 1):
            keys = build_c_str(mkb, extra)
            assert pick_sub_bins(len(keys), cap_of(rb_of(mkb))) == 4
            check_c_model(keys, lambda k: str_sub(k, 4), cap_of(rb_of(mkb)), extra, True)
        for kind in ("near", "wide", "mates8", "mates9"):
            check_d_model(mkb, kind, build_d(mkb, kind))
    for mkb in [None] + MKBS:
        for flags in (0, mrhbm.F_SMALL_BINS):
            keys, S, cap = build_e(mkb, flags)
            check_e_model(keys, S, cap, (lambda k: u64_sub(k, S, False)) if mkb is None else (lambda k: str_sub(k, S)))
        for ok in (True, False):
            keys, S = build_f(mkb, ok)
            check_f_model(keys, S, (lambda k, s: u64_sub(k, s, False)) if mkb is None else str_sub, ok)
