"""The number-sum combiner (MRHBM_COMBINE_FSUM) branch by branch, at the edges between its branches.

Which kernel splits a key's sum is decided by its value count: k_fsum_sum splits a key of 1 or 2 values in one thread
(two_split) and one of 3 .. 4096 values in one warp (warp_acc, then acc_split); k_fsum_big spreads a longer key's
4096-value chunks over every warp of a fixed grid (sm_count * 6 CTAs of 2 warps) and k_fsum_big_split splits it.  A key
whose sum overflows keeps its values, which the host places with k_fsum_copy.  All of it runs over the job's open ranges
cut into 256-record tiles, on a linear-probing set of max(1024, pow2 >= 2n) entries, with a tile scan that takes
several CTAs from 3073 tiles on.  A model (pure Python: the path of a count, the chunk rotation, the tiles, the scan,
the key fingerprint and the probe chain restated) says where each construction lands, and the CPU tests below check the
constructions alone.

The API cannot read a committed value back, so the GPU tests read it through the reducer with residual probes: a key K
with values V whose split is t1 .. tk (expected(V)) has probe keys K.1 .. K.k+1 that carry V too, and a second job adds
-t1 .. -t(j-1) to K.j (all of -t1 .. -tk to K.k+1).  After the shuffle K.j must be exactly t_j and K.k+1 exactly +0.0,
which holds only when the pairs committed for V sum to exactly sum(V).  With pool_read after every commit (the keys in
first-pair order, expected()'s term count per key, fresh consecutive ids) and the bit-identical results of a ctx without
the combiner (run_both), that pins each committed split down."""
import itertools
import math
import random
from fractions import Fraction

import numpy as np
import pytest

import mrhbm_loader
from test_fsum_combiner_host import cases, expected, run_native, split_cases
from test_gpu_fsum_combiner import commit_job, ctx_pair, expected_layout, results, run_both
from test_gpu_fsum_reducer import BIG, INVAL, TINY, bits, enc, oracle, want_sums
from test_gpu_sort_paths import mix64

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402

gpu = pytest.mark.gpu
M64 = (1 << 64) - 1
WARP_VALUES = 4096    # kFsumWarpValues: the longest key one warp splits, and k_fsum_big's chunk
WARPS_PER_SM = 12     # k_fsum_big: sm_count * 6 CTAs of 2 warps
TILE = 256            # kDistinctTile
SCAN_CTA_TILES = 3072  # launch_exscan: one CTA for fewer than 4 x 1024 tile counts
KINDS = [mrhbm.KEY_STR, mrhbm.KEY_U64]


# ---- the placement model ---------------------------------------------------------------------------------------------

def path_of(n):
    """the branch that splits a key of n values"""
    return "thread" if n <= 2 else "warp" if n <= WARP_VALUES else "grid"


def chunk_warps(k, n, W):
    """k_fsum_big's loop for the k-th listed big key of n values on W warps: the warp of each chunk"""
    nch = -(-n // WARP_VALUES)
    out = [None] * nch
    for gw in range(W):
        for ch in range((gw + W - k % W) % W, nch, W):
            assert out[ch] is None
            out[ch] = gw
    return out


def table_entries(n):
    T = 1024
    while T < 2 * n:
        T <<= 1
    return T


def tiles(lengths):
    """(range, first record in the range, records) of every tile of a job whose open ranges hold `lengths` records"""
    return [(k, j, min(TILE, ln - j)) for k, ln in enumerate(lengths) for j in range(0, ln, TILE)]


def scan_ctas(ntiles):
    nb = -(-ntiles // 1024)
    return nb if nb >= 4 else 1


def fp_step(h, x):
    h = ((h ^ x) * 0x9E3779B97F4A7C15) & M64
    return h ^ (h >> 29)


def key_words(rb):
    return 2 if rb == 16 else rb // 4 - 1


def key_fingerprint(words, rb):
    """key_fingerprint<RB> of mrhbm_job_tiles.cuh over the key slot's u32 words"""
    kw = key_words(rb)
    h = 0x5851F42D4C957F2D
    for i in range(0, kw, 2):
        h = fp_step(h, words[i] | (words[i + 1] << 32 if i + 1 < kw else 0))
    h = mix64(h)
    return 0 if h == M64 else h


def slot_words(key, rb):
    """the key slot of a plain key (ASCII without escapes, or a u64) as the pool holds it; the GPU test checks it against
    pool_read"""
    raw = key.to_bytes(8, "little") if rb == 16 else key.ljust(4 * key_words(rb), b"\0")
    return [int.from_bytes(raw[i:i + 4], "little") for i in range(0, len(raw), 4)]


def pool_words(recs):
    return recs.view(np.uint32).reshape(len(recs), -1).tolist()


def place(fps, mask):
    """linear probing of the distinct fingerprints, one after the other: their slots (the cluster a group of keys fills
    does not depend on the order of their claims)"""
    taken, out = {}, {}
    for fp in fps:
        if fp in out:
            continue
        s = fp & mask
        while s in taken:
            s = (s + 1) & mask
        taken[s] = fp
        out[fp] = s
    return out


# ---- values ----------------------------------------------------------------------------------------------------------

def enc_np(vals):
    """enc() of many doubles at once: rows of 11 bytes"""
    b = np.ascontiguousarray(vals, dtype=np.float64).view(np.uint64)
    u = np.where((b >> np.uint64(63)) != 0, ~b, b | np.uint64(1 << 63))
    out = np.empty((b.size, 11), np.uint8)
    out[:, 0] = 0x10
    for k in range(10):
        out[:, 1 + k] = (np.uint64(0x80) | ((u >> np.uint64(63 - 7 * k)) & np.uint64(0x7F))).astype(np.uint8)
    return out


def emit_np(m, ctx, keys, vals, blob=None):
    recs = np.zeros(len(vals), dtype=mrhbm.record_dtype(ctx.key_kind, ctx.cfg.max_key_bytes))
    recs["key"] = keys
    blob = enc_np(vals) if blob is None else blob
    m.emit_batch_values(recs, blob.ravel(), np.arange(len(vals) + 1, dtype=np.uint64) * 11)


def dyadic(rng, n, exps=(0, -40, -80)):
    """n doubles m * 2^e (0 < |m| < 2^20, e in exps) and their class sums, exact doubles (each below 2^53) whose exact
    sum is the values' own: what expected() and oracle() take in place of millions of values"""
    m = rng.integers(1, 1 << 20, n) * rng.choice(np.array([-1, 1]), n)
    e = rng.choice(np.array(exps), n)
    vals = m.astype(np.float64) * np.exp2(e)
    proxy = [float(int(m[e == x].sum())) * 2.0 ** x for x in exps]
    return vals, proxy


def padded(vals, total, rng, z=None):
    """vals among +-z pairs (and one 0.0 when the parity needs it), total values in all, shuffled"""
    out = list(vals)
    if (total - len(out)) % 2:
        out.append(0.0)
    while len(out) < total:
        x = z if z is not None else rng.choice((-1, 1)) * (1 + rng.random()) * 2.0 ** rng.randrange(-60, 60)
        out += [x, -x]
    rng.shuffle(out)
    return out


def key_maker(kind):
    """the key of a case's name and probe number j (0: the case's own key)"""
    if kind == mrhbm.KEY_STR:
        return lambda name, j=0: b"%s.%d" % (name.encode(), j)
    ids = {}
    return lambda name, j=0: (ids.setdefault(name, len(ids) + 1) << 8) | j


def with_probes(named, key, rng=None):
    """job A: each case's values under its key and its probe keys (shuffled when rng is given), job B: the probes'
    subtractions, and what the shuffle must give for each of those keys"""
    a, b, reads = [], [], {}
    for name, vals in named:
        e = expected(vals)
        assert e is not None, name
        k0 = key(name)
        a += [(k0, v) for v in vals]
        reads[k0] = bits(oracle(vals))
        if e == "keep" or not all(math.isfinite(t) for t in e):
            continue
        for j in range(1, len(e) + 2):
            a += [(key(name, j), v) for v in vals]
            b += [(key(name, j), -t) for t in e[:j - 1]]
            reads[key(name, j)] = bits(e[j - 1] if j <= len(e) else 0.0)
    if rng is not None:
        rng.shuffle(a)
    return a, b, reads


def probe_cases():
    """split_cases() + cases() without the ones whose commit fails; their indices name them"""
    return [("c%d" % i, v) for i, v in enumerate(split_cases() + cases()) if expected(v) is not None]


def adversarial_cases():
    """split_cases()'s hand-written edges (ties, half-ulp pairs, 2^1024 - 2^970, subnormals) and every 40th other case"""
    n0 = len([v for v in cases() if len(v) <= 250])
    named = probe_cases()
    hand = {"c%d" % i for i in range(n0, n0 + 33)}
    return [(n, v) for i, (n, v) in enumerate(named) if n in hand or i % 40 == 0]


def pad_cases(total, seed=3):
    rng = random.Random(seed + total)
    pool = probe_cases() if total <= 3 else adversarial_cases()
    return [("p%d.%s" % (total, n), padded(v, total, rng)) for n, v in pool if len(v) <= total]


COUNTS = [1, 2, 3, 32, 33, 4095, 4096, 4097, 8192, 8193]
BIG_KEYS = [WARP_VALUES + 100, 2 * WARP_VALUES + 1, 3 * WARP_VALUES + 4095]  # each with a partial last chunk


def count_cases(seed=5):
    rng = np.random.default_rng(seed)
    return [("n%d" % n, dyadic(rng, n)[0].tolist()) for n in COUNTS] + \
        [("big%d" % n, dyadic(rng, n)[0].tolist()) for n in BIG_KEYS]


def flag_cases():
    """signed zeros, infinities, both ends of the accumulator and exact cancellation, on each path"""
    rng = random.Random(7)
    out = [("negz-1", [-0.0]), ("inf-1", [math.inf])]
    for n in (2, 3000, 9000):
        xs = [rng.choice((-1, 1)) * (1 + rng.random()) * 2.0 ** rng.randrange(-1000, 1000) for _ in range((n - 1) // 2)]
        canc = xs + [-x for x in xs] + [TINY] + [0.0] * (n - 1 - 2 * len(xs))
        if n == 2:
            canc = [2.2250738585072014e-308, -(2.2250738585072014e-308 - TINY)]
        m = n // 4
        ends = [2.0 ** 1023] * m + [-2.0 ** 1023] * m + [TINY] * (n - 2 * m - 1) + [BIG]
        if n == 2:
            ends = [TINY, 2.0 ** 1023]
        for name, vals in (("negz", [-0.0] * n), ("negzpos", [-0.0] * (n - 1) + [0.0]),
                           ("inf", [math.inf] + [rng.uniform(-1e300, 1e300) for _ in range(n - 1)]),
                           ("ends", ends), ("cancel", canc)):
            if name != "negzpos":
                rng.shuffle(vals)
            out.append(("%s-%d" % (name, n), vals))
    return out


def kept_cases():
    """keys whose |sum| >= 2^1024 - 2^970 on every path, and what a later job adds to bring each back into range"""
    keep = [("k2", [BIG, BIG]), ("kn2", [-BIG, -BIG]), ("k3", [BIG, BIG, 2.0 ** 1000]),
            ("k100", [BIG] * 60 + [-BIG] * 40), ("k4096", [BIG] * 2100 + [-BIG] * 1996),
            ("k4097", [-BIG] * 2100 + [BIG] * 1997), ("k6000", [BIG] * 3100 + [-BIG] * 2900)]
    back = {"k2": [-BIG, -1e300], "kn2": [BIG, 0.5], "k3": [-BIG, -BIG], "k100": [-BIG] * 20 + [1.0],
            "k4096": [-BIG] * 104 + [0.5], "k4097": [BIG] * 103 + [TINY], "k6000": [-BIG] * 200 + [-3.0]}
    return keep, back


def kept_job(key):
    """job A in five ranges (the second of one record) with every kept key's values dealt over several of them, among
    split keys and fillers; job B's batches between A's; the job that brings the kept sums back"""
    rng = random.Random(8)
    keep, back = kept_cases()
    split = [("s3", [1.0, 2.0 ** -60, -3.5]), ("s2", [0.1, 0.2]),
             ("s5000", dyadic(np.random.default_rng(2), 5000)[0].tolist())]
    a_chunks = [[] for _ in range(5)]
    for i, (n, vs) in enumerate(keep + split):
        for j, v in enumerate(vs):
            a_chunks[(0, 2, 3, 4)[(i + j) % 4]].append((key(n), v))
    a_chunks[1].append((key("k3"), a_chunks[0].pop(next(j for j, (k, _) in enumerate(a_chunks[0]) if k == key("k3")))[1]))
    for _ in range(800):
        a_chunks[rng.choice((0, 2, 3, 4))].append((key("f%d" % rng.randrange(300)), rng.uniform(-9, 9)))
    for ch in a_chunks:
        rng.shuffle(ch)
    b_chunks = [[(key("f%d" % rng.randrange(300)), rng.uniform(-1, 1)) for _ in range(5)] for _ in a_chunks]
    c = [(key(n), v) for n, vs in back.items() for v in vs]
    return a_chunks, b_chunks, c


def range_chunks(pairs, sizes):
    out, i = [], 0
    for s in sizes:
        out.append(pairs[i:i + s])
        i += s
    assert i == len(pairs)
    return out


# ---- CPU: the constructions alone ------------------------------------------------------------------------------------

def test_numpy_encoding_is_the_bindings():
    vals = [v for vs in split_cases()[:300] for v in vs] + [-0.0, 0.0, math.inf, -math.inf, TINY, -BIG]
    assert [bytes(r) for r in enc_np(vals)] == [enc(v) for v in vals]


@pytest.mark.parametrize("name", ["cases", "counts", "flags", "padded"])
def test_probes_read_each_term(name):
    named = {"cases": probe_cases, "counts": count_cases, "flags": flag_cases,
             "padded": lambda: pad_cases(4097)[::6]}[name]()
    a, b, reads = with_probes(named, key_maker(mrhbm.KEY_STR))
    assert want_sums([a, b]) == reads
    n_probe = sum(1 for k in reads if not k.endswith(b".0"))
    assert n_probe >= len(named) // 2


def test_padding_keeps_each_sum_and_reaches_each_path():
    for total in (3, 4096, 4097, 2 * 4096 + 1):
        named = pad_cases(total)
        assert len(named) >= 40 and all(len(v) == total for _, v in named)
        assert path_of(total) == {3: "warp", 4096: "warp"}.get(total, "grid")
        base = dict(probe_cases())
        for n, v in named[:60]:
            src = base[n.split(".", 1)[1]]
            if all(math.isfinite(x) for x in src):
                assert sum(Fraction(x) for x in v) == sum(Fraction(x) for x in src)
    assert any(len(v) <= 2 for _, v in probe_cases())  # the thread path, unpadded


def test_counts_reach_each_path_and_chunk_edge():
    assert [path_of(n) for n in COUNTS] == ["thread"] * 2 + ["warp"] * 5 + ["grid"] * 3
    for k, n in enumerate(BIG_KEYS):
        assert n % WARP_VALUES and path_of(n) == "grid"
        for W in (114 * WARPS_PER_SM, 132 * WARPS_PER_SM):
            assert chunk_warps(k, n, W) == [(k + j) % W for j in range(-(-n // WARP_VALUES))]
    for W in (114 * WARPS_PER_SM, 132 * WARPS_PER_SM):
        n = W * WARP_VALUES + 4097
        ws = chunk_warps(0, n, W)
        assert len(ws) == W + 2 and n % WARP_VALUES == 1  # a partial last chunk of one value
        twice = [w for w in set(ws) if ws.count(w) == 2]
        assert sorted(twice) == [0, 1] and len(set(ws)) == W  # every warp busy, two of them take a second chunk
        # several big keys: each key's chunks start at its own warp, so a hot key's first chunks never share one
        assert {chunk_warps(k, 5 * WARP_VALUES, W)[0] for k in range(3)} == {0, 1, 2}


def test_dyadic_class_sums_are_exact():
    rng = np.random.default_rng(1)
    for n in (1, 7, 5000):
        vals, proxy = dyadic(rng, n)
        assert sum(Fraction(v) for v in vals.tolist()) == sum(Fraction(p) for p in proxy)
        assert expected(proxy) == expected(vals.tolist())
    vals, proxy = dyadic(rng, 200_000)
    assert len(expected(proxy)) >= 2  # a split of more than one term for the key with the most chunks


def test_tile_model_at_range_edges_and_the_scan_switch():
    ts = tiles([1, 255, 256, 257, 511, 1])
    assert [(k, j, c) for k, j, c in ts] == [(0, 0, 1), (1, 0, 255), (2, 0, 256), (3, 0, 256), (3, 256, 1),
                                             (4, 0, 256), (4, 256, 255), (5, 0, 1)]
    assert len(tiles([SCAN_CTA_TILES * TILE])) == 3072 and scan_ctas(3072) == 1
    assert len(tiles([SCAN_CTA_TILES * TILE + 1])) == 3073 and scan_ctas(3073) == 4
    assert table_entries(40) == 1024 and table_entries(512) == 1024 and table_entries(513) == 2048


def test_flag_and_kept_constructions():
    seen = {}
    for name, vals in flag_cases():
        kind, e = name.split("-")[0], expected(vals)
        if kind == "negzpos":
            assert [bits(t) for t in e] == [bits(0.0)], name
        elif kind == "negz":
            assert [bits(t) for t in e] == [bits(-0.0)], name
        elif kind == "inf":
            assert e == [math.inf], name
        elif kind == "cancel":
            assert e == [TINY], name
        else:
            assert len(e) == 2 and e[0] in (BIG, 2.0 ** 1023) and 0 < e[1] < 2.0 ** -1000, name
        seen.setdefault(kind, set()).add(path_of(len(vals)))
    assert all(p == {"thread", "warp", "grid"} for p in seen.values()), seen
    keep, back = kept_cases()
    assert {path_of(len(v)) for _, v in keep} == {"thread", "warp", "grid"}
    for n, v in keep:
        assert expected(v) == "keep" and math.isinf(oracle(v)), n
        assert math.isfinite(oracle(v + back[n])), n
    key = key_maker(mrhbm.KEY_STR)
    a_chunks, _, _ = kept_job(key)
    assert len(a_chunks[1]) == 1 and a_chunks[1][0][0] == key("k3")
    for n, v in keep:
        assert sum(1 for ch in a_chunks if any(k == key(n) for k, _ in ch)) >= 2, n
        assert sorted(x for ch in a_chunks for k, x in ch if k == key(n)) == sorted(v), n


def test_fingerprint_model_is_the_device_hash(tmp_path):
    rng = random.Random(2)
    lines, want = [], []
    for rb in (16, 32, 64, 128):
        for t in range(200):
            w = [rng.getrandbits(32) if t % 3 else rng.choice((0, 1, M64 >> 32)) for _ in range(key_words(rb))]
            lines.append("%d %s" % (rb, " ".join("%x" % x for x in w)))
            want.append(key_fingerprint(w, rb))
    got = run_native(tmp_path, "fsum_fingerprint_check.cu", "fsum_fingerprint_check", lines)
    assert [int(g, 16) for g in got] == want


def chain_keys(kind):
    """64 keys on one home slot (100) and 8 on the last slot, whose probes wrap to slot 0: (keys, home of each) for a
    job of at most 512 pairs (1024 entries)"""
    rb = 16 if kind == mrhbm.KEY_U64 else 32
    mask = table_entries(512) - 1
    want = {100: 64, mask: 8}
    out = []
    for c in itertools.count():
        k = (c * 0x9E3779B97F4A7C15 + 1) & M64 if rb == 16 else b"chain%d" % c
        h = key_fingerprint(slot_words(k, rb), rb) & mask
        if want.get(h, 0):
            want[h] -= 1
            out.append((k, h))
            if not any(want.values()):
                return out, mask, rb


@pytest.mark.parametrize("kind", KINDS, ids=["str", "u64"])
def test_probe_chain_constructions(kind):
    keys, mask, rb = chain_keys(kind)
    fps = [key_fingerprint(slot_words(k, rb), rb) for k, _ in keys]
    slots = place(fps, mask)
    home100 = sorted(slots[f] for f, (_, h) in zip(fps, keys) if h == 100)
    wrap = sorted(slots[f] for f, (_, h) in zip(fps, keys) if h == mask)
    assert home100 == list(range(100, 164))
    assert wrap == list(range(0, 7)) + [mask]
    pairs = chain_job(keys)
    assert len(pairs) <= 512 and table_entries(len(pairs)) == mask + 1


def chain_job(keys):
    rng = random.Random(4)
    pairs = [(k, rng.uniform(-4, 4) * 2.0 ** rng.randrange(-30, 30)) for i, (k, _) in enumerate(keys)
             for _ in range((1, 2, 3, 5)[i % 4])]
    rng.shuffle(pairs)
    return pairs


# ---- GPU -------------------------------------------------------------------------------------------------------------

def probed_both(named, kind, seed=1):
    """the cases as job A and their probes' subtractions as job B, on both ctxs: run_both checks every key, the probe
    keys included, against the oracle (test_probes_read_each_term: the probes then read each term)"""
    a, b, _ = with_probes(named, key_maker(kind), random.Random(seed))
    run_both([a, b], kind, batch=(0, 1))


@gpu
@pytest.mark.parametrize("kind", KINDS, ids=["str", "u64"])
def test_device_split_on_the_host_cases(kind):
    """every case of split_cases() + cases() as its own key, unpadded: two_split for 1 or 2 values, warp_acc +
    acc_split for more"""
    probed_both(probe_cases(), kind)


@gpu
@pytest.mark.parametrize("kind,total", [(mrhbm.KEY_STR, 3), (mrhbm.KEY_STR, 4096), (mrhbm.KEY_STR, 4097),
                                        (mrhbm.KEY_STR, 2 * 4096 + 1), (mrhbm.KEY_U64, 3), (mrhbm.KEY_U64, 4097)],
                         ids=["str-3", "str-4096", "str-4097", "str-8193", "u64-3", "u64-4097"])
def test_device_split_on_padded_cases(kind, total):
    """the same cases among +-z pairs: 3 and 4096 values on the warp path, 4097 and 8193 on the grid's chunks"""
    probed_both(pad_cases(total), kind)


@gpu
def test_counts_at_every_path_edge_next_to_small_keys():
    rng = random.Random(6)
    small = [("s%d" % i, [rng.uniform(-1, 1) for _ in range(rng.randrange(1, 4))]) for i in range(3000)]
    probed_both(count_cases() + small, mrhbm.KEY_STR)


@gpu
def test_a_key_with_more_chunks_than_the_grid_has_warps():
    import torch
    W = torch.cuda.get_device_properties(0).multi_processor_count * WARPS_PER_SM
    n = W * WARP_VALUES + 4097
    assert len(chunk_warps(0, n, W)) == W + 2
    vals, proxy = dyadic(np.random.default_rng(9), n)
    terms = expected(proxy)
    assert isinstance(terms, list) and len(terms) >= 2
    K, Z = 1 << 40, 1 << 41  # the key, and its probe whose sum must come back to +0.0
    rng = random.Random(9)
    small = [(rng.randrange(1, 1 << 20), rng.uniform(-5, 5)) for _ in range(3000)]
    keys_a = np.concatenate([np.full(n, K, np.uint64), np.full(n, Z, np.uint64),
                             np.array([k for k, _ in small], np.uint64)])
    vals_a = np.concatenate([vals, vals, np.array([v for _, v in small])])
    comb, plain = ctx_pair(mrhbm.KEY_U64)
    with comb, plain:
        for ctx in (comb, plain):
            m = ctx.map_begin("A")
            emit_np(m, ctx, keys_a, vals_a)
            m.commit()
        lay = [(K, len(terms)), (Z, len(terms))] + expected_layout(comb, small)
        nn = sum(c for _, c in lay)
        assert comb.checksum_input()[3] == nn
        recs = comb.pool_read(0, nn)
        assert [int(x) for x in recs["key"]] == [k for k, c in lay for _ in range(c)]
        ids = [int(x) for x in recs["val"]]
        assert ids == list(range(ids[0], ids[0] + nn))
        for ctx in (comb, plain):
            m = ctx.map_begin("B")
            emit_np(m, ctx, np.full(len(terms), Z, np.uint64), -np.array(terms))
            m.commit()
        got, want = results(comb), results(plain)
        assert got == want
        sums = {k: v[1][0] for k, v in got[0].items()}
        assert sums[K] == bits(oracle(proxy)) and sums[Z] == bits(0.0)
        assert {k: sums[k] for k, _ in small} == want_sums([small])


@gpu
def test_flags_and_zeros_on_each_path():
    probed_both(flag_cases(), mrhbm.KEY_STR)


@gpu
@pytest.mark.parametrize("n", [2, 3000, 5000])
@pytest.mark.parametrize("bad", ["nan", "notnum"])
def test_a_failed_commit_keeps_the_earlier_commit(n, bad):
    rng = random.Random(n)
    vals = [rng.uniform(-1, 1) for _ in range(n)]
    good = [(b"k", v) for v in vals] + [(b"o%d" % i, 1.5 * i) for i in range(50)]
    comb, plain = ctx_pair()
    with comb, plain:
        for ctx in (comb, plain):
            commit_job(ctx, "J", good, batch=True)
        before = comb.checksum_input()[3]
        if bad == "nan":
            vals[0], vals[-1] = math.inf, -math.inf
        blob = enc_np(vals)
        if bad == "notnum":
            blob[min(n - 1, 4500), 0] = 0x11  # (in the partial last chunk of the 5000-value key)
        m = comb.map_begin("J")
        emit_np(m, comb, [b"k"] * n, vals, blob)
        with pytest.raises(mrhbm.MrhbmError) as e:
            m.commit()
        assert e.value.code == INVAL
        assert ("+inf and -inf" if bad == "nan" else "not a number") in str(e.value)
        assert comb.checksum_input()[3] == before
        assert results(comb) == results(plain)
        later = [(b"k", 0.25), (b"k", 0.5), (b"o3", -4.5)]
        for ctx in (comb, plain):
            commit_job(ctx, "L", later)
        got = results(comb)
        assert got == results(plain)
        assert {k: v[1][0] for k, v in got[0].items()} == want_sums([good, later])


def run_interleaved(kind, a_chunks, b_chunks, after=()):
    """job A emitted in a_chunks and job B in b_chunks, batch by batch in turn on two open handles (so A's ranges are
    not adjacent), A committed first, then the jobs of `after`: pool layout after each commit, both ctxs bit-identical,
    the sums against the oracle"""
    comb, plain = ctx_pair(kind)
    jobs = [sum(a_chunks, []), sum(b_chunks, [])] + list(after)
    with comb, plain:
        for ctx in (comb, plain):
            ma, mb = ctx.map_begin("A"), ctx.map_begin("B")
            for ca, cb in itertools.zip_longest(a_chunks, b_chunks, fillvalue=[]):
                for m, c in ((ma, ca), (mb, cb)):
                    if c:
                        emit_np(m, ctx, [k for k, _ in c], [v for _, v in c])
            before = 0
            for j, pairs in enumerate(jobs):
                if j == 0:
                    ma.commit()
                elif j == 1:
                    mb.commit()
                else:
                    commit_job(ctx, "C%d" % j, pairs)
                if ctx is comb:
                    lay = expected_layout(comb, pairs)
                    n = sum(c for _, c in lay)
                    assert comb.checksum_input()[3] == before + n
                    recs = comb.pool_read(before, n)
                    keys = [int(x) for x in recs["key"]] if kind == mrhbm.KEY_U64 else [bytes(x) for x in recs["key"]]
                    assert keys == [k for k, c in lay for _ in range(c)], j
                    ids = [int(x) for x in recs["val"]]
                    assert ids == list(range(ids[0], ids[0] + n))
                    before += n
        got, want = results(comb), results(plain)
        assert got == want
        assert {k: v[1][0] for k, v in got[0].items()} == want_sums(jobs)
    return jobs


@gpu
@pytest.mark.parametrize("kind", KINDS, ids=["str", "u64"])
def test_kept_keys_across_ranges_on_every_path(kind):
    """kept keys of 2, 3 .. 4096 and more values, spread over five ranges of one job among split keys: k_fsum_copy's
    list crosses ranges; a later job brings every sum back into range, so each kept value is checked"""
    a_chunks, b_chunks, c = kept_job(key_maker(kind))
    run_interleaved(kind, a_chunks, b_chunks, after=[c])


@gpu
@pytest.mark.parametrize("kind", KINDS, ids=["str", "u64"])
def test_job_ranges_and_tile_edges(kind):
    """job A in six ranges of 1, 255, 256, 257, 511 and 1 records (8 tiles, two of them of one record); keys straddle
    every range edge, one key's first pair lies in the fifth range, one key spans them all"""
    key = key_maker(kind)
    rng = random.Random(12)
    sizes = [1, 255, 256, 257, 511, 1]
    n = sum(sizes)
    names = [None] * n
    edges = list(itertools.accumulate(sizes))[:-1]
    for i, e in enumerate(edges):
        names[e - 1] = names[e] = "edge%d" % i
    for p in range(n):
        if names[p] is None:
            names[p] = "late" if p > edges[3] + 100 and p % 7 == 0 else "all" if p % 3 == 0 else "w%d" % rng.randrange(40)
    a = [(key(nm), rng.uniform(-1, 1) * 2.0 ** rng.randrange(-40, 40)) for nm in names]
    a_chunks = range_chunks(a, sizes)
    first = {}
    for p, nm in enumerate(names):
        first.setdefault(nm, p)
    assert first["late"] > edges[3] and first["all"] < edges[0] + 3
    b_chunks = [[(key("w%d" % rng.randrange(60)), rng.uniform(-1, 1)) for _ in range(1 + i)] for i in range(6)]
    run_interleaved(kind, a_chunks, b_chunks)


@gpu
@pytest.mark.parametrize("n", [SCAN_CTA_TILES * TILE, SCAN_CTA_TILES * TILE + 1], ids=["3072tiles", "3073tiles"])
def test_jobs_on_either_side_of_the_tile_scan_switch(n):
    rng = random.Random(n)
    nkeys = 150_000
    pairs = [(b"t%d" % rng.randrange(nkeys), rng.randrange(-1000, 1000) / 64) for _ in range(n - 1)]
    pairs.append((b"last", 0.5))  # the last tile's only record is a key's first pair
    assert scan_ctas(len(tiles([n]))) == (1 if n == SCAN_CTA_TILES * TILE else 4)
    run_both([pairs], batch=(0,))


@gpu
@pytest.mark.parametrize("kind", KINDS, ids=["str", "u64"])
def test_probe_chains_and_the_wrap(kind):
    keys, mask, rb = chain_keys(kind)
    pairs = chain_job(keys)
    comb, plain = ctx_pair(kind)
    with comb, plain:
        commit_job(plain, "words", pairs)
        words = pool_words(plain.pool_read(0, len(pairs)))
    fps = [key_fingerprint(w[:key_words(rb)], rb) for w in words]
    assert [w[:key_words(rb)] for w in words] == [slot_words(k, rb) for k, _ in pairs]
    home = {k: h for k, h in keys}
    assert [fp & mask for fp in fps] == [home[k] for k, _ in pairs]
    run_both([pairs, pairs[:40]], kind, batch=(1,))


@gpu
def test_scratch_is_reused_from_larger_commits():
    """one ctx: a 1M-pair job, a 40-pair job, a 70,000-pair job with two big keys, a replaced job; each step is checked
    in full, so a stale count, room, accumulator or table entry of a larger earlier commit would show"""
    rng = random.Random(13)
    named = adversarial_cases()
    comb, plain = ctx_pair()
    live, reads = {}, {}

    def step(job, pairs, probes=None):
        for ctx in (comb, plain):
            commit_job(ctx, job, pairs, batch=True)
        live[job] = pairs
        lay = expected_layout(comb, pairs)
        n = sum(c for _, c in lay)
        total = comb.checksum_input()[3]
        recs = comb.pool_read(total - n, n)
        assert [bytes(x) for x in recs["key"]] == [k for k, c in lay for _ in range(c)], job
        ids = [int(x) for x in recs["val"]]
        assert ids == list(range(ids[0], ids[0] + n))
        if probes:
            for ctx in (comb, plain):
                commit_job(ctx, job + "-probes", probes, batch=True)
            live[job + "-probes"] = probes
        got, want = results(comb), results(plain)
        assert got == want, job
        sums = {k: v[1][0] for k, v in got[0].items()}
        assert sums == want_sums(list(live.values())), job
        assert {k: sums[k] for k in reads} == reads, job

    def probed(prefix, sub):
        a, b, r = with_probes(sub, lambda name, j=0: b"%s%s.%d" % (prefix, name.encode(), j))
        reads.update(r)
        return a, b

    with comb, plain:
        a, b = probed(b"a", named[:20])
        big = [(b"h%d" % rng.randrange(50_000), rng.randrange(-99, 99) / 8) for _ in range(1_000_000 - len(a))]
        step("S1", big + a, b)
        a, b = probed(b"b", [("x", [1.0, 2.0 ** -60, 2.0 ** -120])])
        step("S2", a + [(b"h7", 0.5)] * (40 - len(a)), b)
        a, b = probed(b"c", named[20:40])
        vals = np.random.default_rng(3)
        big = [(b"B1", v) for v in dyadic(vals, 9000)[0].tolist()] + [(b"B2", v) for v in dyadic(vals, 30000)[0].tolist()]
        fill = [(b"f%d" % rng.randrange(4000), rng.uniform(-1, 1)) for _ in range(70_000 - len(big) - len(a))]
        s3 = big + fill + a
        rng.shuffle(s3)
        step("S3", s3, b)
        step("R", [(b"r%d" % (i % 900), i / 3) for i in range(5000)])
        step("R", [(b"r%d" % (i % 30), -i / 7) for i in range(700)])
