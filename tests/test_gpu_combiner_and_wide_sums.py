"""String-key sums past 2^32 on every path (hot keys in k_big_bins, the map-side combiner), and the combiner paths
the other tests do not reach: the 64- and 128-byte record classes, keys on the short / long table boundary, table
growth and the fall-back to raw pairs, and several committed ranges combined into one table.  Every expected
result comes from the CPU oracle (u64 sums) on the same seeded records."""
import numpy as np
import pytest

import mrhbm_loader
import oracle as O
from test_gpu_parity import check_vs_oracle_str, check_vs_oracle_u64, u64_records

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402

pytestmark = pytest.mark.gpu
U32MAX = 0xFFFFFFFF
OPART = {mrhbm.PART_FNV_LUA: O.PART_FNV_LUA, mrhbm.PART_WORDHASH: O.PART_FNV64}


def kbytes(mkb):
    return mrhbm.record_dtype(mrhbm.KEY_STR, mkb)["key"].itemsize


def cap_of(mkb, flags=0):
    return 96 if flags & mrhbm.F_SMALL_BINS else 32 * 1024 // (kbytes(mkb) + 4)


def records(keys, vals, mkb):
    """keys: an array of stored (escaped) key slots, vals: u32"""
    recs = np.zeros(len(keys), dtype=mrhbm.record_dtype(mrhbm.KEY_STR, mkb))
    recs["key"] = keys
    recs["val"] = vals
    return recs


def rand_words(rng, count, lo, hi, tag):
    """`count` distinct NUL-free words of lo..hi bytes (hi >= len(tag) + 7)"""
    lens = rng.integers(lo, hi + 1, count)
    fill = rng.integers(97, 123, (count, hi), dtype=np.uint8)
    return [(tag + b"%06d" % i + fill[i].tobytes())[:max(int(lens[i]), len(tag) + 6)] for i in range(count)]


def long_keys(idx, lens, kb):
    """distinct keys of lens[i] (13..kb) bytes built from the numbers idx (< 10^9), vectorised"""
    a = np.full((idx.size, kb), ord("q"), dtype=np.uint8)
    a[:, 0], a[:, 1] = ord("L"), ord("-")
    for d in range(9):
        a[:, 2 + d] = 48 + (idx // 10 ** d) % 10
    a[:, 11:] = 97 + (idx[:, None] + np.arange(kb - 11)) % 26
    a[np.arange(kb)[None, :] >= lens[:, None]] = 0
    return a.view("S%d" % kb).reshape(-1)


def shuffle_str(recs_by_job, mkb, P, partitioner, **kw):
    ctx = mrhbm.Ctx(mrhbm.KEY_STR, P, partitioner, max_key_bytes=mkb, **kw)
    for j, recs in enumerate(recs_by_job):
        m = ctx.map_begin(j)
        m.emit_batch(recs)
        m.commit()
    ctx.shuffle()
    return ctx


def snapshot(ctx):
    return [(p, k, v) for p in ctx.partitions() for k, v in ctx.groups(p)]


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


def check_vs_oracle_escaped(ctx, recs, P, partitioner):
    """check_vs_oracle_str for records whose key slots hold escaped 0x00 / 0x01 bytes: FNV-in-doubles hashes the
    original bytes, so those keys' partitions are recomputed from the unescaped key; the iterator hands keys back
    unescaped, result_copy in the stored form"""
    raw = recs.view(np.uint8).reshape(len(recs), -1)
    okeys, osum, po = O.groupby_rec(raw, OPART[partitioner], P)
    part = np.repeat(np.arange(P), np.diff(po.astype(np.int64)))
    rows = []
    for k, s, p in zip(okeys, osum.tolist(), part.tolist()):
        k = bytes(k).rstrip(b"\0")
        if b"\x01" in k and partitioner == mrhbm.PART_FNV_LUA:
            p = O.part_fnv_lua(unescape(k), P)
        rows.append((p, k, s))
    rows.sort()
    want_po = np.searchsorted([r[0] for r in rows], np.arange(P + 1), side="left")
    assert any(b"\x01" in r[1] for r in rows)
    info = ctx.result_info()
    assert info.groups == len(rows)
    gk, gs, gpo = ctx.result_copy()
    assert (gpo == want_po).all()
    for p in range(P):
        a, b = int(want_po[p]), int(want_po[p + 1])
        assert [(k, [v]) for k, v in ((unescape(r[1]), r[2]) for r in rows[a:b])] == list(ctx.groups(p))
        assert sorted(zip(gk[a:b].tolist(), gs[a:b].tolist())) == [(r[1], r[2]) for r in rows[a:b]]
    cin, cout = ctx.checksum_input(), ctx.checksum_result()
    assert cin[:3] == cout[:3] and cout[3] == len(rows) and cout[4:] == [0, 0]


# ---- A1: hot string keys whose sums pass 2^32, no combiner (k_big_bins) --------------------------------------------

@pytest.mark.parametrize("flags", [0, mrhbm.F_NO_OPTIMISTIC, mrhbm.F_SMALL_BINS])
@pytest.mark.parametrize("mkb", [27, 59, 123])
def test_hot_string_keys_sum_past_32_bits(mkb, flags):
    """A key with more pairs than one bin holds is merged chunk by chunk in k_big_bins.  A chunk of cap pairs at
    0xFFFFFFFF (or at just enough that cap of them pass 2^32) sums past 32 bits in the first merge round; the
    partial sums must stay exact through every round.  Cold keys with 2-3 large values are the control (the
    one-CTA sort)."""
    rng = np.random.default_rng(mkb * 8 + flags)
    P, cap = 15, cap_of(mkb, flags)
    hot_a, hot_b = b"hot", b"H" * mkb
    cold = rand_words(rng, 300, 1, mkb, b"c")
    n_a, n_b = 4 * cap + 7, 5000
    keys = [hot_a] * n_a + [hot_b] * n_b
    vals = [U32MAX] * n_a + [(1 << 32) // cap + 1] * n_b
    for w in cold:
        r = int(rng.integers(2, 4))
        keys += [w] * r
        vals += rng.integers(0xFFFF0000, 1 << 32, r, dtype=np.uint64).tolist()
    perm = rng.permutation(len(keys))
    recs = records(np.array(keys, dtype="S%d" % kbytes(mkb))[perm], np.array(vals, dtype=np.uint64)[perm], mkb)
    with shuffle_str([recs[:3001], recs[3001:]], mkb, P, mrhbm.PART_FNV_LUA, flags=flags) as ctx:
        assert ctx.stats()["big_bins"] >= 1
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)
        got = dict((k, v[0]) for _, k, v in snapshot(ctx))
        assert got[hot_a] == n_a * U32MAX and got[hot_b] == n_b * ((1 << 32) // cap + 1)
    if flags == 0:  # group-only: every value of a hot key arrives untouched
        with shuffle_str([recs], mkb, P, mrhbm.PART_FNV_LUA, reducer=mrhbm.RED_NONE) as ctx:
            want = {}
            for k, v in zip(recs["key"].tolist(), recs["val"].tolist()):
                want.setdefault(k, []).append(v)
            got = {}
            for p, k, v in snapshot(ctx):
                assert k not in got
                got[k] = sorted(v)
            assert got == {k: sorted(v) for k, v in want.items()}


# ---- A2: string sums past 2^32 with the combiner -------------------------------------------------------------------

A2_CASES = ["shared_table", "global_table", "long_table", "single_values"]


@pytest.mark.parametrize("case", A2_CASES)
@pytest.mark.parametrize("mkb", [27, 59, 123])
def test_combiner_string_sums_past_32_bits(mkb, case):
    """>= 2^20 pairs: the combiner runs.  A hot key whose sum passes 2^32 -- summed in the shared-memory tables
    (values <= vcap), straight in the global table (values > 0xFFFF), in the long-key table (> 12 bytes) -- or a
    single value too large for the table's state word must give the exact sum, the same as without combiner."""
    rng = np.random.default_rng(1000 + mkb + A2_CASES.index(case))
    P, n = 15, (1 << 20) + 13
    kb = kbytes(mkb)
    vocab = rand_words(rng, 5000, 1, mkb, b"w")
    if case == "shared_table":
        special = {b"hotshort": (100_000, 50_000)}  # key: (pairs, value)
    elif case == "global_table":
        special = {b"hot-global12": (3000, 3_000_000)}  # exactly 12 bytes: still a short entry
    elif case == "long_table":
        special = {b"hot-long-" + b"k" * (mkb - 9): (3000, 3_000_000), b"hot-long-key-13": (2000, 2_500_000)}
    else:
        special = {b"one-fff0": (1, 0xFFFFFFF0), b"one-ffff": (1, U32MAX), b"one-long-key-ffffffff": (1, U32MAX),
                   b"two-ffff": (2, U32MAX)}
    ns = sum(c for c, _ in special.values())
    keys = np.array(vocab, dtype="S%d" % kb)[rng.integers(0, len(vocab), n - ns)]
    vals = rng.integers(1, 50, n - ns, dtype=np.uint64)
    keys = np.concatenate([keys] + [np.full(c, k, dtype="S%d" % kb) for k, (c, _) in special.items()])
    vals = np.concatenate([vals] + [np.full(c, v, dtype=np.uint64) for c, v in special.values()])
    perm = rng.permutation(n)
    recs = records(keys[perm], vals[perm], mkb)
    results = []
    for combiner in (True, False):
        with shuffle_str([recs], mkb, P, mrhbm.PART_FNV_LUA, combiner=combiner) as ctx:
            if combiner:
                assert ctx.stats()["ms_combine"] > 0
                check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)
            else:
                cin, cout = ctx.checksum_input(), ctx.checksum_result()
                assert cin[:3] == cout[:3]
            results.append(snapshot(ctx))
    assert results[0] == results[1]  # (the oracle's result, above)
    got = dict((k, v[0]) for _, k, v in results[0])
    for k, (c, v) in special.items():
        assert got[k] == c * v


# ---- A3: the combiner on the 64- and 128-byte record classes ---------------------------------------------------------

@pytest.mark.parametrize("partitioner", [mrhbm.PART_FNV_LUA, mrhbm.PART_WORDHASH])
@pytest.mark.parametrize("mkb", [59, 123])
def test_combiner_wide_records_vs_oracle(mkb, partitioner):
    """k_combine<64/128> + k_gtab_compact: Zipf-distributed words from a vocabulary mixed with words of 13..mkb
    bytes, keys at 12 / 13 bytes (the short / long table boundary), at 27 / 28 and at the class maximum, proper
    prefixes across the boundary, keys that escaping makes long, zero values, values past 0xFFFF (pairs x the
    largest value >= 2^32: the checked re-run), an odd pair count."""
    rng = np.random.default_rng(mkb + partitioner)
    P, n = 15, 1_500_017
    kb = kbytes(mkb)
    vocab = rand_words(rng, 20_000, 1, 12, b"") + rand_words(rng, 20_000, 13, mkb, b"long")
    special = [b"abcdefghijkl", b"abcdefghijklm", b"abcdefghijk", b"x" * 12, b"x" * 13, b"y" * 27, b"y" * 28,
               b"z" * mkb, b"z" * (mkb - 1), b"\x00" * 6, b"\x00" * 7, b"\x01" * 7, b"ab\x00cd\x01e", b"\x01" * 12,
               b"abcdefghijk\x00", b"abcdefghij\x01"]
    vocab += [escape(k) for k in special]
    assert max(len(k) for k in vocab) <= mkb
    w = 1.0 / np.arange(1, len(vocab) + 1) ** 1.1
    order = rng.permutation(len(vocab))  # (the Zipf ranks do not follow the vocabulary's order)
    idx = order[rng.choice(len(vocab), n - 400 * len(special), p=w / w.sum())]
    idx = np.concatenate([idx, np.repeat(np.arange(len(vocab) - len(special), len(vocab)), 400)])
    rng.shuffle(idx)
    vals = rng.integers(0, 3000, n).astype(np.uint32)
    vals[::13] = 0
    vals[::97] = 70_000
    recs = records(np.array(vocab, dtype="S%d" % kb)[idx], vals, mkb)
    with shuffle_str([recs], mkb, P, partitioner, combiner=True) as ctx:
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.pairs_recv < n // 4, (info.pairs_recv, n)  # it combined
        check_vs_oracle_escaped(ctx, recs, P, partitioner)


# ---- A4: table growth and the fall-back to raw pairs ----------------------------------------------------------------

def test_combiner_table_growth_u64():
    """2.5 M distinct u64 keys, twice each: more than the 2^21-entry table takes.  The table grows and the stream
    still combines to one record per key (about)."""
    rng = np.random.default_rng(41)
    P, nk = 16, 2_500_000
    k = O.gen_u64(7, 0, nk)[0]
    keys = np.concatenate([k, k])[rng.permutation(2 * nk)]
    vals = rng.integers(0, 1 << 40, keys.size, dtype=np.uint64)
    with mrhbm.Ctx(mrhbm.KEY_U64, P, combiner=True) as ctx:
        m = ctx.map_begin(1)
        m.emit_batch(u64_records(keys, vals))
        m.commit()
        ctx.shuffle()
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.groups <= info.pairs_recv < 0.6 * keys.size
        check_vs_oracle_u64(ctx, keys, vals, P)


def second_shuffle_small_vocab(ctx, mkb, seed):
    """the same ctx after reset(): exact (whether it combines depends on what the ctx learnt)"""
    rng = np.random.default_rng(seed)
    n = (1 << 20) + 77
    vocab = rand_words(rng, 3000, 1, mkb, b"s")
    recs = records(np.array(vocab, dtype="S%d" % kbytes(mkb))[rng.integers(0, 3000, n)],
                   rng.integers(0, 1000, n).astype(np.uint32), mkb)
    ctx.reset()
    m = ctx.map_begin("again")
    m.emit_batch(recs)
    m.commit()
    ctx.shuffle()
    check_vs_oracle_str(ctx, recs, ctx.num_partitions, O.PART_FNV_LUA)


def test_combiner_long_table_growth_strings():
    """150 k distinct keys of 13..27 bytes, 8 pairs each: more than the 2^17-entry long-key table takes"""
    rng = np.random.default_rng(43)
    P, nk, mkb = 15, 150_000, 27
    idx = np.repeat(np.arange(nk), 8)
    rng.shuffle(idx)
    keys = long_keys(np.arange(nk), rng.integers(13, 28, nk), 28)[idx]
    recs = records(keys, rng.integers(1, 1 << 20, idx.size).astype(np.uint32), mkb)
    with shuffle_str([recs], mkb, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.groups <= info.pairs_recv < 0.6 * idx.size
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)
        second_shuffle_small_vocab(ctx, mkb, 44)


def test_combiner_falls_back_to_raw_pairs():
    """2^22 + 300 k distinct long keys, one pair each: more than the long-key table holds at its largest size.
    The combine is given up and the raw pairs take the partition / sort / reduce stages."""
    rng = np.random.default_rng(45)
    P, nk, mkb = 15, (1 << 22) + 300_000, 27
    keys = long_keys(rng.permutation(nk), rng.integers(13, 28, nk), 28)
    recs = records(keys, rng.integers(0, 1 << 31, nk).astype(np.uint32), mkb)
    with shuffle_str([recs], mkb, P, mrhbm.PART_FNV_LUA, combiner=True) as ctx:
        assert ctx.stats()["ms_combine"] > 0 and ctx.result_info().pairs_recv == nk
        check_vs_oracle_str(ctx, recs, P, O.PART_FNV_LUA)
        second_shuffle_small_vocab(ctx, mkb, 46)


# ---- A5: several committed ranges into one table ---------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["str27", "str123", "u64"])
def test_combiner_several_sources(kind):
    """One k_combine launch per committed range, into one table: job A, job B, job A again with other pairs (a hole
    in the pool), an aborted job C, an empty job D.  The result is the oracle's over the live pairs only."""
    rng = np.random.default_rng(len(kind))
    P = 15
    sizes = {"A": 400_001, "B": 700_003, "A2": 500_009, "C": 300_007}
    if kind == "u64":
        vocab = O.gen_u64(9, 0, 40_000)[0]
        make = {j: u64_records(vocab[rng.integers(0, vocab.size, s)], rng.integers(0, 1 << 36, s, dtype=np.uint64))
                for j, s in sizes.items()}
        ctx = mrhbm.Ctx(mrhbm.KEY_U64, P, combiner=True)
    else:
        mkb = 27 if kind == "str27" else 123
        vocab = np.array(rand_words(rng, 20_000, 1, 12, b"") + rand_words(rng, 20_000, 13, mkb, b"lk"),
                         dtype="S%d" % kbytes(mkb))
        make = {j: records(vocab[rng.integers(0, vocab.size, s)], rng.integers(0, 5000, s).astype(np.uint32), mkb)
                for j, s in sizes.items()}
        ctx = mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=mkb, combiner=True)
    with ctx:
        for job, part in (("A", "A"), ("B", "B"), ("A", "A2")):
            m = ctx.map_begin(job)
            m.emit_batch(make[part])
            m.commit()
        m = ctx.map_begin("C")
        m.emit_batch(make["C"])
        m.abort()
        ctx.map_begin("D").commit()
        ctx.shuffle()
        live = np.concatenate([make["B"], make["A2"]])
        info = ctx.result_info()
        assert ctx.stats()["ms_combine"] > 0 and info.pairs_in == live.size and info.pairs_recv < live.size // 2
        if kind == "u64":
            check_vs_oracle_u64(ctx, live["key"], live["val"], P)
        else:
            check_vs_oracle_str(ctx, live, P, O.PART_FNV_LUA)
