"""The range partitioner (MRHBM_PART_RANGE) against the CPU oracle.

Expected results come from the oracle's flat group-by (one partition, so one ascending key list) re-partitioned with
bisect_right over the splitters: partition k holds the keys that k splitters are <= to.  Every case also checks the
device's own parity sums (checksum_result: out[5] counts keys in the wrong partition) and the global key order."""
import bisect
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import mrhbm_loader  # noqa: E402

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm, synth  # noqa: E402

import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
M = mrhbm
U64_MAX = (1 << 64) - 1


def _checksums(ctx):
    cin, cout = ctx.checksum_input(), ctx.checksum_result()
    assert cout[5] == 0, "keys in the wrong partition: %d" % cout[5]
    assert cout[0:3] == cin[0:3], (cin, cout)


def _u64_ctx(P, splitters, combiner=False, flags=0, reducer=M.RED_SUM):
    ctx = M.Ctx(M.KEY_U64, P, M.PART_RANGE, device=0, combiner=combiner, flags=flags, reducer=reducer)
    if splitters is not None:
        ctx.set_splitters(splitters)
    return ctx


def _u64_expect(keys, vals, splitters, P):
    ok, osum, _ = O.groupby_u64(keys, vals, O.PART_MULHASH, 1)  # one partition: every key, ascending
    pid = np.searchsorted(np.asarray(splitters, dtype=np.uint64), ok, side="right")
    po = np.zeros(P + 1, dtype=np.uint64)
    po[1:] = np.cumsum(np.bincount(pid, minlength=P))
    return ok, osum, po


def _u64_check(ctx, keys, vals, splitters, P):
    ok, osum, opo = _u64_expect(keys, vals, splitters, P)
    gk, gs, gpo = ctx.result_copy()
    assert (gpo == opo).all(), "part_off differs"
    if ctx.result_info().sorted:
        assert (gk[1:] > gk[:-1]).all(), "not globally ascending"
    else:  # runs inside a partition: order them (partitions are already in key order)
        pid = np.repeat(np.arange(P), np.diff(gpo).astype(np.int64))
        o = np.lexsort((gk, pid))
        gk, gs = gk[o], gs[o]
    assert (gk == ok).all() and (gs == osum).all()
    _checksums(ctx)


def _emit_u64(ctx, keys, vals, job="m"):
    rec = np.empty(keys.size, dtype=M.record_dtype(M.KEY_U64))
    rec["key"], rec["val"] = keys, vals
    m = ctx.map_begin(job)
    m.emit_batch(rec)
    m.commit()


def _stream(n, extra=()):
    k, v = O.gen_u64(synth.SEED, 0, n)
    if extra:
        k = np.concatenate([k, np.asarray(extra, dtype=np.uint64)])
        v = np.concatenate([v, np.arange(1, len(extra) + 1, dtype=np.uint32)])
    return k, v


def _quantiles(P):
    return [int(((i << 64) // P)) for i in range(1, P)]


@pytest.mark.parametrize("P", [1, 2, 15, 1024])
def test_u64_even_quantiles(P):
    spl = _quantiles(P)
    extra = [0, U64_MAX] + spl[:8] + [s - 1 for s in spl[:8]]
    k, v = _stream(2_000_000, extra)
    with _u64_ctx(P, spl) as ctx:
        _emit_u64(ctx, k, v)
        ctx.shuffle()
        _u64_check(ctx, k, v, spl, P)
        if P > 1:
            assert ctx.result_info().sorted == 1, ctx.stats()  # range-relative key-ordered sub-bins on uniform keys


@pytest.mark.parametrize("flags", [0, M.F_FORCE_RUNS, M.F_SMALL_BINS, M.F_NO_OPTIMISTIC])
@pytest.mark.parametrize("combiner", [False, True])
def test_u64_flags_and_combiner(flags, combiner):
    P = 15
    spl = _quantiles(P)
    k, v = _stream(1_500_000, [0, U64_MAX] + spl)
    k = np.concatenate([k, k[:300_000]])  # repeated keys: the combiner has something to fold
    v = np.concatenate([v, v[:300_000]])
    with _u64_ctx(P, spl, combiner=combiner, flags=flags) as ctx:
        _emit_u64(ctx, k, v)
        ctx.shuffle()
        _u64_check(ctx, k, v, spl, P)


@pytest.mark.parametrize("combiner", [False, True])
def test_single_partition_needs_no_splitters(combiner):
    # P = 1: one key range, nothing to install; enough pairs for the sampled, key-ordered, multi-sub-bin path
    k, v = _stream(2_000_000, [0, U64_MAX])
    with _u64_ctx(1, None, combiner=combiner) as ctx:
        _emit_u64(ctx, k, v)
        ctx.shuffle()
        _u64_check(ctx, k, v, [], 1)
        assert ctx.stats()["sub_bins"] > 1
    words = [b"b", b"a", b"zz" * 20, b"a\x00", b"m"] * 1000
    _, counts = O.naive_wordcount([_words_text(words)])
    with M.Ctx(M.KEY_STR, 1, M.PART_RANGE, device=0) as ctx:
        m = ctx.map_begin("w")
        for w in words:
            m.emit(w, 1)
        m.commit()
        ctx.shuffle()
        assert [(key, vals[0]) for key, vals in ctx.groups(0)] == counts
        _checksums(ctx)


def test_checksum_refuses_other_splitters_than_the_shuffles():
    P = 4
    spl = _quantiles(P)
    k, v = _stream(100_000)
    with _u64_ctx(P, spl) as ctx:
        _emit_u64(ctx, k, v)
        ctx.shuffle()
        _checksums(ctx)
        ctx.set_splitters([1, 2, 3])
        with pytest.raises(M.MrhbmError) as e:
            ctx.checksum_result()
        assert e.value.code == -1
        ctx.set_splitters(spl)  # the shuffle's splitters again
        _checksums(ctx)


def test_u64_narrow_and_duplicate_splitters():
    # all splitters inside a narrow key range: one partition takes almost everything (the exact layout), and
    # duplicated splitters leave partitions empty
    P = 64
    lo = 1 << 62
    spl = sorted([lo + 1000 * (i // 3) for i in range(P - 1)])
    k, v = _stream(1_000_000, spl + [lo - 1, lo, U64_MAX, 0])
    with _u64_ctx(P, spl) as ctx:
        _emit_u64(ctx, k, v)
        ctx.shuffle()
        _u64_check(ctx, k, v, spl, P)
        # the sub-bins are sized from the fullest partition at once, not doubled attempt by attempt
        assert ctx.stats()["attempts"] <= 4, ctx.stats()


def test_u64_red_none():
    P = 15
    spl = _quantiles(P)
    k, v = _stream(200_000, spl[:4])
    k = np.concatenate([k, k[:50_000]])
    v = np.concatenate([v, v[:50_000]])
    with _u64_ctx(P, spl, reducer=M.RED_NONE) as ctx:
        _emit_u64(ctx, k, v)
        ctx.shuffle()
        ok, osum, opo = _u64_expect(k, v, spl, P)
        prev = None
        got_k, got_s = [], []
        for p in range(P):
            for key, vals in ctx.groups(p):
                kk = int.from_bytes(key, "big")
                assert bisect.bisect_right(spl, kk) == p
                assert prev is None or kk > prev
                prev = kk
                got_k.append(kk)
                got_s.append(sum(vals))
        assert got_k == [int(x) for x in ok] and got_s == [int(x) for x in osum]
        _checksums(ctx)


def test_u64_sampled_splitters():
    P, n = 16, 10_000_000
    with _u64_ctx(P, None) as ctx:
        m = ctx.map_begin("s")
        m.gen_u64(synth.SEED, 0, n)
        m.commit()
        spl = ctx.sample_splitters()
        assert spl == ctx.sample_splitters(), "sampling is not deterministic"
        assert len(spl) == P - 1 and spl == sorted(spl)
        ctx.shuffle()
        info = ctx.result_info()
        assert info.sorted == 1
        gk, gs, gpo = ctx.result_copy()
        assert (gk[1:] > gk[:-1]).all(), "result_copy is not globally ascending"
        assert np.diff(gpo).max() <= 1.5 * n / P
        ok, osum, opo = O.groupby_u64_stream(synth.SEED, 0, n, O.PART_MULHASH, 1)
        pid = np.searchsorted(np.asarray(spl, dtype=np.uint64), ok, side="right")
        opo = np.zeros(P + 1, dtype=np.uint64)
        opo[1:] = np.cumsum(np.bincount(pid, minlength=P))
        assert (gpo == opo).all() and (gk == ok).all() and (gs == osum).all()
        _checksums(ctx)
    # the sampled splitters reproduce the result through set_splitters on another ctx
    with _u64_ctx(P, spl) as ctx2:
        m = ctx2.map_begin("s")
        m.gen_u64(synth.SEED, 0, n)
        m.commit()
        ctx2.shuffle()
        gk2, gs2, gpo2 = ctx2.result_copy()
        assert (gk2 == gk).all() and (gs2 == gs).all() and (gpo2 == gpo).all()


# ---- string keys -------------------------------------------------------------------------------------------------
def _words_text(words):
    return b" ".join(words)


def _str_run(words, splitters, max_key_bytes, P, flags=0, combiner=False):
    """emits every word with value 1; compares groups() with naive_wordcount re-partitioned by bisect_right"""
    _, counts = O.naive_wordcount([_words_text(words)])
    want = [[] for _ in range(P)]
    for key, cnt in counts:  # ascending bytewise
        want[bisect.bisect_right(splitters, key)].append((key, cnt))
    with M.Ctx(M.KEY_STR, P, M.PART_RANGE, max_key_bytes=max_key_bytes, device=0, flags=flags, combiner=combiner) as ctx:
        ctx.set_splitters(splitters)
        m = ctx.map_begin("w")
        for w in words:
            m.emit(w, 1)
        m.commit()
        ctx.shuffle()
        got = [[(k, v[0]) for k, v in ctx.groups(p)] for p in range(P)]
        assert got == want
        flat = [k for part in got for k, _ in part]
        assert all(a < b for a, b in zip(flat, flat[1:])), "partitions 0..P-1 are not in one ascending key order"
        _checksums(ctx)


def _word_mix(kb, seed=7):
    """words around the interesting boundaries of a slot of kb bytes"""
    rng = np.random.default_rng(seed)
    letters = b"abcxyz\x00\x01\xff"
    words = []
    for _ in range(20_000):
        ln = int(rng.integers(1, kb + 1))
        words.append(bytes(rng.choice(list(letters[:6]), ln).astype(np.uint8)))
    base = b"m" * (kb - 1)
    words += [b"m", b"mm", base, base + b"m", base + b"mm", b"m" * (kb + 10),  # around a slot-long splitter
              b"a\x00", b"a\x01", b"a\x00\x01", b"a", b"\x00", b"\x01", b"\x01\x01",
              b"q" * (kb - 1) + b"\x00",  # escape pair across the slot boundary: a long key
              b"q" * (kb - 2) + b"\x01", b"q" * (kb - 1), b"q" * kb, b"q" * (kb + 3)]
    words += [b"z" * (kb + 40) + bytes([i]) for i in range(40, 50)]  # long host-side keys
    return words


@pytest.mark.parametrize("max_key_bytes", [27, 59, 123])
def test_str_splitter_shapes(max_key_bytes):
    kb = {27: 28, 59: 60, 123: 124}[max_key_bytes]
    P = 9
    base = b"m" * (kb - 1)
    spl = sorted([b"", b"a\x00", b"b", base, base + b"m", b"m" * (kb + 5), b"q" * (kb - 1) + b"\x00\x01",
                  b"z" * (kb + 40) + bytes([45])])
    _str_run(_word_mix(kb), spl, max_key_bytes, P)


@pytest.mark.parametrize("flags", [M.F_FORCE_RUNS, M.F_SMALL_BINS, M.F_NO_OPTIMISTIC])
def test_str_flags(flags):
    spl = [bytes([c]) for c in range(ord("b"), ord("z") + 1)]
    _str_run(_word_mix(28, seed=3), spl, 27, len(spl) + 1, flags=flags)


def test_str_zipf_sampled_and_combiner():
    P, n = 15, 3_000_000
    table = synth.zipf_table(1 << 14)
    with M.Ctx(M.KEY_STR, P, M.PART_RANGE, device=0, combiner=True) as ctx:
        m = ctx.map_begin("z")
        m.gen_zipf(synth.SEED, 0, n, table)
        m.commit()
        spl = ctx.sample_splitters()
        assert spl == ctx.sample_splitters()
        counts = O.zipf_counts(synth.SEED, 0, n, table, nthreads=4)
        okeys, osum, _ = O.wordcount_from_counts(counts, O.PART_FNV_LUA, 1)
        stream_keys = {bytes(k).rstrip(b"\0") for k in okeys}
        assert all(s in stream_keys for s in spl), "a sampled splitter is not a key of the stream"
        ctx.shuffle()
        want = sorted((bytes(k).rstrip(b"\0"), int(s)) for k, s in zip(okeys, osum))
        got = []
        for p in range(P):
            for k, v in ctx.groups(p):
                assert bisect.bisect_right(spl, k) == p
                got.append((k, v[0]))
        assert got == want
        _checksums(ctx)


# ---- errors -------------------------------------------------------------------------------------------------------
def test_errors_leave_the_ctx_usable():
    P = 4
    k, v = _stream(100_000)
    with _u64_ctx(P, None) as ctx:
        _emit_u64(ctx, k, v)
        with pytest.raises(M.MrhbmError) as e:
            ctx.shuffle()
        assert e.value.code == -1
        for bad in ([1, 2], [3, 2, 1], [b"\x00" * 7, b"\x00" * 8, b"\x01" * 8]):
            with pytest.raises(M.MrhbmError) as e:
                ctx.set_splitters(bad)
            assert e.value.code == -1
        spl = _quantiles(P)
        ctx.set_splitters(spl)
        ctx.shuffle()
        _u64_check(ctx, k, v, spl, P)
    with M.Ctx(M.KEY_STR, 3, M.PART_RANGE, device=0) as ctx:
        with pytest.raises(M.MrhbmError):
            ctx.set_splitters([b"b", b"a"])
        with pytest.raises(M.MrhbmError):
            ctx.set_splitters([b"a"])
        ctx.set_splitters([b"a", b"a"])  # duplicates are allowed
    with M.Ctx(M.KEY_U64, 3, M.PART_MULHASH, device=0) as ctx:
        with pytest.raises(M.MrhbmError):
            ctx.set_splitters([1, 2])  # not a range ctx
