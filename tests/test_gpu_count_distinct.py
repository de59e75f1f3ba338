"""MRHBM_RED_COUNT_DISTINCT: after the shuffle every key holds one value, the number of its distinct value bytes over
all map jobs, encoded as the 11-byte number of tuple.encode_value(float(n)).

Every expected result is computed on the host: len(set(value bytes)) per key over the live commits.  The same commits
also go to a MRHBM_RED_DISTINCT ctx: its keys must come out in the same order, its group sizes equal the counts."""
import ctypes as C
import random

import numpy as np
import pytest

import mrhbm_loader
from conftest import expand_tokens

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce import tuple as T  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.DocumentFrequency import init as DF  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WordCount import init as WordCount  # noqa: E402

gpu = pytest.mark.gpu
P = 7
INVAL = -1
DF_PKG = "lua_mapreduce_b200.mapreduce.examples.DocumentFrequency"
KINDS = [("u64", mrhbm.KEY_U64, 27), ("str27", mrhbm.KEY_STR, 27), ("str59", mrhbm.KEY_STR, 59),
         ("str123", mrhbm.KEY_STR, 123)]
FLAGS = [mrhbm.F_FORCE_RUNS, mrhbm.F_SMALL_BINS, mrhbm.F_NO_OPTIMISTIC,
         mrhbm.F_FORCE_RUNS | mrhbm.F_NO_OPTIMISTIC | mrhbm.F_SMALL_BINS]


def cd_ctx(kind=mrhbm.KEY_STR, max_key_bytes=27, combiner=mrhbm.COMBINE_NONE, flags=0, partitioner=None, parts=P,
           reducer=mrhbm.RED_COUNT_DISTINCT):
    kw = {} if partitioner is None else dict(partitioner=partitioner)
    return mrhbm.Ctx(kind, parts, max_key_bytes=max_key_bytes, device=0, reducer=reducer,
                     flags=mrhbm.F_BYTE_VALUES | flags, combiner=combiner, **kw)


def enc(n):
    return T.encode_value(float(n))


def want_counts(jobs):
    want = {}
    for pairs in jobs:
        for k, v in pairs:
            want.setdefault(k, set()).add(v)
    return {k: len(v) for k, v in want.items()}


def emit_jobs(ctx, jobs, batch=(), names=None):
    for j, pairs in enumerate(jobs):
        m = ctx.map_begin(names[j] if names else "job%d" % j)
        if j in batch:
            recs = np.zeros(len(pairs), dtype=mrhbm.record_dtype(ctx.key_kind, ctx.cfg.max_key_bytes))
            # records carry the stored form of a string key: 0x01 -> 01 02, 0x00 -> 01 01 (mrhbm_emit_str)
            recs["key"] = [k if isinstance(k, int) else k.replace(b"\x01", b"\x01\x02").replace(b"\x00", b"\x01\x01")
                           for k, _ in pairs]
            off = np.zeros(len(pairs) + 1, dtype=np.uint64)
            off[1:] = np.cumsum([len(v) for _, v in pairs])
            m.emit_batch_values(recs, b"".join(v for _, v in pairs), off)
        else:
            for k, v in pairs:
                m.emit(k, v)
        m.commit()


def read_groups(ctx):
    """[(key, values)] over the partitions in order, keys ascending inside each"""
    u64 = ctx.key_kind == mrhbm.KEY_U64
    out = []
    for p in ctx.partitions():
        part = [(int.from_bytes(k, "big") if u64 else k, vals) for k, vals in ctx.groups(p)]
        assert [k for k, _ in part] == sorted(k for k, _ in part)
        out += part
    return out


def check(ctx, want, long_keys=0, shuffle=True, pairs_recv=None):
    """groups, rows and result_info against want = {key: count}; returns the groups and the bulk rows"""
    if shuffle:
        ctx.shuffle()
    u64 = ctx.key_kind == mrhbm.KEY_U64
    groups = read_groups(ctx)
    assert all(len(vals) == 1 for _, vals in groups)
    assert dict((k, vals[0]) for k, vals in groups) == {k: enc(n) for k, n in want.items()}
    assert len(groups) == len(want)
    info = ctx.result_info()
    assert info.groups == len(want) - long_keys
    if pairs_recv is not None:
        assert info.pairs_recv == pairs_recv
    if long_keys:
        return groups, None
    keys, _, po = ctx.result_copy()
    blob, roff = ctx.result_values()
    assert (roff == np.arange(info.groups + 1, dtype=np.uint64) * 11).all()
    raw = blob.tobytes()
    rows = [(int(keys[r]) if u64 else bytes(keys[r]), raw[11 * r:11 * r + 11]) for r in range(info.groups)]
    if u64:
        assert sorted(rows) == sorted((k, enc(n)) for k, n in want.items())
    else:  # result_copy gives the stored (escaped) slots
        assert len(rows) == len(want) and len({k for k, _ in rows}) == len(rows)
    if info.sorted:
        for p in range(ctx.num_partitions):
            part = [k for k, _ in rows[int(po[p]):int(po[p + 1])]]
            assert part == sorted(part)
    return groups, rows


def against_distinct(jobs, kind=mrhbm.KEY_STR, mkb=27, flags=0, batch=()):
    """the same commits in a MRHBM_RED_DISTINCT ctx: [(key, group size)] in iteration order"""
    with cd_ctx(kind, mkb, flags=flags, reducer=mrhbm.RED_DISTINCT) as ctx:
        emit_jobs(ctx, jobs, batch=batch)
        ctx.shuffle()
        return [(k, len(v)) for k, v in read_groups(ctx)]


def as_counts(groups):
    return [(k, int(T.decode_value(v[0]))) for k, v in groups]


def value_mix():
    """strings, numbers (1 and 1.0 share their bytes, -0 and +0 do not), the empty value, prefixes, a value past the 4 MB
    stage"""
    big = random.Random(1).randbytes((4 << 20) + 77)
    mix = [b"", b"\x00", b"\x00\x00", b"a", b"ab", b"abc", b"file-a", b"file-b", big, big[:-1] + b"\x01"]
    mix += [T.encode_value(x) for x in (0, 0.0, -0.0, 1, 1.0, -1, 1.5, 2 ** 40, "file-a", b"file-b")]
    return mix


def mixed_jobs(keys, seed=7):
    rng = random.Random(seed)
    mix = value_mix()
    jobs = []
    for j in range(3):
        pairs = [(k, v) for k in keys[:3] for v in mix]  # every job, every value: the same bytes under many ids
        pairs += [(keys[3], b"one")]
        pairs += [(rng.choice(keys[4:]), rng.choice(mix[:8])) for _ in range(400)]
        pairs += [(keys[0], mix[3])] * 5
        rng.shuffle(pairs)
        jobs.append(pairs)
    return jobs


def str_keys(mkb):
    # keys with 0x00 / 0x01 (stored escaped), the longest key that fits, one byte less
    return [b"k%d" % i for i in range(36)] + [b"z\x00", b"z\x01", b"\x00\x00", b"\x01", b"w" * (mkb - 2),
                                              b"x" * (mkb - 3)]


def keys_of(kind, mkb):
    return list(range(0, 42 * 2 ** 50, 2 ** 50)) if kind == mrhbm.KEY_U64 else str_keys(mkb)


def test_value_mix_equality_rules():
    mix = value_mix()
    assert T.encode_value(1) == T.encode_value(1.0) and T.encode_value(0) == T.encode_value(0.0)
    assert T.encode_value(-0.0) != T.encode_value(0.0)
    assert len(set(mix)) == len(mix) - 2


@gpu
@pytest.mark.parametrize("combiner", [mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT], ids=["none", "distinct"])
@pytest.mark.parametrize("name,kind,mkb", KINDS, ids=[k[0] for k in KINDS])
def test_counts_by_value_bytes(name, kind, mkb, combiner):
    jobs = mixed_jobs(keys_of(kind, mkb))
    want = want_counts(jobs)
    assert want[keys_of(kind, mkb)[0]] == len(value_mix()) - 2
    with cd_ctx(kind, mkb, combiner) as ctx:
        emit_jobs(ctx, jobs, batch=(1,))
        groups, _ = check(ctx, want, pairs_recv=sum(want.values()))
        if combiner == mrhbm.COMBINE_NONE:
            assert ctx.result_info().pairs_in == sum(map(len, jobs))
        assert ctx.stats()["ms_combine"] > 0  # (the dedupe)
    assert as_counts(groups) == against_distinct(jobs, kind, mkb, batch=(1,))


@gpu
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_layout_flags_and_the_combiner_are_bit_identical(kind):
    jobs = mixed_jobs(keys_of(kind, 27), seed=9)
    want = want_counts(jobs)
    results = []
    for flags in [0] + FLAGS:
        for combiner in (mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT):
            with cd_ctx(kind, flags=flags, combiner=combiner) as ctx:
                emit_jobs(ctx, jobs)
                groups, rows = check(ctx, want)
                results.append(sorted((k, v[0]) for k, v in groups))
    assert all(r == results[0] for r in results)


@gpu
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_range_partitioner_one_global_order(kind):
    keys = list(range(0, 2 ** 63, 2 ** 57)) if kind == mrhbm.KEY_U64 else [b"r%03d" % i for i in range(64)]
    jobs = mixed_jobs(keys, seed=3)
    with cd_ctx(kind, partitioner=mrhbm.PART_RANGE, parts=5) as ctx:
        emit_jobs(ctx, jobs)
        ctx.sample_splitters()
        ctx.shuffle()
        assert ctx.result_info().sorted == 1
        groups, rows = check(ctx, want_counts(jobs), shuffle=False)
        assert [k for k, _ in groups] == sorted(want_counts(jobs))
        assert [k for k, _ in rows] == sorted(k for k, _ in rows)


@gpu
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_no_pair_repeats(kind):
    # the pool's value ids must never be summed: every pair survives and still counts 1
    keys = keys_of(kind, 27)
    jobs = [[(keys[i % len(keys)], b"v%d-%d" % (j, i)) for i in range(3000)] for j in range(2)]
    want = want_counts(jobs)
    assert sum(want.values()) == 6000
    with cd_ctx(kind) as ctx:
        emit_jobs(ctx, jobs, batch=(0,))
        check(ctx, want, pairs_recv=6000)


@gpu
@pytest.mark.parametrize("flags", [0, mrhbm.F_SMALL_BINS | mrhbm.F_NO_OPTIMISTIC], ids=["cap", "small-bins"])
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_a_key_over_several_bins(kind, flags):
    hot = 5 if kind == mrhbm.KEY_U64 else b"hot"
    n = 300_000
    vals = [b"visitor-%07d" % i for i in range(n)]
    random.Random(2).shuffle(vals)
    other = [((100 + i) if kind == mrhbm.KEY_U64 else b"o%d" % i, b"v%d" % (i % 3)) for i in range(20000)]
    jobs = [[(hot, v) for v in vals[:2 * n // 3]] + other[:10000], [(hot, v) for v in vals[n // 3:]] + other[10000:]]
    want = want_counts(jobs)
    with cd_ctx(kind, flags=flags) as ctx:
        emit_jobs(ctx, jobs, batch=(0, 1))
        groups, _ = check(ctx, want)
        assert ctx.stats()["big_bins"] >= 1 or flags == 0
    assert dict(as_counts(groups))[hot] == n


@gpu
def test_a_zipf_stream_of_ten_million_pairs():
    n, V, F = 10_000_000, 200_000, 5000
    rng = np.random.default_rng(8)
    w = rng.zipf(1.2, size=n) % V
    f = rng.integers(0, F, size=n)
    keys = np.char.add(b"w", w.astype("S7"))
    vals = np.char.add(b"/corpus/f", f.astype("S5"))
    pairs = np.unique(np.stack([w, f], axis=1), axis=0)
    wk, cnt = np.unique(pairs[:, 0], return_counts=True)
    want = {b"w%d" % a: int(b) for a, b in zip(wk.tolist(), cnt.tolist())}
    results = []
    for combiner in (mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT):
        with cd_ctx(combiner=combiner) as ctx:
            half = n // 2
            for j, (a, b) in enumerate(((0, half), (half, n))):
                m = ctx.map_begin(j)
                recs = np.zeros(b - a, dtype=mrhbm.record_dtype(mrhbm.KEY_STR, 27))
                recs["key"] = keys[a:b]
                lens = np.char.str_len(vals[a:b]).astype(np.uint64)
                off = np.zeros(b - a + 1, dtype=np.uint64)
                off[1:] = np.cumsum(lens)
                m.emit_batch_values(recs, b"".join(vals[a:b].tolist()), off)
                m.commit()
            ctx.shuffle()
            assert ctx.result_info().pairs_recv == len(pairs)
            keys_out, _, po = ctx.result_copy()
            blob, _ = ctx.result_values()
            raw = blob.tobytes()
            got = {bytes(keys_out[r]): int(T.decode_value(raw[11 * r:11 * r + 11])) for r in range(len(keys_out))}
            assert got == want
            results.append(raw)
    assert results[0] == results[1]


@gpu
def test_long_keys_merge_in_key_order():
    long = [b"long-key-%02d-" % i + b"z" * 30 for i in range(4)]
    jobs = [[(long[2], b"v"), (long[2], b"v"), (long[2], b"\x00"), (long[2], b""), (b"short", b"v"), (long[1], b"b"),
             (long[1], b"a"), (long[0], T.encode_value(-0.0)), (long[0], T.encode_value(0)), (b"m", b"2"),
             (long[0], T.encode_value(0.0))],
            [(long[2], b"u"), (long[2], b"v"), (long[3], b"q"), (long[1], b"a"), (b"short", b"a"), (b"m", b"1")]]
    want = want_counts(jobs)
    assert want[long[2]] == 4 and want[long[0]] == 2
    for combiner in (mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT):
        with cd_ctx(combiner=combiner) as ctx:
            emit_jobs(ctx, jobs)
            groups, _ = check(ctx, want, long_keys=4)
            with pytest.raises(mrhbm.MrhbmError) as e:
                ctx.result_copy()
            assert e.value.code == -4


@gpu
def test_words_value_pieces_share_a_value_id():
    words = [b"word%d" % i for i in range(3000)] + [b"the"]
    text = b" ".join(words) + b"\n"
    long = b"L" * 40
    for combiner in (mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT):
        with cd_ctx(combiner=combiner) as ctx:
            for j, name in enumerate((b"file-B", b"file-A", b"file-B", b"file-AB")):
                m = ctx.map_begin(j)
                m.words_value(text * 3, name)  # one device piece: every pair shares one value id
                m.words_value(b"the cat " + long + b" the\n", name)  # a piece on the host tokeniser
                m.commit()
            check(ctx, {w: 3 for w in words + [b"cat", long]}, long_keys=1)


@gpu
def test_ledger_rules_and_repeated_shuffles():
    rng = random.Random(11)

    def pairs(tag, n):
        return [(b"k%d" % rng.randrange(30), tag + b"%d" % rng.randrange(40)) for _ in range(n)]
    for combiner in (mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT):
        with cd_ctx(combiner=combiner) as ctx:
            a, b = pairs(b"a", 800), pairs(b"b", 800)
            emit_jobs(ctx, [a, b])
            check(ctx, want_counts([a, b]))
            check(ctx, want_counts([a, b]))  # a second shuffle of the same commits
            m = ctx.map_begin("job0")  # replace job0
            a2 = pairs(b"A", 500)
            for k, v in a2:
                m.emit(k, v)
            m.commit()
            check(ctx, want_counts([a2, b]))
            m = ctx.map_begin("aborted")
            for k, v in pairs(b"x", 100):
                m.emit(k, v)
            m.abort()
            check(ctx, want_counts([a2, b]))
            ctx.reset()
            c = pairs(b"c", 300)
            emit_jobs(ctx, [c])
            check(ctx, want_counts([c]))


@gpu
def test_accessors():
    jobs = mixed_jobs(str_keys(27), seed=5)
    want = want_counts(jobs)
    with cd_ctx() as ctx:
        emit_jobs(ctx, jobs)
        ctx.shuffle()
        info = ctx.result_info()
        assert info.pairs_in == sum(map(len, jobs)) and info.pairs_recv == sum(want.values())
        assert info.groups == len(want)
        keys, _, po = ctx.result_copy()
        assert int(po[-1]) == len(want)
        out = (C.c_uint64 * 6)()
        assert ctx.L.mrhbm_checksum_result(ctx.h, out) == 0
        assert out[3] == len(want) and out[4] == 0 and out[5] == 0
        # integer sums are refused: result_copy takes sums = NULL, groups are read with groups_next_values
        sums = np.empty(len(want), dtype=np.uint64)
        assert ctx.L.mrhbm_result_copy(ctx.h, keys.ctypes.data, sums.ctypes.data, None) == INVAL
        it = C.c_void_p()
        assert ctx.L.mrhbm_groups_open(ctx.h, ctx.partitions()[0], C.byref(it)) == 0
        kp, kl, vp, vn = C.c_void_p(), C.c_size_t(), C.c_void_p(), C.c_size_t()
        assert ctx.L.mrhbm_groups_next(it, C.byref(kp), C.byref(kl), C.byref(vp), C.byref(vn)) == INVAL
        ctx.L.mrhbm_groups_close(it)
        check(ctx, want, shuffle=False)


@gpu
def test_refusals():
    bad = (dict(flags=0), dict(flags=mrhbm.F_BYTE_VALUES, combiner=mrhbm.COMBINE_REDUCER),
           dict(flags=mrhbm.F_BYTE_VALUES, combiner=mrhbm.COMBINE_FSUM), dict(flags=0, combiner=mrhbm.COMBINE_DISTINCT),
           dict(flags=0, combiner=mrhbm.COMBINE_REDUCER))
    for kind in (mrhbm.KEY_U64, mrhbm.KEY_STR):
        for kw in bad:
            with pytest.raises(mrhbm.MrhbmError) as e:
                mrhbm.Ctx(kind, P, device=0, reducer=mrhbm.RED_COUNT_DISTINCT, **kw)
            assert e.value.code == INVAL
    with pytest.raises(mrhbm.MrhbmError) as e:
        mrhbm.Ctx(mrhbm.KEY_STR, P, device=0, reducer=mrhbm.RED_COUNT_DISTINCT + 1, flags=mrhbm.F_BYTE_VALUES)
    assert e.value.code == INVAL
    with cd_ctx() as ctx:  # integer-valued emits are refused on the byte-values ctx
        m = ctx.map_begin("x")
        with pytest.raises(mrhbm.MrhbmError):
            m.wordcount(b"a b c")
        m.abort()


def golden_corpus(tmp_path, golden_wordcount):
    files = []
    for job in range(4):
        toks = expand_tokens(golden_wordcount, job)
        p = tmp_path / ("file%d.txt" % job)
        p.write_bytes(b"\n".join(b" ".join(toks[i:i + 7]) for i in range(0, len(toks), 7)) + b"\n")
        files.append(str(p))
    files.append(files[1])  # the same file twice: one more job, no more distinct files
    return files


@gpu
def test_document_frequency_example(tmp_path, golden_wordcount):
    WordCount.FILES[:] = golden_corpus(tmp_path, golden_wordcount)
    S = DF_PKG + ".init"
    results = []
    arms = ((S, None, S), (S, DF_PKG + ".combinerfn", S), (DF_PKG + ".reducefn_device", None, S),
            (DF_PKG + ".reducefn_device", DF_PKG + ".combinerfn", DF_PKG + ".mapfn_device"))
    for arm, (reducefn, combinerfn, mapfn) in enumerate(arms):
        DF.RESULT.clear()
        s = server.new("hbm://local", "cd-loop-%d" % arm)  # (a task board, and its ctx, per database name)
        s.configure(dict(taskfn=S, mapfn=mapfn, partitionfn=S, reducefn=reducefn, finalfn=S, combinerfn=combinerfn,
                         storage="hbm", hbm={"value_kind": "bytes"}))
        s.loop()
        results.append(dict(DF.RESULT))
    assert results[0] and all(r == results[0] for r in results[1:])
    assert 1 <= min(results[0].values()) and max(results[0].values()) <= 4
    assert all(type(v) is int for v in results[0].values())
