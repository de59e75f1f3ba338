"""MRHBM_RED_DISTINCT: after the shuffle every key holds its distinct values over all map jobs, ascending by bytes.

Every expected result is computed on the host: sorted(set(...)) of the value bytes per key over the union of all jobs.
Sequences are compared exactly, not as multisets, through Ctx.groups, through result_copy + result_values (each key's
rows contiguous and ascending; with info.sorted a partition's rows ascending by (key, value) as a whole), and through
pairs_recv / groups."""
import random

import numpy as np
import pytest

import mrhbm_loader
from conftest import expand_tokens

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce import tuple as T  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.InvertedIndex import init as II  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WordCount import init as WordCount  # noqa: E402

gpu = pytest.mark.gpu
P = 7
INVAL = -1
STAGE = 4 << 20  # value bytes staged next to the records; a longer value is copied on its own
II_PKG = "lua_mapreduce_b200.mapreduce.examples.InvertedIndex"


def dr_ctx(kind=mrhbm.KEY_STR, max_key_bytes=27, combiner=mrhbm.COMBINE_NONE, flags=0, partitioner=None, parts=P):
    kw = {} if partitioner is None else dict(partitioner=partitioner)
    return mrhbm.Ctx(kind, parts, max_key_bytes=max_key_bytes, device=0, reducer=mrhbm.RED_DISTINCT,
                     flags=mrhbm.F_BYTE_VALUES | flags, combiner=combiner, **kw)


def value(n, seed, last=None):
    rng = random.Random(seed)
    b = bytearray(rng.getrandbits(8) for _ in range(n))
    if last is not None and n:
        b[-1] = last
    return bytes(b)


def want_groups(jobs):
    want = {}
    for pairs in jobs:
        for k, v in pairs:
            want.setdefault(k, set()).add(v)
    return {k: sorted(v) for k, v in want.items()}


def emit_jobs(ctx, jobs, batch=()):
    for j, pairs in enumerate(jobs):
        m = ctx.map_begin("job%d" % j)
        if j in batch:
            recs = np.zeros(len(pairs), dtype=mrhbm.record_dtype(ctx.key_kind, ctx.cfg.max_key_bytes))
            recs["key"] = [k for k, _ in pairs]
            off = np.zeros(len(pairs) + 1, dtype=np.uint64)
            off[1:] = np.cumsum([len(v) for _, v in pairs])
            m.emit_batch_values(recs, b"".join(v for _, v in pairs), off)
        else:
            for k, v in pairs:
                m.emit(k, v)
        m.commit()


def check(ctx, want, long_keys=0, shuffle=True):
    """groups, rows and counts against want = {key: ascending distinct values}"""
    if shuffle:
        ctx.shuffle()
    u64 = ctx.key_kind == mrhbm.KEY_U64
    got = {}
    for p in ctx.partitions():
        keys = []
        for k, vals in ctx.groups(p):
            k = int.from_bytes(k, "big") if u64 else k
            assert k not in got
            keys.append(k)
            got[k] = vals
        assert keys == sorted(keys)
    assert got == want
    info = ctx.result_info()
    short = {k: v for k, v in want.items() if u64 or len(k) <= ctx.record_bytes - 4}
    n = sum(len(v) for v in short.values())
    assert info.groups == n and info.pairs_recv == n
    assert len(short) == len(want) - long_keys
    if long_keys:
        return
    keys, _, po = ctx.result_copy()
    blob, roff = ctx.result_values()
    raw = blob.tobytes()
    rows = [(int(keys[r]) if u64 else bytes(keys[r]), raw[int(roff[r]):int(roff[r + 1])]) for r in range(n)]
    assert sorted(rows) == sorted((k, v) for k, vs in short.items() for v in vs)
    seen = {}
    for i, (k, v) in enumerate(rows):  # a key's rows: contiguous, ascending
        if k in seen:
            assert rows[i - 1][0] == k and rows[i - 1][1] < v
        seen[k] = True
    if info.sorted:
        for p in range(ctx.num_partitions):
            part = rows[int(po[p]):int(po[p + 1])]
            assert all(a < b for a, b in zip(part, part[1:]))
    return rows, po


def value_mix():
    """values that differ past byte 8, past byte 4096 and in their last byte, proper prefixes, the empty value, one
    larger than the 4 MB stage, number and string encodings"""
    big = value(STAGE + 12345, 1)
    big2 = big[:-1] + bytes([big[-1] ^ 1])
    long = value(6000, 2)
    long2 = long[:5000] + bytes([long[5000] ^ 0x80]) + long[5001:]
    pre = b"common-prefix-"
    mix = [b"", b"\x00", b"\x00\x00", b"a", b"ab", b"abc", b"abcdefgh", b"abcdefghi", b"abcdefgh\x00", b"abcdefgh\xff",
           pre + b"1", pre + b"2", pre + b"10", pre, long, long2, big, big2, b"\xff" * 9, b"\x80",
           value(17, 3), value(17, 3, last=0), value(17, 3, last=0xff)]
    mix += [T.encode_value(x) for x in (0, 1, -1, 1.5, 2 ** 40, b"file-a", b"file-b", "file-a")]
    return mix


def mixed_jobs(keys, seed=7):
    rng = random.Random(seed)
    mix = value_mix()
    jobs = []
    for j in range(3):
        pairs = [(k, v) for k in keys[:3] for v in mix]  # every job, every value: the same bytes under many ids
        pairs += [(keys[3], b"one")]
        pairs += [(rng.choice(keys[4:]), rng.choice(mix[:14])) for _ in range(400)]
        pairs += [(keys[0], mix[3])] * 5
        rng.shuffle(pairs)
        jobs.append(pairs)
    return jobs


def str_keys(mkb):
    return [b"k%d" % i for i in range(40)] + [b"w" * mkb, b"x" * (mkb - 1)]


KINDS = [("u64", mrhbm.KEY_U64, 27), ("str27", mrhbm.KEY_STR, 27), ("str59", mrhbm.KEY_STR, 59),
         ("str123", mrhbm.KEY_STR, 123)]


@gpu
@pytest.mark.parametrize("combiner", [mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT], ids=["none", "distinct"])
@pytest.mark.parametrize("name,kind,mkb", KINDS, ids=[k[0] for k in KINDS])
def test_values_ascend_by_bytes(name, kind, mkb, combiner):
    keys = list(range(0, 42 * 2 ** 50, 2 ** 50)) if kind == mrhbm.KEY_U64 else str_keys(mkb)
    jobs = mixed_jobs(keys)
    with dr_ctx(kind, mkb, combiner) as ctx:
        emit_jobs(ctx, jobs, batch=(1,))
        check(ctx, want_groups(jobs))


@gpu
@pytest.mark.parametrize("flags", [mrhbm.F_NO_OPTIMISTIC, mrhbm.F_FORCE_RUNS,
                                   mrhbm.F_NO_OPTIMISTIC | mrhbm.F_FORCE_RUNS])
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_layout_flags(kind, flags):
    keys = list(range(1, 43)) if kind == mrhbm.KEY_U64 else str_keys(27)
    jobs = mixed_jobs(keys, seed=9)
    with dr_ctx(kind, flags=flags) as ctx:
        emit_jobs(ctx, jobs)
        check(ctx, want_groups(jobs))


def many_values(key, n, seed, prefix=b"/data/corpus/file-name-"):
    """n distinct values sharing a 23-byte prefix (prefix ties), shuffled"""
    vals = [prefix + b"%07d" % i for i in range(n)]
    random.Random(seed).shuffle(vals)
    return [(key, v) for v in vals]


@gpu
@pytest.mark.parametrize("flags", [0, mrhbm.F_SMALL_BINS], ids=["cap", "small-bins"])
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_oversized_bins_are_one_run(kind, flags):
    hot, warm = (5, 6) if kind == mrhbm.KEY_U64 else (b"hot", b"warm")
    other = [((100 + i) if kind == mrhbm.KEY_U64 else b"o%d" % i, b"v%d" % (i % 3)) for i in range(20000)]
    jobs = [many_values(hot, 5000, 1)[:3000] + other[:10000], many_values(hot, 5000, 1)[2000:] + other[10000:],
            many_values(warm, 300, 2) + [(hot, b"")], many_values(warm, 300, 2)]
    with dr_ctx(kind, flags=flags | mrhbm.F_NO_OPTIMISTIC) as ctx:
        emit_jobs(ctx, jobs, batch=(0, 1))
        check(ctx, want_groups(jobs))
        assert ctx.stats()["big_bins"] >= 1


@gpu
def test_a_key_with_a_million_values():
    n = 1_000_000
    rng = np.random.default_rng(4)
    ids = rng.permutation(n)
    vals = [b"doc-%07d" % i for i in ids.tolist()]
    with dr_ctx() as ctx:
        for j in range(2):  # two jobs, overlapping halves
            part = vals[j * n // 3: j * n // 3 + 2 * n // 3 + 1]
            m = ctx.map_begin(j)
            recs = np.zeros(len(part) + 1, dtype=mrhbm.record_dtype(ctx.key_kind, 27))
            recs["key"] = [b"big"] * len(part) + [b"small"]
            off = np.zeros(len(part) + 2, dtype=np.uint64)
            off[1:] = np.cumsum([len(v) for v in part] + [1])
            m.emit_batch_values(recs, b"".join(part) + b"s", off)
            m.commit()
        ctx.shuffle()
        got = {k: v for p in ctx.partitions() for k, v in ctx.groups(p)}
        assert got[b"small"] == [b"s"]
        assert got[b"big"] == sorted(set(vals)) and len(got[b"big"]) == n
        assert ctx.result_info().groups == n + 1


@gpu
def test_many_keys_per_bin():
    rng = random.Random(5)
    jobs = [[(b"key%05d" % rng.randrange(30000), b"f%d" % rng.randrange(6)) for _ in range(60000)] for _ in range(3)]
    for combiner in (mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT):
        with dr_ctx(combiner=combiner) as ctx:
            emit_jobs(ctx, jobs, batch=(0, 1, 2))
            check(ctx, want_groups(jobs))


@gpu
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_range_partitioner_one_global_order(kind):
    keys = list(range(0, 2 ** 63, 2 ** 57)) if kind == mrhbm.KEY_U64 else [b"r%03d" % i for i in range(64)]
    jobs = mixed_jobs(keys + keys[:1], seed=3)
    with dr_ctx(kind, partitioner=mrhbm.PART_RANGE, parts=5) as ctx:
        emit_jobs(ctx, jobs)
        ctx.sample_splitters()
        ctx.shuffle()
        assert ctx.result_info().sorted == 1
        rows, po = check(ctx, want_groups(jobs), shuffle=False)
        assert all(a < b for a, b in zip(rows, rows[1:]))


@gpu
def test_ledger_rules_and_repeated_shuffles():
    rng = random.Random(11)

    def pairs(tag, n):
        return [(b"k%d" % rng.randrange(30), tag + value(rng.choice((0, 3, 17, 300)), rng.randrange(4)))
                for _ in range(n)]
    for combiner in (mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT):
        with dr_ctx(combiner=combiner) as ctx:
            a, b = pairs(b"a", 800), pairs(b"b", 800)
            emit_jobs(ctx, [a, b])
            check(ctx, want_groups([a, b]))
            check(ctx, want_groups([a, b]))  # a second shuffle of the same commits
            m = ctx.map_begin("job0")  # replace job0
            a2 = pairs(b"A", 500)
            for k, v in a2:
                m.emit(k, v)
            m.commit()
            check(ctx, want_groups([a2, b]))
            m = ctx.map_begin("aborted")
            for k, v in pairs(b"x", 100):
                m.emit(k, v)
            m.abort()
            check(ctx, want_groups([a2, b]))
            ctx.reset()
            c = pairs(b"c", 300)
            emit_jobs(ctx, [c])
            check(ctx, want_groups([c]))


@gpu
def test_long_keys_merge_in_key_order():
    long = [b"long-key-%02d-" % i + b"z" * 30 for i in range(4)]
    jobs = [[(long[2], b"v"), (long[2], b"v"), (long[2], b"\x00"), (long[2], b""), (b"short", b"v"), (long[1], b"b"),
             (long[1], b"a"), (long[0], value(STAGE + 5, 1)), (long[0], value(STAGE + 5, 1)), (b"m", b"2")],
            [(long[2], b"u"), (long[2], b"v"), (long[3], b"q"), (long[1], b"a"), (b"short", b"a"), (b"m", b"1")]]
    for combiner in (mrhbm.COMBINE_NONE, mrhbm.COMBINE_DISTINCT):
        with dr_ctx(combiner=combiner) as ctx:
            emit_jobs(ctx, jobs)
            check(ctx, want_groups(jobs), long_keys=4)


@gpu
def test_words_value_shared_ids_and_host_fallback():
    words = [b"word%d" % i for i in range(3000)] + [b"the"]
    text = b" ".join(words) + b"\n"
    long = b"L" * 40
    with dr_ctx(combiner=mrhbm.COMBINE_NONE) as ctx:
        for j, name in enumerate((b"file-B", b"file-A", b"file-B", b"file-AB")):
            m = ctx.map_begin(j)
            m.words_value(text * 3, name)  # one device piece: every pair shares one value id
            m.words_value(b"the cat " + long + b" the\n", name)  # a piece on the host tokeniser
            m.commit()
        want = {w: [b"file-A", b"file-AB", b"file-B"] for w in words + [b"cat", long]}
        check(ctx, want, long_keys=1)


@gpu
def test_refusals():
    for kw in (dict(flags=0), dict(flags=mrhbm.F_BYTE_VALUES, combiner=mrhbm.COMBINE_REDUCER)):
        with pytest.raises(mrhbm.MrhbmError) as e:
            mrhbm.Ctx(mrhbm.KEY_STR, P, device=0, reducer=mrhbm.RED_DISTINCT, **kw)
        assert e.value.code == INVAL


def golden_corpus(tmp_path, golden_wordcount):
    files = []
    for job in range(4):
        toks = expand_tokens(golden_wordcount, job)
        p = tmp_path / ("file%d.txt" % job)
        p.write_bytes(b"\n".join(b" ".join(toks[i:i + 7]) for i in range(0, len(toks), 7)) + b"\n")
        files.append(str(p))
    return files


@gpu
def test_inverted_index_loop_with_the_device_reducer(tmp_path, golden_wordcount):
    WordCount.FILES[:] = golden_corpus(tmp_path, golden_wordcount)
    S = II_PKG + ".init"
    results = []
    arms = ((S, II_PKG + ".combinerfn", S), (II_PKG + ".reducefn_device", None, S),
            (II_PKG + ".reducefn_device", II_PKG + ".combinerfn", II_PKG + ".mapfn_device"))
    for arm, (reducefn, combinerfn, mapfn) in enumerate(arms):
        II.RESULT.clear()
        s = server.new("hbm://local", "dr-loop-%d" % arm)  # (a task board, and its ctx, per database name)
        s.configure(dict(taskfn=S, mapfn=mapfn, partitionfn=S, reducefn=reducefn, finalfn=S, combinerfn=combinerfn,
                         storage="hbm", hbm={"value_kind": "bytes"}))
        s.loop()
        results.append(dict(II.RESULT))
    assert results[0] and results[1] == results[0] and results[2] == results[0]
