"""MRHBM_COMBINE_DISTINCT: a byte-values map job keeps one copy of each distinct (key, value bytes) pair at its commit.

Every expected result is computed on the host from the same inputs: a job's distinct pairs in first-occurrence order
(dict.fromkeys), the union of the jobs' sets with the multiplicity across jobs kept.  Rows are compared as a multiset
through result_copy + result_values, groups through Ctx.groups, the committed records through pool_read."""
import random
import sys
import types
from collections import Counter

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


def dd_ctx(kind=mrhbm.KEY_STR, max_key_bytes=27, combiner=mrhbm.COMBINE_DISTINCT):
    return mrhbm.Ctx(kind, P, max_key_bytes=max_key_bytes, device=0, reducer=mrhbm.RED_NONE,
                     flags=mrhbm.F_BYTE_VALUES, combiner=combiner)


def distinct(pairs):
    return list(dict.fromkeys(pairs))


def want_groups(jobs):
    """{key: sorted values} of the union of the jobs' distinct pairs"""
    want = {}
    for pairs in jobs:
        for k, v in distinct(pairs):
            want.setdefault(k, []).append(v)
    return {k: sorted(v) for k, v in want.items()}


def got_groups(ctx):
    got = {}
    for p in ctx.partitions():
        keys = []
        for k, vals in ctx.groups(p):
            assert k not in got
            keys.append(k)
            got[k] = sorted(vals)
        assert keys == sorted(keys)
    return got


def got_rows(ctx):
    keys, sums, _ = ctx.result_copy()
    assert sums is None
    blob, roff = ctx.result_values()
    raw = blob.tobytes()
    u64 = keys.dtype.kind == "u"
    return Counter((int(keys[r]) if u64 else bytes(keys[r]), raw[int(roff[r]):int(roff[r + 1])])
                   for r in range(keys.shape[0]))


def check(ctx, jobs, rows=True):
    """shuffles; groups (and rows) are the union of the jobs' distinct pairs"""
    ctx.shuffle()
    assert ctx.result_info().pairs_in == sum(len(distinct(p)) for p in jobs) - sum(
        1 for p in jobs for k, _ in distinct(p) if isinstance(k, bytes) and len(k) >= ctx.record_bytes - 4)
    assert got_groups(ctx) == want_groups(jobs)
    if rows:
        assert got_rows(ctx) == Counter(x for p in jobs for x in distinct(p))


def value(n, seed, last=None):
    rng = random.Random(seed)
    b = bytearray(rng.getrandbits(8) for _ in range(n))
    if last is not None and n:
        b[-1] = last
    return bytes(b)


def emit_pairs(m, pairs):
    for k, v in pairs:
        m.emit(k, v)


def emit_batch(ctx, m, pairs):
    recs = np.zeros(len(pairs), dtype=mrhbm.record_dtype(ctx.key_kind, ctx.cfg.max_key_bytes))
    recs["key"] = [k for k, _ in pairs]
    off = np.zeros(len(pairs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(v) for _, v in pairs])
    m.emit_batch_values(recs, b"".join(v for _, v in pairs), off)


# =================================================================================================================
# 1. per-emit jobs
# =================================================================================================================
def per_emit_jobs():
    big = value(STAGE + 12345, 1)
    big2 = big[:-1] + bytes([big[-1] ^ 1])  # differs in its last byte only
    mid = value(5000, 2)
    mid2 = mid[:2500] + bytes([mid[2500] ^ 0x80]) + mid[2501:]
    v17 = value(17, 3)
    v17b = value(17, 3, last=v17[-1] ^ 0xFF)
    common = [(b"shared", b"x"), (b"shared", b"y"), (b"e", b"")]
    job0 = [(b"a", b"1"), (b"a", b"1"), (b"a", b"2"), (b"b", b""), (b"b", b""), (b"b", b"\x00"), (b"c", v17),
            (b"c", v17b), (b"c", v17), (b"d", mid), (b"d", mid2), (b"d", mid), (b"g", big), (b"g", big),
            (b"g", big2), (b"a", b"1")] + common + common
    job1 = [(b"k%d" % (i % 5), b"v%d" % (i % 3)) for i in range(60)] + common + [(b"d", mid)]  # (batch: own ids)
    job2 = common + [(b"a", b"1"), (b"zz", b"")] * 3
    return job0, job1, job2


@gpu
def test_per_emit_jobs_keep_their_distinct_pairs():
    jobs = per_emit_jobs()
    with dd_ctx() as ctx:
        for j, pairs in enumerate(jobs):
            m = ctx.map_begin("job%d" % j)
            if j == 1:
                emit_batch(ctx, m, pairs)
            else:
                emit_pairs(m, pairs)
            m.commit()
        # pool_read: each job's survivors in first-occurrence order, with the value id they were emitted under
        n = sum(len(distinct(p)) for p in jobs)
        recs = ctx.pool_read(0, n)
        want_keys, want_ids, base = [], [], 0
        for pairs in jobs:
            first = {}
            for i, x in enumerate(pairs):
                first.setdefault(x, i)
            for x in distinct(pairs):
                want_keys.append(x[0])
                want_ids.append(base + first[x])
            base += len(pairs)
        assert list(recs["key"]) == want_keys
        assert list(recs["val"]) == want_ids
        assert ctx.checksum_input()[3] == n
        check(ctx, jobs)


@gpu
def test_u64_keys():
    rng = random.Random(5)
    jobs = [[(rng.randrange(50) * (1 << 40), b"f%d" % rng.randrange(4)) for _ in range(3000)] for _ in range(3)]
    jobs[1] += [(7, b""), (7, b""), (7, value(STAGE + 1, 9)), (7, value(STAGE + 1, 9))]
    with dd_ctx(mrhbm.KEY_U64) as ctx:
        for j, pairs in enumerate(jobs):
            m = ctx.map_begin(j)
            emit_pairs(m, pairs)
            m.commit()
        ctx.shuffle()
        got = got_groups(ctx)
        want = {k.to_bytes(8, "big"): v for k, v in want_groups(jobs).items()}
        assert got == want
        assert got_rows(ctx) == Counter(x for p in jobs for x in distinct(p))


@gpu
@pytest.mark.parametrize("mkb", [27, 59, 123])
def test_many_pairs_and_record_classes(mkb):
    """enough pairs for many tiles and a table of 2^17 entries; keys at the class maximum"""
    rng = random.Random(mkb)
    words = [b"w%d" % i for i in range(3000)] + [b"m" * mkb, b"n" * mkb]
    vals = [b"", b"f1", b"f2", value(40, 4)]
    jobs = [[(rng.choice(words), rng.choice(vals)) for _ in range(40000)] for _ in range(2)]
    with dd_ctx(max_key_bytes=mkb) as ctx:
        for j, pairs in enumerate(jobs):
            m = ctx.map_begin(j)
            emit_batch(ctx, m, pairs[:20000])
            emit_pairs(m, pairs[20000:])
            m.commit()
        check(ctx, jobs)


# =================================================================================================================
# 2. device tokeniser
# =================================================================================================================
@gpu
def test_words_value_over_three_pieces():
    words = [b"word%d" % i for i in range(2000)] + [b"x", b"y" * 27]
    line = b" ".join(words) + b"\n"
    text = line * ((140 << 20) // len(line) + 1)  # > 2 x 64 MB: three pieces, the same words in every one
    with dd_ctx() as ctx:
        m = ctx.map_begin("big")
        assert m.words_value(text, b"file-A") == len(words) * (len(text) // len(line))
        m.words_value(b"x extra x", b"file-A")  # a second call of the same job: x again, one new word
        m.words_value(b"x", b"file-B")
        m.commit()
        ctx.shuffle()
        want = {w: [b"file-A"] for w in words + [b"extra"]}
        want[b"x"] = [b"file-A", b"file-B"]
        assert ctx.result_info().pairs_in == len(words) + 2
        assert got_groups(ctx) == want
        assert got_rows(ctx) == Counter((w, v) for w, vs in want.items() for v in vs)


@gpu
def test_words_value_host_fallback_piece():
    """a word longer than the record class sends the call's one piece to the host tokeniser"""
    long = b"L" * 40
    text = b"the cat the " + long + b" cat " + long + b" dog the\n"
    with dd_ctx() as ctx:
        m = ctx.map_begin("fallback")
        m.words_value(text, b"doc")
        m.commit()
        ctx.shuffle()
        assert ctx.result_info().pairs_in == 3  # the, cat, dog (the long word waits on the host)
        assert got_groups(ctx) == {b"the": [b"doc"], b"cat": [b"doc"], b"dog": [b"doc"], long: [b"doc"]}


# =================================================================================================================
# 3. the ledger: interleaved handles, replace, abort, reset
# =================================================================================================================
@gpu
@pytest.mark.parametrize("order", ["ab", "ba"])
def test_interleaved_handles_and_ledger_rules(order):
    rng = random.Random(11)

    def pairs(tag, n):
        return [(b"k%d" % rng.randrange(30), tag + value(rng.choice((0, 3, 17, 300)), rng.randrange(4))) for _ in range(n)]
    with dd_ctx() as ctx:
        hs = {"a": ctx.map_begin("A"), "b": ctx.map_begin("B")}
        emitted = {"a": [], "b": []}
        for step in range(6):  # ranges alternate a, b, a, b, ...
            for name in "ab":
                p = pairs(name.encode(), 500)
                if step % 2:
                    emit_batch(ctx, hs[name], p)
                else:
                    emit_pairs(hs[name], p)
                emitted[name] += p
                if step % 2 == 0:  # (staged emits become a range at the next flush: force one)
                    emit_batch(ctx, hs[name], [(b"flush", b"")])
                    emitted[name].append((b"flush", b""))
        for name in order:
            hs[name].commit()
        check(ctx, [emitted["a"], emitted["b"]])
        # replace-by-job-id: job A again
        m = ctx.map_begin("A")
        again = pairs(b"A2", 300)
        emit_pairs(m, again)
        m.commit()
        check(ctx, [again, emitted["b"]])
        # an abort after another handle's commit
        c, d = ctx.map_begin("C"), ctx.map_begin("D")
        emit_batch(ctx, c, pairs(b"c", 200))
        dp = pairs(b"d", 200)
        emit_batch(ctx, d, dp)
        d.commit()
        c.abort()
        check(ctx, [again, emitted["b"], dp])
        e = ctx.map_begin("E")
        ep = pairs(b"e", 100)
        emit_pairs(e, ep)
        e.commit()
        check(ctx, [again, emitted["b"], dp, ep])
        ctx.reset()
        f = ctx.map_begin("F")
        fp = pairs(b"f", 400)
        emit_batch(ctx, f, fp)
        f.commit()
        check(ctx, [fp])


# =================================================================================================================
# 4. long keys
# =================================================================================================================
@gpu
def test_long_keys_are_deduped_on_the_host():
    long = [b"long-key-%02d-" % i + b"z" * 30 for i in range(4)]
    jobs = [[(long[0], b"v"), (long[0], b"v"), (long[0], b"w"), (b"short", b"v"), (long[1], b""), (long[1], b""),
             (b"short", b"v"), (long[2], value(STAGE + 5, 1)), (long[2], value(STAGE + 5, 1))],
            [(long[0], b"v"), (long[3], b"q"), (long[3], b"q"), (b"short", b"v")]]
    with dd_ctx() as ctx:
        for j, pairs in enumerate(jobs):
            m = ctx.map_begin(j)
            emit_pairs(m, pairs)
            m.commit()
        check(ctx, jobs, rows=False)


# =================================================================================================================
# 5. refusals and the path without the combiner
# =================================================================================================================
@gpu
def test_refusals():
    for kw in (dict(flags=0), dict(flags=0, reducer=mrhbm.RED_SUM), dict(flags=mrhbm.F_BYTE_VALUES, reducer=mrhbm.RED_SUM)):
        kw = dict(dict(reducer=mrhbm.RED_NONE), **kw)
        with pytest.raises(mrhbm.MrhbmError) as e:
            mrhbm.Ctx(mrhbm.KEY_STR, P, device=0, combiner=mrhbm.COMBINE_DISTINCT, **kw)
        assert e.value.code == INVAL


@gpu
def test_without_the_combiner_every_pair_stays():
    jobs = per_emit_jobs()
    with dd_ctx(combiner=mrhbm.COMBINE_NONE) as ctx:
        for j, pairs in enumerate(jobs):
            m = ctx.map_begin(j)
            emit_pairs(m, pairs)
            m.commit()
        ctx.shuffle()
        assert ctx.result_info().pairs_in == sum(len(p) for p in jobs)
        assert got_rows(ctx) == Counter(x for p in jobs for x in p)


# =================================================================================================================
# 6. end to end: the InvertedIndex example
# =================================================================================================================
def run_inverted_index(mapfn, combinerfn, name):
    S = II_PKG + ".init"
    II.RESULT.clear()
    s = server.new("hbm://local", name)
    s.configure(dict(taskfn=S, mapfn=mapfn, partitionfn=S, reducefn=S, finalfn=S, combinerfn=combinerfn,
                     storage="hbm", hbm={"value_kind": "bytes"}))
    s.loop()
    return dict(II.RESULT), s.stats["shuffle"]["pairs"]


def golden_corpus(tmp_path, golden_wordcount):
    files = []
    for job in range(4):
        toks = expand_tokens(golden_wordcount, job)
        p = tmp_path / ("file%d.txt" % job)
        p.write_bytes(b"\n".join(b" ".join(toks[i:i + 7]) for i in range(0, len(toks), 7)) + b"\n")
        files.append(str(p))
    return files


def synthetic_corpus(tmp_path):
    rng = random.Random(3)
    vocab = [b"t%d" % i for i in range(400)]
    files = []
    for j in range(6):
        p = tmp_path / ("syn%d.txt" % j)
        p.write_bytes(b" ".join(vocab[min(int(rng.paretovariate(1.1)) - 1, 399)] for _ in range(20000)) + b"\n")
        files.append(str(p))
    return files


@gpu
@pytest.mark.parametrize("corpus", ["wordcount", "synthetic"])
def test_inverted_index_end_to_end(tmp_path, golden_wordcount, corpus):
    files = golden_corpus(tmp_path, golden_wordcount) if corpus == "wordcount" else synthetic_corpus(tmp_path)
    WordCount.FILES[:] = files
    want = {}
    for f in files:
        for w in set(open(f, "rb").read().split()):
            want.setdefault(w, []).append(f.encode())
    want = {k: sorted(v) for k, v in want.items()}
    plain, n_plain = run_inverted_index(II_PKG + ".init", None, corpus + "-plain")
    assert plain == want
    for mapfn in (II_PKG + ".init", II_PKG + ".mapfn_device"):
        got, n = run_inverted_index(mapfn, II_PKG + ".combinerfn", corpus + "-distinct")
        assert got == want
        assert n == sum(len(v) for v in want.values()) < n_plain


# =================================================================================================================
# 7. configure (CPU, stand-in ctx)
# =================================================================================================================
class StandIn:
    made = []

    def __init__(self, h):
        type(self).made.append(dict(h))


def plugin(monkeypatch, name, combinerfn, decl="distinct"):
    mod = types.ModuleType(name)
    mod.init = lambda arg=None: None
    mod.combinerfn = combinerfn
    mod.hbm_combinerfn = decl
    monkeypatch.setitem(sys.modules, name, mod)
    return name


def configure(combinerfn, value_kind="bytes"):
    S = II_PKG + ".init"
    s = server.new("hbm://local", "dd-configure")
    s.ctx_factory = StandIn
    s.configure(dict(taskfn=S, mapfn=S, partitionfn=S, reducefn=S, finalfn=S, combinerfn=combinerfn, storage="hbm",
                     hbm={"value_kind": value_kind}))
    return s


def test_configure_selects_the_distinct_combiner():
    s = configure(II_PKG + ".combinerfn")
    assert s.config["hbm"]["combiner"] == "distinct"
    assert configure(None).config["hbm"]["combiner"] is False


def test_configure_refuses_a_combinerfn_that_does_not_dedupe(monkeypatch):
    def summing(key, values, emit):
        emit(sum(len(v) if isinstance(v, bytes) else v for v in values))

    def dropping(key, values, emit):
        for v in sorted(set(values))[1:]:
            emit(v)

    def identity(key, values, emit):
        for v in values:
            emit(v)
    for fn in (summing, dropping, identity):
        with pytest.raises(ValueError, match="distinct"):
            configure(plugin(monkeypatch, "dd_plugin_" + fn.__name__, fn))
    with pytest.raises(ValueError, match="hbm_combinerfn"):
        configure(plugin(monkeypatch, "dd_plugin_unknown", II.reducefn, decl="unique"))


def test_configure_refuses_distinct_on_integer_values():
    with pytest.raises(ValueError, match="value_kind"):
        configure(II_PKG + ".combinerfn", value_kind="int")


def test_probe_values_encode_as_the_shuffle_compares_them():
    assert len({T.encode_value(v) for v in server._DISTINCT_PROBES[0]}) == 4
    assert len({T.encode_value(v) for v in server._DISTINCT_PROBES[1]}) == 3
