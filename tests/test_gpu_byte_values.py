"""Byte-string values (MRHBM_F_BYTE_VALUES) through the group-only shuffle on the GPU.  The expected result is a plain
Python group-by: every key maps to the sorted multiset of its values (the reference semantics of a general reducer);
partition ids come from the oracle's partitioners."""
import random

import numpy as np
import pytest

import mrhbm_loader
import oracle as O
from conftest import expand_tokens

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.InvertedIndex import init as II  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WordCount import init as WordCount  # noqa: E402

P = 7
FLAGS = [0, mrhbm.F_FORCE_RUNS, mrhbm.F_NO_OPTIMISTIC, mrhbm.F_SMALL_BINS]


def byte_ctx(kind, max_key_bytes=27, flags=0, P=P):
    return mrhbm.Ctx(kind, P, max_key_bytes=max_key_bytes, device=0, reducer=mrhbm.RED_NONE,
                     flags=flags | mrhbm.F_BYTE_VALUES)


def key_bytes(kind, k):
    return k.to_bytes(8, "big") if kind == mrhbm.KEY_U64 else k


def expected(kind, pairs):
    want = {}
    for k, v in pairs:
        want.setdefault(key_bytes(kind, k), []).append(bytes(v))
    return {k: sorted(v) for k, v in want.items()}


def pid(kind, kb):
    return O.part_mulhash(int.from_bytes(kb, "big"), P) if kind == mrhbm.KEY_U64 else O.part_fnv_lua(kb, P)


def check(ctx, kind, pairs, bulk=True):
    """iteration == expected group-by, keys ascending, partitions right; result_values agrees row by row"""
    got = {}
    for p in ctx.partitions():
        keys = [k for k, _ in ctx.groups(p)]
        assert keys == sorted(keys)
        for k, vals in ctx.groups(p):
            assert pid(kind, k) == p
            assert k not in got
            got[k] = sorted(vals)
    assert got == expected(kind, pairs)
    if not bulk:
        return got
    keys, sums, po = ctx.result_copy()
    assert sums is None
    blob, roff = ctx.result_values()
    assert roff.shape[0] == keys.shape[0] + 1 and int(roff[0]) == 0 and int(roff[-1]) == blob.shape[0]
    rows = {}
    raw = blob.tobytes()
    for r in range(keys.shape[0]):
        # (string key slots hold the stored form: 0x00 / 0x01 escaped as 01 01 / 01 02)
        k = int(keys[r]).to_bytes(8, "big") if kind == mrhbm.KEY_U64 else \
            bytes(keys[r]).replace(b"\x01\x01", b"\x00").replace(b"\x01\x02", b"\x01")
        rows.setdefault(k, []).append(raw[int(roff[r]):int(roff[r + 1])])
    assert {k: sorted(v) for k, v in rows.items()} == got
    assert ctx.checksum_input()[:3] == ctx.checksum_result()[:3]
    return got


def random_pairs(kind, klen, n, nkeys, seed, vmax=300):
    rng = random.Random(seed)
    if kind == mrhbm.KEY_U64:
        keys = [rng.getrandbits(64) for _ in range(nkeys)]
    else:
        keys = [bytes(rng.randrange(2, 256) for _ in range(rng.randint(1, klen))) for _ in range(nkeys)]
        keys[0] = b"\x00\x01" + keys[0][:max(0, klen - 4)]  # escaped bytes take two slot bytes each
    pairs = [(keys[rng.randrange(nkeys)], bytes(rng.getrandbits(8) for _ in range(rng.randint(0, vmax))))
             for _ in range(n)]
    pairs.append((keys[1], bytes(range(256))))  # every byte value
    return pairs


@pytest.mark.gpu
@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("kind,klen", [(mrhbm.KEY_STR, 27), (mrhbm.KEY_STR, 59), (mrhbm.KEY_STR, 123), (mrhbm.KEY_U64, 8)])
def test_round_trip(kind, klen, flags):
    pairs = random_pairs(kind, klen, 6000, 700, seed=klen + flags)
    with byte_ctx(kind, klen, flags) as ctx:
        m = ctx.map_begin("j")
        for k, v in pairs:
            m.emit(k, v)
        m.commit()
        ctx.shuffle()
        check(ctx, kind, pairs)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [0, mrhbm.F_SMALL_BINS])
def test_awkward_sizes_and_a_key_with_5000_values(flags):
    rng = random.Random(5)
    pairs = []
    for size in (4096, 4097, 65536 + 3, (1 << 20) + 5, 1 << 20, 13):
        for _ in range(3):
            pairs.append((b"big%d" % rng.randrange(4), rng.randbytes(size)))
            pairs.append((b"one", rng.randbytes(1)))
    pairs += [(b"crowded", rng.randbytes(rng.choice((1, 7, 17, 33, 100)))) for _ in range(5000)]
    rng.shuffle(pairs)
    with byte_ctx(mrhbm.KEY_STR, flags=flags) as ctx:
        m = ctx.map_begin("j")
        for k, v in pairs:
            m.emit(k, v)
        m.commit()
        ctx.shuffle()
        check(ctx, mrhbm.KEY_STR, pairs)


@pytest.mark.gpu
def test_long_keys_merge_in_key_order():
    rng = random.Random(3)
    keys = [b"k%02d" % i for i in range(20)] + [b"k%02d" % i + b"x" * 40 for i in range(0, 20, 3)]
    pairs = [(rng.choice(keys), rng.randbytes(rng.randint(0, 40))) for _ in range(3000)]
    with byte_ctx(mrhbm.KEY_STR, 27) as ctx:
        m = ctx.map_begin("j")
        for k, v in pairs:
            m.emit(k, v)
        m.commit()
        ctx.shuffle()
        check(ctx, mrhbm.KEY_STR, pairs, bulk=False)
        with pytest.raises(mrhbm.MrhbmError) as e:
            ctx.result_values()
        assert e.value.code == -4


def emit_all(ctx, job, pairs):
    m = ctx.map_begin(job)
    for k, v in pairs:
        m.emit(k, v)
    return m


@pytest.mark.gpu
def test_abort_replace_and_reset():
    a = random_pairs(mrhbm.KEY_STR, 27, 2000, 100, seed=1)
    b = random_pairs(mrhbm.KEY_STR, 27, 1500, 100, seed=2)
    c = random_pairs(mrhbm.KEY_STR, 27, 1000, 100, seed=3)
    with byte_ctx(mrhbm.KEY_STR) as ctx:
        emit_all(ctx, "a", a).commit()
        emit_all(ctx, "x", c).abort()  # at the end of the pool: its room is taken back
        emit_all(ctx, "b", c).commit()
        emit_all(ctx, "b", b).commit()  # replaces job b
        emit_all(ctx, "y", c).abort()
        ctx.shuffle()
        check(ctx, mrhbm.KEY_STR, a + b)
        ctx.reset()
        emit_all(ctx, "c", c).commit()
        ctx.shuffle()
        check(ctx, mrhbm.KEY_STR, c)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [mrhbm.KEY_STR, mrhbm.KEY_U64])
def test_batch_values_pinned_and_pageable_match_single_emits(kind):
    pairs = random_pairs(kind, 27, 5000, 300, seed=11)
    if kind == mrhbm.KEY_STR:  # (batch records hold keys in the stored form: keep to keys without 0x00 / 0x01)
        pairs = [(k, v) for k, v in pairs if b"\x00" not in k and b"\x01" not in k]
    dt = mrhbm.record_dtype(kind)
    recs = np.zeros(len(pairs), dtype=dt)
    recs["key"] = [k for k, _ in pairs]
    recs["val"] = 12345  # ignored
    blob = b"".join(v for _, v in pairs)
    voff = np.zeros(len(pairs) + 1, dtype=np.uint64)
    voff[1:] = np.cumsum([len(v) for _, v in pairs])
    results = []
    for mode in ("single", "pageable", "pinned"):
        with byte_ctx(kind) as ctx:
            m = ctx.map_begin("j")
            if mode == "single":
                for k, v in pairs:
                    m.emit(k, v)
            elif mode == "pageable":
                m.emit_batch_values(recs[:100], blob, voff[:101])  # two calls: the second one's offsets start past 0
                m.emit_batch_values(recs[100:], blob, voff[100:])
            else:
                pr = ctx.pinned_array(recs.shape[0], dt)
                pb = ctx.pinned_array(len(blob), np.uint8)
                po = ctx.pinned_array(voff.shape[0], np.uint64)
                pr[:], pb[:], po[:] = recs, np.frombuffer(blob, np.uint8), voff
                m.emit_batch_values(pr, pb, po)
            m.commit()
            if mode == "pinned":
                for a in (pr, pb, po):
                    ctx.host_free(a.ctypes.data)
            ctx.shuffle()
            results.append(check(ctx, kind, pairs))
    assert results[0] == results[1] == results[2]


def code_of(fn):
    with pytest.raises(mrhbm.MrhbmError) as e:
        fn()
    return e.value.code


@pytest.mark.gpu
def test_refusals():
    inval = -1
    for kw in (dict(reducer=mrhbm.RED_SUM), dict(reducer=mrhbm.RED_NONE, combiner=True)):
        assert code_of(lambda: mrhbm.Ctx(mrhbm.KEY_STR, P, device=0, flags=mrhbm.F_BYTE_VALUES, **kw)) == inval
    table = np.arange(1, 17, dtype=np.uint64) << np.uint64(60)
    with byte_ctx(mrhbm.KEY_STR) as ctx:
        m = ctx.map_begin("j")
        L = ctx.L
        assert L.mrhbm_emit_str(m.h, b"k", 1, 1) == inval
        assert L.mrhbm_emit_batch(m.h, np.zeros(1, mrhbm.record_dtype(mrhbm.KEY_STR)).ctypes.data, 1) == inval
        assert L.mrhbm_map_gen_zipf(m.h, 1, 0, 10, table.ctypes.data, table.size) == inval
        assert L.mrhbm_map_wordcount(m.h, b"a b", 3, None) == inval
        assert code_of(lambda: m.emit(b"k", b"x" * ((1 << 30) + 1))) == inval
        m.emit(b"k", b"")
        m.emit(b"k", b"v")
        m.commit()
        ctx.shuffle()
        assert L.mrhbm_result_copy(ctx.h, None, np.zeros(4, np.uint64).ctypes.data, None) == inval
        it = mrhbm.C.c_void_p()
        assert L.mrhbm_groups_open(ctx.h, ctx.partitions()[0], mrhbm.C.byref(it)) == 0
        kp, kl, vp, vn = mrhbm.C.c_void_p(), mrhbm.C.c_size_t(), mrhbm.C.c_void_p(), mrhbm.C.c_size_t()
        assert L.mrhbm_groups_next(it, mrhbm.C.byref(kp), mrhbm.C.byref(kl), mrhbm.C.byref(vp), mrhbm.C.byref(vn)) == inval
        L.mrhbm_groups_close(it)
        vals = dict(ctx.groups(ctx.partitions()[0]))[b"k"]
        assert sorted(vals) == [b"", b"v"]
    with byte_ctx(mrhbm.KEY_U64) as ctx:
        m = ctx.map_begin("j")
        assert ctx.L.mrhbm_emit_u64(m.h, 1, 1) == inval
        assert ctx.L.mrhbm_map_gen_u64(m.h, 1, 0, 10) == inval
        assert ctx.L.mrhbm_emit_device(m.h, None, 0) == inval
        m.abort()
    with mrhbm.Ctx(mrhbm.KEY_STR, P, device=0, reducer=mrhbm.RED_NONE) as ctx:  # the new calls need the flag
        m = ctx.map_begin("j")
        L = ctx.L
        assert L.mrhbm_emit_str_value(m.h, b"k", 1, b"v", 1) == inval
        assert L.mrhbm_emit_u64_value(m.h, 1, b"v", 1) == inval
        assert L.mrhbm_emit_batch_values(m.h, None, 0, None, None) == inval
        m.emit(b"k", 1)
        m.commit()
        ctx.shuffle()
        need = mrhbm.C.c_size_t()
        assert L.mrhbm_result_values(ctx.h, None, 0, None, mrhbm.C.byref(need)) == inval
        it = mrhbm.C.c_void_p()
        assert L.mrhbm_groups_open(ctx.h, ctx.partitions()[0], mrhbm.C.byref(it)) == 0
        kp, kl, vp, op, vn = (mrhbm.C.c_void_p(), mrhbm.C.c_size_t(), mrhbm.C.c_void_p(), mrhbm.C.c_void_p(),
                              mrhbm.C.c_size_t())
        assert L.mrhbm_groups_next_values(it, *(mrhbm.C.byref(x) for x in (kp, kl, vp, op, vn))) == inval
        L.mrhbm_groups_close(it)


@pytest.fixture
def corpus(tmp_path, golden_wordcount):
    files = []
    for job in range(4):
        toks = expand_tokens(golden_wordcount, job)
        p = tmp_path / ("file%d.txt" % job)
        p.write_bytes(b"\n".join(b" ".join(toks[i:i + 7]) for i in range(0, len(toks), 7)) + b"\n")
        files.append(str(p))
    WordCount.FILES[:] = files
    II.RESULT.clear()
    return files


@pytest.mark.gpu
def test_inverted_index_through_server_loop(tmp_path, corpus, golden_wordcount):
    S = "lua_mapreduce_b200.mapreduce.examples.InvertedIndex.init"
    s = server.new("hbm://local", "inverted-index")
    s.configure(dict(taskfn=S, mapfn=S, partitionfn=S, reducefn=S, finalfn=S, storage="hbm", hbm={"value_kind": "bytes"}))
    s.loop()
    want = {k: sorted(corpus[j].encode() for j in range(4) if c[j] > 0) for k, _, c in golden_wordcount}
    assert II.RESULT == want
    out = tmp_path / "results"
    out.mkdir()
    names = s.export_results(str(out))
    lines = set()
    for n in names:
        lines.update((out / n).read_bytes().splitlines())
    assert lines == {b"return " + O.escape(k) + b"," + O.serialize_table_ipairs(v) for k, v in want.items()}


@pytest.mark.gpu
def test_numbers_and_strings_keep_their_lua_type():
    from lua_mapreduce_b200.mapreduce import tuple as T
    vals = [-3, 0.5, 2 ** 53, -(2 ** 53), -0.0, 0, 1e308, -1e-300, float("inf"), float("-inf"), b"", b"str", "text",
            b"\x00\x01\xff"]
    with byte_ctx(mrhbm.KEY_STR) as ctx:
        m = ctx.map_begin("j")
        for i, v in enumerate(vals):
            m.emit(b"k%d" % (i % 3), T.encode_value(v))
        m.commit()
        ctx.shuffle()
        got = [T.decode_value(v) for p in ctx.partitions() for _, vs in ctx.groups(p) for v in vs]
    want = [v.encode() if isinstance(v, str) else v for v in vals]
    key = lambda v: (type(v).__name__, repr(v))  # noqa: E731  (type and value, -0.0 apart from 0)
    assert sorted(got, key=key) == sorted(want, key=key)
