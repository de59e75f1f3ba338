"""mrhbm_map_words_value: the device tokeniser on a byte-values ctx, emitting (word, value) for every word of a text.

The expected result is a host tokenisation: the text split on the six C-locale white-space bytes, every word paired
with the call's value.  Results are compared as key -> sorted multiset of values through Ctx.groups and, where every
key fits a record slot, row by row through result_copy + result_values.  Partition ids come from the oracle."""
import random
import re
from collections import Counter

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

gpu = pytest.mark.gpu
P = 7
INVAL, KEY = -1, -4
PIECE = 1 << 26  # bytes per device piece of one tokeniser call
STAGE = 4 << 20  # value bytes staged next to the records; a longer value is copied on its own
WS = b" \t\n\v\f\r"  # C-locale isspace (Lua's %s)
IS_WS = np.zeros(256, dtype=bool)
IS_WS[list(WS)] = True


def byte_ctx(kind=mrhbm.KEY_STR, max_key_bytes=27, P=P):
    return mrhbm.Ctx(kind, P, max_key_bytes=max_key_bytes, device=0, reducer=mrhbm.RED_NONE, flags=mrhbm.F_BYTE_VALUES)


# ---- helpers (the same rules as test_tokeniser_pieces.py) ---------------------------------------------------------
def tokens(text):
    """split on the six C-locale white-space bytes only (str.split would also split on 0x1c-0x1f)"""
    return [w for w in re.split(rb"[ \t\n\v\f\r]+", bytes(text)) if w]


def escape(k):
    return k.replace(b"\x01", b"\x01\x02").replace(b"\x00", b"\x01\x01")


def unescape(k):
    return k.replace(b"\x01\x01", b"\x00").replace(b"\x01\x02", b"\x01")


def put(t, x, b):
    t[x:x + len(b)] = np.frombuffer(b, dtype=np.uint8)


def piece_end(t, p):
    """a piece starting at p ends at min(len, p + 2^26), moved back to just after the last white-space byte before it"""
    e = min(len(t), p + PIECE)
    if e == len(t):
        return e
    hit = np.flatnonzero(IS_WS[t[p:e]])
    return p + int(hit[-1]) + 1 if hit.size else e


def piece_cuts(t):
    cuts = [0]
    while cuts[-1] < len(t):
        cuts.append(piece_end(t, cuts[-1]))
    return cuts


def word_starts(t):
    nonws = ~IS_WS[t]
    start = nonws.copy()
    start[1:] &= ~nonws[:-1]
    return start


def expected(calls, pairs=()):
    """{word: sorted values} of (text, value) calls plus single pairs"""
    want = {}
    for text, v in calls:
        for w in tokens(text):
            want.setdefault(w, []).append(v)
    for k, v in pairs:
        want.setdefault(k, []).append(v)
    return {k: sorted(v) for k, v in want.items()}


def check(ctx, want, rows=True):
    """groups == want (keys ascending, partitions right); with rows, result_copy + result_values agree row by row"""
    got = {}
    for p in ctx.partitions():
        keys = []
        for k, vals in ctx.groups(p):
            assert O.part_fnv_lua(k, P) == p
            assert k not in got
            keys.append(k)
            got[k] = sorted(vals)
        assert keys == sorted(keys)
    assert got == want
    if not rows:
        with pytest.raises(mrhbm.MrhbmError) as e:  # long keys live on the host: no bulk result
            ctx.result_copy()
        assert e.value.code == KEY
        return
    keys, sums, _ = ctx.result_copy()
    assert sums is None
    blob, roff = ctx.result_values()
    raw = blob.tobytes()
    by_row = {}
    for r in range(keys.shape[0]):
        by_row.setdefault(unescape(bytes(keys[r])), []).append(raw[int(roff[r]):int(roff[r + 1])])
    assert {k: sorted(v) for k, v in by_row.items()} == want


def code_of(fn):
    with pytest.raises(mrhbm.MrhbmError) as e:
        fn()
    return e.value.code


# =================================================================================================================
# record classes, values, short texts
# =================================================================================================================
def class_words(kb):
    """(words whose escaped form fits the kb-byte slot with its zero byte, words that do not)"""
    fits = [b"sep%d" % i for i in range(12)]
    for b in (0x00, 0x01, 0x02, 0x1C, 0x7F, 0x80, 0xFF):
        c = bytes([b])
        fits += [c, b"w" + c, c + b"v", b"x" + c * 3 + b"y"]
    fits += [b"a" * (kb - 1), b"b" * (kb - 3) + b"\x00", b"c" * (kb - 3) + b"\x01", b"\x00" * ((kb - 2) // 2) + b"d",
             b"\x01" * ((kb - 2) // 2), b"\xff" * (kb - 1)]
    long = [b"a" * kb, b"b" * (kb - 2) + b"\x00", b"\x00" * (kb // 2), b"\x01" + b"f" * (kb - 2)]
    assert all(len(escape(w)) <= kb - 1 for w in fits) and all(len(escape(w)) >= kb for w in long)
    assert sum(len(escape(w)) == kb - 1 for w in fits) == 5  # (at the class maximum)
    return fits, long


def class_text(words, rng):
    """every word 1..3 times in random order, between random runs of white space, with white space at both ends"""
    toks = [w for w in words for _ in range(rng.randint(1, 3))]
    rng.shuffle(toks)
    return b"\t " + b"".join(w + bytes(rng.choice(WS) for _ in range(rng.randint(1, 3))) for w in toks)


def value_of(n, seed):
    rng = random.Random(seed)
    return b"\x00" + bytes(rng.getrandbits(8) for _ in range(n - 1)) if n else b""


VALUES = [b"", b"\x00", bytes(range(16)), b"\x00v\x00" * 5 + b"\x00\x00", value_of(4097, 1)]  # 0, 1, 16, 17, 4 KiB + 1


@gpu
@pytest.mark.parametrize("mkb", [27, 59, 123])
def test_record_classes_and_values(mkb):
    kb = mrhbm.record_dtype(mrhbm.KEY_STR, mkb)["key"].itemsize
    fits, long = class_words(kb)
    rng = random.Random(mkb)
    dev = class_text(fits, rng)  # every word fits: the device emits the records
    mixed = class_text(fits + long, rng)  # words that do not fit: the call goes through the host
    with byte_ctx(max_key_bytes=mkb) as ctx:
        assert ctx.record_bytes == kb + 4
        for v in VALUES:
            ctx.reset()
            m = ctx.map_begin("dev")
            assert m.words_value(dev, v) == len(tokens(dev))
            m.commit()
            ctx.shuffle()
            check(ctx, expected([(dev, v)]))
        ctx.reset()
        m = ctx.map_begin("mixed")
        assert m.words_value(dev, VALUES[3]) + m.words_value(mixed, VALUES[4]) == len(tokens(dev)) + len(tokens(mixed))
        m.commit()
        ctx.shuffle()
        check(ctx, expected([(dev, VALUES[3]), (mixed, VALUES[4])]), rows=False)


@gpu
def test_a_value_larger_than_the_value_stage():
    big = value_of(STAGE + 5, 2)
    dev = b"alpha beta\tgamma alpha\n\x00zero delta "
    host = b"beta " + b"L" * 40 + b" epsilon"  # a word over 27 bytes: this call goes through the host
    with byte_ctx() as ctx:
        m = ctx.map_begin("big")
        assert m.words_value(dev, big) == 6
        assert m.words_value(b"alpha omega", VALUES[2]) == 2
        m.commit()
        ctx.shuffle()
        check(ctx, expected([(dev, big), (b"alpha omega", VALUES[2])]))
        ctx.reset()
        m = ctx.map_begin("big")
        assert m.words_value(host, big) == 3
        assert m.words_value(dev, big) == 6
        m.commit()
        ctx.shuffle()
        check(ctx, expected([(host, big), (dev, big)]), rows=False)


@gpu
def test_empty_and_white_space_texts():
    edged = b" \n\tlead and trail\r\v\f "
    with byte_ctx() as ctx:
        m = ctx.map_begin("j")
        assert m.words_value(b"", b"e") == 0
        assert ctx.L.mrhbm_map_words_value(m.h, None, 0, b"e", 1, None) == 0
        assert m.words_value(WS * 50, b"w") == 0
        assert m.words_value(edged, b"v") == 3
        assert m.words_value(b"one-word-no-white-space", b"") == 1
        m.commit()
        ctx.shuffle()
        check(ctx, expected([(edged, b"v"), (b"one-word-no-white-space", b"")]))


# =================================================================================================================
# a text of three pieces: words at the piece cuts, every piece on the device, then the middle one on the host
# =================================================================================================================
LONG = b"long-word-in-the-middle-piece-".ljust(40, b"x")
BIG_VALUE = b"\x00file\x00name\x01.txt\x00\x00"  # 17 bytes


@pytest.fixture(scope="module")
def big_text():
    """2 * 2^26 + 1 MiB bytes of words of a 3000-word vocabulary (1 to 27 bytes, some holding 0x00 / 0x01) between
    runs of white space; the first piece ends just before a word that reaches its 2^26 mark, the third piece starts
    with a word right after a white-space byte at the second piece's mark.  Returns (text, piece cuts, middle)."""
    rng = random.Random(17)
    letters = b"abcdefghijklmnopqrstuvwxyz"
    vocab = {bytes(rng.choice(letters) for _ in range(rng.choice((1, 2, 27)) if i < 60 else rng.randint(6, 27)))
             for i in range(2900)}
    vocab |= {b"%c\x00%c\x01" % (rng.choice(letters), rng.choice(letters)) + b"q" * rng.randint(0, 20) for _ in range(100)}
    vocab = sorted(vocab)
    seps = [b" ", b" ", b" ", b"\n", b"\t", b" \r\n", b"\v", b"\f "]
    combos = [w + s for w in vocab for s in seps]
    n = 2 * PIECE + (1 << 20)
    nrng = np.random.default_rng(17)
    pick = nrng.integers(0, len(combos), n // 12).tolist()
    t = np.frombuffer(b"".join([combos[i] for i in pick]), dtype=np.uint8)
    assert t.nbytes > n
    t = t[:n].copy()
    t[-1] = ord(" ")
    x = PIECE
    put(t, x - 6, b" edged\n")  # a word whose last byte is x - 1: the cut moves back before it
    c1 = piece_end(t, 0)
    assert c1 == x - 5
    x = c1 + PIECE
    put(t, x - 3, b"ab\vcd")  # one white-space byte at x - 1: the cut stays at x, "cd..." starts the third piece
    cuts = piece_cuts(t)
    assert cuts == [0, c1, x, n]
    return t, cuts, c1 + PIECE // 2


def id_runs(ids):
    """sorted lengths of the runs of equal value ids in pool order; every run's id is the pool index of its first pair"""
    ids = ids.astype(np.int64)
    starts = np.concatenate([[0], np.flatnonzero(np.diff(ids)) + 1])
    assert (ids[starts] == starts).all()
    return sorted(np.diff(np.concatenate([starts, [ids.size]])).tolist())


def check_big(ctx, want, value, rows):
    """groups: key -> count, every value == value; rows: result_copy + result_values, vectorised"""
    got = {}
    for p in ctx.partitions():
        prev = None
        for k, vals in ctx.groups(p):
            assert prev is None or prev < k
            prev = k
            assert O.part_fnv_lua(k, P) == p
            assert vals.count(value) == len(vals)
            got[k] = len(vals)
    assert got == want
    if not rows:
        assert code_of(ctx.result_copy) == KEY
        return
    keys, _, _ = ctx.result_copy()
    blob, roff = ctx.result_values()
    assert (np.diff(roff.astype(np.int64)) == len(value)).all()
    assert (blob.reshape(-1, len(value)) == np.frombuffer(value, dtype=np.uint8)).all()
    uk, cnt = np.unique(keys, return_counts=True)
    assert {unescape(bytes(k)): int(c) for k, c in zip(uk, cnt)} == want


@gpu
def test_three_pieces_then_a_host_piece_in_the_middle(big_text):
    t, cuts, mid = big_text
    start = word_starts(t)
    per_piece = [int(start[a:b].sum()) for a, b in zip(cuts[:-1], cuts[1:])]
    want = Counter(tokens(t))
    assert sum(want.values()) == sum(per_piece)
    with byte_ctx() as ctx:
        # every piece on the device: the pairs of a piece share the id of its first pair
        m = ctx.map_begin("big")
        assert m.words_value(t, BIG_VALUE) == sum(per_piece)
        m.commit()
        ids = ctx.pool_read(0, sum(per_piece))["val"]
        first = np.concatenate([[0], np.cumsum(per_piece)[:-1]])
        assert (ids == np.repeat(first, per_piece)).all()
        ctx.shuffle()
        check_big(ctx, dict(want), BIG_VALUE, rows=True)
        # a word too long for the record class in the middle of piece 2: that piece goes through the host, its long
        # key is merged into the groups at its place in key order
        t2 = t.copy()
        put(t2, mid, b" " + LONG + b" ")
        assert piece_cuts(t2) == cuts
        per2 = [int(word_starts(t2[a:b]).sum()) for a, b in zip(cuts[:-1], cuts[1:])]
        want2 = Counter(tokens(t2))
        assert want2[LONG] == 1
        ctx.reset()
        m = ctx.map_begin("big")
        assert m.words_value(t2, BIG_VALUE) == sum(per2)
        m.commit()
        # device pieces: one id per piece; host-staged pairs: one id per pair (the long word is not in the pool)
        n = sum(per2) - 1
        assert id_runs(ctx.pool_read(0, n)["val"]) == sorted([per2[0], per2[2]] + [1] * (per2[1] - 1))
        assert code_of(lambda: ctx.pool_read(0, n + 1)) == INVAL
        ctx.shuffle()
        check_big(ctx, dict(want2), BIG_VALUE, rows=False)


@gpu
def test_failed_call_leaves_pool_arena_and_long_keys_as_before(big_text):
    """a 2 MB word (over the 1 MB key limit) in the second piece of a call, after a long word: the call fails with
    MRHBM_E_KEY after its first piece went to the device; none of its pairs, value bytes or long keys survive"""
    t, cuts, _ = big_text
    bad = t[:cuts[1] + (16 << 20)].copy()
    put(bad, cuts[1] + (1 << 20), b" " + LONG + b" ")
    y = cuts[1] + (8 << 20)
    bad[y:y + (2 << 20)] = ord("z")
    bad[y - 1] = bad[y + (2 << 20)] = ord(" ")
    assert piece_cuts(bad)[:2] == cuts[:2]
    early = b"one two two " + b"E" * 40 + b" three"  # a long word: this call goes through the host
    with byte_ctx() as ctx:
        m = ctx.map_begin("undo")
        m.emit(b"before", b"b0")
        assert m.words_value(early, b"early") == 5
        assert code_of(lambda: m.words_value(bad, b"BAD")) == KEY
        m.emit(b"after", b"a1")
        m.commit()
        assert ctx.pool_read(0, 6)["val"].tolist() == [0, 1, 2, 3, 4, 5]  # before, 4 words of early, after
        assert code_of(lambda: ctx.pool_read(0, 7)) == INVAL
        ctx.shuffle()
        check(ctx, expected([(early, b"early")], [(b"before", b"b0"), (b"after", b"a1")]), rows=False)


# =================================================================================================================
# ids, mixing with the other emits, commit / abort / replace / reset
# =================================================================================================================
def batch(keys, vals):
    recs = np.zeros(len(keys), dtype=mrhbm.record_dtype(mrhbm.KEY_STR))
    recs["key"] = keys
    voff = np.zeros(len(keys) + 1, dtype=np.uint64)
    voff[1:] = np.cumsum([len(v) for v in vals])
    return recs, b"".join(vals), voff


@gpu
def test_pairs_of_a_call_share_the_id_of_its_first_pair():
    recs, blob, voff = batch([b"x", b"y"], [b"X", b"YY"])
    with byte_ctx() as ctx:
        m = ctx.map_begin("ids")
        m.emit(b"first", b"f")  # id 0
        assert m.words_value(b"a b c d e", b"V1") == 5  # ids 1 (x5)
        m.emit_batch_values(recs, blob, voff)  # ids 6, 7
        assert m.words_value(b"f\tg\nh", b"") == 3  # id 8 (x3)
        m.emit(b"last", b"l")  # id 11
        m.commit()
        assert ctx.pool_read(0, 12)["val"].tolist() == [0, 1, 1, 1, 1, 1, 6, 7, 8, 8, 8, 11]
        ctx.shuffle()
        check(ctx, expected([(b"a b c d e", b"V1"), (b"f\tg\nh", b"")],
                            [(b"first", b"f"), (b"x", b"X"), (b"y", b"YY"), (b"last", b"l")]))


T1 = b"the quick brown fox\njumps over the lazy dog " + b"Q" * 30 + b" end"  # a long word: host piece
T2 = b"the dog sleeps\tthe fox runs\n"


def mixed_job(ctx, job, tag):
    """two calls with different values, a single emit and a batch emit; returns the handle and the expected pairs"""
    recs, blob, voff = batch([b"fox", b"batch-" + tag], [b"b1" + tag, b"\x00b2" + tag])
    m = ctx.map_begin(job)
    assert m.words_value(T1, b"v1" + tag) == 11
    m.emit(b"single", b"s" + tag)
    m.emit_batch_values(recs, blob, voff)
    assert m.words_value(T2, b"\x00v2" + tag) == 6
    calls = [(T1, b"v1" + tag), (T2, b"\x00v2" + tag)]
    pairs = [(b"single", b"s" + tag), (b"fox", b"b1" + tag), (b"batch-" + tag, b"\x00b2" + tag)]
    return m, calls, pairs


@gpu
def test_mixed_emits_abort_replace_and_reset():
    with byte_ctx() as ctx:
        m, calls_a, pairs_a = mixed_job(ctx, "a", b"A")
        m.commit()
        mixed_job(ctx, "x", b"X")[0].abort()  # at the end of the pool: its room is taken back
        mixed_job(ctx, "b", b"B")[0].commit()
        m, calls_b, pairs_b = mixed_job(ctx, "b", b"C")
        m.commit()  # replaces job b
        mixed_job(ctx, "y", b"Y")[0].abort()
        ctx.shuffle()
        check(ctx, expected(calls_a + calls_b, pairs_a + pairs_b), rows=False)
        ctx.reset()
        m = ctx.map_begin("c")
        assert m.words_value(T2, b"after reset") == 6
        m.commit()
        ctx.shuffle()
        check(ctx, expected([(T2, b"after reset")]))


@gpu
def test_refusals():
    with mrhbm.Ctx(mrhbm.KEY_STR, P, device=0, reducer=mrhbm.RED_NONE) as ctx:  # integer values
        m = ctx.map_begin("j")
        assert ctx.L.mrhbm_map_words_value(m.h, b"a b", 3, b"v", 1, None) == INVAL
        assert code_of(lambda: m.words_value(b"a b", b"v")) == INVAL
        m.abort()
    with byte_ctx(mrhbm.KEY_U64) as ctx:
        m = ctx.map_begin("j")
        assert ctx.L.mrhbm_map_words_value(m.h, b"a b", 3, b"v", 1, None) == INVAL
        m.abort()
    with byte_ctx() as ctx:
        m = ctx.map_begin("j")
        L = ctx.L
        n = mrhbm.C.c_uint64(99)
        assert L.mrhbm_map_words_value(m.h, b"a b", 3, None, 1, mrhbm.C.byref(n)) == INVAL
        assert n.value == 0
        assert L.mrhbm_map_words_value(m.h, b"a b", 3, b"x", (1 << 30) + 1, None) == INVAL
        assert L.mrhbm_map_wordcount(m.h, b"a b", 3, None) == INVAL  # the integer-valued call stays refused
        assert L.mrhbm_map_words_value(m.h, b"a b", 3, None, 0, mrhbm.C.byref(n)) == 0  # (no value bytes: empty)
        assert n.value == 2
        m.commit()
        ctx.shuffle()
        check(ctx, {b"a": [b""], b"b": [b""]})


# =================================================================================================================
# the mirror: InvertedIndex with the device tokeniser declared
# =================================================================================================================
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


def run_inverted_index(tmp_path, mapfn, name):
    S = "lua_mapreduce_b200.mapreduce.examples.InvertedIndex.init"
    II.RESULT.clear()
    s = server.new("hbm://local", name)
    s.configure(dict(taskfn=S, mapfn=mapfn, partitionfn=S, reducefn=S, finalfn=S, storage="hbm",
                     hbm={"value_kind": "bytes"}))
    s.loop()
    out = tmp_path / name
    out.mkdir()
    files = {n: (out / n).read_bytes() for n in s.export_results(str(out))}
    return dict(II.RESULT), files


@gpu
def test_inverted_index_device_mapfn_matches_the_host_mapfn(tmp_path, corpus, golden_wordcount):
    host = run_inverted_index(tmp_path, "lua_mapreduce_b200.mapreduce.examples.InvertedIndex.init", "host")
    dev = run_inverted_index(tmp_path, "lua_mapreduce_b200.mapreduce.examples.InvertedIndex.mapfn_device", "device")
    want = {k: sorted(corpus[j].encode() for j in range(4) if c[j] > 0) for k, _, c in golden_wordcount}
    assert host[0] == want
    assert dev[0] == want
    assert dev[1] == host[1] and len(host[1]) > 0


def test_words_file_mapfn_needs_byte_values():
    S = "lua_mapreduce_b200.mapreduce.examples.InvertedIndex.init"
    s = server.new("hbm://local", "words-file-int")
    with pytest.raises(ValueError, match="words_file"):
        s.configure(dict(taskfn=S, mapfn="lua_mapreduce_b200.mapreduce.examples.InvertedIndex.mapfn_device",
                         partitionfn=S, reducefn=S, finalfn=S, storage="hbm"))
