"""The device tokeniser (mrhbm_map_wordcount) at the sizes the end-to-end word count runs at: calls of several 64 MiB
pieces, edge patterns at the piece cuts and at 256-byte block edges, every record class and byte value, the host
fall-back and the undo of a failed call inside a call of several pieces, and two contexts driven at once from two
threads.  Part A (no GPU) pins the host-side text generator to the word stream the oracle counts.

Every expected result comes from the CPU oracle (O.naive_wordcount, O.zipf_counts + O.wordcount_from_counts,
O.groupby_u64) or from words the test placed itself, and every result is compared in full."""
import contextlib
import re
import threading
import time
from collections import Counter

import numpy as np
import pytest

import mrhbm_loader
import oracle as O
from test_gpu_combiner_and_wide_sums import escape

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm, synth  # noqa: E402

gpu = pytest.mark.gpu
SEED = synth.SEED
P = 15
PIECE = 1 << 26  # kTokPiece: bytes per device piece of one wordcount call
WS = b" \t\n\v\f\r"  # C-locale isspace (Lua's %s)
IS_WS = np.zeros(256, dtype=bool)
IS_WS[list(WS)] = True
SP, NL = ord(" "), ord("\n")
N_WORDS = 30_000_000  # the Zipf text: about 200 MB, more than 2 pieces


def tokens(text):
    """split on the six C-locale white-space bytes only (str.split would also split on 0x1c-0x1f)"""
    return [w for w in re.split(rb"[ \t\n\v\f\r]+", bytes(text)) if w]


def stream_words(first, n, table):
    recs = O.gen_zipf_rec32(SEED, first, n, table)
    return [bytes(r[:28]).rstrip(b"\0") for r in recs]


def first_diff(got, want):
    for i, (a, b) in enumerate(zip(got, want)):
        if a != b:
            return "row %d: got %r, want %r" % (i, a, b)
    return "%d rows, want %d" % (len(got), len(want))


# ---- the piece rule of mrhbm_map_wordcount, restated ------------------------------------------------------------
def piece_end(t, p):
    """a piece starting at p ends at min(len, p + 2^26), moved back to just after the last white-space byte before it"""
    e = min(len(t), p + PIECE)
    if e == len(t):
        return e
    w = 4096
    while True:
        a = max(p, e - w)
        hit = np.flatnonzero(IS_WS[t[a:e]])
        if hit.size:
            return a + int(hit[-1]) + 1
        if a == p:
            return e
        w *= 16


def piece_cuts(t):
    cuts = [0]
    while cuts[-1] < len(t):
        cuts.append(piece_end(t, cuts[-1]))
    return cuts


# ---- comparisons --------------------------------------------------------------------------------------------------
def result_of(ctx, keys=None, sums=None):
    """(keys, sums, part_off) of result_copy, each partition in ascending key order"""
    keys, sums, po = ctx.result_copy(keys, sums)
    keys, sums = keys.copy(), sums.copy()
    if not ctx.result_info().sorted:  # a partition is several ascending runs: sort each
        order = np.lexsort((keys, np.repeat(np.arange(P), np.diff(po.astype(np.int64)))))
        keys, sums = keys[order], sums[order]
    return keys, sums, po


def check_arrays(got, want):
    keys, sums, po = got
    okeys, osums, opo = want
    assert (po == opo).all()
    assert keys.shape == okeys.shape
    bad = np.flatnonzero((keys != okeys) | (sums != osums))
    assert bad.size == 0, "%d groups differ, first: got %r %d, want %r %d" % (
        bad.size, keys[bad[0]], sums[bad[0]], okeys[bad[0]], osums[bad[0]])


def check_vs_words(ctx, counts):
    """every (partition, key, [sum]) from groups() against word counts {key: count}; when every key fits a record
    slot also result_copy's keys (stored escaped), sums and part_off"""
    rows = sorted((O.part_fnv_lua(k, P), k, c) for k, c in counts.items())
    got = [(p, k, v) for p in ctx.partitions() for k, v in ctx.groups(p)]
    want = [(p, k, [c]) for p, k, c in rows]
    assert got == want, first_diff(got, want)
    kb = ctx.result_info().key_bytes
    if all(len(escape(k)) < kb for _, k, _ in rows):
        keys, sums, po = ctx.result_copy()
        assert (po == np.searchsorted([r[0] for r in rows], np.arange(P + 1))).all()
        part = np.repeat(np.arange(P), np.diff(po.astype(np.int64)))
        got = sorted(zip(part.tolist(), keys.tolist(), sums.tolist()))
        want = [(p, escape(k), c) for p, k, c in rows]
        assert got == want, first_diff(got, want)


def naive_counts(*texts):
    ntok, wc = O.naive_wordcount([bytes(t) for t in texts])
    return dict(wc), ntok


def count_text(ctx, *calls):
    """one map job of wordcount calls (each a uint8 array or bytes), committed and shuffled; returns the words"""
    ctx.reset()
    m = ctx.map_begin("text")
    n = sum(m.wordcount(c) for c in calls)
    m.commit()
    ctx.shuffle()
    return n


# =================================================================================================================
# A. the end-to-end text generator is the oracle's word stream (host only)
# =================================================================================================================
@pytest.fixture(scope="module")
def table():
    return synth.zipf_table()


@pytest.mark.parametrize("first,n,wpl", [(0, 1000, 25), (10**9 + 7, 1003, 25), (10**9 + 7, 7, 25), (31, 500, 1),
                                         (0, 4096, 7)])
def test_synth_text_is_the_oracle_stream(table, first, n, wpl):
    words = stream_words(first, n, table)
    text = mrhbm.synth_zipf_text(SEED, first, n, table, words_per_line=wpl, threads=4)
    assert tokens(text) == words
    lines = [b" ".join(words[i:i + wpl]) for i in range(0, n, wpl)]  # a line end after every wpl words and the last
    assert text.tobytes() == b"\n".join(lines) + b"\n"


@pytest.mark.parametrize("n", [100, 101])
def test_synth_text_does_not_depend_on_threads(table, n):
    """more threads than lines (4 or 5 lines): every thread count writes the same bytes"""
    texts = [mrhbm.synth_zipf_text(SEED, 999, n, table, threads=th).tobytes() for th in (1, 3, 64, 256)]
    assert texts[0] == texts[1] == texts[2] == texts[3]
    assert tokens(texts[0]) == stream_words(999, n, table)


def test_synth_text_empty_and_short_buffer(table):
    assert mrhbm.synth_zipf_text(SEED, 5, 0, table).nbytes == 0
    need = mrhbm.synth_zipf_text(SEED, 5, 333, table).nbytes
    out = np.full(need - 1, 0xAA, dtype=np.uint8)
    with pytest.raises(mrhbm.MrhbmError) as e:
        mrhbm.synth_zipf_text(SEED, 5, 333, table, out=out)
    assert e.value.code == -1 and ("needs %d bytes" % need) in str(e.value)
    assert (out == 0xAA).all()
    out = np.empty(need, dtype=np.uint8)
    assert mrhbm.synth_zipf_text(SEED, 5, 333, table, out=out).nbytes == need


def test_zipf_counts_count_the_text_words(table):
    """the identity the end-to-end check relies on: O.zipf_counts over words [first, first + n) counts the words of
    synth_zipf_text(first, n)"""
    first, n = 77_777, 20_000
    counts = O.zipf_counts(SEED, first, n, table, nthreads=3)
    want = {O.rank_to_key(r + 1): int(counts[r]) for r in np.flatnonzero(counts)}
    assert Counter(tokens(mrhbm.synth_zipf_text(SEED, first, n, table))) == want


# =================================================================================================================
# B. one call over several pieces: the bench's Zipf text in four ways of feeding it
# =================================================================================================================
@pytest.fixture(scope="module")
def zipf_text(table):
    text = mrhbm.synth_zipf_text(SEED, 0, N_WORDS, table)
    okeys, osums, opo = O.wordcount_from_counts(O.zipf_counts(SEED, 0, N_WORDS, table), O.PART_FNV_LUA, P)
    assert text.nbytes > 2 * PIECE and len(piece_cuts(text)) - 1 >= 3
    return text, (okeys.view("S28").reshape(-1), osums, opo)


@pytest.fixture(scope="module")
def ctxs():
    """the word-count context with and without the map-side combiner (with: the bench's config 3 context)"""
    cs = {comb: mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, combiner=comb) for comb in (False, True)}
    yield cs
    for c in cs.values():
        c.close()


def ws_cuts(text, targets, rng):
    """call boundaries at random white space inside lines near the targets: just before or just after a space"""
    cuts = [0]
    for i, q in enumerate(targets):
        q += int(rng.integers(0, 1 << 16))
        q += int(np.flatnonzero(text[q:q + 4096] == SP)[0]) + (i & 1)
        cuts.append(q)
    return cuts + [text.nbytes]


def padded_calls(text, size):
    """the text as calls of exactly `size` bytes (the last one shorter): each call holds the text up to its last
    white space that fits and is filled up with spaces, so every call boundary falls on white space"""
    calls, p, n = [], 0, text.nbytes
    while n - p > size:
        q = p + int(np.flatnonzero(IS_WS[text[p:p + size]])[-1]) + 1
        calls.append(np.concatenate([text[p:q], np.full(size - (q - p), SP, dtype=np.uint8)]))
        p = q
    return calls + [text[p:]]


@gpu
@pytest.mark.parametrize("combiner", [False, True])
def test_zipf_text_in_one_call_and_cut_at_white_space(ctxs, zipf_text, combiner):
    ctx, (text, want) = ctxs[combiner], zipf_text
    # (a) one call of > 2 pieces
    assert count_text(ctx, text) == N_WORDS
    check_arrays(result_of(ctx), want)
    # (b) calls cut at random spaces inside lines: a short call, one of > 2 pieces, a short one and the rest
    rng = np.random.default_rng(5)
    cuts = ws_cuts(text, [1 << 20, (1 << 20) + int(2.2 * PIECE), (6 << 20) + int(2.2 * PIECE)], rng)
    assert all(text[c - 1] == SP or text[c] == SP for c in cuts[1:-1])
    assert cuts[2] - cuts[1] > 2 * PIECE
    assert count_text(ctx, *[text[a:b] for a, b in zip(cuts[:-1], cuts[1:])]) == N_WORDS
    check_arrays(result_of(ctx), want)


@gpu
@pytest.mark.parametrize("combiner", [False, True])
@pytest.mark.parametrize("size", [PIECE - 1, PIECE, PIECE + 1])
def test_zipf_text_in_calls_of_one_piece_size(ctxs, zipf_text, combiner, size):
    ctx, (text, want) = ctxs[combiner], zipf_text
    calls = padded_calls(text, size)
    assert len(calls) >= 3 and all(c.nbytes == size for c in calls[:-1])
    assert count_text(ctx, *calls) == N_WORDS
    check_arrays(result_of(ctx), want)


@gpu
@pytest.mark.parametrize("combiner", [False, True])
def test_zipf_text_from_pinned_memory_at_every_alignment(ctxs, zipf_text, combiner):
    ctx, (text, want) = ctxs[combiner], zipf_text
    n = text.nbytes
    buf = ctx.pinned_array(n + 16, np.uint8)
    try:
        for off in range(16):  # 0: a pinned_array; 1..15: a pinned address off bytes past the buffer start
            buf[off:off + n] = text
            ctx.reset()
            m = ctx.map_begin("pinned")
            assert m.wordcount(buf[:n] if off == 0 else buf.ctypes.data + off, n) == N_WORDS
            m.commit()
            ctx.shuffle()
            check_arrays(result_of(ctx), want)
    finally:
        ctx.host_free(buf.ctypes.data)


# =================================================================================================================
# C. edge patterns at the piece cuts, at multiples of 2^26 and at 256-byte block edges
# =================================================================================================================
@pytest.fixture(scope="module")
def filler():
    """words of 1..6 letters a..d (5,460 distinct) between random runs of the six white-space bytes"""
    n = int(3.6 * PIECE)
    rng = np.random.default_rng(7)
    t = rng.integers(ord("a"), ord("e"), n, dtype=np.uint8)
    ws = rng.integers(0, 100, n, dtype=np.uint8) < 22
    pos = np.cumsum(rng.integers(1, 8, n // 3, dtype=np.int32))  # white space at least every 7 bytes, no period
    ws[pos[pos < n]] = True
    t[ws] = np.frombuffer(WS, dtype=np.uint8)[rng.integers(0, 6, int(ws.sum()))]
    t[0] = ord("b")  # the text starts with a word
    return t


def put(t, x, b):
    t[x:x + len(b)] = np.frombuffer(b, dtype=np.uint8)


# each pattern: (writer, window (lo, hi) relative to x, where the piece whose 2^26 mark is x then ends, relative to x)
def word_ends_at(t, x):  # a word whose last byte is x - 1: the cut moves back before it
    put(t, x - 6, b" edged\n")


def ws_byte_before(t, x):  # one white-space byte at x - 1 between two words: the cut stays at x
    put(t, x - 3, b"ab\vcd")


def ws_run_across(t, x):
    put(t, x - 3, b"\t \r\n\f ")


def word27_over(t, x):  # the longest word of the 32-byte class across the mark
    put(t, x - 14, b" " + b"abcdefghijklmnopqrstuvwxyz0"[:27] + b" ")


def one_letter_words(t, x):  # "a a a ...": 128 word starts in every 256-byte block
    t[x - 2048:x + 2048:2] = ord("a")
    t[x - 2047:x + 2048:2] = SP


def ws_run_over_a_piece(t, x):  # a whole piece of white space: the piece has no words
    t[x - 100:x + PIECE + 900] = np.frombuffer(WS, dtype=np.uint8)[np.arange(PIECE + 1000) % 6]


PATTERNS = {"word_ends_at_mark": (word_ends_at, (-6, 1), -5), "ws_byte_before_mark": (ws_byte_before, (-3, 2), 0),
            "ws_run_across_mark": (ws_run_across, (-3, 3), 0), "word27_over_mark": (word27_over, (-14, 15), -13),
            "one_letter_words": (one_letter_words, (-2048, 2048), 0),
            "ws_run_over_a_piece": (ws_run_over_a_piece, (-100, PIECE + 900), 0)}
ENDINGS = {"ends_inside_a_word": b" xyz", "ends_in_a_one_byte_word": b" q", "ends_in_a_ws_run": b"z\t \n\r\v\f"}
MARK_OFFSETS = [0, -1, 1, -255, 255, -256, 256]


def edge_text(filler, name, ending):
    """2^27 + 1 MiB bytes of filler with the pattern where every piece's 2^26 mark falls (pieces computed with the
    rule after each placement), then at every multiple of 2^26 plus each offset whose window is still free
    (the order of the offsets turns from mark to mark), and the ending at the end"""
    write, (lo, hi), shift = PATTERNS[name]
    t = filler[:2 * PIECE + (1 << 20)].copy()
    taken, cuts = [], [0]
    while cuts[-1] + PIECE < len(t):
        x = cuts[-1] + PIECE
        if x + hi < len(t) - 64:
            write(t, x)
            taken.append((x + lo, x + hi))
            cuts.append(piece_end(t, cuts[-1]))
            assert cuts[-1] == x + shift
        else:
            cuts.append(piece_end(t, cuts[-1]))
    for j, m in enumerate(range(PIECE, len(t), PIECE)):
        for d in MARK_OFFSETS[j:] + MARK_OFFSETS[:j]:
            a, b = m + d + lo, m + d + hi
            if b < len(t) - 64 and all(b <= a2 - 2 or a >= b2 + 2 for a2, b2 in taken):
                write(t, m + d)
                taken.append((a, b))
    put(t, len(t) - len(ENDINGS[ending]), ENDINGS[ending])
    assert piece_cuts(t)[:len(cuts)] == cuts and len(piece_cuts(t)) - 1 >= 3
    return t


@gpu
@pytest.mark.parametrize("name", list(PATTERNS))
def test_edge_patterns_at_piece_cuts(ctxs, filler, name):
    ctx = ctxs[False]
    ending = list(ENDINGS)[list(PATTERNS).index(name) % len(ENDINGS)]
    t = edge_text(filler, name, ending)
    want, ntok = naive_counts(t)
    assert count_text(ctx, t) == ntok
    check_vs_words(ctx, want)


@gpu
def test_short_and_piece_sized_texts(ctxs, filler):
    ctx = ctxs[False]
    for texts in ([b"a"], [b"a", b" ", b"\xff", b"\x00"], [filler[:PIECE]], [filler[:PIECE + 1]]):
        want, ntok = naive_counts(*texts)
        assert count_text(ctx, *texts) == ntok
        check_vs_words(ctx, want)


# =================================================================================================================
# D. bytes and record classes 32 / 64 / 128
# =================================================================================================================
ODD_BYTES = [0x00, 0x01, 0x02, 0x1C, 0x1D, 0x1E, 0x1F, 0x7F] + list(range(0x80, 0x100))


def class_words(kb):
    """(words whose stored, escaped form fits the kb-byte slot with its zero byte, words that do not)"""
    fits = [b"sep%d" % i for i in range(12)]
    for b in ODD_BYTES:
        c = bytes([b])
        fits += [c, b"w" + c, c + b"v", b"x" + c * 3 + b"y"]
    fits += [b"a" * (kb - 1), b"b" * (kb - 3) + b"\x00", b"c" * (kb - 3) + b"\x01", b"\x00" * ((kb - 2) // 2) + b"d",
             b"\x01" * ((kb - 2) // 2), b"\xff" * (kb - 1), b"e\x1c" * ((kb - 1) // 2)]
    long = [b"a" * kb, b"b" * (kb - 2) + b"\x00", b"c" * (kb - 2) + b"\x01", b"\x00" * (kb // 2),
            b"e" * (kb - 1) + b"\x00", b"\x01" + b"f" * (kb - 2), b"\x80" * (kb + 5)]
    assert all(len(escape(w)) <= kb - 1 for w in fits) and all(len(escape(w)) >= kb for w in long)
    return fits, long


def class_text(words, rng):
    """every word 1..4 times in random order, between random runs of white space; every separator byte also alone"""
    toks = [w for w in words for _ in range(int(rng.integers(1, 5)))]
    toks = [toks[i] for i in rng.permutation(len(toks))]
    seps = [rng.choice(np.frombuffer(WS, dtype=np.uint8), int(rng.integers(1, 4))).tobytes() for _ in toks]
    alone = b"".join(b"sep%d" % i + bytes([WS[i % 6]]) + b"sep%d" % (i + 6) + bytes([WS[i % 6]]) for i in range(6))
    return alone + b"".join(w + s for w, s in zip(toks, seps))


@gpu
@pytest.mark.parametrize("mkb", [27, 59, 123])
def test_every_byte_and_slot_edge_in_each_record_class(mkb):
    kb = mrhbm.record_dtype(mrhbm.KEY_STR, mkb)["key"].itemsize
    fits, long = class_words(kb)
    rng = np.random.default_rng(mkb)
    dev = class_text(fits, rng)  # every word fits: the device emits the records
    mixed = class_text(fits + long, rng)  # words that do not fit: the call goes through the host
    with mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=mkb) as ctx:
        assert ctx.record_bytes == kb + 4
        want, ntok = naive_counts(dev)
        assert set(want) == set(fits)
        assert count_text(ctx, dev) == ntok
        check_vs_words(ctx, want)
        want, ntok = naive_counts(dev, mixed)
        assert set(want) == set(fits + long)
        assert count_text(ctx, dev, mixed) == ntok
        check_vs_words(ctx, want)


# =================================================================================================================
# E. host fall-back and undo inside a call of several pieces
# =================================================================================================================
def long_word(i, n=40):
    return (b"long-word-%d-" % i).ljust(n, b"x")


@gpu
def test_host_fall_back_piece_between_device_pieces(ctxs, filler):
    """pieces 2 and 4 of 4 hold words too long for the 32-byte class (first word of piece 2, one in its middle, the
    last word of piece 4): those pieces are tokenised on the host, pieces 1 and 3 on the device"""
    ctx = ctxs[False]
    t = filler[:int(3.5 * PIECE)].copy()
    put(t, PIECE - 21, b" " + long_word(0) + b" ")  # across the first mark: the first piece ends before it
    c1 = piece_end(t, 0)
    assert c1 == PIECE - 20
    put(t, c1 + PIECE // 2 - 1, b" " + long_word(1) + b" ")
    put(t, len(t) - 41, b" " + long_word(2))
    cuts = piece_cuts(t)
    assert len(cuts) == 5 and cuts[1] == c1 and cuts[2] > c1 + PIECE // 2 + 40 and cuts[3] < len(t) - 41
    want, ntok = naive_counts(t)
    assert all(want[long_word(i)] == 1 for i in range(3))
    assert count_text(ctx, t) == ntok
    check_vs_words(ctx, want)


@gpu
def test_failed_call_leaves_nothing_of_itself(ctxs, filler):
    """a 2 MB word (over the 1 MB key limit) in piece 3 of a call whose piece 2 went through the host: the call
    fails with MRHBM_E_KEY and none of its pairs, staged words or long keys survive; the job's earlier emits and an
    earlier wordcount call stay, the job commits, and later emits count"""
    ctx = ctxs[False]
    t = filler[:int(2.5 * PIECE)].copy()
    c1 = piece_end(t, 0)
    put(t, c1 + PIECE // 2 - 1, b" " + long_word(1) + b" ")
    c2 = piece_end(t, c1)
    y = c2 + (8 << 20)
    t[y:y + (2 << 20)] = ord("z")
    t[y - 1] = t[y + (2 << 20)] = SP
    cuts = piece_cuts(t)
    assert cuts[:3] == [0, c1, c2] and c1 + PIECE // 2 + 40 < c2 and y + (2 << 20) < cuts[3]
    early = b"one two two three " + b"q" * 30 + b" tail\n"  # a word over 27 bytes: this call goes through the host
    ctx.reset()
    m = ctx.map_begin("undo")
    m.emit(b"before", 3)
    m.emit(b"E" * 50, 2)
    assert m.wordcount(early) == 6
    with pytest.raises(mrhbm.MrhbmError) as e:
        m.wordcount(t)
    assert e.value.code == -4
    m.emit(b"after", 5)
    m.commit()
    ctx.shuffle()
    want, _ = naive_counts(early)
    want.update({b"before": 3, b"E" * 50: 2, b"after": 5})
    check_vs_words(ctx, want)


# =================================================================================================================
# F. two contexts at once (the bench's two-worker mode)
# =================================================================================================================
@contextlib.contextmanager
def two_contexts(*args, **kw):
    """two contexts of the same configuration and pin(w, n, dtype), pinned host arrays of worker w's context; all
    freed and closed on the way out"""
    cs, held = [mrhbm.Ctx(*args, **kw) for _ in range(2)], []

    def pin(w, n, dtype):
        a = cs[w].pinned_array(n, dtype)
        held.append((cs[w], a))
        return a
    try:
        yield cs, pin
    finally:
        for c, a in held:
            c.host_free(a.ctypes.data)
        for c in cs:
            c.close()


def two_workers(step, steps=3):
    """step(w) once for each worker w (the allocations), then `steps` times for each from its own thread, the second
    worker about half a step behind; returns the results of every step of both"""
    t0 = time.perf_counter()
    out = [[step(0)], [step(1)]]
    half = 0.4 * (time.perf_counter() - t0) / 2
    errs, start = [], threading.Barrier(2)

    def loop(w):
        try:
            start.wait()
            if w:
                time.sleep(half)
            for _ in range(steps):
                out[w].append(step(w))
        except BaseException as e:  # re-raised in the calling thread
            errs.append(e)
    th = [threading.Thread(target=loop, args=(w,)) for w in (0, 1)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    if errs:
        raise errs[0]
    assert [len(o) for o in out] == [steps + 1] * 2
    return out[0] + out[1]


@gpu
def test_two_contexts_count_words_at_once(zipf_text):
    """the bench's two-worker word count: calls of 1.5 pieces from one pinned text, ending at line ends, on two
    combiner contexts; result_copy into pinned arrays"""
    text, want = zipf_text
    cuts, p = [0], 0
    while p + PIECE * 3 // 2 < text.nbytes:
        p += PIECE * 3 // 2
        p += int(np.argmax(text[p:p + 4096] == NL)) + 1
        cuts.append(p)
    cuts.append(text.nbytes)
    with two_contexts(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, combiner=True) as (cs, pin):
        src = pin(0, text.nbytes, np.uint8)
        src[:] = text
        outs = [(pin(w, want[1].size + 4096, "S28"), pin(w, want[1].size + 4096, np.uint64)) for w in (0, 1)]

        def step(w):
            cs[w].reset()
            m = cs[w].map_begin("e2e")
            words = sum(m.wordcount(src.ctypes.data + a, b - a) for a, b in zip(cuts[:-1], cuts[1:]))
            m.commit()
            cs[w].shuffle()
            return words, result_of(cs[w], *outs[w])
        for words, got in two_workers(step):
            assert words == N_WORDS
            check_arrays(got, want)


@gpu
def test_two_contexts_shuffle_u64_records_at_once():
    """the bench's two-worker u64 run: emit_batch_ptr in 4 Mi-record chunks from one pinned record array"""
    n, chunk = 3 * (1 << 22) + 12_345, 1 << 22
    keys, vals = O.gen_u64(SEED, 555, n)
    want = O.groupby_u64(keys, vals, O.PART_MULHASH, P)
    with two_contexts(mrhbm.KEY_U64, P) as (cs, pin):
        recs = pin(0, n, mrhbm.record_dtype(mrhbm.KEY_U64))
        recs["key"], recs["val"] = keys, vals
        rb = recs.dtype.itemsize
        outs = [(pin(w, want[1].size + 4096, np.uint64), pin(w, want[1].size + 4096, np.uint64)) for w in (0, 1)]

        def step(w):
            cs[w].reset()
            m = cs[w].map_begin("e2e")
            for s in range(0, n, chunk):
                m.emit_batch_ptr(recs.ctypes.data + s * rb, min(chunk, n - s))
            m.commit()
            cs[w].shuffle()
            return result_of(cs[w], *outs[w])
        for got in two_workers(step):
            check_arrays(got, want)
