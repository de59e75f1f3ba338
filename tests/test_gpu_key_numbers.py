"""mrhbm_map_key_numbers: lines "key number" parsed on the device into (key, 11-byte number) pairs.

The oracle is Python: the text split into lines at '\\n', each line into fields at the six C-locale white-space bytes,
a strict regex for the number, float() and tuple.encode_value.  Records are compared through pool_read (keys in text
order, each pair's value id its own pool index) and values through a RED_NONE shuffle, pair for pair where every key is
unique.  The sums go through MRHBM_RED_FSUM with and without MRHBM_COMBINE_FSUM against float(sum(Fraction))."""
import math
import random
import re
import struct
from collections import Counter, defaultdict
from fractions import Fraction

import numpy as np
import pytest

import mrhbm_loader

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.KeyNumberSum import init as KNS  # noqa: E402
from lua_mapreduce_b200.mapreduce.tuple import encode_value  # noqa: E402

gpu = pytest.mark.gpu
P = 7
INVAL = -1
PIECE = 1 << 26
FIX_CAP = 1 << 16  # tokens per device piece that the host may round before the piece goes to the host
NUMBER = re.compile(rb"[+-]?([0-9]+(\.[0-9]*)?|\.[0-9]+)([eE][+-]?[0-9]+)?\Z")
FIELD = re.compile(rb"[^ \t\n\v\f\r]+")
MAXF = Fraction(2) ** 1024 - Fraction(2) ** 970


def byte_ctx(max_key_bytes=27, reducer=mrhbm.RED_NONE, combiner=False, kind=mrhbm.KEY_STR):
    return mrhbm.Ctx(kind, P, max_key_bytes=max_key_bytes, device=0, reducer=reducer, combiner=combiner,
                     flags=mrhbm.F_BYTE_VALUES)


def oracle(text):
    """[(key, number)] of the text's lines, in text order"""
    out = []
    for line in bytes(text).split(b"\n"):
        f = FIELD.findall(line)
        if not f:
            continue
        assert len(f) == 2 and NUMBER.match(f[1]), line
        out.append((f[0], float(f[1])))
    return out


def escape(k):
    return k.replace(b"\x01", b"\x01\x02").replace(b"\x00", b"\x01\x01")


def number_token(rng):
    """one decimal token of every class the parser has a path for"""
    c = rng.randrange(14)
    x = rng.uniform(-1e6, 1e6)
    if c == 0:
        return b"%.2f" % x
    if c == 1:
        return b"%d" % int(x)
    if c == 2:
        return repr(x * 10 ** rng.randint(-30, 30)).encode()
    if c == 3:  # random bits: subnormals to near DBL_MAX
        v = math.inf
        while not math.isfinite(v):
            v = struct.unpack("<d", struct.pack("<Q", rng.getrandbits(63)))[0]
        return repr(-v if rng.random() < 0.5 else v).encode()
    if c == 4:  # more than 19 significant digits: rounded on the host
        return (b"%d" % rng.randrange(10 ** 19, 10 ** 30)) + b"e%d" % rng.randint(-340, 280)
    if c == 5:
        return rng.choice([b"-0", b"+0", b"0.0", b"-0.000e5", b"+.5", b"5.", b"-.25", b"1e-400", b"-1e400", b"1e309",
                           b"0e999999999", b"4.9e-324", b"2.4703282292062328e-324", b"1.7976931348623158e308",
                           b"1.7976931348623159e308", b"9007199254740993", b"2.2250738585072011e-308"])
    if c == 6:
        return b"%de%d" % (rng.randrange(1, 10 ** rng.randint(1, 19)), rng.randint(-360, 320))
    if c == 7:
        return b"%.17e" % x
    return b"%.*f" % (rng.randint(0, 6), x)


def key_bytes(rng, i):
    k = b"k%d" % i
    if rng.random() < 0.1:
        k += bytes([rng.choice([0, 1])]) + b"x"  # escaped in the slot
    return k


def messy_text(pairs, rng, final_newline=True):
    """pairs as lines with tabs, CRLF, blank and white-space-only lines, leading and trailing blanks"""
    ws = [b" ", b"\t", b"  \t", b"\v", b"\f"]
    lines = []
    for k, n in pairs:
        if rng.random() < 0.1:
            lines.append(rng.choice([b"", b"   ", b"\t\r", b"\r"]))
        lines.append(rng.choice([b"", b" ", b"\t"]) + k + rng.choice(ws) + n + rng.choice([b"", b" ", b"\r", b"\t "]))
    t = b"\n".join(lines)
    return t + b"\n" if final_newline else t


def check_pool(ctx, first, want):
    """pool_read from first: keys in text order, each value id its own pool index"""
    recs = ctx.pool_read(first, len(want))
    assert [bytes(k) for k in recs["key"]] == [escape(k) for k, _ in want]
    assert (recs["val"] == np.arange(first, first + len(want), dtype=np.uint32)).all()


def groups(ctx):
    ctx.shuffle()
    return {k: v for p in ctx.partitions() for k, v in ctx.groups(p)}


@gpu
@pytest.mark.parametrize("mkb", [27, 59, 123])
def test_record_classes_pair_for_pair(mkb):
    rng = random.Random(mkb)
    pairs = [(key_bytes(rng, i), number_token(rng)) for i in range(20000)]  # unique keys: one value per group
    for final_newline in (True, False):
        text = messy_text(pairs, rng, final_newline)
        want = oracle(text)
        assert len(want) == len(pairs)
        with byte_ctx(mkb) as ctx:
            m = ctx.map_begin("j")
            assert m.key_numbers(text) == len(want)
            m.commit()
            check_pool(ctx, 0, want)
            got = groups(ctx)
            assert got == {k: [encode_value(v)] for k, v in want}


@gpu
def test_many_values_per_key_and_several_calls():
    rng = random.Random(5)
    keys = [b"url/%d" % i for i in range(300)]
    texts = [messy_text([(rng.choice(keys), number_token(rng)) for _ in range(5000)], rng) for _ in range(3)]
    with byte_ctx() as ctx:
        m = ctx.map_begin("j")
        n = 0
        for t in texts:
            assert m.key_numbers(t) == len(oracle(t))
            n += len(oracle(t))
        m.key_numbers(b"")
        m.key_numbers(b"\n \t\r\n")
        m.commit()
        want = [p for t in texts for p in oracle(t)]
        check_pool(ctx, 0, want)
        exp = defaultdict(list)
        for k, v in want:
            exp[k].append(encode_value(v))
        assert {k: sorted(v) for k, v in groups(ctx).items()} == {k: sorted(v) for k, v in exp.items()}


@gpu
def test_fix_up_list_on_the_device_and_its_overflow_to_the_host():
    """a piece with a few 20-digit numbers (rounded on the host, patched on the device) and a piece with more of them
    than the list holds (the whole piece parsed on the host): the same pairs as the oracle either way"""
    rng = random.Random(6)
    few = [(b"f%d" % i, b"%d.%d" % (rng.randrange(10 ** 10, 10 ** 11), rng.randrange(10 ** 14, 10 ** 15)))
           for i in range(3000)]
    many = [(b"m%d" % i, b"%de-%d" % (rng.randrange(10 ** 19, 10 ** 20), rng.randint(0, 330)))
            for i in range(FIX_CAP + 100)]
    for pairs in (few, many):
        text = messy_text(pairs, rng)
        want = oracle(text)
        with byte_ctx() as ctx:
            m = ctx.map_begin("j")
            assert m.key_numbers(text) == len(want)
            m.commit()
            check_pool(ctx, 0, want)
            assert groups(ctx) == {k: [encode_value(v)] for k, v in want}


@pytest.fixture(scope="module")
def big_text():
    """> 2 pieces of lines with 1000 keys; the second piece holds one key longer than the record class"""
    rng = np.random.default_rng(7)
    n = 6_000_000
    keys = rng.integers(0, 1000, n)
    cents = rng.integers(0, 10 ** 9, n)
    lines = [b"customer-%06d %d.%02d" % (k, c // 100, c % 100) for k, c in zip(keys.tolist(), cents.tolist())]
    long_key = b"L" * 60
    lines[len(lines) // 2] = long_key + b" 12.5"
    text = b"\n".join(lines)  # no final newline
    assert len(text) > 2 * PIECE
    return text, long_key


@gpu
def test_pieces_with_lines_across_the_cut_and_a_host_piece(big_text):
    text, long_key = big_text
    want = oracle(text)
    with byte_ctx() as ctx:
        m = ctx.map_begin("j")
        assert m.key_numbers(text) == len(want)
        m.commit()
        short = [p for p in want if p[0] != long_key]
        recs = ctx.pool_read(0, len(short))
        assert (recs["key"] == np.array([k for k, _ in short], dtype="S28")).all()
        assert (recs["val"] == np.arange(len(short), dtype=np.uint32)).all()
        exp = defaultdict(Counter)
        for k, v in want:
            exp[k][encode_value(v)] += 1
        got = groups(ctx)
        assert got.keys() == exp.keys()
        for k, vs in got.items():
            assert Counter(vs) == exp[k], k


def bad(ctx, m, text, at):
    with pytest.raises(mrhbm.MrhbmError) as e:
        m.key_numbers(text)
    assert e.value.code == INVAL and ("byte %d " % at) in str(e.value), str(e.value)


@gpu
def test_refusals_leave_pool_arena_and_long_keys_as_they_were():
    good = b"a 1\nb 2.5\n" + b"L" * 40 + b" 3\n"
    with byte_ctx() as ctx:
        m = ctx.map_begin("j")
        m.key_numbers(good)
        for t, at in [(b"a 1\nb\n", 4), (b"a 1\nb 2 3\n", 4), (b"x 0x10", 0), (b"x inf", 0), (b"x nan", 0),
                      (b"x 1e", 0), (b"x 1_0", 0), (b"a 1\n\n  x 1e5.5\n", 5), (b"a 1\n 1\n", 4), (b"x ,5", 0),
                      (b"L" * 40 + b" 1\n" + b"y 1 2", 43), (b"a 1\nq 12345678901234567890123 4\n", 4)]:
            bad(ctx, m, t, at)
        # a failure in the third piece, after a device piece and a host piece
        rng = random.Random(8)
        body = b"".join(b"k%d %d\n" % (rng.randrange(100), rng.randrange(10 ** 6)) for _ in range(7_000_000))
        assert len(body) > PIECE
        cut = body.rindex(b"\n", 0, PIECE - 100) + 1
        mid = body[:cut] + b"L" * 40 + b" 7\n" + body[cut:]
        text = mid + body + b"z 1 2\n"
        bad(ctx, m, text, len(mid) + len(body))
        # a line longer than a piece
        bad(ctx, m, b"a 1\n" + b"x" * (PIECE + 10) + b" 1\nb 2\n", 4)
        m.commit()
        want = oracle(good)
        check_pool(ctx, 0, want[:2])
        assert groups(ctx) == {k: [encode_value(v)] for k, v in want}
    with mrhbm.Ctx(mrhbm.KEY_STR, P, device=0) as ctx:  # no byte values
        with pytest.raises(mrhbm.MrhbmError) as e:
            ctx.map_begin("j").key_numbers(b"a 1\n")
        assert e.value.code == INVAL
    with byte_ctx(kind=mrhbm.KEY_U64) as ctx:
        with pytest.raises(mrhbm.MrhbmError) as e:
            ctx.map_begin("j").key_numbers(b"1 1\n")
        assert e.value.code == INVAL


@gpu
def test_abort_replace_and_reset():
    with byte_ctx() as ctx:
        m = ctx.map_begin("a")
        m.key_numbers(b"x 1\ny 2\n")
        m.abort()
        m = ctx.map_begin("b")
        m.key_numbers(b"x 3\n")
        m.commit()
        m = ctx.map_begin("b")  # replaces the first commit of b
        m.key_numbers(b"x 4\nz 5\n")
        m.commit()
        assert groups(ctx) == {b"x": [encode_value(4.0)], b"z": [encode_value(5.0)]}
        ctx.reset()
        m = ctx.map_begin("c")
        m.key_numbers(b"y -0\n")
        m.commit()
        check_pool(ctx, 0, [(b"y", -0.0)])
        assert groups(ctx) == {b"y": [encode_value(-0.0)]}


def fsum_oracle(values):
    pinf, ninf = math.inf in values, -math.inf in values
    if pinf or ninf:
        return math.inf if pinf else -math.inf
    s = sum(Fraction(v) for v in values)
    if s == 0:
        return -0.0 if all(math.copysign(1, v) < 0 for v in values) else 0.0
    if abs(s) >= MAXF:
        return math.inf if s > 0 else -math.inf
    return float(s)


@gpu
@pytest.mark.parametrize("combiner", [False, mrhbm.COMBINE_FSUM])
def test_number_sum_end_to_end(combiner):
    rng = random.Random(9)
    keys = [b"p%d" % i for i in range(500)]
    texts = []
    for j in range(4):
        pairs = []
        for _ in range(20000):
            tok = number_token(rng)
            if math.isinf(float(tok)):
                tok = b"1e300"
            pairs.append((rng.choice(keys), tok))
        texts.append(messy_text(pairs, rng))
    with byte_ctx(reducer=mrhbm.RED_FSUM, combiner=combiner) as ctx:
        for j, t in enumerate(texts):
            m = ctx.map_begin("j%d" % j)
            m.key_numbers(t)
            m.commit()
        got = groups(ctx)
    vals = defaultdict(list)
    for t in texts:
        for k, v in oracle(t):
            vals[k].append(v)
    assert got == {k: [encode_value(fsum_oracle(v))] for k, v in vals.items()}


def run_kns(tmp_path, mapfn, name, combiner):
    S = "lua_mapreduce_b200.mapreduce.examples.KeyNumberSum"
    KNS.RESULT.clear()
    s = server.new("hbm://local", name)
    s.configure(dict(taskfn=S + ".init", mapfn=S + mapfn, partitionfn=S + ".init", reducefn=S + ".reducefn_device",
                     finalfn=S + ".init", combinerfn=S + ".combinerfn" if combiner else None, storage="hbm",
                     hbm={"value_kind": "bytes"}))
    s.loop()
    return dict(KNS.RESULT)


@gpu
@pytest.mark.parametrize("combiner", [False, True])
def test_key_number_sum_device_mapfn_matches_the_host_mapfn(tmp_path, combiner):
    rng = random.Random(10)
    files = []
    for j in range(3):
        p = tmp_path / ("sales%d.txt" % j)
        p.write_bytes(messy_text([(b"product%d" % rng.randrange(200), b"%.2f" % rng.uniform(0, 500))
                                  for _ in range(20000)], rng))
        files.append(str(p))
    KNS.FILES[:] = files
    host = run_kns(tmp_path, ".init", "kns-host-%d" % combiner, combiner)
    dev = run_kns(tmp_path, ".mapfn_device", "kns-dev-%d" % combiner, combiner)
    vals = defaultdict(list)
    for f in files:
        for k, v in oracle(open(f, "rb").read()):
            vals[k].append(v)
    assert host == dev == {k: fsum_oracle(v) for k, v in vals.items()}
