"""MRHBM_RED_FSUM: after the shuffle every key holds one value, the exact sum of its numbers rounded once.

The oracle is the exact rational sum (Fraction) rounded by float(), overflow to +-inf, with the inf and -0 rules of
include/mrhbm.h.  Results are compared as exact bit patterns through Ctx.groups, through result_copy + result_values,
and through the counts."""
import math
import random
import struct
from fractions import Fraction

import numpy as np
import pytest

import mrhbm_loader
from conftest import expand_tokens

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce import tuple as T  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WeightedWordCount import init as WWC  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WordCount import init as WordCount  # noqa: E402

gpu = pytest.mark.gpu
P = 7
INVAL = -1
WWC_PKG = "lua_mapreduce_b200.mapreduce.examples.WeightedWordCount"
TINY, BIG = 5e-324, 1.7976931348623157e308
MAXF = Fraction(2) ** 1024 - Fraction(2) ** 970  # sums this large round to inf


def fs_ctx(kind=mrhbm.KEY_STR, max_key_bytes=27, flags=0, partitioner=None, parts=P):
    kw = {} if partitioner is None else dict(partitioner=partitioner)
    return mrhbm.Ctx(kind, parts, max_key_bytes=max_key_bytes, device=0, reducer=mrhbm.RED_FSUM,
                     flags=mrhbm.F_BYTE_VALUES | flags, **kw)


def enc(x):
    """a number value as the bindings encode it (bit-exact, -0 included)"""
    return T.encode_value(x)


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def oracle(values):
    pinf, ninf = math.inf in values, -math.inf in values
    assert not (pinf and ninf)
    if pinf or ninf:
        return math.inf if pinf else -math.inf
    s = sum(Fraction(v) for v in values)
    if s == 0:
        return -0.0 if all(math.copysign(1, v) < 0 for v in values) else 0.0
    if abs(s) >= MAXF:
        return math.inf if s > 0 else -math.inf
    return float(s)


def want_sums(jobs):
    acc = {}
    for pairs in jobs:
        for k, v in pairs:
            acc.setdefault(k, []).append(v)
    return {k: bits(oracle(v)) for k, v in acc.items()}


def emit_jobs(ctx, jobs, batch=()):
    for j, pairs in enumerate(jobs):
        m = ctx.map_begin("job%d" % j)
        if j in batch:
            recs = np.zeros(len(pairs), dtype=mrhbm.record_dtype(ctx.key_kind, ctx.cfg.max_key_bytes))
            recs["key"] = [k for k, _ in pairs]
            blob = b"".join(enc(v) for _, v in pairs)
            off = np.arange(len(pairs) + 1, dtype=np.uint64) * 11
            m.emit_batch_values(recs, blob, off)
        else:
            for k, v in pairs:
                m.emit(k, enc(v))
        m.commit()


def dec(b):
    assert len(b) == 11 and b[0] == 0x10
    u = 0
    for c in b[1:]:
        assert c & 0x80
        u = (u << 7) | (c & 0x7F)
    u &= (1 << 64) - 1
    return u & ~(1 << 63) if u >> 63 else ~u & ((1 << 64) - 1)


def short_pairs(ctx, jobs):
    """the committed pairs whose keys fit a record slot: what the device's pool holds"""
    return sum(1 for pairs in jobs for k, _ in pairs
               if ctx.key_kind == mrhbm.KEY_U64 or len(k) <= ctx.record_bytes - 4)


def check(ctx, want, long_keys=0, shuffle=True, pairs=None):
    """groups, rows and counts against want = {key: double bits} (and pairs = committed pairs, when given); returns
    the rows"""
    if shuffle:
        ctx.shuffle()
    info = ctx.result_info()
    committed = ctx.checksum_input()[3]
    assert info.pairs_in == committed and info.pairs_recv == committed  # every pair is carried, none is dropped
    if pairs is not None:
        assert committed == pairs
    u64 = ctx.key_kind == mrhbm.KEY_U64
    got = {}
    for p in ctx.partitions():
        keys = []
        for k, vals in ctx.groups(p):
            k = int.from_bytes(k, "big") if u64 else k
            assert k not in got and len(vals) == 1
            keys.append(k)
            got[k] = dec(vals[0])
        assert keys == sorted(keys)
    assert got == want
    info = ctx.result_info()
    short = {k: v for k, v in want.items() if u64 or len(k) <= ctx.record_bytes - 4}
    assert info.groups == len(short) and len(short) == len(want) - long_keys
    if long_keys:
        return None
    keys, _, po = ctx.result_copy()
    blob, roff = ctx.result_values()
    raw = blob.tobytes()
    assert [int(x) for x in roff] == [11 * r for r in range(len(short) + 1)]
    rows = [(int(keys[r]) if u64 else bytes(keys[r]), dec(raw[11 * r:11 * r + 11])) for r in range(len(short))]
    assert dict(rows) == short and len(rows) == len(short)
    if info.sorted:
        for p in range(ctx.num_partitions):
            part = [k for k, _ in rows[int(po[p]):int(po[p + 1])]]
            assert part == sorted(part)
    return rows


ARITH = {
    b"cancel": [1e308, -1e308, 5e-324],
    b"sub": [TINY, TINY * 3, -TINY, 2.2250738585072014e-308, -2.225073858507201e-308],
    b"tie-even": [1.0, 2.0 ** -53],                       # halfway, 1.0 is even: stays
    b"tie-odd": [1.0 + 2.0 ** -52, 2.0 ** -53],           # halfway, odd: rounds up
    b"tie-sticky": [1.0, 2.0 ** -53, 2.0 ** -110],        # just past halfway: up
    b"below-max": [BIG, 2.0 ** 969, -TINY],               # just under the threshold: DBL_MAX
    b"at-max": [BIG, 2.0 ** 970, -2.0 ** 900],            # under the tie: DBL_MAX
    b"over": [BIG, 2.0 ** 970],                           # the tie at DBL_MAX + half an ulp: inf
    b"over-neg": [-BIG, -BIG, BIG / 2],
    b"pinf": [math.inf, 1.0, -BIG, math.inf],
    b"ninf": [-math.inf, 3.5],
    b"neg0": [-0.0, -0.0, -0.0],
    b"mixed0": [-0.0, 0.0, -0.0],
    b"exact0": [1.5, -1.5],
    b"one": [0.1],
    b"one-neg0": [-0.0],
    b"tenth": [0.1] * 10,
    b"weights": [1 / 3, 1 / 7, 1 / 7, 1 / 3, 1 / 11, 2 / 3, 0.25, 1e-17],
    b"int": [3, 4, 2 ** 52, -7],
}


@gpu
@pytest.mark.parametrize("flags", [0, mrhbm.F_NO_OPTIMISTIC, mrhbm.F_SMALL_BINS | mrhbm.F_NO_OPTIMISTIC],
                         ids=["fast", "exact", "small"])
def test_arithmetic_cases(flags):
    rng = random.Random(1)
    jobs = [[], []]
    for k, vals in ARITH.items():
        for v in vals:
            jobs[rng.randrange(2)].append((k, v))
    for j in jobs:
        rng.shuffle(j)
    with fs_ctx(flags=flags) as ctx:
        emit_jobs(ctx, jobs, batch=(1,))
        check(ctx, want_sums(jobs), pairs=short_pairs(ctx, jobs))


@gpu
def test_integers_equal_the_builtin_sum():
    rng = random.Random(2)
    pairs = [(b"w%d" % rng.randrange(3000), rng.randrange(1, 1000)) for _ in range(60000)]
    with fs_ctx() as ctx:
        emit_jobs(ctx, [pairs], batch=(0,))
        ctx.shuffle()
        fs = {k: dec(v[0]) for p in ctx.partitions() for k, v in ctx.groups(p)}
    with mrhbm.Ctx(mrhbm.KEY_STR, P, max_key_bytes=27, device=0) as ctx:
        m = ctx.map_begin("j")
        for k, v in pairs:
            m.emit(k, v)
        m.commit()
        ctx.shuffle()
        ref = {k: v[0] for p in ctx.partitions() for k, v in ctx.groups(p)}
    assert fs == {k: bits(float(v)) for k, v in ref.items()}


def random_jobs(keys, n, seed, jobs=3, skew=True):
    """Zipf-like keys (skew) or uniform ones, with weights, wide-range doubles and cancellation"""
    rng = random.Random(seed)
    out = []
    for _ in range(jobs):
        pairs = []
        for _ in range(n):
            k = keys[min(int(rng.paretovariate(1.1)) - 1, len(keys) - 1)] if skew else rng.choice(keys)
            r = rng.random()
            v = (1 / rng.randrange(1, 50) if r < 0.5 else rng.uniform(-1e6, 1e6) if r < 0.8
                 else rng.choice((-1, 1)) * rng.random() * 2.0 ** rng.randrange(-1000, 1000))
            pairs.append((k, v))
        out.append(pairs)
    return out


KINDS = [("u64", mrhbm.KEY_U64, 27), ("str27", mrhbm.KEY_STR, 27), ("str59", mrhbm.KEY_STR, 59),
         ("str123", mrhbm.KEY_STR, 123)]


@gpu
@pytest.mark.parametrize("name,kind,mkb", KINDS, ids=[k[0] for k in KINDS])
def test_key_classes(name, kind, mkb):
    keys = list(range(7, 7 + 500 * 2 ** 50, 2 ** 50)) if kind == mrhbm.KEY_U64 else \
        [b"k%d" % i for i in range(498)] + [b"w" * mkb, b"x" * (mkb - 1)]
    jobs = random_jobs(keys, 4000, 3)
    with fs_ctx(kind, mkb) as ctx:
        emit_jobs(ctx, jobs, batch=(0,))
        check(ctx, want_sums(jobs), pairs=short_pairs(ctx, jobs))


@gpu
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_layout_flags_are_bit_identical(kind):
    keys = list(range(1, 20001)) if kind == mrhbm.KEY_U64 else [b"key%05d" % i for i in range(20000)]
    jobs = random_jobs(keys, 50000, 4)
    want = want_sums(jobs)
    rows = []
    for flags in (0, mrhbm.F_SMALL_BINS, mrhbm.F_NO_OPTIMISTIC, mrhbm.F_FORCE_RUNS,
                  mrhbm.F_SMALL_BINS | mrhbm.F_NO_OPTIMISTIC | mrhbm.F_FORCE_RUNS):
        with fs_ctx(kind, flags=flags) as ctx:
            emit_jobs(ctx, jobs, batch=(1, 2))
            rows.append(sorted(check(ctx, want, pairs=short_pairs(ctx, jobs))))
    assert all(r == rows[0] for r in rows)


@gpu
@pytest.mark.parametrize("flags", [0, mrhbm.F_SMALL_BINS], ids=["cap", "small-bins"])
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_oversized_bins_and_chunk_crossing_groups(kind, flags):
    """hot keys of thousands of values next to many small keys in the same bins: groups cross cap-row chunks"""
    rng = random.Random(6)
    key = (lambda i: 1000 + i) if kind == mrhbm.KEY_U64 else (lambda i: b"o%d" % i)
    hot = [key(i) for i in range(0, 40, 7)]
    pairs = [(rng.choice(hot), rng.uniform(-5, 5) * 2.0 ** rng.randrange(-60, 60)) for _ in range(30000)]
    pairs += [(key(rng.randrange(40, 3000)), 1 / rng.randrange(1, 9)) for _ in range(20000)]
    pairs += [(hot[0], math.inf), (hot[1], -0.0)]
    rng.shuffle(pairs)
    jobs = [pairs[:25000], pairs[25000:]]
    with fs_ctx(kind, flags=flags | mrhbm.F_NO_OPTIMISTIC, parts=1 if flags else 2) as ctx:
        emit_jobs(ctx, jobs, batch=(0, 1))
        check(ctx, want_sums(jobs), pairs=short_pairs(ctx, jobs))
        assert ctx.stats()["big_bins"] >= 1


@gpu
def test_a_key_with_a_million_values():
    n = 1_000_000
    rng = np.random.default_rng(4)
    vals = (rng.standard_normal(n) * 2.0 ** rng.integers(-40, 40, n)).tolist()
    with fs_ctx() as ctx:
        m = ctx.map_begin(0)
        recs = np.zeros(n + 1, dtype=mrhbm.record_dtype(ctx.key_kind, 27))
        recs["key"] = [b"big"] * n + [b"small"]
        off = np.arange(n + 2, dtype=np.uint64) * 11
        m.emit_batch_values(recs, b"".join(enc(v) for v in vals) + enc(2.5), off)
        m.commit()
        check(ctx, {b"big": bits(oracle(vals)), b"small": bits(2.5)}, pairs=n + 1)


@gpu
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_range_partitioner_one_global_order(kind):
    keys = list(range(0, 2 ** 63, 2 ** 57)) if kind == mrhbm.KEY_U64 else [b"r%03d" % i for i in range(64)]
    jobs = random_jobs(keys, 500, 5, skew=False)  # (few pairs: one sub-bin per partition, one run)
    with fs_ctx(kind, partitioner=mrhbm.PART_RANGE, parts=5) as ctx:
        emit_jobs(ctx, jobs)
        ctx.sample_splitters()
        ctx.shuffle()
        assert ctx.result_info().sorted == 1
        rows = check(ctx, want_sums(jobs), pairs=short_pairs(ctx, jobs), shuffle=False)
        assert [k for k, _ in rows] == sorted(k for k, _ in rows)


@gpu
def test_ledger_rules_and_repeated_shuffles():
    rng = random.Random(11)

    def pairs(n):
        return [(b"k%d" % rng.randrange(30), rng.uniform(-10, 10)) for _ in range(n)]
    with fs_ctx() as ctx:
        a, b = pairs(800), pairs(800)
        emit_jobs(ctx, [a, b])
        check(ctx, want_sums([a, b]), pairs=short_pairs(ctx, [a, b]))
        check(ctx, want_sums([a, b]), pairs=short_pairs(ctx, [a, b]))  # a second shuffle of the same commits
        m = ctx.map_begin("job0")  # replace job0
        a2 = pairs(500)
        for k, v in a2:
            m.emit(k, enc(v))
        m.commit()
        check(ctx, want_sums([a2, b]), pairs=short_pairs(ctx, [a2, b]))
        m = ctx.map_begin("aborted")
        for k, v in pairs(100):
            m.emit(k, enc(v))
        m.abort()
        check(ctx, want_sums([a2, b]), pairs=short_pairs(ctx, [a2, b]))
        ctx.reset()
        c = pairs(300)
        emit_jobs(ctx, [c])
        check(ctx, want_sums([c]), pairs=short_pairs(ctx, [c]))


@gpu
def test_long_keys_are_summed_on_the_host():
    long = [b"long-key-%02d-" % i + b"z" * 30 for i in range(3)]
    jobs = [[(long[0], 1e308), (long[0], -1e308), (long[0], TINY), (long[1], -0.0), (b"short", 0.5), (long[2], 1.0)],
            [(long[1], -0.0), (long[2], 2.0 ** -53), (b"short", 0.25)]]
    with fs_ctx() as ctx:
        emit_jobs(ctx, jobs)
        check(ctx, want_sums(jobs), pairs=short_pairs(ctx, jobs), long_keys=3)


@gpu
def test_failures_leave_no_result():
    for bad in ([(b"a", 1.0), (b"b", None)], [(b"a", math.inf), (b"a", -math.inf), (b"b", 1.0)]):
        for long in (False, True):
            with fs_ctx() as ctx:
                m = ctx.map_begin(0)
                for k, v in bad:
                    k = k * 40 if long else k
                    m.emit(k, T.encode_value(b"str") if v is None else enc(v))
                m.emit(b"fill", enc(1.0))
                m.commit()
                with pytest.raises(mrhbm.MrhbmError) as e:
                    ctx.shuffle()
                assert e.value.code == INVAL
                with pytest.raises(mrhbm.MrhbmError):
                    ctx.result_info()


@gpu
@pytest.mark.parametrize("where", ["warp", "crossing"])
def test_both_infinities_on_one_key_fail_on_every_path(where):
    """+inf and -inf among a key's values: in a group of more than two values (a warp's accumulator), and in a group
    that crosses a chunk of an oversized bin (the merge of the partial accumulators)"""
    rng = random.Random(8)
    if where == "warp":
        pairs, flags = [(b"k", 1.0)] * 5 + [(b"k", math.inf), (b"k", -math.inf)], 0
    else:
        pairs = [(b"hot", rng.uniform(-1, 1)) for _ in range(3000)] + [(b"k%d" % i, 1.0) for i in range(200)]
        pairs[10] = (b"hot", math.inf)
        pairs[2900] = (b"hot", -math.inf)
        flags = mrhbm.F_SMALL_BINS | mrhbm.F_NO_OPTIMISTIC
    with fs_ctx(flags=flags, parts=1) as ctx:
        emit_jobs(ctx, [pairs])
        with pytest.raises(mrhbm.MrhbmError) as e:
            ctx.shuffle()
        assert e.value.code == INVAL and "NaN" in str(e.value)
        with pytest.raises(mrhbm.MrhbmError):
            ctx.result_info()
        m = ctx.map_begin("job0")  # the job replaced without the infinities: the next shuffle succeeds
        for k, v in pairs:
            if math.isfinite(v):
                m.emit(k, enc(v))
        m.commit()
        kept = [(k, v) for k, v in pairs if math.isfinite(v)]
        check(ctx, want_sums([kept]), pairs=len(kept))
        if where == "crossing":
            assert ctx.stats()["big_bins"] >= 1


@gpu
def test_refusals_at_init():
    for kw in (dict(flags=0), dict(flags=mrhbm.F_BYTE_VALUES, combiner=mrhbm.COMBINE_REDUCER),
               dict(flags=mrhbm.F_BYTE_VALUES, combiner=mrhbm.COMBINE_DISTINCT)):
        with pytest.raises(mrhbm.MrhbmError) as e:
            mrhbm.Ctx(mrhbm.KEY_STR, P, device=0, reducer=mrhbm.RED_FSUM, **kw)
        assert e.value.code == INVAL


@gpu
def test_weighted_word_count_loop(tmp_path, golden_wordcount):
    """the declared device arm against the oracle, and the host reducefn where its left-to-right sum is exact: lines of
    1, 2, 4 or 8 words give weights that are powers of two"""
    files, acc = [], {}
    for job in range(4):
        toks = expand_tokens(golden_wordcount, job)
        lines, i, n = [], 0, 0
        while i < len(toks):
            w = max(x for x in (1, 2, 4, 8) if x <= min((1, 2, 4, 8)[n % 4], len(toks) - i))
            lines.append(toks[i:i + w])
            i, n = i + w, n + 1
        for ln in lines:
            for t in ln:
                acc.setdefault(t, []).append(1 / len(ln))
        p = tmp_path / ("file%d.txt" % job)
        p.write_bytes(b"\n".join(b" ".join(ln) for ln in lines) + b"\n")
        files.append(str(p))
    WordCount.FILES[:] = files
    want = {k: oracle(v) for k, v in acc.items()}
    S = WWC_PKG + ".init"
    results = []
    for arm, reducefn in enumerate((WWC_PKG + ".reducefn_device", S)):
        WWC.RESULT.clear()
        s = server.new("hbm://local", "fsum-loop-%d" % arm)
        s.configure(dict(taskfn=S, mapfn=S, partitionfn=S, reducefn=reducefn, finalfn=S, storage="hbm",
                         hbm={"value_kind": "bytes"}))
        s.loop()
        results.append({k: bits(float(v)) for k, v in WWC.RESULT.items()})
    assert results[0] == {k: bits(v) for k, v in want.items()}
    assert results[1] == results[0]
