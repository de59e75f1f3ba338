"""MRHBM_COMBINE_FSUM: at each commit a key's numbers become the greedy expansion of their exact sum, and every result
of the shuffle is bit-identical to the same commits on a MRHBM_RED_FSUM ctx without the combiner.

The main oracle is that second ctx, compared bit for bit through Ctx.groups, result_copy + result_values and the group
count; the Fraction oracle of the reducer and the split rule of tests/test_fsum_combiner_host.py check the sums and the
committed pairs (pool_read) themselves."""
import math
import random

import numpy as np
import pytest

import mrhbm_loader
from conftest import expand_tokens
from test_fsum_combiner_host import expected
from test_gpu_fsum_reducer import (ARITH, BIG, INVAL, KINDS, P, TINY, WWC_PKG, bits, dec, enc, oracle, random_jobs,
                                   want_sums)

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm  # noqa: E402
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WeightedWordCount import init as WWC  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WordCount import init as WordCount  # noqa: E402

gpu = pytest.mark.gpu


def ctx_pair(kind=mrhbm.KEY_STR, max_key_bytes=27, flags=0, partitioner=None, parts=P):
    kw = {} if partitioner is None else dict(partitioner=partitioner)
    return [mrhbm.Ctx(kind, parts, max_key_bytes=max_key_bytes, device=0, reducer=mrhbm.RED_FSUM,
                      flags=mrhbm.F_BYTE_VALUES | flags, combiner=comb, **kw)
            for comb in (mrhbm.COMBINE_FSUM, mrhbm.COMBINE_NONE)]


def slot_fits(ctx, k):
    return ctx.key_kind == mrhbm.KEY_U64 or len(k) <= ctx.record_bytes - 4


def commit_job(ctx, job_id, pairs, batch=False):
    m = ctx.map_begin(job_id)
    if batch:
        short = [(k, v) for k, v in pairs if slot_fits(ctx, k)]
        recs = np.zeros(len(short), dtype=mrhbm.record_dtype(ctx.key_kind, ctx.cfg.max_key_bytes))
        recs["key"] = [k for k, _ in short]
        m.emit_batch_values(recs, b"".join(enc(v) for _, v in short), np.arange(len(short) + 1, dtype=np.uint64) * 11)
        for k, v in pairs:
            if not slot_fits(ctx, k):
                m.emit(k, enc(v))
    else:
        for k, v in pairs:
            m.emit(k, enc(v))
    m.commit()


def expected_layout(ctx, pairs):
    """the survivors of one job as the combiner lays them out: (key, number of values), keys by first pair"""
    vals = {}
    for k, v in pairs:
        if slot_fits(ctx, k):
            vals.setdefault(k, []).append(v)
    out = []
    for k, vs in vals.items():
        e = expected(vs)
        assert e is not None
        out.append((k, len(vs) if e == "keep" else len(e)))
    return out


def results(ctx):
    """everything a shuffle hands out: groups (key -> its values' bits, by partition), the rows as (key slot, value
    bytes), the group count.  (The rows' order follows info.sorted, which the shuffle picks from the pairs it carries,
    so it is not compared.)"""
    ctx.shuffle()
    u64 = ctx.key_kind == mrhbm.KEY_U64
    groups = {}
    for p in ctx.partitions():
        for k, vals in ctx.groups(p):
            groups[int.from_bytes(k, "big") if u64 else k] = (p, [dec(v) for v in vals])
    info = ctx.result_info()
    keys, _, _ = ctx.result_copy()
    blob, roff = ctx.result_values()
    raw, keys = blob.tobytes(), keys.tolist()
    rows = sorted((keys[r], raw[int(roff[r]):int(roff[r + 1])]) for r in range(len(keys)))
    return groups, rows, info.groups


def run_both(jobs, kind=mrhbm.KEY_STR, mkb=27, flags=0, partitioner=None, parts=P, batch=(), check_pool=True,
             splitters=False):
    """the jobs on both ctxs: bit-identical results, the sums against the Fraction oracle, and after each commit the
    combined ctx's new pairs (pool_read) against the split rule"""
    comb, plain = ctx_pair(kind, mkb, flags, partitioner, parts)
    with comb, plain:
        before = 0
        for j, pairs in enumerate(jobs):
            for ctx in (comb, plain):
                commit_job(ctx, "job%d" % j, pairs, batch=j in batch)
            if check_pool:
                lay = expected_layout(comb, pairs)
                n = sum(c for _, c in lay)
                assert comb.checksum_input()[3] == before + n
                recs = comb.pool_read(before, n)
                keys = [int(x) for x in recs["key"]] if kind == mrhbm.KEY_U64 else [bytes(x) for x in recs["key"]]
                assert keys == [k for k, c in lay for _ in range(c)]
                ids = [int(x) for x in recs["val"]]
                assert ids == list(range(ids[0], ids[0] + n))  # fresh ids: each new pair's own pool index
                before += n
        if splitters:  # (sampled from the uncombined pairs: a sample of the survivors would split elsewhere)
            comb.set_splitters(plain.sample_splitters())
        got, want = results(comb), results(plain)
        assert got[0] == want[0] and got[2] == want[2]
        diff = [(x, y) for x, y in zip(got[1], want[1]) if x != y][:3]
        assert got[1] == want[1], (flags, len(got[1]), len(want[1]), diff)
        assert {k: v[1][0] for k, v in got[0].items()} == want_sums(jobs)
        assert comb.result_info().pairs_in == comb.checksum_input()[3] == comb.result_info().pairs_recv
        return comb.result_info().pairs_in, plain.result_info().pairs_in


@gpu
@pytest.mark.parametrize("flags", [0, mrhbm.F_NO_OPTIMISTIC, mrhbm.F_SMALL_BINS | mrhbm.F_NO_OPTIMISTIC],
                         ids=["fast", "exact", "small"])
def test_arithmetic_cases_over_jobs(flags):
    rng = random.Random(1)
    jobs = [[], [], []]
    for k, vals in ARITH.items():
        for v in vals:
            jobs[rng.randrange(3)].append((k, v))
    # a partial sum that overflows in one job and comes back in range with another
    jobs[0] += [(b"back", 1e308), (b"back", 1e308)]
    jobs[1] += [(b"back", -1e308)]
    jobs[2] += [(b"pair", 1.0), (b"pair", 2.0 ** -80), (b"zero", -0.0), (b"zero", -0.0), (b"inf", math.inf)]
    for j in jobs:
        rng.shuffle(j)
    run_both(jobs, flags=flags, batch=(1,))


@gpu
@pytest.mark.parametrize("name,kind,mkb", KINDS, ids=[k[0] for k in KINDS])
def test_key_classes(name, kind, mkb):
    keys = list(range(7, 7 + 500 * 2 ** 50, 2 ** 50)) if kind == mrhbm.KEY_U64 else \
        [b"k%d" % i for i in range(498)] + [b"w" * mkb, b"x" * (mkb - 1)]
    jobs = random_jobs(keys, 4000, 3)
    kept, raw = run_both(jobs, kind, mkb, batch=(0,))
    assert kept < raw


@gpu
def test_long_keys_are_combined_on_the_host():
    long = [b"long-key-%02d-" % i + b"z" * 30 for i in range(4)]
    jobs = [[(long[0], 1e308), (long[0], -1e308), (long[0], TINY), (long[1], -0.0), (b"short", 0.5), (long[2], 1.0),
             (long[3], BIG), (long[3], BIG)],
            [(long[1], -0.0), (long[2], 2.0 ** -53), (b"short", 0.25), (long[3], -BIG)]]
    comb, plain = ctx_pair()
    with comb, plain:
        for j, pairs in enumerate(jobs):
            for ctx in (comb, plain):
                commit_job(ctx, "job%d" % j, pairs)
        for ctx in (comb, plain):
            ctx.shuffle()
        g = [{k: [dec(v) for v in vs] for p in ctx.partitions() for k, vs in ctx.groups(p)} for ctx in (comb, plain)]
        assert g[0] == g[1]
        assert {k: v[0] for k, v in g[0].items()} == want_sums(jobs)


@gpu
def test_words_value_jobs_get_fresh_ids():
    """the pairs of a tokeniser piece share one value id; their survivors each hold a value and an id of their own"""
    texts = [(b"a bb a ccc bb a\n" * 3000, 0.1), (b"a dd", -0.1)]
    pairs = [(w, v) for t, v in texts for w in t.split()]
    comb, plain = ctx_pair()
    with comb, plain:
        for ctx in (comb, plain):
            m = ctx.map_begin("w")
            for t, v in texts:
                m.words_value(t, enc(v))
            m.commit()
        lay = expected_layout(comb, pairs)
        n = comb.checksum_input()[3]
        assert n == sum(c for _, c in lay)
        recs = comb.pool_read(0, n)
        assert [bytes(k) for k in recs["key"]] == [k for k, c in lay for _ in range(c)]
        ids = [int(x) for x in recs["val"]]
        assert ids == list(range(ids[0], ids[0] + n))
        got = results(comb)
        assert got == results(plain)
        assert {k: v[1][0] for k, v in got[0].items()} == want_sums([pairs])


@gpu
def test_a_hot_key_with_a_million_values():
    n = 1_000_000
    rng = np.random.default_rng(4)
    vals = (rng.standard_normal(n) * 2.0 ** rng.integers(-40, 40, n)).tolist()
    pairs = [(b"big", v) for v in vals] + [(b"k%d" % i, 1 / (i + 1)) for i in range(5000)]
    kept, raw = run_both([pairs], batch=(0,))
    assert raw == n + 5000 and kept <= 5000 + 1 + 2 * 5000


@gpu
@pytest.mark.parametrize("kind", [mrhbm.KEY_U64, mrhbm.KEY_STR])
def test_layout_flags_and_the_range_partitioner(kind):
    keys = list(range(1, 5001)) if kind == mrhbm.KEY_U64 else [b"key%05d" % i for i in range(5000)]
    jobs = random_jobs(keys, 20000, 4)
    for flags in (0, mrhbm.F_SMALL_BINS, mrhbm.F_NO_OPTIMISTIC, mrhbm.F_FORCE_RUNS,
                  mrhbm.F_SMALL_BINS | mrhbm.F_NO_OPTIMISTIC | mrhbm.F_FORCE_RUNS):
        run_both(jobs, kind, flags=flags, batch=(1, 2), check_pool=flags == 0)
    run_both(jobs, kind, partitioner=mrhbm.PART_RANGE, parts=5, splitters=True, check_pool=False)


@gpu
def test_ledger_rules_failed_commits_and_interleaved_handles():
    rng = random.Random(11)

    def pairs(n, nkeys=30):
        return [(b"k%d" % rng.randrange(nkeys), rng.uniform(-10, 10)) for _ in range(n)]
    comb, plain = ctx_pair()
    with comb, plain:
        a, b, c = pairs(800), pairs(800), pairs(300)
        for ctx in (comb, plain):
            ma, mb = ctx.map_begin("A"), ctx.map_begin("B")  # interleaved handles
            for x, y in zip(a, b):
                ma.emit(x[0], enc(x[1]))
                mb.emit(y[0], enc(y[1]))
            mb.commit()
            ma.commit()
        assert results(comb) == results(plain)
        assert results(comb) == results(plain)  # a second shuffle of the same commits
        a2 = pairs(500)
        for ctx in (comb, plain):
            commit_job(ctx, "A", a2)  # replace A
            m = ctx.map_begin("aborted")
            for k, v in pairs(100):
                m.emit(k, enc(v))
            m.abort()
        assert results(comb) == results(plain)
        assert {k: v[1][0] for k, v in results(comb)[0].items()} == want_sums([a2, b])
        n_before = comb.checksum_input()[3]
        for bad in ([(b"k1", 1.0), (b"k2", None)], [(b"k1", math.inf), (b"k3", 2.0), (b"k1", -math.inf)],
                    [(b"long" * 20, 1.0), (b"long" * 20, None)], [(b"long" * 20, math.inf), (b"long" * 20, -math.inf)]):
            m = comb.map_begin("B")  # a failed commit: B's earlier commit stays
            for k, v in bad:
                m.emit(k, b"str" if v is None else enc(v))
            with pytest.raises(mrhbm.MrhbmError) as e:
                m.commit()
            assert e.value.code == INVAL
            assert comb.checksum_input()[3] == n_before
        assert results(comb) == results(plain)
        for ctx in (comb, plain):
            ctx.reset()
            commit_job(ctx, "C", c)
        assert results(comb) == results(plain)


@gpu
def test_infinities_of_both_signs_in_two_jobs_fail_the_shuffle():
    comb, plain = ctx_pair()
    with comb, plain:
        for ctx in (comb, plain):
            commit_job(ctx, "j0", [(b"k", math.inf), (b"k", 1.0), (b"x", 2.0)])
            commit_job(ctx, "j1", [(b"k", -math.inf), (b"x", 3.0)])
            with pytest.raises(mrhbm.MrhbmError) as e:
                ctx.shuffle()
            assert e.value.code == INVAL and "NaN" in str(e.value)


@gpu
def test_refusals_at_init():
    for kw in (dict(flags=0, reducer=mrhbm.RED_FSUM), dict(flags=mrhbm.F_BYTE_VALUES, reducer=mrhbm.RED_NONE),
               dict(flags=mrhbm.F_BYTE_VALUES, reducer=mrhbm.RED_DISTINCT), dict(flags=0, reducer=mrhbm.RED_SUM)):
        with pytest.raises(mrhbm.MrhbmError) as e:
            mrhbm.Ctx(mrhbm.KEY_STR, P, device=0, combiner=mrhbm.COMBINE_FSUM, **kw)
        assert e.value.code == INVAL


@gpu
def test_weighted_word_count_loop_with_the_combiner(tmp_path, golden_wordcount):
    files, acc = [], {}
    rng = random.Random(5)
    for job in range(4):
        toks = expand_tokens(golden_wordcount, job)
        lines, i = [], 0
        while i < len(toks):
            w = rng.randrange(1, 12)
            lines.append(toks[i:i + w])
            i += w
        for ln in lines:
            for t in ln:
                acc.setdefault(t, []).append(1 / len(ln))
        p = tmp_path / ("file%d.txt" % job)
        p.write_bytes(b"\n".join(b" ".join(ln) for ln in lines) + b"\n")
        files.append(str(p))
    WordCount.FILES[:] = files
    S = WWC_PKG + ".init"
    results_ = []
    for arm, combinerfn in enumerate((WWC_PKG + ".combinerfn", None)):
        WWC.RESULT.clear()
        s = server.new("hbm://local", "fsum-comb-loop-%d" % arm)
        s.configure(dict(taskfn=S, mapfn=S, partitionfn=S, reducefn=WWC_PKG + ".reducefn_device", finalfn=S,
                         combinerfn=combinerfn, storage="hbm", hbm={"value_kind": "bytes"}))
        assert s.config["hbm"]["combiner"] == ("fsum" if combinerfn else False)
        s.loop()
        results_.append({k: bits(float(v)) for k, v in WWC.RESULT.items()})
    assert results_[0] == results_[1]
    assert results_[0] == {k: bits(oracle(v)) for k, v in acc.items()}
