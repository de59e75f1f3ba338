"""Pins the CPU oracle (oracle/mr_oracle.c) to the reference's own test vectors and to the
golden word count derived from the reference's test.sh corpus (tests/golden/make_golden.py)."""
import hashlib

import numpy as np
import pytest

import oracle as O
from conftest import expand_tokens


def test_escape_vectors(golden_vectors):  # mapreduce/utils.lua:345-347
    for v, want in golden_vectors["escape"]:
        got = O.escape(v if isinstance(v, (int, float)) else v.encode())
        assert got == want.encode()
    assert O.escape(2.0**53) == b"9.007199254741e+15"  # SURVEY A.4: %.14g
    assert O.escape(b'a"b\\c') == b'"a\\"b\\\\c"'
    assert O.escape(b"\x001") == b'"\\0001"' and O.escape(b"\x00a") == b'"\\0a"'


def test_serialize_and_keys_sorted(golden_vectors):  # utils.lua:348-349
    for vals, want in golden_vectors["serialize_table_ipairs"]:
        got = O.serialize_table_ipairs([v if isinstance(v, int) else v.encode() for v in vals])
        assert got == want.encode()
    e = O.Engine(nparts=1, reducer=O.RED_IDENTITY, aci=False)
    e.map_job(1, pairs=[(b"c", 1), (b"a", 2), (b"b", 3)])
    (name, data), = e.files().items()
    assert data == b'return "a",{2}\nreturn "b",{3}\nreturn "c",{1}\n'
    # C-locale order: unsigned bytes, proper prefix first (SURVEY A.3)
    e = O.Engine(nparts=1, reducer=O.RED_IDENTITY, aci=False)
    e.map_job(1, pairs=[(b"\xff", 1), (b"a\x00", 1), (b"a", 1), (b"B", 1), (b"", 1)])
    keys = [l.split(b",{")[0] for l in list(e.files().values())[0].splitlines()]
    assert keys == [b'return ""', b'return "B"', b'return "a"', b'return "a\\0"', b'return "\xff"']


def test_merge_fixture(golden_vectors):  # utils.lua:360-380
    m = golden_vectors["merge"]
    e = O.Engine(nparts=1, reducer=O.RED_IDENTITY, aci=False)
    for i, (name, lines) in enumerate(sorted(m["files"].items())):
        e.add_file("map_results.P0.M%s" % name, "\n".join(lines).encode())
    e.reduce_all()
    got = [[k, v] for _, k, v in e.final_pairs()]
    assert got == [[float(k), [float(x) for x in v]] for k, v in m["result"]]


def test_heap_and_count_digits(golden_vectors):  # heap.lua:99-118, server.lua:630-636
    assert O.heap_sort(golden_vectors["heap"]["push"]) == golden_vectors["heap"]["pop"]
    rng = np.random.default_rng(1)
    x = rng.integers(0, 1000, 500).astype(float)
    assert O.heap_sort(x) == sorted(x.tolist())
    for n, d in golden_vectors["count_digits"]:
        assert O.lib().mro_count_digits(n) == d


def test_partitionfn_known_answers(golden_vectors, golden_wordcount):
    for k, (p, h) in golden_vectors["partitionfn_known_answers"].items():
        assert O.part_fnv_lua(k.encode()) == p and O.fnv_lua(k.encode()) == h
    for k, p, _ in golden_wordcount:  # all 1,577 keys of the corpus
        assert O.part_fnv_lua(k) == p


@pytest.mark.parametrize("combiner,aci", [(O.RED_SUM, True), (-1, True), (-1, False)])
def test_wordcount_golden(golden_vectors, golden_wordcount, combiner, aci):
    """test.sh:8-53: the three plugin configurations == misc/naive.lua, per partition too."""
    e = O.Engine(O.PART_FNV_LUA, 15, combiner=combiner, reducer=O.RED_SUM, aci=aci)
    for job in range(4):
        e.map_job(job + 1, pairs=[(t, 1) for t in expand_tokens(golden_wordcount, job)])
    assert e.reduce_all(2) == 15
    pairs = list(e.final_pairs())
    assert [p for p, _, _ in pairs] == sorted(p for p, _, _ in pairs)  # server.lua:367
    for p in range(15):
        ks = [k for q, k, _ in pairs if q == p]
        assert ks == sorted(ks)  # ascending inside a partition (utils.lua:214)
    got = {k: (p, int(v[0])) for p, k, v in pairs}
    assert all(len(v) == 1 for _, _, v in pairs)
    assert got == {k: (p, sum(c)) for k, p, c in golden_wordcount}
    per = [sum(1 for k in got if got[k][0] == p) for p in range(15)]
    assert per == golden_vectors["distinct_per_partition"]
    lines = sorted(b"%d %s\n" % (c, k) for k, (_, c) in got.items())
    assert hashlib.sha256(b"".join(lines)).hexdigest() == golden_vectors["sha256_sorted_count_word_lines"]
    assert [n for n, _, _ in e.results()] == ["result.P%02d" % p for p in range(15)]  # server.lua:313-321


def test_naive_matches_golden(golden_vectors, golden_wordcount):
    toks = [t for job in range(4) for t in expand_tokens(golden_wordcount, job)]
    ntok, wc = O.naive_wordcount([b" \t".join(toks[:100]) + b"\n", b"\n".join(toks[100:])])
    assert ntok == golden_vectors["tokens"] and len(wc) == golden_vectors["distinct"]
    assert wc == [(k, sum(c)) for k, _, c in golden_wordcount]


def test_combiner_trigger():
    """job.lua:89-96: the combiner fires when #values (before the append) exceeds 5000."""
    e = O.Engine(nparts=1, combiner=O.RED_SUM, reducer=O.RED_IDENTITY, aci=False)
    e.map_job(1, pairs=[(b"k", 1)] * 5001 + [(b"j", 2)] * 3)
    assert list(e.files().values())[0] == b'return "j",{6}\nreturn "k",{5001}\n'
    e = O.Engine(nparts=1, combiner=-1, reducer=O.RED_IDENTITY, aci=False)
    e.map_job(1, pairs=[(b"j", 2)] * 3)
    assert list(e.files().values())[0] == b'return "j",{2,2,2}\n'


def test_recommit_replaces_and_empty_partitions():
    """job.lua:217-221 remove_file+build; server.lua:300-324 only non-empty partitions."""
    e = O.Engine(O.PART_FNV_LUA, 15, combiner=-1)
    e.map_job(1, pairs=[(b"a", 1), (b"a", 1)])
    e.map_job(1, pairs=[(b"a", 5)])
    e.map_job(2, pairs=[])
    assert e.reduce_all() == 1
    assert [(p, k, v) for p, k, v in e.final_pairs()] == [(10, b"a", [5.0])]


def test_synthetic_selftests(golden_vectors):
    s = golden_vectors["splitmix64"]
    assert [hex(O.splitmix64(s["seed"] + i)) for i in range(3)] == [hex(int(x, 16)) for x in s["out"]]
    for r, k in golden_vectors["rank_to_key"].items():
        assert O.rank_to_key(int(r)) == k.encode()
    keys = {O.rank_to_key(r) for r in range(1, 20001)}
    assert len(keys) == 20000 and max(map(len, keys)) <= 27


def test_flat_groupby_matches_engine():
    """The flat oracles used at 10^6..10^7 give the engine's results."""
    rng = np.random.default_rng(5)
    keys = rng.integers(0, 300, 4000).astype(np.uint64) * np.uint64(0x0123456789ABCDEF)
    vals = rng.integers(0, 1000, 4000).astype(np.uint32)
    ok, osum, po = O.groupby_u64(keys, vals, O.PART_MULHASH, 16)
    e = O.Engine(O.PART_MULHASH, 16, combiner=O.RED_SUM)
    for j in range(4):
        sl = slice(j * 1000, (j + 1) * 1000)
        e.map_job(j, pairs=[(int(k).to_bytes(8, "big"), int(v)) for k, v in zip(keys[sl], vals[sl])])
    e.reduce_all()
    eng = [(p, int.from_bytes(k, "big"), int(v[0])) for p, k, v in e.final_pairs()]
    flat = [(int(np.searchsorted(po, i, side="right")) - 1, int(ok[i]), int(osum[i])) for i in range(len(ok))]
    assert eng == flat
    # string slots
    words = [O.rank_to_key(int(r)) for r in rng.integers(1, 200, 3000)]
    recs = np.zeros((3000, 32), dtype=np.uint8)
    for i, w in enumerate(words):
        recs[i, :len(w)] = np.frombuffer(w, dtype=np.uint8)
        recs[i, 28] = 1
    okk, osum, po = O.groupby_rec(recs, O.PART_FNV_LUA, 15)
    e = O.Engine(O.PART_FNV_LUA, 15, combiner=-1)
    e.map_job(1, pairs=[(w, 1) for w in words])
    e.reduce_all()
    eng = [(p, k, int(v[0])) for p, k, v in e.final_pairs()]
    flat = [(int(np.searchsorted(po, i, side="right")) - 1, bytes(okk[i]).rstrip(b"\0"), int(osum[i]))
            for i in range(len(osum))]
    assert eng == flat


def test_job_size_oracles_agree_with_the_flat_ones():
    """the threaded stream oracles bench.py uses at 10^8..10^9 pairs are the flat group-by oracles
    (themselves pinned to the engine above) on the same pairs, incl. the per-rank partition filter"""
    import mrhbm_loader
    mrhbm_loader.load()
    from lua_mapreduce_b200 import synth
    S, n = synth.SEED, 400_000
    k, v = O.gen_u64(S, 11, n)
    flat = O.groupby_u64(k, v, O.PART_MULHASH, 1024)
    mt = O.groupby_u64_stream(S, 11, n, O.PART_MULHASH, 1024, nthreads=5)
    assert all((a == b).all() for a, b in zip(flat, mt))
    flat7 = O.groupby_u64(k, v, O.PART_MULHASH, 7)
    for rank in range(3):
        keys, sums, po = O.groupby_u64_stream(S, 11, n, O.PART_MULHASH, 7, world=3, rank=rank, nthreads=2)
        want_k = [flat7[0][int(flat7[2][p]):int(flat7[2][p + 1])] for p in range(7) if p % 3 == rank]
        want_s = [flat7[1][int(flat7[2][p]):int(flat7[2][p + 1])] for p in range(7) if p % 3 == rank]
        assert (np.concatenate(want_k) == keys).all() and (np.concatenate(want_s) == sums).all()
        for p in range(7):
            assert int(po[p + 1] - po[p]) == (int(flat7[2][p + 1] - flat7[2][p]) if p % 3 == rank else 0)
    table = synth.zipf_table(1 << 13)
    recs = O.gen_zipf_rec32(S, 3, 150_000, table)
    fk, fs, fpo = O.groupby_rec(recs, O.PART_FNV_LUA, 15)
    counts = O.zipf_counts(S, 3, 150_000, table, nthreads=3)
    assert int(counts.sum()) == 150_000
    wk, ws, wpo = O.wordcount_from_counts(counts, O.PART_FNV_LUA, 15)
    assert (wk == fk).all() and (ws == fs).all() and (wpo == fpo).all()
    wk1, ws1, wpo1 = O.wordcount_from_counts(counts, O.PART_FNV_LUA, 15, world=2, rank=1)
    sel = np.concatenate([np.arange(int(fpo[p]), int(fpo[p + 1])) for p in range(15) if p % 2 == 1])
    assert (wk1 == fk[sel]).all() and (ws1 == fs[sel]).all()


@pytest.mark.parametrize("rb", [32, 64, 128])
def test_groupby_rec_sums_past_32_bits(rb):
    """the GPU suite checks string-key sums past 2^32 against O.groupby_rec: pin it against a plain dict sum with
    values near 2^32 and sums up to about 2^45, keys up to the record class's full slot"""
    rng = np.random.default_rng(rb)
    kb = rb - 4
    vocab = [b"k%d" % i + b"x" * int(rng.integers(0, kb - 6)) for i in range(300)] + [b"z" * kb, b"z" * (kb - 1)]
    idx = np.concatenate([rng.integers(0, len(vocab), 20_000), np.full(8192, len(vocab) - 2)])  # one key: 2^13 pairs
    vals = rng.integers(0xF0000000, 1 << 32, idx.size, dtype=np.uint64).astype(np.uint32)
    recs = np.zeros(idx.size, dtype=[("key", "S%d" % kb), ("val", "<u4")])
    recs["key"] = np.array(vocab, dtype="S%d" % kb)[idx]
    recs["val"] = vals
    P = 7
    okeys, osum, po = O.groupby_rec(recs.view(np.uint8).reshape(idx.size, rb), O.PART_FNV_LUA, P)
    want = {}
    for k, v in zip(idx.tolist(), vals.tolist()):
        want[vocab[k]] = want.get(vocab[k], 0) + v
    assert max(want.values()) > 1 << 44
    got = {}
    for p in range(P):
        ks = [bytes(k).rstrip(b"\0") for k in okeys[int(po[p]):int(po[p + 1])]]
        assert ks == sorted(ks)
        for k, s in zip(ks, osum[int(po[p]):int(po[p + 1])].tolist()):
            assert O.part_fnv_lua(k, P) == p and k not in got
            got[k] = s
    assert got == want
