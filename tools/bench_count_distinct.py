"""COUNT(DISTINCT) per key on the device: MRHBM_RED_COUNT_DISTINCT against MRHBM_RED_DISTINCT followed by counting
each key's rows on the host.

Two streams, each on string keys in 32-byte records, P = 15, FNV partitioner, byte values:
  words   the corpus of tools/bench_inverted_index.py (Zipf(1.1) words of mrhbm_synth_zipf_text, 25 per line), --files
          files of --lines lines, every file one map job: words_value(file bytes, encode_value(file name)), so the
          result is every word's document frequency (>= 10^8 pairs at the defaults)
  visits  (url, visitor) pairs from emit_batch_values: --visits pairs over Zipf(1.1) urls of 10^5 pages and
          visitor ids drawn from 2^24 (8-byte big-endian values), plus one hot url holding --hot distinct visitors
          (each seen twice), in --jobs map jobs
Four arms per stream, every run on a ctx of its own:
  distinct          COMBINE_NONE,     RED_DISTINCT, then the group sizes from result_copy + result_values
  distinct+comb     COMBINE_DISTINCT, RED_DISTINCT, the same
  count             COMBINE_NONE,     RED_COUNT_DISTINCT
  count+comb        COMBINE_DISTINCT, RED_COUNT_DISTINCT
Reported per arm and run: commit time (the dedupe with the combiner), the shuffle's wall time, ms_total, ms_combine,
ms_bigbins and launches, the first result access (mrhbm_result_values sizing: compaction, and the value gather or
the count encoding) and, for the distinct arms, the host time to turn the rows into counts.  Parity: every key's
count, as a sorted hash of (key, count) rows, is identical across the four arms.

The card's name and power limit are read in one nvidia-smi query.  Prints ONE JSON line.

    python tools/bench_count_distinct.py [--files 400] [--lines 10000] [--visits 50000000] [--hot 1500000] [--reps 2]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mrhbm_loader  # noqa: E402

mrhbm_loader.load()
from bench_words_value import KB, P, WORDS_PER_LINE, card, file_name, hash_rows  # noqa: E402
from lua_mapreduce_b200 import mrhbm, synth  # noqa: E402
from lua_mapreduce_b200.mapreduce import tuple as T  # noqa: E402

ARMS = {"distinct": (mrhbm.COMBINE_NONE, mrhbm.RED_DISTINCT),
        "distinct+comb": (mrhbm.COMBINE_DISTINCT, mrhbm.RED_DISTINCT),
        "count": (mrhbm.COMBINE_NONE, mrhbm.RED_COUNT_DISTINCT),
        "count+comb": (mrhbm.COMBINE_DISTINCT, mrhbm.RED_COUNT_DISTINCT)}


def words_jobs(files, lines):
    table = synth.zipf_table()
    per_file = lines * WORDS_PER_LINE
    texts = [mrhbm.synth_zipf_text(synth.SEED, f * per_file, per_file, table, words_per_line=WORDS_PER_LINE)
             for f in range(files)]
    values = [T.encode_value(file_name(f)) for f in range(files)]
    return [("words", t, v) for t, v in zip(texts, values)], files * per_file


def visit_jobs(visits, hot, jobs):
    rng = np.random.default_rng(12)
    urls = (rng.zipf(1.1, size=visits) % 100_000).astype(np.int64)
    who = rng.integers(0, 1 << 24, size=visits, dtype=np.uint64)
    hot_who = np.concatenate([np.arange(hot, dtype=np.uint64)] * 2) + np.uint64(1 << 40)
    urls = np.concatenate([urls, np.full(2 * hot, -1, dtype=np.int64)])
    who = np.concatenate([who, hot_who])
    order = rng.permutation(len(urls))
    urls, who = urls[order], who[order]
    keys = np.char.add(b"/page/", urls.astype("S7"))
    keys[urls < 0] = b"/"
    out = []
    for j in range(jobs):
        a, b = len(urls) * j // jobs, len(urls) * (j + 1) // jobs
        recs = np.zeros(b - a, dtype=mrhbm.record_dtype(mrhbm.KEY_STR, KB - 1))
        recs["key"] = keys[a:b]
        out.append(("visits", recs, (who[a:b].astype(">u8").tobytes(), np.arange(b - a + 1, dtype=np.uint64) * 8)))
    return out, len(urls)


def run(jobs, arm):
    combiner, reducer = ARMS[arm]
    ctx = mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=KB - 1, device=0, reducer=reducer,
                    flags=mrhbm.F_BYTE_VALUES, combiner=combiner)
    commit_s = 0.0
    for j, (kind, x, v) in enumerate(jobs):
        m = ctx.map_begin(str(j))
        if kind == "words":
            m.words_value(x, v)
        else:
            m.emit_batch_values(x, v[0], v[1])
        t0 = time.perf_counter()
        m.commit()
        commit_s += time.perf_counter() - t0
    t0 = time.perf_counter()
    ctx.shuffle()
    shuffle_ms = (time.perf_counter() - t0) * 1e3
    st = ctx.stats()
    need = C.c_size_t()
    t0 = time.perf_counter()
    ctx._chk(ctx.L.mrhbm_result_values(ctx.h, None, 0, None, C.byref(need)))
    first_access_ms = (time.perf_counter() - t0) * 1e3
    info = ctx.result_info()
    r = dict(commit_s=commit_s, shuffle_wall_ms=shuffle_ms, ms_total=st["ms_total"], ms_combine=st["ms_combine"],
             ms_bigbins=st["ms_bigbins"], launches=st["launches"], attempts=st["attempts"], pairs_in=info.pairs_in,
             pairs_recv=info.pairs_recv, rows=info.groups, first_access_ms=first_access_ms)
    t0 = time.perf_counter()
    keys, _, _ = ctx.result_copy()
    k = np.ascontiguousarray(keys).view(np.uint8).reshape(-1, KB)
    if reducer == mrhbm.RED_DISTINCT:  # a key's rows are adjacent in its run: the group sizes are the counts
        heads = np.flatnonzero(np.concatenate([[True], np.any(k[1:] != k[:-1], axis=1)]))
        counts = np.diff(np.append(heads, len(k)))
        k = k[heads]
        r["count_on_host_ms"] = (time.perf_counter() - t0) * 1e3
    else:  # one 11-byte number per key: the sign-folded double in ten 7-bit groups
        blob, _ = ctx.result_values()
        g = blob.reshape(-1, 11)[:, 1:].astype(np.uint64) & np.uint64(0x7F)
        u = np.zeros(len(k), dtype=np.uint64)
        for j in range(10):
            u = (u << np.uint64(7)) | g[:, j]
        counts = (u & np.uint64(0x7FFFFFFFFFFFFFFF)).view(np.float64).astype(np.int64)
    ctx.close()
    r["keys"] = int(len(k))
    r["max_count"] = int(counts.max(initial=0))
    return r, np.sort(hash_rows(k, counts.astype(np.uint64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=400)
    ap.add_argument("--lines", type=int, default=10_000)
    ap.add_argument("--visits", type=int, default=50_000_000)
    ap.add_argument("--hot", type=int, default=1_500_000)
    ap.add_argument("--jobs", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    name, power = card()
    res = dict(bench="count_distinct", gpu=name, power_limit=power, streams={})
    for stream in ("words", "visits"):
        if stream == "words":
            jobs, pairs = words_jobs(a.files, a.lines)
        else:
            jobs, pairs = visit_jobs(a.visits, a.hot, a.jobs)
        runs, hashes = {arm: [] for arm in ARMS}, {}
        for rep in range(a.reps):
            for arm in ARMS:
                r, h = run(jobs, arm)
                runs[arm].append(r)
                if rep == 0:
                    hashes[arm] = h
        ref = hashes["distinct"]
        res["streams"][stream] = dict(pairs=pairs, runs=runs,
                                      parity=bool(len(ref) and all(np.array_equal(ref, hashes[arm]) for arm in ARMS)))
        del jobs
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
