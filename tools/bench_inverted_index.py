"""An inverted index with the device's distinct combiner (MRHBM_COMBINE_DISTINCT) and distinct reducer
(MRHBM_RED_DISTINCT).

The corpus is the one of tools/bench_words_value.py, config 1 of bench.py in shape (SURVEY App. B): 197 files of
10,000 lines of 25 Zipf(1.1) words from mrhbm_synth_zipf_text, in host memory.  Three arms alternate in one process,
--reps times each, every run on a byte-values ctx of its own (string keys in 32-byte records, P = 15, FNV
partitioner):
  combine_host     COMBINE_DISTINCT, RED_NONE: each job's repeated pairs dropped at commit, the reducefn on the host
  combine_device   COMBINE_DISTINCT, RED_DISTINCT: the same, and every key's distinct values ordered on the device
  device           COMBINE_NONE, RED_DISTINCT: the whole dedupe at the shuffle
A run makes every file one map job, words_value(file bytes, encode_value(file name)) then commit, then one shuffle
and the first result access (mrhbm_result_values sizing only: compaction, value-length scan and gather).  Reported
per arm and run: map side and commit time (the commit includes the dedupe with the combiner), pairs after commit, the
shuffle's ms_total, ms_combine (the shuffle's dedupe), ms_bigbins (the value ordering) and attempts, and the first
result access, all with the host clock (the calls synchronise before they return).

Then, once per arm, server.loop() end to end through the InvertedIndex example (mapfn_device; combinerfn module
examples/InvertedIndex/combinerfn with the combiner; reducefn module reducefn_device with the device reducer) over the
files written to a temporary directory, split into its map phase (until the last map job is done), its shuffle (up to
the first reduce job) and its reduce phase (the reduce jobs: the host reducefn, or only the groups' hand-out).

--profile: one more run of each device-reducer arm under torch.profiler, reporting the CUDA time of the ordering
kernels (k_value_order, k_value_merge) and of the distinct set's kernels (k_distinct_*) of the whole run.

Parity: the rows of the three arms (result_copy + result_values) as sets of (key, value) are identical and all
different, and the three loops give the identical RESULT.

The card's name and power limit are read in one nvidia-smi query.  Prints ONE JSON line.

    python tools/bench_inverted_index.py [--files 197] [--lines 10000] [--reps 3] [--no-loop] [--profile]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mrhbm_loader  # noqa: E402

mrhbm_loader.load()
from bench_words_value import KB, P, WORDS_PER_LINE, card, file_name, hash_rows  # noqa: E402
from lua_mapreduce_b200 import mrhbm, synth  # noqa: E402
from lua_mapreduce_b200.mapreduce import server  # noqa: E402
from lua_mapreduce_b200.mapreduce import tuple as T  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.InvertedIndex import init as II  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.WordCount import init as WordCount  # noqa: E402

# (combiner, reducer) per arm
ARMS = {"combine_host": (mrhbm.COMBINE_DISTINCT, mrhbm.RED_NONE),
        "combine_device": (mrhbm.COMBINE_DISTINCT, mrhbm.RED_DISTINCT),
        "device": (mrhbm.COMBINE_NONE, mrhbm.RED_DISTINCT)}
II_PKG = "lua_mapreduce_b200.mapreduce.examples.InvertedIndex"


def run(texts, values, arm, keep_rows):
    combiner, reducer = ARMS[arm]
    ctx = mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=KB - 1, device=0, reducer=reducer,
                    flags=mrhbm.F_BYTE_VALUES, combiner=combiner)
    map_s = commit_s = 0.0
    for f, t in enumerate(texts):
        t0 = time.perf_counter()
        m = ctx.map_begin(str(f))
        m.words_value(t, values[f])
        t1 = time.perf_counter()
        m.commit()
        t2 = time.perf_counter()
        map_s += t1 - t0
        commit_s += t2 - t1
    t0 = time.perf_counter()
    ctx.shuffle()
    shuffle_s = time.perf_counter() - t0
    st = ctx.stats()
    need = C.c_size_t()
    t0 = time.perf_counter()
    ctx._chk(ctx.L.mrhbm_result_values(ctx.h, None, 0, None, C.byref(need)))
    first_access_ms = (time.perf_counter() - t0) * 1e3
    r = dict(map_s=map_s, commit_s=commit_s, pairs_after_commit=ctx.result_info().pairs_in, shuffle_wall_ms=shuffle_s * 1e3,
             ms_total=st["ms_total"], ms_combine=st["ms_combine"], ms_bigbins=st["ms_bigbins"], attempts=st["attempts"],
             pairs_recv=ctx.result_info().pairs_recv, first_access_ms=first_access_ms)
    rows = None
    if keep_rows:
        keys, _, _ = ctx.result_copy()
        blob, roff = ctx.result_values()
        vlen = len(values[0])
        assert (np.diff(roff.astype(np.int64)) == vlen).all()
        names = blob.reshape(-1, vlen)[:, -7:-4]  # the three digits of europarl_XXX.txt
        fidx = (names[:, 0] - 48).astype(np.int64) * 100 + (names[:, 1] - 48) * 10 + (names[:, 2] - 48)
        rows = np.sort(hash_rows(keys.view(np.uint8).reshape(-1, KB), fidx))
    ctx.close()
    return r, rows


def loop(paths, arm):
    WordCount.FILES[:] = paths
    II.RESULT.clear()
    s = server.new("hbm://local", "bench-inverted-index-" + arm)
    combiner, reducer = ARMS[arm]
    s.configure(dict(taskfn=II_PKG + ".init", mapfn=II_PKG + ".mapfn_device", partitionfn=II_PKG + ".init",
                     reducefn=II_PKG + (".reducefn_device" if reducer == mrhbm.RED_DISTINCT else ".init"),
                     finalfn=II_PKG + ".init", combinerfn=II_PKG + ".combinerfn" if combiner else None, storage="hbm",
                     hbm={"value_kind": "bytes"}))
    waits = {}
    wait = s._wait

    def timed_wait(ns):  # the map jobs, then (after the shuffle) the reduce jobs
        t = time.perf_counter()
        r = wait(ns)
        waits[ns] = (t, time.perf_counter())
        return r
    s._wait = timed_wait
    t0 = time.perf_counter()
    s.loop()
    secs = time.perf_counter() - t0
    st = s.stats["shuffle"]
    s.board.ctx.close()
    (_, map_end), (red_start, red_end) = waits["map_jobs"], waits["red_jobs"]
    return dict(loop_s=secs, map_s=map_end - t0, shuffle_s=red_start - map_end, reduce_s=red_end - red_start,
                pairs=st["pairs"], ms_total=st["ms_total"]), dict(II.RESULT)


def profile(texts, values, arm):
    """CUDA time (ms) of the distinct set's and the ordering kernels over one whole run"""
    import torch
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as tprofile
    torch.cuda.init()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        run(texts, values, arm, keep_rows=False)
        torch.cuda.synchronize()
    ms = {}
    for e in prof.key_averages():
        for name in ("k_value_order", "k_value_merge", "k_distinct_mark", "k_distinct_count", "k_distinct_scatter"):
            if name in e.key:
                t = getattr(e, "device_time_total", None)
                t = getattr(e, "cuda_time_total", 0) if t is None else t
                ms[name] = ms.get(name, 0.0) + t / 1e3
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=197)
    ap.add_argument("--lines", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-loop", action="store_true")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    name, power = card()
    table = synth.zipf_table()
    per_file = a.lines * WORDS_PER_LINE
    texts = [mrhbm.synth_zipf_text(synth.SEED, f * per_file, per_file, table, words_per_line=WORDS_PER_LINE)
             for f in range(a.files)]
    values = [T.encode_value(file_name(f)) for f in range(a.files)]
    out = {arm: [] for arm in ARMS}
    rows = {}
    for rep in range(a.reps):
        for arm in ARMS:
            r, h = run(texts, values, arm, keep_rows=rep == 0)
            out[arm].append(r)
            if h is not None:
                rows[arm] = h
    ref = rows["combine_host"]
    parity_rows = bool(len(np.unique(ref)) == len(ref) and all(np.array_equal(ref, rows[arm]) for arm in ARMS))
    res = dict(bench="inverted_index", gpu=name, power_limit=power, files=a.files, words=a.files * per_file,
               runs=out, parity_rows=parity_rows)
    if a.profile:
        res["kernel_ms"] = {arm: profile(texts, values, arm) for arm in ARMS if ARMS[arm][1] == mrhbm.RED_DISTINCT}
    if not a.no_loop:
        d = tempfile.mkdtemp(prefix="mrhbm_inverted_index_")
        try:
            paths = []
            for f, t in enumerate(texts):
                p = os.path.join(d, file_name(f))
                t.tofile(p)
                paths.append(p)
            del texts
            loops, results = {}, {}
            for arm in ARMS:
                loops[arm], results[arm] = loop(paths, arm)
            res["loop"] = loops
            res["parity_result"] = all(results[arm] == results["combine_host"] for arm in ARMS)
        finally:
            shutil.rmtree(d, ignore_errors=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
