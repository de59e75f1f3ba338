"""An inverted index with and without the device's distinct combiner (MRHBM_COMBINE_DISTINCT).

The corpus is the one of tools/bench_words_value.py, config 1 of bench.py in shape (SURVEY App. B): 197 files of
10,000 lines of 25 Zipf(1.1) words from mrhbm_synth_zipf_text, in host memory.  Two arms alternate in one process,
--reps times each, every run on a byte-values ctx of its own (string keys in 32-byte records, P = 15, FNV
partitioner) that differs only in its combiner: 0, or COMBINE_DISTINCT.  A run makes every file one map job,
words_value(file bytes, encode_value(file name)) then commit, then one shuffle and the first result access
(mrhbm_result_values sizing only: compaction, value-length scan and gather).  Reported per arm and run: map side and
commit time (the commit includes the dedupe in the distinct arm), pairs after commit, the shuffle's ms_total,
ms_bigbins and attempts, and the first result access, all with the host clock (the calls synchronise before they
return).

Then, once per arm, server.loop() end to end through the InvertedIndex example (mapfn_device; combinerfn module
examples/InvertedIndex/combinerfn in the distinct arm) over the files written to a temporary directory: the host
reducefn runs on every value that reaches it.

Parity: the rows of the two arms (result_copy + result_values) as sets of (key, value) are identical, the distinct
arm's rows are all different, and the two loops give the identical RESULT.

The card's name and power limit are read in one nvidia-smi query.  Prints ONE JSON line.

    python tools/bench_inverted_index.py [--files 197] [--lines 10000] [--reps 3] [--no-loop]
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

ARMS = {"none": mrhbm.COMBINE_NONE, "distinct": mrhbm.COMBINE_DISTINCT}
II_PKG = "lua_mapreduce_b200.mapreduce.examples.InvertedIndex"


def run(texts, values, combiner, keep_rows):
    ctx = mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=KB - 1, device=0, reducer=mrhbm.RED_NONE,
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
             ms_total=st["ms_total"], ms_bigbins=st["ms_bigbins"], attempts=st["attempts"],
             first_access_ms=first_access_ms)
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


def loop(paths, combinerfn):
    WordCount.FILES[:] = paths
    II.RESULT.clear()
    s = server.new("hbm://local", "bench-inverted-index")
    s.configure(dict(taskfn=II_PKG + ".init", mapfn=II_PKG + ".mapfn_device", partitionfn=II_PKG + ".init",
                     reducefn=II_PKG + ".init", finalfn=II_PKG + ".init", combinerfn=combinerfn, storage="hbm",
                     hbm={"value_kind": "bytes"}))
    t0 = time.perf_counter()
    s.loop()
    secs = time.perf_counter() - t0
    s.board.ctx.close()
    return dict(loop_s=secs, pairs=s.stats["shuffle"]["pairs"]), dict(II.RESULT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=197)
    ap.add_argument("--lines", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-loop", action="store_true")
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
        for arm, comb in ARMS.items():
            r, h = run(texts, values, comb, keep_rows=rep == 0)
            out[arm].append(r)
            if h is not None:
                rows[arm] = h
    parity_rows = bool(np.array_equal(np.unique(rows["none"]), rows["distinct"]))
    res = dict(bench="inverted_index", gpu=name, power_limit=power, files=a.files, words=a.files * per_file,
               runs=out, parity_rows=parity_rows)
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
                loops[arm], results[arm] = loop(paths, II_PKG + ".combinerfn" if arm == "distinct" else None)
            res["loop"] = loops
            res["parity_result"] = results["none"] == results["distinct"]
        finally:
            shutil.rmtree(d, ignore_errors=True)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
