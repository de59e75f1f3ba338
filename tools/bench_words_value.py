"""The map side of an inverted index on the device: mrhbm_map_words_value against the Python per-emit path.

The text has the shape of config 1 of bench.py (SURVEY App. B): 197 files of 10,000 lines of 25 Zipf(1.1) words from
mrhbm_synth_zipf_text, held in host memory.  On one byte-values ctx (string keys in 32-byte records, P = 15, FNV
partitioner) every file is one map job: words_value(file bytes, encode_value(file name)), then commit.  Then one
shuffle and the first result access (mrhbm_result_values sizing only: the compaction, the value-length scan and the
gather, nothing copied to the host).  Every step is timed with the host clock; the calls synchronise before they
return.  The map side is also given as words/s.

The Python arm is the InvertedIndex mapfn loop (a regex over each line, emit(word, file path) per token, each emit one
tuple.encode_value and one mrhbm_emit_str_value) over the first --py-files files, written to a temporary directory,
on a ctx of its own: map and commit time and words/s, the same per-word rate as the device arm.

Parity: the device arm's rows (result_copy + result_values) against a host tokenisation of the same text (numpy, split
on the six C-locale white-space bytes), as multisets of (key, value): the row counts must match and the sorted 64-bit
hashes of (key bytes, file index) must be equal.

The card's name and power limit are read in one nvidia-smi query.  Prints ONE JSON line.

    python tools/bench_words_value.py [--files 197] [--lines 10000] [--py-files 2]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mrhbm_loader  # noqa: E402

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm, synth  # noqa: E402
from lua_mapreduce_b200.mapreduce import tuple as T  # noqa: E402
from lua_mapreduce_b200.mapreduce.examples.InvertedIndex import init as II  # noqa: E402

P = 15
WORDS_PER_LINE = 25
KB = 28  # key bytes of a 32-byte record
IS_WS = np.zeros(256, dtype=bool)
IS_WS[list(b" \t\n\v\f\r")] = True


def card():
    """name and power limit of GPU 0, read in one query"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return None, "unavailable (%s)" % e


def byte_ctx():
    return mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, max_key_bytes=KB - 1, device=0, reducer=mrhbm.RED_NONE,
                     flags=mrhbm.F_BYTE_VALUES)


def file_name(f):
    return "europarl_%03d.txt" % f


def hash_rows(keys, file_idx):
    """a 64-bit hash of each (KB key bytes zero padded, file index) row"""
    w = np.ascontiguousarray(keys).view(np.uint32).reshape(-1, KB // 4).astype(np.uint64)
    h = np.full(w.shape[0], 0xCBF29CE484222325, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for j in range(w.shape[1]):
            h = (h ^ w[:, j]) * np.uint64(0x100000001B3)
            h ^= h >> np.uint64(29)
        h = (h ^ file_idx.astype(np.uint64)) * np.uint64(0x9E3779B97F4A7C15)
    return h


def host_tokens(t):
    """the words of t as an (n, KB) zero-padded byte matrix"""
    ws = IS_WS[t]
    starts = np.flatnonzero(~ws & np.concatenate([[True], ws[:-1]]))
    ends = np.flatnonzero(~ws & np.concatenate([ws[1:], [True]])) + 1
    assert (ends - starts).max(initial=0) < KB
    col = np.arange(KB)
    idx = np.minimum(starts[:, None] + col[None, :], t.size - 1)
    return np.where(col[None, :] < (ends - starts)[:, None], t[idx], 0).astype(np.uint8)


def device_arm(texts, values):
    ctx = byte_ctx()
    map_s = commit_s = 0.0
    words = 0
    for f, t in enumerate(texts):
        t0 = time.perf_counter()
        m = ctx.map_begin(str(f))
        words += m.words_value(t, values[f])
        t1 = time.perf_counter()
        m.commit()
        t2 = time.perf_counter()
        map_s += t1 - t0
        commit_s += t2 - t1
    t0 = time.perf_counter()
    ctx.shuffle()
    shuffle_ms = (time.perf_counter() - t0) * 1e3
    stats = ctx.stats()
    need = C.c_size_t()
    t0 = time.perf_counter()
    ctx._chk(ctx.L.mrhbm_result_values(ctx.h, None, 0, None, C.byref(need)))  # compaction + value gather, sizing only
    first_access_ms = (time.perf_counter() - t0) * 1e3
    r = dict(words=words, map_s=map_s, commit_s=commit_s, words_per_s=words / map_s, shuffle_ms=shuffle_ms,
             first_access_ms=first_access_ms, value_bytes=need.value, stats=stats)
    return ctx, r


def parity(ctx, texts, values):
    keys, _, _ = ctx.result_copy()
    blob, roff = ctx.result_values()
    vlen = len(values[0])
    if not (np.diff(roff.astype(np.int64)) == vlen).all():
        return False
    names = blob.reshape(-1, vlen)[:, -7:-4]  # the three digits of europarl_XXX.txt
    file_idx = ((names[:, 0] - 48).astype(np.int64) * 100 + (names[:, 1] - 48) * 10 + (names[:, 2] - 48))
    if not all(bytes(blob[i * vlen:(i + 1) * vlen]) == values[int(file_idx[i])] for i in range(0, keys.shape[0], 99991)):
        return False
    got = np.sort(hash_rows(keys.view(np.uint8).reshape(-1, KB), file_idx))
    del keys, blob
    want = []
    for f, t in enumerate(texts):
        mat = host_tokens(t)
        want.append(hash_rows(mat, np.full(mat.shape[0], f)))
    want = np.sort(np.concatenate(want))
    return bool(got.shape == want.shape and (got == want).all())


def python_arm(texts, nfiles):
    d = tempfile.mkdtemp(prefix="mrhbm_words_value_")
    try:
        paths = []
        for f in range(nfiles):
            p = os.path.join(d, file_name(f))
            texts[f].tofile(p)
            paths.append(p)
        ctx = byte_ctx()
        map_s = commit_s = 0.0
        words = 0
        for f, p in enumerate(paths):
            t0 = time.perf_counter()
            m = ctx.map_begin(str(f))
            count = [0]

            def emit(key, value):  # mapreduce/job.py's emit on a value_kind = "bytes" job
                count[0] += 1
                m.emit(key, T.encode_value(value))
            II.mapfn(f, p, emit)
            t1 = time.perf_counter()
            m.commit()
            t2 = time.perf_counter()
            words += count[0]
            map_s += t1 - t0
            commit_s += t2 - t1
        ctx.close()
        return dict(files=nfiles, words=words, map_s=map_s, commit_s=commit_s, words_per_s=words / map_s)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=197)
    ap.add_argument("--lines", type=int, default=10_000)
    ap.add_argument("--py-files", type=int, default=2)
    a = ap.parse_args()
    name, power = card()
    table = synth.zipf_table()
    per_file = a.lines * WORDS_PER_LINE
    texts = [mrhbm.synth_zipf_text(synth.SEED, f * per_file, per_file, table, words_per_line=WORDS_PER_LINE)
             for f in range(a.files)]
    values = [T.encode_value(file_name(f)) for f in range(a.files)]
    ctx, dev = device_arm(texts, values)
    ok = parity(ctx, texts, values)
    ctx.close()
    py = python_arm(texts, min(a.py_files, a.files))
    print(json.dumps(dict(bench="words_value", gpu=name, power_limit=power, files=a.files, words=dev["words"],
                          text_bytes=int(sum(t.nbytes for t in texts)), device=dev, python=py,
                          speedup_words_per_s=dev["words_per_s"] / py["words_per_s"], parity=ok)), flush=True)


if __name__ == "__main__":
    main()
