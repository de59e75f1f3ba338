"""Byte values (MRHBM_F_BYTE_VALUES) on an inverted-index-shaped stream: Zipf(1.1) word keys in 32-byte records with
a document id per pair as its value.  One JSON line per value kind:

  int     today's group-only mode, the document id as an integer value (the baseline)
  docid   the document id as a 6-10 byte decimal string
  b100    a 100-byte value per pair

shuffle_ms is mrhbm_stats.ms_total.  compact_ms is a host clock around the first result access, which compacts the
rows (and, with byte values, scans the value lengths and gathers the value bytes) and ends in a stream synchronise;
it copies nothing to the host and includes the allocation of the result buffers.  The shuffle then runs again and
torch.profiler (CUDA activities) times the kernels of a second first access: kernel_ms per kernel, gather_ms = the
k_value_* kernels (length scan, gather, pieces of long values).  gather_bytes counts what the gather has to move: per
row its value id (8), its two value offsets (16) and its row offset read and written (16), plus the value bytes read
and written; gather_tbs = gather_bytes / gather_ms.

    python bench_values.py [--pairs 100000000] [--chunk 10000000] [--kinds int,docid,b100]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import mrhbm_loader  # noqa: E402

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm, synth  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet
P = 15


def card():
    """name and power limit of GPU 0, read in one query"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return None, "unavailable (%s)" % e


def doc_ids(start, n):
    """document id of pair i: a splitmix64 hash, printed in 6 to 10 decimal digits"""
    h = synth.splitmix64_np(np.arange(start, start + n, dtype=np.uint64) + np.uint64(1 << 42))
    ndig = (6 + h % np.uint64(5)).astype(np.int64)
    v = (h >> np.uint64(8)) % (np.uint64(10) ** ndig.astype(np.uint64))
    return v, ndig


def docid_blob(v, ndig):
    """decimal strings, zero padded to their digit count, packed, and their offsets"""
    n = v.shape[0]
    mat = np.empty((n, 10), dtype=np.uint8)
    x = v.copy()
    for j in range(9, -1, -1):  # right-aligned digits
        mat[:, j] = (x % np.uint64(10)).astype(np.uint8) + ord("0")
        x //= np.uint64(10)
    mask = np.arange(10)[None, :] >= (10 - ndig)[:, None]
    voff = np.zeros(n + 1, dtype=np.uint64)
    voff[1:] = np.cumsum(ndig)
    return mat[mask], voff


def run(kind, pairs, chunk, table):
    flags = mrhbm.F_BYTE_VALUES if kind != "int" else 0
    gen = mrhbm.Ctx(mrhbm.KEY_STR, 1, device=0, reducer=mrhbm.RED_NONE)
    ctx = mrhbm.Ctx(mrhbm.KEY_STR, P, device=0, reducer=mrhbm.RED_NONE, flags=flags, reserve_pairs=pairs)
    m = ctx.map_begin("bench")
    value_bytes = 0
    rng = np.random.default_rng(7)
    for start in range(0, pairs, chunk):
        n = min(chunk, pairs - start)
        g = gen.map_begin("keys")
        g.gen_zipf(synth.SEED, start, n, table)
        g.commit()
        recs = gen.pool_read(0, n)
        gen.reset()
        v, ndig = doc_ids(start, n)
        if kind == "int":
            recs["val"] = (v & np.uint64(0xFFFFFFFF)).astype(np.uint32)
            m.emit_batch(recs)
            continue
        if kind == "docid":
            blob, voff = docid_blob(v, ndig)
        else:
            blob = rng.integers(0, 256, size=n * 100, dtype=np.uint8)
            voff = np.arange(n + 1, dtype=np.uint64) * np.uint64(100)
        value_bytes += int(voff[-1])
        m.emit_batch_values(recs, blob, voff)
    m.commit()
    gen.close()
    ctx.shuffle()
    st = ctx.stats()
    t0 = time.perf_counter()
    if kind == "int":
        rc = ctx.L.mrhbm_result_copy(ctx.h, None, None, None)  # compaction only, nothing copied
    else:
        need = C.c_size_t()
        rc = ctx.L.mrhbm_result_values(ctx.h, None, 0, None, C.byref(need))  # compaction + value gather, sizing only
        assert need.value == value_bytes, (need.value, value_bytes)
    compact_ms = (time.perf_counter() - t0) * 1e3
    ctx._chk(rc)
    rows = ctx.result_info().groups
    ctx.shuffle()  # again: a fresh result, its first access under the profiler
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        if kind == "int":
            ctx._chk(ctx.L.mrhbm_result_copy(ctx.h, None, None, None))
        else:
            ctx._chk(ctx.L.mrhbm_result_values(ctx.h, None, 0, None, C.byref(need)))
    kernel_ms = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t and ("k_compact" in e.key or "k_value" in e.key):
            kernel_ms[e.key] = round(t / 1e3, 4)
    ctx.close()
    gather = sum(v for k, v in kernel_ms.items() if "k_value" in k)
    return dict(shuffle_ms=st["ms_total"], compact_ms=compact_ms, rows=rows, value_bytes=value_bytes,
                kernel_ms=kernel_ms, gather_ms=gather if kind != "int" else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=10 ** 8)
    ap.add_argument("--chunk", type=int, default=10 ** 7)
    ap.add_argument("--kinds", default="int,docid,b100")
    ap.add_argument("--vocab", type=int, default=1 << 20)
    a = ap.parse_args()
    name, power = card()
    table = synth.zipf_table(a.vocab)
    for kind in a.kinds.split(","):
        r = run(kind, a.pairs, a.chunk, table)
        line = dict(bench="byte_values", gpu=name, power_limit=power, kind=kind, pairs=a.pairs, zipf_s=synth.ZIPF_S,
                    vocab=a.vocab, **r)
        g = r["gather_ms"]
        if g:
            moved = r["rows"] * (8 + 16 + 16) + 2 * r["value_bytes"]
            line.update(gather_bytes=moved, gather_tbs=moved / (g * 1e-3) / 1e12,
                        gather_share_of_hbm=moved / (g * 1e-3) / 1e12 / HBM_TBS)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
