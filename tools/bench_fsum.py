"""The device's number-sum reducer (MRHBM_RED_FSUM) against today's path for a summing reducefn over Lua numbers.

Input: --pairs (default 10^8) Zipf(1.1) words over 2^20 ranks (mrhbm_map_gen_zipf's stream, 32-byte records), each
with a seeded random double (weights 1/k, wide-range values and negatives) encoded as a number value, one map job, on
a byte-values ctx with P = 15 and the FNV partitioner.  Two arms alternate, --reps times each, on a fresh ctx per run:
  fsum        RED_FSUM: the shuffle sums every key's numbers exactly and rounds once; then the first result access
              (result_copy + result_values: compaction and the 11-byte encoding of every sum), host clock
  none_fsum   RED_NONE: the group-only shuffle; then result_copy + result_values of every pair, the values decoded and
              grouped by key on the host and math.fsum per group (a correctly rounded sum, as the device's), host clock
Reported per run: ms_total and ms_bigbins of the shuffle (ms_bigbins holds the summing kernels), the first access,
and for none_fsum the host reduce.  Parity: every key's sum of the two arms bit-identical (checked on the first rep).
The card's name and power limit are read in the same call.  Prints ONE JSON line.

    python tools/bench_fsum.py [--pairs 100000000] [--chunk 10000000] [--reps 2]
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mrhbm_loader  # noqa: E402

mrhbm_loader.load()
from bench_words_value import card  # noqa: E402
from lua_mapreduce_b200 import mrhbm, synth  # noqa: E402

P = 15
V = 1 << 20


def encode(x):
    """float64 array -> (n, 11) uint8 number encodings (mapreduce/tuple.py _enc_num, -0 kept)"""
    u = x.view(np.uint64)
    u = np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))
    out = np.empty((x.size, 11), dtype=np.uint8)
    out[:, 0] = 0x10
    for k in range(10):
        out[:, 1 + k] = (np.uint64(0x80) | ((u >> np.uint64(63 - 7 * k)) & np.uint64(0x7F))).astype(np.uint8)
    return out


def decode(blob):
    """(n, 11) uint8 -> float64"""
    g = blob[:, 1:].astype(np.uint64) & np.uint64(0x7F)
    u = np.zeros(blob.shape[0], dtype=np.uint64)
    for k in range(10):
        u = (u << np.uint64(7)) | g[:, k]
    return np.where(u >> np.uint64(63), u & np.uint64((1 << 63) - 1), ~u).view(np.float64)


def key_hash(keys):
    """a 64-bit hash of every key slot (the host groups by it: a sort of u64 instead of 28-byte strings)"""
    w = np.frombuffer(keys.tobytes(), dtype=np.uint32).reshape(keys.size, -1).astype(np.uint64)
    h = np.full(keys.size, 0x9E3779B97F4A7C15, dtype=np.uint64)
    for j in range(w.shape[1]):
        h = synth.splitmix64_np(h ^ w[:, j])
    return h


def values(start, n):
    rng = np.random.default_rng(start + 17)
    kind = rng.integers(0, 3, n)
    w = 1.0 / rng.integers(1, 64, n)
    wide = rng.standard_normal(n) * np.exp2(rng.integers(-30, 30, n).astype(np.float64))
    return np.where(kind == 0, w, np.where(kind == 1, wide, -w))


def fill(ctx, pairs, chunk, table, gen):
    m = ctx.map_begin("bench")
    for start in range(0, pairs, chunk):
        n = min(chunk, pairs - start)
        g = gen.map_begin("keys")
        g.gen_zipf(synth.SEED, start, n, table)
        g.commit()
        recs = gen.pool_read(0, n)
        gen.reset()
        m.emit_batch_values(recs, encode(values(start, n)).reshape(-1), np.arange(n + 1, dtype=np.uint64) * np.uint64(11))
    m.commit()


def run(arm, pairs, chunk, table, gen, want=None):
    red = mrhbm.RED_FSUM if arm == "fsum" else mrhbm.RED_NONE
    with mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, device=0, reducer=red, flags=mrhbm.F_BYTE_VALUES,
                   reserve_pairs=pairs) as ctx:
        fill(ctx, pairs, chunk, table, gen)
        ctx.shuffle()
        st = ctx.stats()
        t0 = time.perf_counter()
        keys, _, _ = ctx.result_copy()
        blob, roff = ctx.result_values()
        access_ms = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        vals = decode(blob.reshape(-1, 11))
        if arm == "fsum":
            sums = vals
            reduce_ms = 0.0
        else:  # today's path: every pair's value on the host, grouped by key, one math.fsum per group
            h = key_hash(keys)
            order = np.argsort(h, kind="stable")
            hs = h[order]
            first = np.flatnonzero(np.r_[True, hs[1:] != hs[:-1]])
            bounds = np.r_[first, hs.size]
            sv = vals[order].tolist()
            keys = keys[order[first]]
            sums = np.array([math.fsum(sv[bounds[i]:bounds[i + 1]]) for i in range(first.size)])
            reduce_ms = (time.perf_counter() - t0) * 1e3
        res = dict(ms_total=round(st["ms_total"], 3), ms_bigbins=round(st["ms_bigbins"], 3),
                   attempts=st["attempts"], big_bins=st["big_bins"], groups=int(keys.size),
                   first_access_ms=round(access_ms, 3), host_reduce_ms=round(reduce_ms, 1))
        got = None
        if want is not None or arm == "fsum":
            order = np.argsort(keys, kind="stable")
            got = (keys[order], sums[order].view(np.uint64))
        return res, got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=100_000_000)
    ap.add_argument("--chunk", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    name, power = card()
    table = synth.zipf_table(V)
    out = {"card": name, "power_limit": power, "pairs": a.pairs, "zipf_ranks": V, "partitions": P, "runs": []}
    parity = None
    with mrhbm.Ctx(mrhbm.KEY_STR, 1, device=0, reducer=mrhbm.RED_NONE) as gen:
        for rep in range(a.reps):
            ref = None
            for arm in ("fsum", "none_fsum"):
                res, got = run(arm, a.pairs, a.chunk, table, gen, want=ref if rep == 0 else None)
                out["runs"].append(dict(arm=arm, rep=rep, **res))
                print(json.dumps(out["runs"][-1]), file=sys.stderr, flush=True)
                if rep == 0 and arm == "fsum":
                    ref = got
                elif rep == 0:
                    parity = bool(np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1]))
    out["parity_bit_identical"] = parity
    print(json.dumps(out))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
