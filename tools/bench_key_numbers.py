"""The map side of a number sum on the device: mrhbm_map_key_numbers against the host's ways of emitting the same pairs.

Input: --lines (default 10^8) seeded text lines "key number", drawn uniformly from a pool of 2^20 distinct lines whose
keys are Zipf(1.1) over 2^18 ranks and whose numbers are, in turn, "%.2f", integers and repr() of a double (the pool is
formatted once; the text is assembled from it with numpy).  Arms, each on a fresh byte-values ctx with P = 15:
  device       one key_numbers call over the whole text: map time (host clock; the call ends in a synchronise) and
               text GB/s, after a warm-up call; then commit and the RED_FSUM shuffle
  device_comb  the same with COMBINE_FSUM: map time, commit (the combine) and shuffle
  numpy        the same pairs encoded with numpy (not timed) and uploaded with one emit_batch_values call (timed)
  python       the KeyNumberSum host mapfn (regex + float + emit) on the first --py-lines lines (pairs/s)
Parity: the first 10^6 committed records of the device arm against the pool (keys in text order, value id = pool
index), and every key's sum in both device arms against float(sum(Fraction)) of its numbers.  The card's name and power
limit are read in the same call.  Prints ONE JSON line.

    python tools/bench_key_numbers.py [--lines 100000000] [--py-lines 1000000]
"""
import argparse
import json
import os
import re
import sys
import time
from fractions import Fraction

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mrhbm_loader  # noqa: E402

mrhbm_loader.load()
from bench_fsum import decode, encode  # noqa: E402
from bench_words_value import card  # noqa: E402
from lua_mapreduce_b200 import mrhbm  # noqa: E402
from lua_mapreduce_b200.mapreduce.tuple import encode_value  # noqa: E402

P = 15
POOL = 1 << 20
RANKS = 1 << 18
SEED = 20261018
FIELD = re.compile(rb"[^ \t\n\v\f\r]+")
NUMBER = re.compile(rb"[+-]?([0-9]+(\.[0-9]*)?|\.[0-9]+)([eE][+-]?[0-9]+)?\Z")


def pool_lines(rng):
    """POOL distinct lines: (line bytes with '\\n', key id, value)"""
    ranks = np.minimum(rng.zipf(1.1, POOL), RANKS).tolist()
    cents = rng.integers(-10 ** 8, 10 ** 8, POOL).tolist()
    reals = (rng.standard_normal(POOL) * 10.0 ** rng.integers(-6, 9, POOL)).tolist()
    lines, keys, vals = [], [], []
    for j in range(POOL):
        kind = j % 3
        tok = b"%.2f" % (cents[j] / 100) if kind == 0 else b"%d" % (cents[j] // 7) if kind == 1 else repr(reals[j]).encode()
        lines.append(b"key-%d %s\n" % (ranks[j], tok))
        keys.append(ranks[j])
        vals.append(float(tok))
    return lines, np.array(keys), np.array(vals)


def assemble(lines, idx):
    """the text of pool lines idx, built in chunks with numpy gathers"""
    blob = np.frombuffer(b"".join(lines), dtype=np.uint8)
    ln = np.array([len(x) for x in lines], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]])
    lens = ln[idx]
    out = np.empty(int(lens.sum()), dtype=np.uint8)
    pos = 0
    for c in range(0, idx.size, 1 << 20):
        i = idx[c:c + (1 << 20)]
        L = ln[i]
        tot = int(L.sum())
        first = np.concatenate([[0], np.cumsum(L)[:-1]])
        src = np.repeat(off[i] - first, L) + np.arange(tot)
        out[pos:pos + tot] = blob[src]
        pos += tot
    return out


def ctx(comb):
    return mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, device=0, reducer=mrhbm.RED_FSUM,
                     combiner=mrhbm.COMBINE_FSUM if comb else mrhbm.COMBINE_NONE, flags=mrhbm.F_BYTE_VALUES)


def sums_of(c):
    return {k: decode(np.frombuffer(v[0], dtype=np.uint8).reshape(1, 11))[0]
            for p in c.partitions() for k, v in c.groups(p)}


def device_arm(text, comb, warm, check_pool=None):
    with ctx(comb) as c:
        m = c.map_begin("warm")
        m.key_numbers(warm)
        m.abort()
        m = c.map_begin("job")
        t0 = time.perf_counter()
        n = m.key_numbers(text)
        t_map = time.perf_counter() - t0
        t0 = time.perf_counter()
        m.commit()
        t_commit = time.perf_counter() - t0
        pool_ok = check_pool(c) if check_pool else None
        t0 = time.perf_counter()
        c.shuffle()
        t_shuffle = time.perf_counter() - t0
        return dict(pairs=n, map_ms=1e3 * t_map, text_GBps=text.size / t_map / 1e9, commit_ms=1e3 * t_commit,
                    shuffle_ms=1e3 * t_shuffle, pairs_after_commit=c.result_info().pairs_in), sums_of(c), pool_ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=100_000_000)
    ap.add_argument("--py-lines", type=int, default=1_000_000)
    a = ap.parse_args()
    name, power = card()
    rng = np.random.default_rng(SEED)
    lines, pkeys, pvals = pool_lines(rng)
    idx = rng.integers(0, POOL, a.lines)
    text = assemble(lines, idx)
    warm = assemble(lines, np.arange(20000))
    # the oracle: every key's exact sum, from each pool line's count
    cnt = np.bincount(idx, minlength=POOL)
    exact = {}
    for j in np.flatnonzero(cnt).tolist():
        k = b"key-%d" % pkeys[j]
        exact[k] = exact.get(k, 0) + Fraction(pvals[j]) * int(cnt[j])
    want = {k: float(s) for k, s in exact.items()}
    slot = np.array([b"key-%d" % k for k in pkeys], dtype="S28")

    def check_pool(c):
        n = min(a.lines, 1_000_000)
        r = c.pool_read(0, n)
        return bool((r["key"] == slot[idx[:n]]).all() and (r["val"] == np.arange(n, dtype=np.uint32)).all())

    dev, got, pool_ok = device_arm(text, False, warm, check_pool)
    comb, got_c, _ = device_arm(text, True, warm)
    parity = {"pool_first_1e6": pool_ok, "fsum": got == want, "comb_fsum": got_c == want}
    # numpy arm: the same pairs as records, 11-byte values and offsets (built before the clock), one upload
    rec = np.zeros(a.lines, dtype=mrhbm.record_dtype(mrhbm.KEY_STR))
    rec["key"] = slot[idx]
    vals = encode(pvals[idx]).reshape(-1)
    voff = np.arange(a.lines + 1, dtype=np.uint64) * np.uint64(11)
    with ctx(False) as c:
        m = c.map_begin("warm")
        m.emit_batch_values(rec[:1000], vals[:11000], voff[:1001])
        m.abort()
        m = c.map_begin("job")
        t0 = time.perf_counter()
        m.emit_batch_values(rec, vals, voff)
        m.commit()
        t_np = time.perf_counter() - t0
    del rec, vals, voff
    # python arm: the host mapfn of examples/KeyNumberSum on the first py-lines lines
    npy = min(a.py_lines, a.lines)
    sub = assemble(lines, idx[:npy]).tobytes()
    with ctx(False) as c:
        m = c.map_begin("py")
        t0 = time.perf_counter()
        for line in sub.split(b"\n"):
            f = FIELD.findall(line)
            if not f:
                continue
            if len(f) != 2 or not NUMBER.match(f[1]):
                raise ValueError(line)
            m.emit(f[0], encode_value(float(f[1])))
        m.commit()
        t_py = time.perf_counter() - t0
    print(json.dumps(dict(bench="key_numbers", gpu=name, power_limit=power, lines=a.lines, text_bytes=int(text.size),
                          keys=len(want), device=dev, device_comb=comb,
                          numpy_upload=dict(ms=1e3 * t_np, pairs_per_s=a.lines / t_np),
                          python_mapfn=dict(lines=npy, ms=1e3 * t_py, pairs_per_s=npy / t_py), parity=parity)))
    return 0 if all(parity.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
