"""Cost of the range partitioner against the hash partitioners it sits beside, on one GPU.

  config 2: 1e8 uniform u64 pairs, P = 1024: MULHASH against RANGE with evenly spaced given splitters (the cost of the
            range search on the optimistic layout) and RANGE with sampled splitters (mrhbm_sample_splitters), each
            on its own ctx
  config 3: Zipf(1.1) word pairs with the combiner, P = 15: FNV_LUA against RANGE with 14 two-letter splitters

The arms alternate inside one process (warm-up steps first, then --steps rounds of every arm), so clock and
thermal drift fall on all arms alike.  Prints ONE JSON line: the card name and power limit, per-arm medians of the
shuffle's stages (level 1 = ms_plan, level 2 = ms_scatter, sort/reduce, total; sampling for the sampled arm), the
result_info().sorted flag, and parity of every arm against the CPU oracle (flat group-by, re-partitioned with
bisect_right for the range arms).

    python tools/bench_range.py --steps 5 --warmup 1
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import mrhbm_loader  # noqa: E402

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm as M, synth  # noqa: E402

import oracle as O  # noqa: E402


def card():
    try:
        import pynvml as N
        N.nvmlInit()
        h = N.nvmlDeviceGetHandleByIndex(0)
        name = N.nvmlDeviceGetName(h)
        return {"gpu": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": N.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
                "sm_max_mhz": N.nvmlDeviceGetMaxClockInfo(h, N.NVML_CLOCK_SM),
                "sm_mhz_now": N.nvmlDeviceGetClockInfo(h, N.NVML_CLOCK_SM)}
    except Exception as e:  # the numbers are then unlabelled: say so
        return {"gpu": None, "nvml": repr(e)}


def two_letter_splitters(P):
    out = []
    for i in range(1, P):
        v = i * 676 // P
        out.append(bytes([97 + v // 26, 97 + v % 26]))
    return out


def run_arm(ctx, fill, sample):
    ctx.reset()
    fill(ctx)
    ms_sample = None
    if sample:
        t = time.perf_counter()
        ctx.sample_splitters()
        ms_sample = (time.perf_counter() - t) * 1e3
    ctx.shuffle()
    st = ctx.stats()
    return {"l1": st["ms_plan"], "l2": st["ms_scatter"], "split": st["ms_plan"] + st["ms_scatter"],
            "sort": st["ms_sort_reduce"], "total": st["ms_total"], "sample": ms_sample, "attempts": st["attempts"]}


def med(rows, k):
    v = [r[k] for r in rows if r[k] is not None]
    return round(float(np.median(v)), 3) if v else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--u64-pairs", type=int, default=100_000_000)
    ap.add_argument("--zipf-pairs", type=int, default=200_000_000)
    a = ap.parse_args()
    out = {"card": card(), "steps": a.steps, "warmup": a.warmup}

    # ---- config 2
    n, P = a.u64_pairs, 1024

    def fill_u64(ctx):
        m = ctx.map_begin("u64")
        m.gen_u64(synth.SEED, 0, n)
        m.commit()

    given = [(i << 64) // P for i in range(1, P)]
    arms = {"mulhash": (M.Ctx(M.KEY_U64, P, M.PART_MULHASH, device=0), False),
            "range_given": (M.Ctx(M.KEY_U64, P, M.PART_RANGE, device=0), False),
            "range_sampled": (M.Ctx(M.KEY_U64, P, M.PART_RANGE, device=0), True)}
    arms["range_given"][0].set_splitters(given)
    rows = {k: [] for k in arms}
    for step in range(a.warmup + a.steps):
        for k, (ctx, smp) in arms.items():
            r = run_arm(ctx, fill_u64, smp)
            if step >= a.warmup:
                rows[k].append(r)
    ok, osum, _ = O.groupby_u64_stream(synth.SEED, 0, n, O.PART_MULHASH, 1)
    c2 = {"workload": "config2: 1e8 uniform u64 pairs, P = 1024" if n == 100_000_000 else "%d uniform u64 pairs, P = 1024" % n}
    for k, (ctx, smp) in arms.items():
        gk, gs, gpo = ctx.result_copy()
        if not ctx.result_info().sorted:  # several ascending runs per partition: order each partition
            pid = np.repeat(np.arange(P), np.diff(gpo).astype(np.int64))
            o = np.lexsort((gk, pid))
            gk, gs = gk[o], gs[o]
        if k != "mulhash":
            spl = np.asarray(ctx.sample_splitters() if smp else given, dtype=np.uint64)
            pid = np.searchsorted(spl, ok, side="right")
            opo = np.zeros(P + 1, dtype=np.uint64)
            opo[1:] = np.cumsum(np.bincount(pid, minlength=P))
            parity = bool((gpo == opo).all() and (gk == ok).all() and (gs == osum).all())
        else:
            hk, hs, hpo = O.groupby_u64_stream(synth.SEED, 0, n, O.PART_MULHASH, P)
            parity = bool((gpo == hpo).all() and (gk == hk).all() and (gs == hs).all())
        c2[k] = {s: med(rows[k], s) for s in ("l1", "l2", "split", "sort", "total", "sample")}
        c2[k].update(sorted=int(ctx.result_info().sorted), attempts=max(r["attempts"] for r in rows[k]), parity=parity)
        ctx.close()
    for k in ("range_given", "range_sampled"):
        c2["split_ratio_%s_over_mulhash" % k] = round(c2[k]["split"] / c2["mulhash"]["split"], 3)
    out["config2"] = c2

    # ---- config 3
    nz, P3 = a.zipf_pairs, 15
    table = synth.zipf_table()
    spl3 = two_letter_splitters(P3)

    def fill_zipf(ctx):
        m = ctx.map_begin("zipf")
        step = 1 << 27
        for s in range(0, nz, step):
            m.gen_zipf(synth.SEED, s, min(step, nz - s), table)
        m.commit()

    fnv = M.Ctx(M.KEY_STR, P3, M.PART_FNV_LUA, device=0, combiner=True, reserve_pairs=nz)
    rng = M.Ctx(M.KEY_STR, P3, M.PART_RANGE, device=0, combiner=True, reserve_pairs=nz)
    rng.set_splitters(spl3)
    arms = {"fnv_lua": fnv, "range_2letter": rng}
    rows = {k: [] for k in arms}
    for step in range(a.warmup + a.steps):
        for k, ctx in arms.items():
            r = run_arm(ctx, fill_zipf, False)
            if step >= a.warmup:
                rows[k].append(r)
    counts = O.zipf_counts(synth.SEED, 0, nz, table)
    c3 = {"workload": "config3 shape: %d Zipf(1.1) word pairs, combiner, P = 15" % nz}
    for k, ctx in arms.items():
        gk, gs, gpo = ctx.result_copy()
        if k == "fnv_lua":
            okeys, osum3, opo3 = O.wordcount_from_counts(counts, O.PART_FNV_LUA, P3)
            want = {(bytes(x).rstrip(b"\0"), int(s)) for x, s in zip(okeys, osum3)}
            parity = bool((gpo == opo3).all())
        else:
            okeys, osum3, _ = O.wordcount_from_counts(counts, O.PART_FNV_LUA, 1)
            want = {(bytes(x).rstrip(b"\0"), int(s)) for x, s in zip(okeys, osum3)}
            import bisect
            opo3 = np.zeros(P3 + 1, dtype=np.uint64)
            for x, _ in want:
                opo3[bisect.bisect_right(spl3, x) + 1] += 1
            parity = bool((gpo == np.cumsum(opo3)).all())
        got = {(bytes(x), int(s)) for x, s in zip(gk.tolist(), gs.tolist())}
        parity = parity and got == want
        c3[k] = {s: med(rows[k], s) for s in ("l1", "l2", "split", "sort", "total")}
        c3[k].update(sorted=int(ctx.result_info().sorted), attempts=max(r["attempts"] for r in rows[k]), parity=parity)
        ctx.close()
    out["config3"] = c3
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
