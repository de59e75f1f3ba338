"""The number-sum combiner (MRHBM_COMBINE_FSUM) in front of the number-sum reducer (MRHBM_RED_FSUM).

Input: bench_fsum.py's stream, --pairs (default 10^8) Zipf(1.1) words over 2^20 ranks with its seeded number values, cut
into --jobs map jobs (default 400 x 250,000 pairs, config 1's job size), on a byte-values ctx with P = 15 and the FNV
partitioner.  Two arms alternate, --reps times each, on a fresh ctx per run:
  fsum        RED_FSUM alone
  comb_fsum   RED_FSUM with COMBINE_FSUM: each job's numbers per key become the exact expansion of their sum at commit
Reported per run: the total commit time (host clock around each commit, which ends in a synchronise), the pairs after
commit, the shuffle's ms_total, ms_bigbins and attempts, the first result access (result_copy + result_values) and the
end-to-end time from the first emit to the first access.  Parity: every key's sum bit-identical across the arms (first
rep).  The card's name and power limit are read in the same call.  --profile instead runs each arm once under
torch.profiler (CUDA activity) and reports the kernel time by kernel name; its times are not the arms' times.  Prints
ONE JSON line.

    python tools/bench_fsum_combiner.py [--pairs 100000000] [--jobs 400] [--reps 2] [--profile]
"""
import argparse
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
from bench_fsum import P, V, decode, encode, values  # noqa: E402
from bench_words_value import card  # noqa: E402
from lua_mapreduce_b200 import mrhbm, synth  # noqa: E402


def make_jobs(pairs, jobs, table, gen):
    """the stream cut into jobs: (records, encoded values, offsets) each, generated before any timing"""
    out, per = [], (pairs + jobs - 1) // jobs
    for start in range(0, pairs, per):
        n = min(per, pairs - start)
        g = gen.map_begin("keys")
        g.gen_zipf(synth.SEED, start, n, table)
        g.commit()
        recs = gen.pool_read(0, n)
        gen.reset()
        out.append((recs, encode(values(start, n)).reshape(-1), np.arange(n + 1, dtype=np.uint64) * np.uint64(11)))
    return out


def run(arm, jobs, pairs):
    comb = mrhbm.COMBINE_FSUM if arm == "comb_fsum" else mrhbm.COMBINE_NONE
    with mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_FNV_LUA, device=0, reducer=mrhbm.RED_FSUM, combiner=comb,
                   flags=mrhbm.F_BYTE_VALUES, reserve_pairs=pairs) as ctx:
        commit_s = 0.0
        t_start = time.perf_counter()
        for j, (recs, blob, off) in enumerate(jobs):
            m = ctx.map_begin("job%d" % j)
            m.emit_batch_values(recs, blob, off)
            t0 = time.perf_counter()
            m.commit()
            commit_s += time.perf_counter() - t0
        pairs_after = ctx.checksum_input()[3]
        ctx.shuffle()
        st = ctx.stats()
        t0 = time.perf_counter()
        keys, _, _ = ctx.result_copy()
        blob, _ = ctx.result_values()
        t1 = time.perf_counter()
        res = dict(commit_ms=round(commit_s * 1e3, 1), pairs_after_commit=int(pairs_after),
                   ms_total=round(st["ms_total"], 3), ms_bigbins=round(st["ms_bigbins"], 3), attempts=st["attempts"],
                   big_bins=st["big_bins"], groups=int(keys.size), first_access_ms=round((t1 - t0) * 1e3, 3),
                   end_to_end_ms=round((t1 - t_start) * 1e3, 1))
        order = np.argsort(keys, kind="stable")
        return res, (keys[order], decode(blob.reshape(-1, 11))[order].view(np.uint64))


def profile(jobs, pairs, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    out = {}
    for arm in ("fsum", "comb_fsum"):
        run(arm, jobs[:2], pairs)  # warm-up: module load, first launches
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            run(arm, jobs, pairs)
            torch.cuda.synchronize()
        tot = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" and e.device_time_total > 0:
                tot[e.key] = tot.get(e.key, 0.0) + e.device_time_total / 1e3
        top = sorted(tot.items(), key=lambda kv: -kv[1])[:20]
        out[arm] = {"kernel_ms_total": round(sum(tot.values()), 1), "top": [(k[:80], round(v, 2)) for k, v in top]}
        if out_dir:
            prof.export_chrome_trace(os.path.join(out_dir, "bench_fsum_combiner_%s.pt.trace.json" % arm))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=100_000_000)
    ap.add_argument("--jobs", type=int, default=400)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--trace-dir", default=None)
    a = ap.parse_args()
    name, power = card()
    table = synth.zipf_table(V)
    out = {"card": name, "power_limit": power, "pairs": a.pairs, "jobs": a.jobs, "zipf_ranks": V, "partitions": P}
    with mrhbm.Ctx(mrhbm.KEY_STR, 1, device=0, reducer=mrhbm.RED_NONE) as gen:
        jobs = make_jobs(a.pairs, a.jobs, table, gen)
    if a.profile:
        out["profile"] = profile(jobs, a.pairs, a.trace_dir)
        print(json.dumps(out))
        return 0
    out["runs"], parity = [], None
    for rep in range(a.reps):
        got = {}
        for arm in ("fsum", "comb_fsum"):
            res, got[arm] = run(arm, jobs, a.pairs)
            out["runs"].append(dict(arm=arm, rep=rep, **res))
            print(json.dumps(out["runs"][-1]), file=sys.stderr, flush=True)
        if rep == 0:
            parity = all(np.array_equal(x, y) for x, y in zip(got["fsum"], got["comb_fsum"]))
    out["parity_bit_identical"] = parity
    print(json.dumps(out))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
