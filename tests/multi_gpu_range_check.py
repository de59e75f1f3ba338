"""Launched by torchrun (one rank per GPU) from tests/test_gpu_multi_range.py: the range partitioner across ranks.
Given and sampled splitters, u64 and string keys; every rank's partitions (p % world == rank) are checked against the
oracle's flat group-by re-partitioned with bisect_right, sampled splitters must agree on every rank, and splitters
that differ between ranks must fail the shuffle on every rank with MRHBM_E_INVAL."""
import bisect
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import mrhbm_loader  # noqa: E402

mrhbm_loader.load()
from lua_mapreduce_b200 import mrhbm, parallel, synth  # noqa: E402

import oracle as O  # noqa: E402


def check(name, cond):
    if not cond:
        raise AssertionError("rank %d: %s" % (dist.get_rank(), name))


def all_same(x):
    box = [None] * dist.get_world_size()
    dist.all_gather_object(box, x)
    return all(b == box[0] for b in box)


def run_u64(rank, world, n_per, P, sample, flags=0):
    dev = int(os.environ["LOCAL_RANK"])
    with mrhbm.Ctx(mrhbm.KEY_U64, P, mrhbm.PART_RANGE, device=dev, flags=flags) as ctx:
        parallel.init_comm(ctx, dist)
        m = ctx.map_begin("r%d" % rank)
        m.gen_u64(synth.SEED, rank * n_per, n_per)
        m.commit()
        if sample:
            spl = ctx.sample_splitters()
            check("sampled splitters agree across ranks", all_same(spl))
        else:
            spl = [(i << 64) // P for i in range(1, P)]
            ctx.set_splitters(spl)
        ctx.shuffle()
        gk, gs, gpo = ctx.result_copy()
        cin, cout = ctx.checksum_input(), ctx.checksum_result()
        check("partition membership", cout[5] == 0)
        ok, osum, _ = O.groupby_u64_stream(synth.SEED, 0, n_per * world, O.PART_MULHASH, 1)
        pid = np.searchsorted(np.asarray(spl, dtype=np.uint64), ok, side="right")
        po = np.zeros(P + 1, dtype=np.int64)
        po[1:] = np.cumsum(np.bincount(pid, minlength=P))
        sorted_ = ctx.result_info().sorted
        for p in range(P):
            a, b = int(gpo[p]), int(gpo[p + 1])
            if p % world != rank:
                check("foreign partition empty", a == b)
                continue
            k, s = gk[a:b], gs[a:b]
            if not sorted_:
                o = np.argsort(k, kind="stable")
                k, s = k[o], s[o]
            check("partition %d" % p, (k == ok[po[p]:po[p + 1]]).all() and (s == osum[po[p]:po[p + 1]]).all())
        box = [None] * world
        dist.all_gather_object(box, (cin[:3], cout[:3]))
        tin = [sum(b[0][i] for b in box) % 2**64 for i in range(3)]
        tout = [sum(b[1][i] for b in box) % 2**64 for i in range(3)]
        check("sum linearity across ranks", tin == tout)


def run_str(rank, world, P, sample):
    dev = int(os.environ["LOCAL_RANK"])
    rng = np.random.default_rng(11 + rank)
    alphabet = list(b"abcdefgmnopqz\x00\x01")
    words = [bytes(rng.choice(alphabet, int(rng.integers(1, 40))).astype(np.uint8)) for _ in range(20_000)]
    with mrhbm.Ctx(mrhbm.KEY_STR, P, mrhbm.PART_RANGE, device=dev) as ctx:
        parallel.init_comm(ctx, dist)
        m = ctx.map_begin("r%d" % rank)
        for w in words:
            m.emit(w, 1)
        m.commit()
        if sample:
            spl = ctx.sample_splitters()
            check("sampled splitters agree across ranks", all_same(spl))
        else:
            spl = sorted([b"b", b"d\x00", b"g" * 30, b"m", b"o\x01", b"q"] + [b"z"] * (P - 7))
            ctx.set_splitters(spl)
        ctx.shuffle()
        got = {p: list(ctx.groups(p)) for p in ctx.partitions()}
        everyone = [None] * world
        dist.all_gather_object(everyone, words)
        _, counts = O.naive_wordcount([b" ".join(w for ws in everyone for w in ws)])
        for p in range(rank, P, world):
            want = [(k, [c]) for k, c in counts if bisect.bisect_right(spl, k) == p]
            check("string partition %d" % p, got.get(p, []) == want)
        check("only owned partitions", all(p % world == rank for p in got))


def run_mismatch(rank, world):
    dev = int(os.environ["LOCAL_RANK"])
    with mrhbm.Ctx(mrhbm.KEY_U64, 4, mrhbm.PART_RANGE, device=dev) as ctx:
        parallel.init_comm(ctx, dist)
        m = ctx.map_begin("r%d" % rank)
        m.gen_u64(synth.SEED, rank * 50_000, 50_000)
        m.commit()
        ctx.set_splitters([1 << 62, 1 << 63, (3 << 62) + (rank == world - 1)])  # the last rank differs
        try:
            ctx.shuffle()
            failed = None
        except mrhbm.MrhbmError as e:
            failed = e.code
        check("differing splitters fail on every rank", failed == -1)
        # the ctx still works once the splitters agree
        ctx.set_splitters([1 << 62, 1 << 63, 3 << 62])
        ctx.shuffle()
        check("usable after the mismatch", ctx.checksum_result()[5] == 0)


def main():
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    import datetime
    dist.init_process_group("nccl", device_id=torch.device("cuda", local), timeout=datetime.timedelta(seconds=120))
    rank, world = dist.get_rank(), dist.get_world_size()
    run_u64(rank, world, 1_000_000, 1024, sample=False)
    run_u64(rank, world, 2_000_000, 16, sample=True)
    run_u64(rank, world, 500_000, 16, sample=True, flags=mrhbm.F_NO_OPTIMISTIC)
    run_str(rank, world, 12, sample=False)
    run_str(rank, world, 12, sample=True)
    run_mismatch(rank, world)
    dist.barrier()
    if rank == 0:
        print("MULTI_GPU_RANGE_CHECK_OK world=%d" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
