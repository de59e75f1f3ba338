"""The split plan (csrc/mrhbm_split_plan.h) on the CPU: every field of plan_split and the level-2 CTAs per region,
against a pure-Python restatement of the planner, over bin counts at the edges between one level and two, the exact
layout's edges, every record class's bin capacity, several destinations with unequal bins, and region sizes near the
8-slot rounding and the 4e9 refusal.  tests/test_gpu_split_paths.py builds its inputs with this model; the driver
tests/native/split_plan_check.cu is host-compiled from the same header."""
import math
import os
import random
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_BINS = 1024  # kSplitMaxBins: bins one level distinguishes
TILE_BYTES = 40 * 1024  # kSplitTileBytes
RBS = (16, 32, 64, 128)
CAPS = tuple(32 * 1024 // rb for rb in RBS) + (96,)  # every record class's bin capacity, and F_SMALL_BINS'


# ---- the model ---------------------------------------------------------------------------------------------------------

def plan_split(Bl, me, cap, nmax, exact):
    """plan_split for the bins Bl[d] of every destination d as seen by rank me: None when the split does not take
    them, else a dict of levels, F, C1, C1_local, rbase[9], fbase[9], sub_stride"""
    ndest, B = len(Bl), sum(Bl)
    levels = 1 if not exact and ndest == 1 and B <= MAX_BINS else 2
    if exact and B < 2048:
        return None
    F = 1
    if levels == 2:
        while F * F < B:
            F <<= 1
        while F <= MAX_BINS and sum(-(-b // F) for b in Bl) > MAX_BINS:
            F <<= 1
        if F > MAX_BINS:
            return None
    rbase, fbase = [0], [0]
    for d in range(8):
        bl = Bl[d] if d < ndest else 0
        rbase.append(rbase[-1] + -(-bl // F))
        fbase.append(fbase[-1] + bl)
    ss = float(F) * float(cap)
    if not exact and levels == 2:  # the same double arithmetic as the C++
        mean = float(nmax) * float(F) / float(B)
        ss = mean + 8.0 * math.sqrt(mean) + 64.0
    if ss >= 4.0e9:
        return None
    return dict(levels=levels, F=F, C1=rbase[ndest], C1_local=rbase[me + 1] - rbase[me], rbase=rbase, fbase=fbase,
                sub_stride=(int(ss) + 7) & ~7)


def l2_ctas(regions, sub_stride, ndest, rb, ctas):
    """level-2 CTAs per region: the first x in 1 .. min(16, max(1, tiles / 4)) whose waves of `ctas` resident CTAs
    are fuller by more than 0.02 than every smaller x's"""
    tiles = ndest * -(-(sub_stride * rb) // TILE_BYTES)
    x, best = 1, 0.0
    for cand in range(1, min(16, max(1, tiles // 4)) + 1):
        total = cand * regions
        eff = total / (-(-total // ctas) * ctas)
        if eff > best + 0.02:
            best, x = eff, cand
    return x


# ---- the driver ----------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path_factory.mktemp("split_plan") / "split_plan_check")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "lua-mapreduce_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "split_plan_check.cu")])

    def run(cmds):
        text = "".join(" ".join(map(str, c)) + "\n" for c in cmds)
        out = subprocess.run([exe], input=text, capture_output=True, text=True, timeout=300, check=True)
        lines = out.stdout.splitlines()
        assert len(lines) == len(cmds)
        return [[int(x) for x in ln.split()] for ln in lines]
    return run


def check_plans(driver, cases):
    """cases: (Bl, me, cap, nmax, exact); every field the driver prints against the model"""
    outs = driver([("P", int(ex), cap, nmax, len(Bl), me, *Bl) for Bl, me, cap, nmax, ex in cases])
    for (Bl, me, cap, nmax, ex), out in zip(cases, outs):
        want = plan_split(Bl, me, cap, nmax, ex)
        if want is None:
            assert out == [0], (Bl, me, cap, nmax, ex, out)
            continue
        got = dict(levels=out[0], F=out[1], C1=out[2], C1_local=out[3], sub_stride=out[4], rbase=out[5:14],
                   fbase=out[14:23])
        assert got == want, (Bl, me, cap, nmax, ex)
    return [plan_split(*c) for c in cases]


def test_one_destination_every_bin_count_to_1025(driver):
    cases = [([B], 0, cap, nmax, False) for B in range(1, 1026) for cap in (2048, 96)
             for nmax in (B * 1776, 7 * B + 3)]
    cases += [([B], 0, cap, 0, True) for B in range(1, 1026, 41) for cap in (2048, 1024)]
    plans = check_plans(driver, cases)
    for (Bl, _, _, _, ex), p in zip(cases, plans):
        if ex:
            assert p is None  # the exact layout scatters below 2048 bins
        else:
            assert p["levels"] == (1 if Bl[0] <= 1024 else 2)
    # 1025 bins: F = 64, C1 = 17, the last region holds one bin
    p = plan_split([1025], 0, 2048, 1025 * 1776, False)
    assert (p["levels"], p["F"], p["C1"], 1025 - (p["C1"] - 1) * p["F"]) == (2, 64, 17, 1)


def test_one_destination_near_2048_and_2_pow_20(driver):
    Bs = [1026, 1100, 1148, 2046, 2047, 2048, 2049, 3000, 4096, 4097, 65536, 65537,
          (1 << 20) - 1, 1 << 20, (1 << 20) + 1, (1 << 21)]
    cases = [([B], 0, cap, nmax, ex) for B in Bs for cap in CAPS for ex in (False, True)
             for nmax in (0, B * 37, B * (cap - 6 * int(math.sqrt(cap))))]
    plans = check_plans(driver, cases)
    for (Bl, _, cap, _, ex), p in zip(cases, plans):
        B = Bl[0]
        if B > 1 << 20 or (ex and B < 2048):
            assert p is None
        else:
            assert p["levels"] == 2 and p["F"] * p["F"] >= B > (p["F"] // 2) ** 2
            if ex:
                assert p["sub_stride"] == p["F"] * cap
    p = plan_split([1 << 20], 0, 96, 0, True)
    assert (p["F"], p["C1"]) == (1024, 1024)  # the largest plan two levels reach


def test_several_destinations(driver):
    rng = random.Random(5)
    cases = []
    for ndest in range(1, 9):
        for _ in range(12):
            Bl = [rng.choice([0, 1, 3, 64, 65, 1000, 1024, 1025, 4096, 40000, 131072, rng.randrange(0, 200000)])
                  for _ in range(ndest)]
            if not sum(Bl):
                Bl[0] = 1
            for me in range(ndest):
                for cap in (2048, 1024, 96):
                    cases.append((Bl, me, cap, rng.choice([1, 1000, 10 ** 6, 10 ** 8]), False))
                    cases.append((Bl, me, cap, 0, True))
    # the doubling of F: at F = 1024 the partial last regions of the ranks can need more than 1024 regions although
    # B <= 2^20 (F = 2048: refused); one region short of that, and more than 2^20 bins
    cases += [([1] * 7 + [1017 * 1024 + 1], me, 2048, 10 ** 7, False) for me in range(8)]
    cases += [([1] * 7 + [1017 * 1024], me, 2048, 10 ** 7, False) for me in range(8)]
    cases += [([1, 1, 1, 1 << 20], me, 2048, 10 ** 7, False) for me in range(4)]
    cases += [([1023] * 8, me, 2048, 10 ** 7, False) for me in range(8)]
    cases += [([0, 5000, 0, 70000, 3, 0, 1, 262144], me, 512, 10 ** 6, False) for me in range(8)]
    plans = check_plans(driver, cases)
    refused_by_regions = 0
    for (Bl, me, _, _, ex), p in zip(cases, plans):
        if p is None:
            refused_by_regions += sum(Bl) <= 1 << 20
            continue
        F = p["F"]
        assert sum(-(-b // F) for b in Bl) == p["C1"] <= MAX_BINS
        assert p["C1_local"] == -(-Bl[me] // F)
        assert p["fbase"][len(Bl)] == sum(Bl) and p["rbase"][8] == p["C1"]
    assert refused_by_regions >= 8
    p = plan_split([1] * 7 + [1017 * 1024], 7, 2048, 10 ** 7, False)
    assert (p["F"], p["C1"], p["C1_local"]) == (1024, 1024, 1017)


def test_sub_stride_rounding_and_refusal(driver):
    cases = []
    for B, cap in ((1025, 2048), (1148, 1024), (3000, 512), (1 << 20, 96)):
        F = plan_split([B], 0, cap, 1, False)["F"]
        raw = lambda n: (lambda m: m + 8.0 * math.sqrt(m) + 64.0)(float(n) * F / B)
        # nmax where int(ss) is a multiple of 8, one more, and one less
        hits = {}
        for n in range(B * 1000, B * 1000 + 4000 * B // F):
            hits.setdefault(int(raw(n)) % 8, n)
        for r in (0, 1, 7):
            cases.append(([B], 0, cap, hits[r], False))
        # the largest nmax below the refusal, and the smallest at it
        lo, hi = 1, 1 << 62
        while hi - lo > 1:
            mid = (lo + hi) // 2
            lo, hi = (mid, hi) if raw(mid) < 4.0e9 else (lo, mid)
        cases += [([B], 0, cap, lo, False), ([B], 0, cap, hi, False)]
    plans = check_plans(driver, cases)
    assert sum(p is None for p in plans) == 4
    assert all(p["sub_stride"] % 8 == 0 for p in plans if p)


def test_level2_ctas_per_region(driver):
    rng = random.Random(7)
    cases = []
    for ctas in (264, 232, 2):
        for rb in RBS:
            for regions in (1, 2, 17, 18, 47, 131, 132, 133, 220, 264, 265, 1024):
                for ss in (8, 640, 2560, 10240, 64504, 116424, 131072, 2097152):
                    cases.append((regions, ss, rng.choice([1, 1, 2, 8]), rb, ctas))
    outs = driver([("X",) + c for c in cases])
    xs = [l2_ctas(*c) for c in cases]
    assert [o[0] for o in outs] == xs
    assert set(xs) & {1} and max(xs) > 2
