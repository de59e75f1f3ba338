// mrhbm_split_plan.h -- the geometry of the two-level split (k_split_tma) as plain host functions (no CUDA runtime
// calls, no ctx): the plan both layouts split by, and the level-2 CTAs per coarse region.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>

#include "mrhbm_kernels.h"  // SplitPlan, kSplitMaxBins, kSplitTileBytes

namespace mrhbm {

// The geometry of the split (k_split_tma) into the fine bins of ndest destination ranks, Bl[d] of them on rank d, as
// seen by rank me: B, F, C1, C1_local, cap, rbase, fbase, ndest, me, sub_stride.  Returns the number of levels, or 0
// when the split does not take these bins.
//   optimistic layout: one level on one GPU with at most kSplitMaxBins bins (level 1 writes the fine bins, regions
//     of `cap` slots); else F = the smallest power of two >= sqrt(B) (both levels see about the same fan-out), doubled
//     until the regions of all ranks fit one level, and a region gets mean + 8 sigma + 64 slots for one rank's share
//     (at most nmax records, hash balanced over the B bins).
//   exact layout (one destination, also on several GPUs: the destination-major send buffer): two levels from 2048
//     bins on; the regions are sized by their bins' capacity, F * cap.
// (With one destination ceil(B / F) <= F, so the doubling never runs and F > kSplitMaxBins alone ends the search.)
inline int plan_split(SplitPlan& pl, const uint64_t* Bl, uint32_t ndest, uint32_t me, uint32_t cap, uint64_t nmax, bool exact) {
  uint64_t B = 0;
  for (uint32_t d = 0; d < ndest; d++) B += Bl[d];
  const int levels = !exact && ndest == 1 && B <= kSplitMaxBins ? 1 : 2;
  if (exact && B < 2048) return 0;
  uint32_t F = 1;
  if (levels == 2) {
    while ((uint64_t)F * F < B) F <<= 1;
    for (; F <= kSplitMaxBins; F <<= 1) {
      uint64_t c1 = 0;
      for (uint32_t d = 0; d < ndest; d++) c1 += (Bl[d] + F - 1) / F;
      if (c1 <= kSplitMaxBins) break;
    }
    if (F > kSplitMaxBins) return 0;  // more bins than two levels reach
  }
  pl.rbase[0] = pl.fbase[0] = 0;
  for (uint32_t d = 0; d < 8; d++) {
    const uint64_t bl = d < ndest ? Bl[d] : 0;
    pl.rbase[d + 1] = pl.rbase[d] + (uint32_t)((bl + F - 1) / F);
    pl.fbase[d + 1] = pl.fbase[d] + (uint32_t)bl;
  }
  pl.B = (uint32_t)B;
  pl.F = F;
  pl.C1 = pl.rbase[ndest];
  pl.C1_local = pl.rbase[me + 1] - pl.rbase[me];
  pl.cap = cap;
  pl.ndest = ndest;
  pl.me = me;
  double ss = (double)F * cap;
  if (!exact && levels == 2) {  // one rank's contribution to one region: F of the B bins, hash balanced
    const double mean = (double)nmax * (double)F / (double)B;
    ss = mean + 8.0 * std::sqrt(mean) + 64.0;
  }
  if (ss >= 4.0e9) return 0;
  pl.sub_stride = ((uint64_t)ss + 7u) & ~7ull;
  return levels;
}

// Level 2 runs x CTAs per coarse region (each takes every x-th tile of all the region's streams), x <= 16 and at most
// a quarter of a region's tiles, chosen so that all CTAs fill whole waves of `ctas` resident CTAs (e.g. 220 regions,
// x = 2 on 264 slots would run 440 CTAs = 1.67 waves: a third of the second wave idle).  `regions`: the regions this
// rank splits (C1_local), `rb`: record bytes.
inline int split_l2_ctas_per_region(uint32_t regions, uint64_t sub_stride, uint32_t ndest, int rb, int ctas) {
  int x = 1;
  double best = 0;
  const uint64_t tiles = ndest * ((sub_stride * rb + kSplitTileBytes - 1) / kSplitTileBytes);
  for (int cand = 1; cand <= 16 && (uint64_t)cand <= std::max<uint64_t>(1, tiles / 4); cand++) {
    uint64_t total = (uint64_t)cand * regions, waves = (total + ctas - 1) / ctas;
    double eff = (double)total / (double)(waves * ctas);
    if (eff > best + 0.02) {
      best = eff;
      x = cand;
    }
  }
  return x;
}

}  // namespace mrhbm
