// mrhbm_job_tiles.cuh -- one map job's records as the commit-time kernels see them: the job's open ranges cut into
// tiles of kDistinctTile records (DistinctRange, mrhbm_kernels.h), one CTA per tile, one thread per record.  Shared by
// MRHBM_COMBINE_DISTINCT (mrhbm_distinct.cu) and MRHBM_COMBINE_FSUM (mrhbm_num_combine.cu).
#pragma once
#include <cstdint>

#include "mrhbm_dev.cuh"
#include "mrhbm_valbytes.cuh"

namespace mrhbm {

// tile t lies in the range k with rg[k].tbase <= t < rg[k + 1].tbase (no range is empty)
__device__ __forceinline__ uint32_t range_of_tile(const DistinctRange* __restrict__ rg, uint32_t nr, uint32_t t) {
  uint32_t lo = 0, hi = nr;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (rg[mid].tbase <= t) lo = mid;
    else hi = mid;
  }
  return lo;
}

// this thread's record of tile blockIdx.x: its pool index p and its index g among the job's records; false past the
// end of the range
__device__ __forceinline__ bool tile_record(const DistinctRange* __restrict__ rg, uint32_t nr, uint64_t* p, uint64_t* g) {
  const uint32_t t = blockIdx.x, k = range_of_tile(rg, nr, t);
  const uint64_t j = (uint64_t)(t - rg[k].tbase) * kDistinctTile + threadIdx.x;
  if (j >= rg[k + 1].vbase - rg[k].vbase) return false;
  *p = rg[k].off + j;
  *g = rg[k].vbase + j;
  return true;
}

// (host-callable, so that tests/native/fsum_fingerprint_check.cu can check the tests' model of the hash set)
__host__ __device__ __forceinline__ uint64_t fp_step(uint64_t h, uint64_t x) {
  h = (h ^ x) * 0x9E3779B97F4A7C15ull;
  return h ^ (h >> 29);
}

// MRHBM_COMBINE_FSUM's 64-bit fingerprint of the key slot words (never ~0, the empty entry)
template <int RB>
__host__ __device__ __forceinline__ uint64_t key_fingerprint(const uint32_t* r) {
  uint64_t h = 0x5851F42D4C957F2Dull;
#pragma unroll
  for (int i = 0; i < Rec<RB>::kKeyWords; i += 2)
    h = fp_step(h, (uint64_t)r[i] | (i + 1 < Rec<RB>::kKeyWords ? (uint64_t)r[i + 1] << 32 : 0ull));
  h = mix64(h);
  return h == ~0ull ? 0 : h;
}

// MRHBM_COMBINE_DISTINCT's (and the distinct reducer's) 64-bit fingerprint of the key slot words and the value bytes
// (never ~0, the empty entry); host-callable for tests/native/distinct_fingerprint_check.cu
template <int RB>
__host__ __device__ __forceinline__ uint64_t pair_fingerprint(const uint32_t* r, const ValView& v) {
  uint64_t h = fp_step(0x5851F42D4C957F2Dull, v.len);
#pragma unroll
  for (int i = 0; i < Rec<RB>::kKeyWords; i += 2)
    h = fp_step(h, (uint64_t)r[i] | (i + 1 < Rec<RB>::kKeyWords ? (uint64_t)r[i + 1] << 32 : 0ull));
  const uint64_t nw = (v.len + 3) / 4;
  for (uint64_t i = 0; i < nw; i += 2)
    h = fp_step(h, (uint64_t)val_word(v, i) | (i + 1 < nw ? (uint64_t)val_word(v, i + 1) << 32 : 0ull));
  h = mix64(h);
  return h == ~0ull ? 0 : h;
}

template <int RB>
__device__ __forceinline__ void load_record(const unsigned char* __restrict__ pool, uint64_t p, uint32_t* r) {
  const uint4* src = (const uint4*)(pool + p * RB);
#pragma unroll
  for (int i = 0; i < Rec<RB>::kVec; i++) {
    const uint4 x = __ldg(src + i);
    r[4 * i] = x.x;
    r[4 * i + 1] = x.y;
    r[4 * i + 2] = x.z;
    r[4 * i + 3] = x.w;
  }
}

}  // namespace mrhbm
