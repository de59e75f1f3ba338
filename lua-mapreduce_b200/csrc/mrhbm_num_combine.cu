// mrhbm_num_combine.cu -- MRHBM_COMBINE_FSUM: at the commit of a map job on a byte-values ctx, each key's numbers are
// replaced by the greedy expansion of their exact sum (acc_split / two_split, mrhbm_numsum.cuh): usually one or two
// doubles whose exact sum is the key's, so that the shuffle's exact sum over them is the sum over the raw values.
//   k_fsum_mark       every record joins a hash set on its key slot alone: entries {fingerprint, smallest pool index of
//                     the key}, claimed and lowered as k_distinct_mark does; slot_of[g] its entry, vbits[g] its value's
//                     double bits, and the entry's count grows by one (one atomic per key and warp)
//   k_fsum_alloc      each used entry gets a room of its count in vals (a bump counter: the rooms' order is free)
//   k_fsum_gather     every value's bits into its key's room
//   k_fsum_sum        a key of one or two values is split by one thread (two_split), one of up to kFsumWarpValues by a
//                     warp through lane-private shared-memory accumulators (warp_acc, then acc_split): alike values of
//                     a hot key would serialise shared 64-bit atomics; the terms overwrite the room's first values.
//                     Longer keys are listed for
//   k_fsum_big        every warp of the grid takes chunks of kFsumWarpValues values of the listed keys and adds each
//                     chunk's accumulator into its key's global one, so a hot key is spread over the whole GPU
//   k_fsum_big_split  one thread per listed key splits its accumulator
//   k_fsum_count      per tile, the new pairs of the keys whose first pair the tile holds
//   (launch_exscan of the tile counts; the host reads the total, takes room at the tail of the pool and goes on)
//   k_fsum_write      the new pairs in the order of their keys' first pairs, each key's terms in order
//   k_fsum_copy       the pairs of the keys that keep their values, in the order the host gives (pool order)
#include <cstdint>

#include "mrhbm_dev.cuh"
#include "mrhbm_job_tiles.cuh"
#include "mrhbm_numsum.cuh"
#include "mrhbm_valbytes.cuh"

namespace mrhbm {

namespace {
constexpr unsigned long long kEmpty = ~0ull;  // an entry's fingerprint and index before the claim (memset to 0xff)
constexpr int kThreads = 256;
// the kernels that add a key's values by warp: 2 warps per CTA, each with 32 lane-private accumulators of an odd
// stride (a half warp's 8-byte words in different banks), so that the adds need no atomics however alike the values
constexpr int kAccThreads = 64, kAccWarps = kAccThreads / 32, kAccStride = kAccWords + 1;

struct Words {
  uint32_t *cnt, *start, *cursor, *nterm;
  __device__ Words(const FsumScratch& fs) {
    const uint64_t T = fs.mask + 1;
    cnt = fs.words;
    start = fs.words + T;
    cursor = fs.words + 2 * T;
    nterm = fs.words + 3 * T;
  }
};

// a key's split (terms k > 0 in its room already, 0: it keeps its n values, < 0: NaN) into its term count and the flags
__device__ __forceinline__ void put_terms(const FsumScratch& fs, uint32_t* nterm, uint32_t e, int k, uint32_t n) {
  if (k > 0) {
    nterm[e] = (uint32_t)k;
  } else {
    nterm[e] = n | kFsumKeep;
    atomicOr(fs.small, k < 0 ? (uint32_t)ERRF_NAN : kFsumKeep);
  }
}

// v[i0 .. i1) summed by the warp: each lane adds its share into its own accumulator of la (32 x kAccStride words),
// then lane l sums word l, l + 32, ... over the 32 and leaves it in la[0 .. kAccWords)
__device__ __forceinline__ void warp_acc(int64_t* la, const uint64_t* v, uint32_t i0, uint32_t i1) {
  const uint32_t lane = threadIdx.x & 31;
  int64_t* my = la + lane * kAccStride;
  for (int k = 0; k < kAccWords; k++) my[k] = 0;
  for (uint32_t i = i0 + lane; i < i1; i += 32) {
    const NumTerm t = num_term(v[i]);
#pragma unroll
    for (int k = 0; k < 3; k++) my[t.i + k] += t.d[k];
    my[kAccFlags] |= (int64_t)t.flag;
  }
  __syncwarp();
  int64_t sum[3];
#pragma unroll
  for (int j = 0; j < 3; j++) {
    const int d = lane + 32 * j;
    sum[j] = 0;
    if (d < kAccWords)
      for (int l = 0; l < 32; l++) sum[j] = d == kAccFlags ? sum[j] | la[l * kAccStride + d] : sum[j] + la[l * kAccStride + d];
  }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 3; j++)
    if (lane + 32 * j < kAccWords) la[lane + 32 * j] = sum[j];
  __syncwarp();
}

// a record's value id
template <int RB>
__device__ __forceinline__ void set_value_id(uint32_t* r, uint64_t id) {
  if constexpr (Rec<RB>::kU64) {
    r[2] = (uint32_t)id;
    r[3] = (uint32_t)(id >> 32);
  } else {
    r[Rec<RB>::kKeyWords] = (uint32_t)id;
  }
}
// the record r as new pair first + i: its slot, its voff entry and its encoded value
template <int RB>
__device__ __forceinline__ void put_pair(unsigned char* pool, uint32_t* r, uint64_t first, uint64_t i, uint64_t aoff,
                                         uint64_t* voff, unsigned char* arena, uint64_t bits) {
  set_value_id<RB>(r, first + i);
  uint4* dst = (uint4*)(pool + (first + i) * RB);
#pragma unroll
  for (int v = 0; v < Rec<RB>::kVec; v++) dst[v] = make_uint4(r[4 * v], r[4 * v + 1], r[4 * v + 2], r[4 * v + 3]);
  voff[first + i] = aoff + kNumBytes * i;
  num_encode(bits, arena + aoff + kNumBytes * i);
}
}  // namespace

template <int RB>
__global__ void __launch_bounds__(kDistinctTile) k_fsum_mark(const unsigned char* __restrict__ pool,
                                                             const DistinctRange* __restrict__ rg, uint32_t nr,
                                                             const unsigned char* __restrict__ arena,
                                                             const uint64_t* __restrict__ voff, FsumScratch fs) {
  uint64_t p = 0, g = 0;
  const bool valid = tile_record(rg, nr, &p, &g);
  uint32_t slot = 0;
  if (valid) {
    uint32_t r[Rec<RB>::kWords];
    load_record<RB>(pool, p, r);
    const ValView v = val_view(arena, voff, rec_value<RB>(r));
    uint64_t bits = 0;
    if (v.len != kNumBytes || !num_decode_words(val_word(v, 0), val_word(v, 1), val_word(v, 2), &bits)) {
      atomicOr(fs.small, (uint32_t)ERRF_NOTNUM);
      bits = 0;
    }
    fs.vbits[g] = bits;
    const uint64_t fp = key_fingerprint<RB>(r);
    for (uint64_t s = fp & fs.mask;; s = (s + 1) & fs.mask) {
      unsigned long long* e = (unsigned long long*)((ulonglong2*)fs.tab + s);
      unsigned long long f = *(volatile unsigned long long*)e;
      if (f == kEmpty) {
        f = atomicCAS(e, kEmpty, (unsigned long long)fp);
        if (f == kEmpty) {
          atomicMin(e + 1, (unsigned long long)p);
          slot = (uint32_t)s;
          break;
        }
      }
      if (f != fp) continue;
      unsigned long long q;
      while ((q = *(volatile unsigned long long*)(e + 1)) == kEmpty) {
      }
      if (key_eq<RB>(r, (const uint32_t*)(pool + q * RB))) {
        if (p < q) atomicMin(e + 1, (unsigned long long)p);
        slot = (uint32_t)s;
        break;
      }
    }
    fs.slot_of[g] = slot;
  }
  const unsigned vm = __ballot_sync(0xffffffffu, valid);
  if (valid) {
    const unsigned peers = __match_any_sync(vm, slot);
    if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(Words(fs).cnt + slot, (uint32_t)__popc(peers));
  }
}

__global__ void __launch_bounds__(kThreads) k_fsum_alloc(FsumScratch fs) {
  const Words w(fs);
  const uint64_t T = fs.mask + 1;  // (a multiple of kThreads)
  const uint32_t lane = threadIdx.x & 31;
  for (uint64_t e = blockIdx.x * (uint64_t)kThreads + threadIdx.x; e < T; e += (uint64_t)gridDim.x * kThreads) {
    const uint32_t c = w.cnt[e], incl = warp_inscan(c), tot = __shfl_sync(0xffffffffu, incl, 31);
    uint32_t b = 0;
    if (lane == 31 && tot) b = atomicAdd(fs.small + 1, tot);
    b = __shfl_sync(0xffffffffu, b, 31) + incl - c;
    if (c) {
      w.start[e] = b;
      w.cursor[e] = b;
    }
  }
}

__global__ void __launch_bounds__(kThreads) k_fsum_gather(uint64_t n, FsumScratch fs) {
  const Words w(fs);
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t n_up = (n + kThreads - 1) / kThreads * kThreads;
  for (uint64_t g = blockIdx.x * (uint64_t)kThreads + threadIdx.x; g < n_up; g += (uint64_t)gridDim.x * kThreads) {
    const bool valid = g < n;
    const uint32_t s = valid ? fs.slot_of[g] : 0u;
    const unsigned vm = __ballot_sync(0xffffffffu, valid);
    if (valid) {
      const unsigned peers = __match_any_sync(vm, s);
      const int leader = __ffs(peers) - 1;
      uint32_t b = 0;
      if ((int)lane == leader) b = atomicAdd(w.cursor + s, (uint32_t)__popc(peers));
      b = __shfl_sync(peers, b, leader);
      fs.vals[b + __popc(peers & ((1u << lane) - 1))] = fs.vbits[g];
    }
  }
}

__global__ void __launch_bounds__(kAccThreads) k_fsum_sum(FsumScratch fs) {
  __shared__ int64_t s_acc[kAccWarps][32 * kAccStride];
  const Words w(fs);
  const uint64_t T = fs.mask + 1;
  const uint32_t lane = threadIdx.x & 31;
  int64_t* la = s_acc[threadIdx.x >> 5];
  for (uint64_t e = blockIdx.x * (uint64_t)kAccThreads + threadIdx.x; e < T; e += (uint64_t)gridDim.x * kAccThreads) {
    const uint32_t c = w.cnt[e];
    if (c == 1 || c == 2) {
      uint64_t* v = fs.vals + w.start[e];
      uint64_t t[2];
      const int k = two_split(v[0], c == 2 ? v[1] : 0ull, (int)c, t);
      if (k > 0) v[0] = t[0];
      if (k > 1) v[1] = t[1];
      put_terms(fs, w.nterm, (uint32_t)e, k, c);
    } else if (c > kFsumWarpValues) {
      fs.big[atomicAdd(fs.small + 2, 1u)] = (uint32_t)e;
    }
    for (unsigned todo = __ballot_sync(0xffffffffu, c > 2 && c <= kFsumWarpValues); todo; todo &= todo - 1) {
      const int l = __ffs(todo) - 1;
      const uint32_t ee = __shfl_sync(0xffffffffu, (uint32_t)e, l), cc = __shfl_sync(0xffffffffu, c, l);
      uint64_t* v = fs.vals + w.start[ee];
      warp_acc(la, v, 0, cc);
      if (lane == 0) put_terms(fs, w.nterm, ee, acc_split(la, v, (int)cc), cc);
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(kAccThreads) k_fsum_big(FsumScratch fs) {
  __shared__ int64_t s_acc[kAccWarps][32 * kAccStride];
  const Words w(fs);
  const uint32_t lane = threadIdx.x & 31, nbig = fs.small[2];
  const uint32_t W = gridDim.x * kAccWarps, gw = blockIdx.x * kAccWarps + (threadIdx.x >> 5);
  int64_t* la = s_acc[threadIdx.x >> 5];
#pragma unroll 1
  for (uint32_t k = 0; k < nbig; k++) {
    const uint32_t e = fs.big[k], c = w.cnt[e];
    const uint64_t* v = fs.vals + w.start[e];
    const uint32_t nch = (c + kFsumWarpValues - 1) / kFsumWarpValues;
#pragma unroll 1
    for (uint32_t ch = (gw + W - k % W) % W; ch < nch; ch += W) {  // key k's chunk j goes to warp (k + j) % W
      warp_acc(la, v, ch * kFsumWarpValues, min(c, (ch + 1) * kFsumWarpValues));
      unsigned long long* dst = (unsigned long long*)(fs.gacc + (uint64_t)k * kAccWords);
      for (int d = lane; d < kAccDigits; d += 32)
        if (la[d]) atomicAdd(dst + d, (unsigned long long)la[d]);
      if (lane == 0 && la[kAccFlags]) atomicOr(dst + kAccFlags, (unsigned long long)la[kAccFlags]);
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(kThreads) k_fsum_big_split(FsumScratch fs) {
  const Words w(fs);
  const uint32_t k = blockIdx.x * kThreads + threadIdx.x;
  if (k >= fs.small[2]) return;
  const uint32_t e = fs.big[k], c = w.cnt[e];
  put_terms(fs, w.nterm, e, acc_split(fs.gacc + (uint64_t)k * kAccWords, fs.vals + w.start[e], (int)c), c);
}

// the term count (kFsumKeep: the value count, flagged) of the key whose first pair is this thread's record, else 0
__device__ __forceinline__ uint32_t first_pair_terms(const DistinctRange* __restrict__ rg, uint32_t nr,
                                                     const FsumScratch& fs, uint32_t* slot, uint64_t* p) {
  uint64_t g;
  if (!tile_record(rg, nr, p, &g)) return 0;
  *slot = fs.slot_of[g];
  return ((const ulonglong2*)fs.tab)[*slot].y == *p ? Words(fs).nterm[*slot] : 0u;
}

__global__ void __launch_bounds__(kDistinctTile) k_fsum_count(const DistinctRange* __restrict__ rg, uint32_t nr,
                                                              FsumScratch fs, uint32_t* __restrict__ tile_cnt) {
  uint32_t slot = 0;
  uint64_t p = 0;
  const uint32_t t = first_pair_terms(rg, nr, fs, &slot, &p) & ~kFsumKeep;
  const uint32_t total = cta_exscan<kDistinctTile>(t).total;
  if (threadIdx.x == 0) tile_cnt[blockIdx.x] = total;
}

template <int RB>
__global__ void __launch_bounds__(kDistinctTile) k_fsum_write(unsigned char* pool, const DistinctRange* __restrict__ rg,
                                                              uint32_t nr, uint32_t ntiles, FsumScratch fs,
                                                              const uint32_t* __restrict__ tile_off, uint64_t first,
                                                              uint64_t aoff, uint64_t* voff, unsigned char* arena) {
  uint32_t slot = 0;
  uint64_t p = 0;
  const uint32_t t = first_pair_terms(rg, nr, fs, &slot, &p), n = t & ~kFsumKeep;
  const uint64_t o = tile_off[blockIdx.x] + cta_exscan<kDistinctTile>(n).excl;
  if (blockIdx.x == 0 && threadIdx.x == 0) voff[first + tile_off[ntiles]] = aoff + kNumBytes * (uint64_t)tile_off[ntiles];
  if (!n) return;
  const Words w(fs);
  if (t & kFsumKeep) {
    w.cursor[slot] = (uint32_t)o;
    return;
  }
  uint32_t r[Rec<RB>::kWords];
  load_record<RB>(pool, p, r);
  const uint64_t* v = fs.vals + w.start[slot];
  for (uint32_t i = 0; i < n; i++) put_pair<RB>(pool, r, first, o + i, aoff, voff, arena, v[i]);
}

template <int RB>
__global__ void __launch_bounds__(kThreads) k_fsum_copy(unsigned char* pool, const uint64_t* __restrict__ cp, uint64_t m,
                                                        FsumScratch fs, uint64_t first, uint64_t aoff, uint64_t* voff,
                                                        unsigned char* arena) {
  for (uint64_t i = blockIdx.x * (uint64_t)kThreads + threadIdx.x; i < m; i += (uint64_t)gridDim.x * kThreads) {
    uint32_t r[Rec<RB>::kWords];
    load_record<RB>(pool, cp[3 * i + 1], r);
    put_pair<RB>(pool, r, first, cp[3 * i], aoff, voff, arena, fs.vbits[cp[3 * i + 2]]);
  }
}

#define DISPATCH_RB(rb, CALL) \
  switch (rb) {               \
    case 16: {                \
      constexpr int RB = 16;  \
      CALL;                   \
    } break;                  \
    case 32: {                \
      constexpr int RB = 32;  \
      CALL;                   \
    } break;                  \
    case 64: {                \
      constexpr int RB = 64;  \
      CALL;                   \
    } break;                  \
    default: {                \
      constexpr int RB = 128; \
      CALL;                   \
    } break;                  \
  }

int launch_fsum_split(int rb, const void* pool, const DistinctRange* rg, uint32_t nr, uint32_t ntiles, uint64_t n,
                      const unsigned char* arena, const uint64_t* voff, const FsumScratch& fs, uint32_t* tile_cnt,
                      int sm_count, cudaStream_t s) {
  if (!ntiles) return 0;
  const unsigned char* P = (const unsigned char*)pool;
  const uint64_t T = fs.mask + 1;
  const unsigned grid_t = (unsigned)(T / kThreads < (uint64_t)sm_count * 8 ? T / kThreads : (uint64_t)sm_count * 8);
  const unsigned grid_a = (unsigned)(T / kAccThreads < (uint64_t)sm_count * 6 ? T / kAccThreads : (uint64_t)sm_count * 6);
  const uint64_t nb = (n + kThreads - 1) / kThreads;
  const unsigned grid_n = (unsigned)(nb < (uint64_t)sm_count * 8 ? nb : (uint64_t)sm_count * 8);
  const uint64_t maxbig = n / kFsumWarpValues + 1;
  DISPATCH_RB(rb, (k_fsum_mark<RB><<<ntiles, kDistinctTile, 0, s>>>(P, rg, nr, arena, voff, fs)));
  k_fsum_alloc<<<grid_t, kThreads, 0, s>>>(fs);
  k_fsum_gather<<<grid_n, kThreads, 0, s>>>(n, fs);
  k_fsum_sum<<<grid_a, kAccThreads, 0, s>>>(fs);
  k_fsum_big<<<(unsigned)sm_count * 6, kAccThreads, 0, s>>>(fs);
  k_fsum_big_split<<<(unsigned)((maxbig + kThreads - 1) / kThreads), kThreads, 0, s>>>(fs);
  k_fsum_count<<<ntiles, kDistinctTile, 0, s>>>(rg, nr, fs, tile_cnt);
  return 7;
}

int launch_fsum_write(int rb, void* pool, const DistinctRange* rg, uint32_t nr, uint32_t ntiles, const FsumScratch& fs,
                      const uint32_t* tile_off, uint64_t first, uint64_t aoff, uint64_t* voff, unsigned char* arena,
                      cudaStream_t s) {
  if (!ntiles) return 0;
  unsigned char* P = (unsigned char*)pool;
  DISPATCH_RB(rb, (k_fsum_write<RB><<<ntiles, kDistinctTile, 0, s>>>(P, rg, nr, ntiles, fs, tile_off, first, aoff, voff, arena)));
  return 1;
}

int launch_fsum_copy(int rb, void* pool, const uint64_t* cp, uint64_t m, const FsumScratch& fs, uint64_t first,
                     uint64_t aoff, uint64_t* voff, unsigned char* arena, cudaStream_t s) {
  if (!m) return 0;
  unsigned char* P = (unsigned char*)pool;
  const uint64_t nb = (m + kThreads - 1) / kThreads;
  const unsigned grid = (unsigned)(nb < 4096 ? nb : 4096);
  DISPATCH_RB(rb, (k_fsum_copy<RB><<<grid, kThreads, 0, s>>>(P, cp, m, fs, first, aoff, voff, arena)));
  return 1;
}

}  // namespace mrhbm
