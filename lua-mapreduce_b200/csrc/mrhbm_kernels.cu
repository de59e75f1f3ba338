// mrhbm_kernels.cu -- hand-written sm_90a kernels of the in-HBM shuffle:
//   k_hist / k_exscan / k_scatter : hash-partition into (partition, sub-bin) bins
//                                   (replaces partitionfn + per-partition spill files,
//                                    mapreduce/job.lua:203-221)
//   k_sort_reduce / k_big_bins    : per-bin shared-memory sort by key + segmented sum
//                                   (replaces keys_sorted + heap merge + reducer loop,
//                                    mapreduce/utils.lua:123-128,206-271, job.lua:264-284)
//   k_compact, k_checksum_*       : result gathering and parity properties
//   k_gen_*                       : synthetic device-side mapfn (SURVEY App. B)
// HBM-bound integer work: no tensor cores.  Grids are multiples of the SM count.
#include "mrhbm_kernels.h"

#include <algorithm>
#include <type_traits>

#include "mrhbm_decimal.cuh"
#include "mrhbm_dev.cuh"
#include "mrhbm_sort.cuh"
#include "mrhbm_split_plan.h"

namespace mrhbm {

static int g_sm_count = 132;

// ============================================================================
// synthetic device-side mapfn
// ============================================================================
__global__ void k_gen_u64(uint4* dst, uint64_t seed, uint64_t start, uint64_t n) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    uint64_t k = splitmix64(seed + start + i);
    uint32_t v = (uint32_t)(splitmix64(seed + (1ull << 40) + start + i) >> 32);
    stg_stream(dst + i, make_uint4((uint32_t)k, (uint32_t)(k >> 32), v, 0u));
  }
}

__device__ __forceinline__ int rank_to_key_dev(uint64_t rank, unsigned char* out /*28, zeroed*/) {
  unsigned char tmp[16];
  int n = 0;
  uint64_t r = rank;
  while (r > 0) {
    r -= 1;
    tmp[n++] = (unsigned char)('a' + (r % 26));
    r /= 26;
  }
  int o = 0;
  while (n > 0) out[o++] = tmp[--n];
  uint64_t h = splitmix64(rank ^ 0xA5A5A5A5A5A5A5A5ull);
  unsigned l = (unsigned)(h % 8);
  if (((h >> 8) % 64) == 0) l = 8 + (unsigned)((h >> 16) % 15);
  for (unsigned j = 0; j < l; j++) out[o++] = (unsigned char)('A' + (splitmix64(h + j) % 26));
  return o;
}

__global__ void k_gen_zipf32(uint4* dst, uint64_t seed, uint64_t start, uint64_t n,
                             const uint64_t* __restrict__ table, uint64_t V) {
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    uint64_t u = splitmix64(seed + (1ull << 41) + start + i);
    uint64_t lo = 0, hi = V;
    while (lo < hi) {
      uint64_t mid = (lo + hi) >> 1;
      if (__ldg(table + mid) < u)
        lo = mid + 1;
      else
        hi = mid;
    }
    uint64_t rank = lo + 1 > V ? V : lo + 1;
    union {
      unsigned char b[32];
      uint4 v[2];
    } rec;
    rec.v[0] = make_uint4(0, 0, 0, 0);
    rec.v[1] = make_uint4(0, 0, 0, 0);
    rank_to_key_dev(rank, rec.b);
    rec.v[1].w = 1u;  // value
    stg_stream(dst + 2 * i, rec.v[0]);
    stg_stream(dst + 2 * i + 1, rec.v[1]);
  }
}

// ============================================================================
// device-side WordCount mapfn: text -> (word, 1) records
// ============================================================================
// Lua's %s in the C locale == isspace: ' ', \t \n \v \f \r (examples/WordCount/mapfn.lua:5)
__device__ __forceinline__ bool tok_space(unsigned char c) { return c == ' ' || (c >= 9 && c <= 13); }
__device__ __forceinline__ bool tok_start(const unsigned char* t, uint64_t i) {
  return !tok_space(t[i]) && (i == 0 || tok_space(t[i - 1]));
}
// one thread per byte, one count per 256-byte block
__global__ void __launch_bounds__(256) k_tok_count(const unsigned char* __restrict__ t, uint64_t len,
                                                   uint32_t* __restrict__ block_counts) {
  uint64_t nb = (len + 255) / 256;
  for (uint64_t blk = blockIdx.x; blk < nb; blk += gridDim.x) {
    uint64_t i = blk * 256 + threadIdx.x;
    int st = i < len && tok_start(t, i);
    int c = __syncthreads_count(st);
    if (threadIdx.x == 0) block_counts[blk] = (uint32_t)c;
  }
}
template <int RB>
__global__ void __launch_bounds__(256) k_tok_emit(const unsigned char* __restrict__ t, uint64_t len,
                                                  const uint32_t* __restrict__ block_off, uint4* __restrict__ recs,
                                                  uint32_t value, uint32_t* __restrict__ flags) {
  constexpr int KB = Rec<RB>::kKeyBytes;
  __shared__ uint32_t wcount[8];
  uint64_t nb = (len + 255) / 256;
  for (uint64_t blk = blockIdx.x; blk < nb; blk += gridDim.x) {
    uint64_t i = blk * 256 + threadIdx.x;
    bool st = i < len && tok_start(t, i);
    // rank of this word start inside the block: ballot prefix within the warp + warp totals
    uint32_t m = __ballot_sync(0xffffffffu, st);
    uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) wcount[warp] = __popc(m);
    __syncthreads();
    uint32_t before = __popc(m & ((1u << lane) - 1u));
    for (uint32_t w = 0; w < warp; w++) before += wcount[w];
    __syncthreads();
    if (!st) continue;
    union {
      unsigned char b[RB];
      uint4 v[RB / 16];
    } rec;
#pragma unroll
    for (int v = 0; v < RB / 16; v++) rec.v[v] = make_uint4(0, 0, 0, 0);
    int l = 0;  // bytes written to the key slot
    uint64_t p = i;
    while (p < len && !tok_space(t[p]) && l < KB) {
      const unsigned char ch = t[p++];
      if (ch <= 1) {  // 0x00 / 0x01 inside a word travel escaped, like mrhbm_emit_str does it
        rec.b[l++] = 1;
        if (l < KB) rec.b[l++] = (unsigned char)(ch + 1);
        else l = KB + 1;
      } else {
        rec.b[l++] = ch;
      }
    }
    if (l >= KB || (p < len && !tok_space(t[p]))) {  // does not fit (one zero byte must remain)
      atomicOr(flags, (uint32_t)ERRF_KEYLEN);
      l = KB - 1;
      rec.b[KB - 1] = 0;
    }
    rec.v[RB / 16 - 1].w = value;  // the u32 value field, bytes KB .. RB - 1
    uint4* d = recs + ((uint64_t)block_off[blk] + before) * (RB / 16);
#pragma unroll
    for (int v = 0; v < RB / 16; v++) d[v] = rec.v[v];
  }
}

// ============================================================================
// device-side key-number mapfn (mrhbm_map_key_numbers): lines "key number" -> (key, 11-byte number)
// ============================================================================
// The start of a line's first field: a field start with only white space other than '\n' back to the line's start
// (the piece starts at a line start).  *ls: the line's start.
__device__ __forceinline__ bool kn_first(const unsigned char* t, uint64_t i, uint64_t* ls) {
  if (!tok_start(t, i)) return false;
  uint64_t j = i;
  while (j > 0 && t[j - 1] != '\n' && tok_space(t[j - 1])) j--;
  *ls = j;
  return j == 0 || t[j - 1] == '\n';
}
// one thread per byte, one count of first fields per 256-byte block
__global__ void __launch_bounds__(256) k_kn_count(const unsigned char* __restrict__ t, uint64_t len,
                                                  uint32_t* __restrict__ block_counts) {
  uint64_t nb = (len + 255) / 256, ls;
  for (uint64_t blk = blockIdx.x; blk < nb; blk += gridDim.x) {
    uint64_t i = blk * 256 + threadIdx.x;
    int st = i < len && kn_first(t, i, &ls);
    int c = __syncthreads_count(st);
    if (threadIdx.x == 0) block_counts[blk] = (uint32_t)c;
  }
}
// The thread at a first field walks its line: key, white space, number, white space up to '\n'.  Pair idx (its rank
// among the piece's lines) gets record recs[idx] with value id first + idx, and its encoded number at vals + 11 idx.
template <int RB>
__global__ void __launch_bounds__(256) k_kn_emit(const unsigned char* __restrict__ t, uint64_t len,
                                                 const uint32_t* __restrict__ block_off, KnOut o) {
  constexpr int KB = Rec<RB>::kKeyBytes;
  __shared__ uint32_t wcount[8];
  uint64_t nb = (len + 255) / 256;
  for (uint64_t blk = blockIdx.x; blk < nb; blk += gridDim.x) {
    uint64_t i = blk * 256 + threadIdx.x, ls = 0;
    bool st = i < len && kn_first(t, i, &ls);
    uint32_t m = __ballot_sync(0xffffffffu, st);
    uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) wcount[warp] = __popc(m);
    __syncthreads();
    uint32_t before = __popc(m & ((1u << lane) - 1u));
    for (uint32_t w = 0; w < warp; w++) before += wcount[w];
    __syncthreads();
    if (!st) continue;
    const uint64_t idx = (uint64_t)block_off[blk] + before;
    union {
      unsigned char b[RB];
      uint4 v[RB / 16];
    } rec;
#pragma unroll
    for (int v = 0; v < RB / 16; v++) rec.v[v] = make_uint4(0, 0, 0, 0);
    int l = 0;
    uint64_t p = i;
    while (p < len && !tok_space(t[p]) && l < KB) {
      const unsigned char ch = t[p++];
      if (ch <= 1) {  // escaped, as mrhbm_emit_str does it
        rec.b[l++] = 1;
        if (l < KB) rec.b[l++] = (unsigned char)(ch + 1);
        else l = KB + 1;
      } else {
        rec.b[l++] = ch;
      }
    }
    if (l >= KB || (p < len && !tok_space(t[p]))) {  // does not fit (one zero byte must remain): a host piece
      atomicOr(o.flags, (uint32_t)ERRF_KEYLEN);
      rec.b[KB - 1] = 0;
      while (p < len && !tok_space(t[p])) p++;
    }
    while (p < len && t[p] != '\n' && tok_space(t[p])) p++;
    const uint64_t s = p;
    while (p < len && !tok_space(t[p])) p++;
    const uint64_t ns = p - s;
    while (p < len && t[p] != '\n' && tok_space(t[p])) p++;
    DecScan d;
    uint64_t bits = 0;
    if (ns == 0 || (p < len && t[p] != '\n') || !dec_scan(t + s, ns, &d)) {  // not "key number"
      atomicOr(o.flags, (uint32_t)ERRF_LINE);
      atomicMin(o.flags + 1, (uint32_t)ls);
    } else if (dec_to_bits(d, o.pow5, &bits) != DEC_EXACT) {  // the host rounds it and patches the 11 bytes
      const uint32_t slot = atomicAdd(o.flags + 2, 1u);
      if (slot < o.fix_cap) o.fix[slot] = make_uint4((uint32_t)idx, (uint32_t)s, (uint32_t)ns, 0);
    }
    unsigned char enc[kNumBytes];
    num_encode(bits, enc);
#pragma unroll
    for (int k = 0; k < kNumBytes; k++) o.vals[idx * kNumBytes + k] = enc[k];
    o.voff[idx + 1] = o.aoff + (idx + 1) * kNumBytes;
    if (idx == 0) o.voff[0] = o.aoff;
    rec.v[RB / 16 - 1].w = (uint32_t)(o.first + idx);
    uint4* dst = o.recs + idx * (RB / 16);
#pragma unroll
    for (int v = 0; v < RB / 16; v++) dst[v] = rec.v[v];
  }
}
// the host's values of the fix-up list: {pair index, double bits}
__global__ void __launch_bounds__(256) k_kn_patch(const ulonglong2* __restrict__ fix, uint32_t n,
                                                  unsigned char* __restrict__ vals) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const ulonglong2 f = fix[i];
    unsigned char enc[kNumBytes];
    num_encode(f.y, enc);
#pragma unroll
    for (int k = 0; k < kNumBytes; k++) vals[f.x * kNumBytes + k] = enc[k];
  }
}

// ============================================================================
// histogram + scatter
// ============================================================================
template <int RB>
__device__ __forceinline__ void load_rec(const uint4* p, uint32_t* w) {
#pragma unroll
  for (int v = 0; v < Rec<RB>::kVec; v++) {
    uint4 x = ldg_stream(p + v);
    w[4 * v + 0] = x.x;
    w[4 * v + 1] = x.y;
    w[4 * v + 2] = x.z;
    w[4 * v + 3] = x.w;
  }
}

// U records per thread per iteration: all loads first, then all atomics, then all stores, so
// that each thread keeps U independent memory chains in flight (the loop is latency-bound:
// load -> L2 atomic -> store).
template <int RB>
struct Unroll {
  static constexpr int U = RB == 16 ? 8 : RB == 32 ? 4 : RB == 64 ? 2 : 1;
};

template <int RB, typename BP = BinParams>
__global__ void __launch_bounds__(256) k_hist(const uint4* __restrict__ recs, uint64_t n, BP bp,
                                              uint32_t* __restrict__ hist) {
  constexpr int U = Unroll<RB>::U;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; base < n; base += stride * U) {
    uint32_t w[U][Rec<RB>::kWords];
#pragma unroll
    for (int k = 0; k < U; k++)
      if (base + k * stride < n) load_rec<RB>(recs + (base + k * stride) * Rec<RB>::kVec, w[k]);
#pragma unroll
    for (int k = 0; k < U; k++) {
      if (base + k * stride < n) {
        uint32_t bin = bin_of<RB>(w[k], bp, nullptr);
        atomicAdd(hist + ((size_t)bin << bp.ctr_shift), 1u);  // RED
      }
    }
  }
}

template <int RB, typename BP = BinParams>
__global__ void __launch_bounds__(256) k_scatter(const uint4* __restrict__ recs, uint64_t n, BP bp,
                                                 uint32_t* __restrict__ cursor, uint4* __restrict__ mid) {
  constexpr int U = Unroll<RB>::U;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; base < n; base += stride * U) {
    uint32_t w[U][Rec<RB>::kWords];
    uint32_t pos[U];
#pragma unroll
    for (int k = 0; k < U; k++)
      if (base + k * stride < n) load_rec<RB>(recs + (base + k * stride) * Rec<RB>::kVec, w[k]);
#pragma unroll
    for (int k = 0; k < U; k++) {
      if (base + k * stride < n) {
        uint32_t bin = bin_of<RB>(w[k], bp, nullptr);
        pos[k] = atomicAdd(cursor + ((size_t)bin << bp.ctr_shift), 1u);
      }
    }
#pragma unroll
    for (int k = 0; k < U; k++) {
      if (base + k * stride < n) {
        uint4* d = mid + (uint64_t)pos[k] * Rec<RB>::kVec;
#pragma unroll
        for (int v = 0; v < Rec<RB>::kVec; v++)
          stg_stream(d + v, make_uint4(w[k][4 * v], w[k][4 * v + 1], w[k][4 * v + 2], w[k][4 * v + 3]));
      }
    }
  }
}

// Strided sample of the u64 keys, histogram of their top 8 bits: decides BEFORE any record moves whether
// key-ordered sub-bins (sub = mulhi(key, S)) would be balanced.  Sequential or clustered keys show up as
// overfull buckets and the shuffle uses hash sub-bins from the start instead of paying a discarded attempt.
__global__ void __launch_bounds__(256) k_sample_u64(const uint4* __restrict__ recs, uint64_t n, uint32_t nsample,
                                                    uint32_t* __restrict__ hist256) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  for (uint32_t i = blockIdx.x * 256 + threadIdx.x; i < nsample; i += gridDim.x * 256) {
    const uint64_t idx = (uint64_t)(((unsigned __int128)i * n) / nsample);
    const uint4 r = __ldg(recs + idx);
    atomicAdd(&h[r.y >> 24], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(hist256 + threadIdx.x, h[threadIdx.x]);
}

// The same decision for MRHBM_PART_RANGE: the top 8 bits of each sampled key's position inside its partition, the
// source of the range-relative key-ordered sub-bin (bin_of).
__global__ void __launch_bounds__(256) k_sample_range_u64(const uint4* __restrict__ recs, uint64_t n, uint32_t nsample,
                                                          RangeBinParams bp, uint32_t* __restrict__ hist256) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  for (uint32_t i = blockIdx.x * 256 + threadIdx.x; i < nsample; i += gridDim.x * 256) {
    const uint64_t idx = (uint64_t)(((unsigned __int128)i * n) / nsample);
    const uint4 r = __ldg(recs + idx);
    const uint32_t w[2] = {r.x, r.y};
    const uint32_t pid = range_pid<16>(w, bp);
    atomicAdd(&h[range_pos(bp, (uint64_t)r.x | ((uint64_t)r.y << 32), pid) >> 56], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(hist256 + threadIdx.x, h[threadIdx.x]);
}

// Key slots of `nsample` evenly spaced records (the positions k_sample_u64 takes), for the splitter sample of
// MRHBM_PART_RANGE: one thread per key word.
template <int RB>
__global__ void __launch_bounds__(256) k_sample_keys(const uint32_t* __restrict__ recs, uint64_t n, uint32_t nsample,
                                                     uint32_t* __restrict__ out) {
  constexpr int KW = Rec<RB>::kKeyWords;
  const uint64_t total = (uint64_t)nsample * KW;
  for (uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x; j < total; j += (uint64_t)gridDim.x * 256) {
    const uint32_t i = (uint32_t)(j / KW), k = (uint32_t)(j % KW);
    const uint64_t idx = (uint64_t)(((unsigned __int128)i * n) / nsample);
    out[j] = __ldg(recs + idx * Rec<RB>::kWords + k);
  }
}

// ============================================================================
// two-level coalesced split (many bins)
// ============================================================================
// A per-pair scatter pays one L2 round trip (cursor claim) and one scattered store per pair.
// k_split_tma instead partitions a TILE of records inside shared memory (one shared-memory atomic
// per pair, cheaper than ranking with warp-match instructions), claims global
// space once per (tile, bin) and copies the tile out bin by bin, so stores are contiguous runs.
// With F fine bins per coarse region it runs twice:
//   level 1: source -> coarse regions (local memory), level 2: coarse region -> its F fine bins.
// On several GPUs level 2 IS the exchange: a coarse region belongs to the rank that owns its
// partitions; every rank's level 1 fills its own copy of ALL regions, and level 2 of the owner pulls
// region y from every rank's buffer (peer-mapped memory over NVLink) with the same 40 KB bulk copies
// that feed it on one GPU, tile by tile, while it splits the previous tile -- transfer and split
// overlap inside one kernel, and the sort then runs on local data only.  Replaces
// mapreduce/job.lua:203-221 (partitionfn + spill) and the GridFS / scp transport (job.lua:255-260,
// fs.lua:143-160).

constexpr int kTmaSplitThreads = 512;
__host__ __device__ constexpr size_t tma_split_smem(int rb) {
  return 2 * (size_t)kSplitTileBytes + (size_t)(kSplitTileBytes / rb) * sizeof(uint32_t);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// one thread: arm the barrier with the byte count and start the bulk copy global -> shared
__device__ __forceinline__ void bulk_load(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // earlier generic reads of dst are done
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// One thread issues ONE cp.async.bulk per tile (global -> shared, completion on an mbarrier),
// double-buffered, so tile t+1 lands while tile t is split; the tile is not re-staged: a
// permutation says which raw record goes to which output position, and the copy-out reads the raw
// tile through it.
// The kernel is issue bound (its time follows the instruction count), so
// what is known at launch time is folded at compile time.  SPEC = 0: level, number of GPUs and layout are read from
// the plan (exact layouts, the rare paths).  Otherwise the optimistic layout with bits 0-1 = level and
// bit 2 = several GPUs.  Bit 3 (added to either form) = MRHBM_PART_RANGE: those instances take a RangeBinParams and
// carry the range search, the hash instances keep their parameters and code.
// Arguments: the plan as the host made it, the level (1 or 2; folded when SPEC != 0) and, at level 1, the records
// it splits (src, n).  Level 2 reads the regions of the plan's region buffers (l1, peer[]).
template <int RB, int SPEC = 0>
__global__ void __launch_bounds__(kTmaSplitThreads, 2)
    k_split_tma(SplitPlan pl, uint32_t level_arg, const uint4* src, uint64_t n,
                typename std::conditional<(SPEC & 8) != 0, RangeBinParams, BinParams>::type bp) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  using R = Rec<RB>;
  constexpr int THREADS = kTmaSplitThreads;
  constexpr int T = kSplitTileBytes / RB;            // records per tile
  constexpr int U = (T + THREADS - 1) / THREADS;     // records per thread
  constexpr int IPT = kSplitMaxBins / THREADS;       // bins per thread in the scan
  constexpr int SP = SPEC & 7;
  constexpr int WORLD = SP ? ((SP & 4) ? 2 : 1) : 0;
  constexpr bool DYN = SP != 0 && (SP & 3) == 1;  // tiles from a ticket counter (level 1, optimistic layout)
  static_assert(T < 65536 && kSplitMaxBins <= 65536, "perm packs (raw index, bin) into 16 + 16 bits");
  uint32_t* perm = (uint32_t*)(smem_raw + 2 * kSplitTileBytes);  // output position -> raw index | bin << 16
  __shared__ uint32_t scnt[kSplitMaxBins], soff[kSplitMaxBins];
  // this tile: the slot (record index in dst, 32-bit wrap-around arithmetic) output position 0 would have in the bin's run
  __shared__ uint32_t sbase[kSplitMaxBins];
  __shared__ uint32_t s_rbase[9], s_fbase[9];  // (kernel-parameter arrays indexed by a register would be copied to local memory)
  __shared__ unsigned long long s_src[8];      // byte address and length (records) of the tile streams of this CTA
  __shared__ uint32_t s_n[8];
  __shared__ __align__(8) uint64_t mbar[2];
  __shared__ uint32_t s_next_len[2];
  const uint32_t tid = threadIdx.x;
  const uint32_t level = SP ? (uint32_t)(SP & 3) : level_arg;
  const bool exact = SP ? false : pl.base_off != nullptr;
  const bool multi = SP ? (SP & 4) != 0 : pl.ndest > 1;
#pragma unroll
  for (int i = 0; i < 9; i++)
    if (tid == (uint32_t)i) {
      s_rbase[i] = pl.rbase[i];
      s_fbase[i] = pl.fbase[i];
    }
  // This level: level 1 claims slots in the coarse regions of l1 (sub_stride slots each) through cursor1, level 2 in
  // the fine bins of mid (cap slots each) through cursor; in the optimistic layout a destination takes at most
  // dst_stride records.  (The two pointers are picked where they are used, once per tile: held in registers across
  // the tile loop they cost the run-time form more registers than the parameter reads.)
  const uint32_t dst_stride = level == 1 ? (uint32_t)pl.sub_stride : pl.cap;
  const uint32_t logF = __ffs(pl.F) - 1;
  uint32_t region_first = pl.rbase[0], fine_base = pl.fbase[0];  // first coarse region / fine bin of this rank
  if (multi) {
#pragma unroll
    for (int z = 1; z < 8; z++)
      if (pl.me == (uint32_t)z) {
        region_first = pl.rbase[z];
        fine_base = pl.fbase[z];
      }
  }
  uint32_t coarse = 0;
  if (level == 2) {
    coarse = blockIdx.y;
    if (exact) {  // the coarse region is the union of its fine bins
      uint32_t f0 = coarse * pl.F, f1 = f0 + pl.F < pl.B ? f0 + pl.F : pl.B;
      uint32_t o0 = pl.base_off[f0], o1 = pl.base_off[f1];
      src = (const uint4*)pl.l1 + (size_t)o0 * R::kVec;
      n = o1 - o0;
    }
  }
  // The tile streams this CTA splits: one (the source range) or, for optimistic level 2, region `coarse` as every
  // rank filled it -- ndest streams, the remote ones read over NVLink: sub_stride slots at peer[z] + (region_first +
  // coarse) * sub_stride holding l1_counts[z * l1_zstride + ((region_first + coarse) << ctr_shift)] records.  The CTA
  // takes tiles x, x + gridDim.x, ... of EVERY stream, round-robin over the streams, so that its remote bulk copies
  // fly while it splits local tiles (with one CTA per source the ranks first did all their local tiles, then sat on
  // the link: level 2 took local time + link time).
  const bool region_streams = level == 2 && !exact;
  const uint32_t nsrc = (region_streams && multi) ? pl.ndest : 1u;
#pragma unroll
  for (int z = 0; z < 8; z++) {
    if (tid == (uint32_t)z && (uint32_t)z < nsrc) {
      if (!region_streams) {
        s_src[0] = (unsigned long long)(uintptr_t)src;
        s_n[0] = (uint32_t)n;
      } else {
        s_src[z] = pl.peer[z] + (unsigned long long)(region_first + coarse) * pl.sub_stride * RB;
        const uint32_t c = pl.l1_counts[(size_t)z * pl.l1_zstride + ((size_t)(region_first + coarse) << bp.ctr_shift)];
        s_n[z] = c < pl.sub_stride ? c : (uint32_t)pl.sub_stride;
      }
    }
  }
  if (tid == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (uint32_t b = tid; b < kSplitMaxBins; b += THREADS) scnt[b] = 0;
  __syncthreads();
  uint32_t ntmax = 0;
  for (uint32_t z = 0; z < nsrc; z++) ntmax = max(ntmax, (s_n[z] + T - 1) / T);
  // (tiles x, x + gridDim.x, ...: interleaved rather than a contiguous range of tiles per CTA)
  const uint32_t rounds = ntmax > blockIdx.x ? (ntmax - blockIdx.x + gridDim.x - 1) / gridDim.x : 0u;
  // the CTA's steps in order: round r = 0, 1, ... (tile blockIdx.x + r * gridDim.x), inside a round the streams
  // zrot, zrot + 1, ... (mod nsrc); kept as counters, advanced without a division
  const uint32_t zrot = nsrc > 1 ? (blockIdx.x + pl.me) % nsrc : 0u;
  uint32_t st_r = 0, st_zi = 0, st_z = zrot;
  const uint4* cur_p = nullptr;
  uint32_t cur_len = 0;
  // describes the step the counters stand on (cur_p, cur_len), skipping empty ones; false when the CTA is done
  auto settle = [&]() -> bool {
    while (st_r < rounds) {
      const uint64_t t0 = (uint64_t)(blockIdx.x + st_r * gridDim.x) * T;
      const uint32_t nz = s_n[st_z];
      if (t0 < nz) {
        cur_p = (const uint4*)(uintptr_t)s_src[st_z] + t0 * R::kVec;
        cur_len = (nz - t0) < (uint64_t)T ? (uint32_t)(nz - t0) : (uint32_t)T;
        return true;
      }
      if (++st_zi == nsrc) {
        st_zi = 0;
        st_r++;
      }
      if (++st_z == nsrc) st_z = 0;
    }
    cur_len = 0;
    return false;
  };
  auto advance = [&]() -> bool {
    if (++st_zi == nsrc) {
      st_zi = 0;
      st_r++;
    }
    if (++st_z == nsrc) st_z = 0;
    return settle();
  };
  bool more = DYN ? false : settle();
  if (!DYN && tid == 0 && more) bulk_load(smem_raw, cur_p, cur_len * RB, &mbar[0]);

  // one tile of tn records in `raw`; FULL: tn == T, no per-record bounds checks
  auto split_tile = [&](auto full_c, const uint4* raw, const uint32_t tn) {
    constexpr bool FULL = decltype(full_c)::value;
    uint32_t sub[U], rk[U];
#pragma unroll
    for (int k = 0; k < U; k++) {
      const uint32_t i = tid + k * THREADS;
      if (((k + 1) * THREADS <= T || i < (uint32_t)T) && (FULL || i < tn)) {
        uint32_t dest;
        const uint32_t fine = bin_of<RB, WORLD>((const uint32_t*)(raw + (size_t)i * R::kVec), bp, nullptr, &dest);
        if (level == 1) {
          if (multi)
            sub[k] = s_rbase[dest] + ((fine - s_fbase[dest]) >> logF);
          else
            sub[k] = fine >> logF;
        } else {
          sub[k] = (fine - fine_base) & (pl.F - 1u);
        }
        rk[k] = atomicAdd(scnt + sub[k], 1u);
      }
    }
    __syncthreads();
    // exclusive scan of the per-bin counts; the thread that owns a bin also claims its global space
    uint32_t v[IPT], ex[IPT], g[IPT], s = 0;
#pragma unroll
    for (int i = 0; i < IPT; i++) {
      v[i] = scnt[IPT * tid + i];  // (bins past this level's C1 / F stay zero)
      scnt[IPT * tid + i] = 0;     // ready for the next tile: every count of this one has been taken
      s += v[i];
    }
#pragma unroll
    for (int i = 0; i < IPT; i++) {
      g[i] = 0;
      const uint32_t b = IPT * tid + i;
      if (v[i]) {
        const uint32_t dbin = level == 1 ? b : coarse * pl.F + b;
        g[i] = atomicAdd((level == 1 ? pl.cursor1 : pl.cursor) + ((size_t)dbin << pl.ctr_shift), v[i]);  // result needed only after the placement
      }
    }
    {
      uint32_t e = cta_exscan<THREADS>(s).excl;
#pragma unroll
      for (int i = 0; i < IPT; i++) {
        ex[i] = e;
        soff[IPT * tid + i] = e;
        e += v[i];
      }
    }
    __syncthreads();
    // which raw record goes to which output position
#pragma unroll
    for (int k = 0; k < U; k++) {
      const uint32_t i = tid + k * THREADS;
      if (((k + 1) * THREADS <= T || i < (uint32_t)T) && (FULL || i < tn)) perm[soff[sub[k]] + rk[k]] = i | (sub[k] << 16);
    }
#pragma unroll
    for (int i = 0; i < IPT; i++) {
      const uint32_t b = IPT * tid + i;
      if (v[i]) {
        const uint32_t dbin = level == 1 ? b : coarse * pl.F + b;
        uint32_t gg = g[i], first;
        if (exact) {  // absolute start of the destination region, always large enough
          const uint32_t f = level == 1 ? b * pl.F : dbin;
          first = pl.base_off[f];
        } else {
          first = dbin * dst_stride;
          if (gg + v[i] > dst_stride) {
            // The run does not fit: the whole attempt is abandoned (ERRF_CAPACITY, the host redoes the shuffle with
            // the exact layout from the untouched input), so these records only have to land INSIDE the buffer:
            // at the start of the bin's region (the buffers carry one tile of slack behind the last region).
            atomicOr(pl.err_flags, (uint32_t)ERRF_CAPACITY);
            gg = 0;
          }
        }
        sbase[b] = first + gg - ex[i];  // output position p of this tile goes to slot sbase[b] + p
      }
    }
    __syncthreads();
    // copy out: consecutive output positions of one bin are consecutive in global memory
#pragma unroll
    for (int k = 0; k < U; k++) {
      const uint32_t p = tid + k * THREADS;
      if (((k + 1) * THREADS <= T || p < (uint32_t)T) && (FULL || p < tn)) {
        const uint32_t pb = perm[p];
        const uint32_t slot = sbase[pb >> 16] + p;
        const uint4* r = raw + (size_t)(pb & 0xffffu) * R::kVec;
        uint4* d = (uint4*)(level == 1 ? pl.l1 : pl.mid) + (size_t)slot * R::kVec;
#pragma unroll
        for (int vv = 0; vv < R::kVec; vv++) stg_stream(d + vv, r[vv]);
      }
    }
    __syncthreads();  // the raw tile may be overwritten, perm / soff / sbase reused
  };

  if (!DYN) {
    for (uint32_t it = 0; more; it++) {
      const uint32_t tn = cur_len;
      const uint4* raw = (const uint4*)(smem_raw + (it & 1) * kSplitTileBytes);
      // the other buffer was last read by the copy-out of the previous iteration (barrier at its end)
      more = advance();
      if (tid == 0 && more) bulk_load(smem_raw + ((it & 1) ^ 1) * kSplitTileBytes, cur_p, cur_len * RB, &mbar[(it & 1) ^ 1]);
      mbar_wait(&mbar[it & 1], (it >> 1) & 1);
      if (tn == (uint32_t)T)
        split_tile(std::true_type{}, raw, tn);
      else
        split_tile(std::false_type{}, raw, tn);
    }
  } else {
    // Level 1 of the optimistic layout: ONE stream, and the CTAs do not run at one speed (with equal static shares
    // the first CTA ends well before the last).  After its first tile
    // (blockIdx.x) a CTA takes the next tile nobody has from a ticket counter; thread 0 fetches the ticket one
    // iteration before it needs it, so the L2 round trip is not waited for.
    const uint64_t nrec = s_n[0];
    const uint4* base = (const uint4*)(uintptr_t)s_src[0];
    auto tile_len = [&](uint32_t t) -> uint32_t {
      const uint64_t t0 = (uint64_t)t * T;
      return t0 < nrec ? ((nrec - t0) < (uint64_t)T ? (uint32_t)(nrec - t0) : (uint32_t)T) : 0u;
    };
    uint32_t tn = tile_len(blockIdx.x);
    uint32_t tk = 0;  // (thread 0) the tile to prefetch next
    if (tid == 0) {
      if (tn) bulk_load(smem_raw, base + (uint64_t)blockIdx.x * T * R::kVec, tn * RB, &mbar[0]);
      tk = gridDim.x + atomicAdd(pl.ticket, 1u);
    }
    for (uint32_t it = 0; tn; it++) {
      const uint4* raw = (const uint4*)(smem_raw + (it & 1) * kSplitTileBytes);
      if (tid == 0) {  // the other buffer was last read by the copy-out of the previous iteration (barrier at its end)
        const uint32_t len = tile_len(tk);
        s_next_len[(it & 1) ^ 1] = len;
        if (len) {
          bulk_load(smem_raw + ((it & 1) ^ 1) * kSplitTileBytes, base + (uint64_t)tk * T * R::kVec, len * RB, &mbar[(it & 1) ^ 1]);
          tk = gridDim.x + atomicAdd(pl.ticket, 1u);
        }
      }
      mbar_wait(&mbar[it & 1], (it >> 1) & 1);
      if (tn == (uint32_t)T)
        split_tile(std::true_type{}, raw, tn);
      else
        split_tile(std::false_type{}, raw, tn);
      tn = s_next_len[(it & 1) ^ 1];  // (written before the barriers of split_tile)
    }
    // the last CTA to leave resets the counters for the next launch on the stream
    if (tid == 0 && atomicAdd(pl.ticket + 1, 1u) == gridDim.x - 1) {
      pl.ticket[0] = 0;
      pl.ticket[1] = 0;
    }
  }
}

// single-CTA exclusive scan (B <= a few million, 1024 threads): out_excl[0..n], optional copy into
// out_copy (scatter cursors), optional list of entries larger than cap
__device__ __forceinline__ void exscan_body(const uint32_t* __restrict__ in, uint32_t n,
                                            uint32_t* __restrict__ out_excl, uint32_t* __restrict__ out_copy,
                                            uint32_t* __restrict__ out_dense, uint32_t cap,
                                            uint32_t* __restrict__ big_list, uint32_t* nbig, uint32_t* total,
                                            uint32_t shift) {
  const uint32_t T = blockDim.x, tid = threadIdx.x;
  uint32_t per = (n + T - 1) / T;
  uint32_t b0 = tid * per, b1 = min(n, b0 + per);
  uint32_t s = 0;
  for (uint32_t i = b0; i < b1; i++) s += in[(size_t)i << shift];
  uint32_t run = cta_exscan<1024>(s).excl;
  for (uint32_t i = b0; i < b1; i++) {
    uint32_t c = in[(size_t)i << shift];
    out_excl[i] = run;
    if (out_copy) out_copy[(size_t)i << shift] = run;
    if (out_dense) out_dense[i] = c;
    if (big_list && c > cap) big_list[atomicAdd(nbig, 1u)] = i;
    run += c;
  }
  if (tid == T - 1) {
    out_excl[n] = run;
    if (total) *total = run;
  }
}
__global__ void __launch_bounds__(1024) k_exscan(const uint32_t* __restrict__ in, uint32_t n,
                                                 uint32_t* __restrict__ out_excl,
                                                 uint32_t* __restrict__ out_copy,
                                                 uint32_t* __restrict__ out_dense, uint32_t cap,
                                                 uint32_t* __restrict__ big_list, uint32_t* nbig,
                                                 uint32_t* total, uint32_t shift) {
  exscan_body(in, n, out_excl, out_copy, out_dense, cap, big_list, nbig, total, shift);
}
// Multi-CTA exclusive scan (bins in the tens of thousands made the single-CTA scan a visible slice of
// the shuffle): block b owns elements [1024 b, 1024 b + 1024), one per thread.  Pass 1 writes the block
// sums, pass 2 adds up the sums of the preceding blocks (<= 4096 of them), scans its own elements and
// writes the same outputs as exscan_body.
__global__ void __launch_bounds__(1024) k_exscan_partials(const uint32_t* __restrict__ in, uint32_t n, uint32_t shift,
                                                          uint32_t* __restrict__ partials) {
  __shared__ uint32_t warp_sums[32];
  const uint32_t tid = threadIdx.x, i = blockIdx.x * 1024u + tid;
  uint32_t v = i < n ? in[(size_t)i << shift] : 0u;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  if ((tid & 31) == 0) warp_sums[tid >> 5] = v;
  __syncthreads();
  if (tid < 32) {
    uint32_t w = warp_sums[tid];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) w += __shfl_xor_sync(0xffffffffu, w, d);
    if (tid == 0) partials[blockIdx.x] = w;
  }
}
__global__ void __launch_bounds__(1024) k_exscan_apply(const uint32_t* __restrict__ in, uint32_t n,
                                                       uint32_t* __restrict__ out_excl, uint32_t* __restrict__ out_copy,
                                                       uint32_t* __restrict__ out_dense, uint32_t cap,
                                                       uint32_t* __restrict__ big_list, uint32_t* nbig, uint32_t* total,
                                                       uint32_t shift, const uint32_t* __restrict__ partials) {
  __shared__ uint32_t warp_pre[32];
  const uint32_t tid = threadIdx.x, lane = tid & 31, i = blockIdx.x * 1024u + tid;
  uint32_t pre = 0;  // sum of the preceding blocks
  for (uint32_t b = tid; b < blockIdx.x; b += 1024u) pre += partials[b];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) pre += __shfl_xor_sync(0xffffffffu, pre, d);
  const uint32_t c = i < n ? in[(size_t)i << shift] : 0u;
  if (lane == 0) warp_pre[tid >> 5] = pre;  // read behind the barrier of the scan
  const uint32_t excl = cta_exscan<1024>(c).excl;
  uint32_t p = warp_pre[lane];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) p += __shfl_xor_sync(0xffffffffu, p, d);
  const uint32_t run = p + excl;  // exclusive prefix of element i
  if (i < n) {
    out_excl[i] = run;
    if (out_copy) out_copy[(size_t)i << shift] = run;
    if (out_dense) out_dense[i] = c;
    if (big_list && c > cap) big_list[atomicAdd(nbig, 1u)] = i;
    if (i == n - 1) {
      out_excl[n] = run + c;
      if (total) *total = run + c;
    }
  }
}
// one CTA per source rank: exclusive scan of that rank's counts for this rank's bins
__global__ void __launch_bounds__(1024) k_exscan_rows(const uint32_t* __restrict__ all, uint32_t stride, uint32_t base,
                                                      uint32_t n, uint32_t* __restrict__ out, uint32_t* __restrict__ totals) {
  uint32_t r = blockIdx.x;
  exscan_body(all + (size_t)r * stride + base, n, out + (size_t)r * (n + 1), nullptr, nullptr, 0xffffffffu, nullptr, nullptr,
              totals + r, 0);
}

// ============================================================================
// map-side combiner (mapreduce/job.lua:92-96,198-202 with the built-in sum)
// ============================================================================
// Two hash tables of whole records.
//  * Every CTA keeps an open-addressing table in SHARED memory for its lifetime: hot keys (Zipf) are summed
//    there with shared-memory atomics and never travel further.
//  * Whatever does not find a place there -- the long tail -- is added to ONE open-addressing table in GLOBAL
//    memory sized to stay resident in the 50 MB L2 (25 MB of two-entry buckets): one L2 atomic per pair
//    instead of a partition pass, a sort pass and a reduce pass over that pair.  At its end every CTA flushes
//    its shared table into the global one; k_gtab_compact then emits one record per table entry.
// The result (one record per distinct key, in the common case) is what the partition/sort/reduce stages see.
// The global table does not have to be perfect: two entries for one key only mean that the sort+reduce stage
// adds them up, so reads of a slot another thread is publishing need no stronger ordering than "state first".
// A full table raises ERRF_SKEW and the host retries with a larger one (not L2 resident any more) or without
// the combiner; a u32 sum about to wrap raises ERRF_OVERFLOW (string records carry u32 values), and the host then
// hands the raw pairs on, whose sums the sort / reduce stages keep in u64.
constexpr int kCombineThreads = 1024;
// Warp roles (see k_combine): the first kCombineStreamWarps warps stream the pairs, the last kCombineTableWarps
// warps alone talk to the global table.
constexpr int kCombineTableWarps = 8;
constexpr int kCombineStreamWarps = kCombineThreads / 32 - kCombineTableWarps;
constexpr uint32_t kCombineStreamThreads = 32u * kCombineStreamWarps;
constexpr uint32_t kHandoffSlots = 128;  // entries of one table warp's handoff queue
// Who walks the keys longer than 12 bytes: the stream warp that read them (true) or a table warp (false).
// Measured per record size (DESIGN §4.4): with 64-byte records long pairs can arrive faster than 8 table warps walk
// them (a stream of long keys only took 5.1 ms per 4·10^7 pairs that way, 4.1 with the stream warps walking);
// with 32- and 128-byte records the table warps walk them faster than the stream warps would.
template <int RB>
constexpr bool kStreamWalksLong = RB == 64;
// the shared table; the rest of the 227 KB holds the handoff queues (8 x 128 x 20 bytes) and the table warps'
// probe rings (8 x 1.2 KB): 188 + 30 = 218 KB
constexpr int kCombineSmem = 188 * 1024;

// cheap 32-bit hash of KW key words (one IMAD per word); the shared table (over the words of a key of up to 12
// bytes) and the long entries of the global table (over all key words) take its top bits
template <int KW>
__device__ __forceinline__ uint32_t slot_hash(const uint32_t* w) {
  uint32_t h = 0x9E3779B9u;
#pragma unroll
  for (int k = 0; k < KW; k++) h = (h ^ w[k]) * 0x85EBCA6Bu + (h >> 15);
  h ^= h >> 16;
  h *= 0xC2B2AE35u;
  return h ^ (h >> 13);
}
// L2 residency: the global table only stays in the 50 MB L2 if the 32 GB of pairs streaming through the
// same L2 do not push it out (without policies the table walk waits on DRAM).  The pair
// stream is read with an evict_first policy, every table access carries evict_last.  Table reads are relaxed
// gpu-scope loads (L2 is the point of coherence; `volatile` would compile to system-scope loads).
struct L2Policy {
  uint64_t stream, keep;
};
__device__ __forceinline__ L2Policy l2_policies() {
  L2Policy p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p.stream));
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p.keep));
  return p;
}
// The loads of one record are 16 bytes each, lanes one record apart: every load touches all sectors of the warp's
// records and uses part of each.  They are allocated in L1 so that the record's next loads find those sectors
// there (with L1::no_allocate, config 3 took 4-5 % longer on an H100, DESIGN §4.4).
__device__ __forceinline__ uint4 ldg_stream_hint(const uint4* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void bulk_prefetch_l2(const void* p, uint32_t bytes, uint64_t pol) {
  asm volatile("cp.async.bulk.prefetch.L2.global.L2::cache_hint [%0], %1, %2;" ::"l"(p), "r"(bytes), "l"(pol) : "memory");
}
// Distance in trips of the L2 bulk prefetch ahead of the trip in hand (0: none).  Prefetched pairs compete with the
// global table for the 50 MB L2.  Config 3 (32-byte records, with the earlier 32 MB table) on one H100 SXM at 700 W,
// ms of k_combine per 10^9 pairs, alternating runs in one call: no prefetch 15.47 against 16.61 with 2 trips (earlier
// sweep, 1 / 2 / 3 / 4 trips: 17.3 / 17.1 / 17.7 / 19.0).  Records of 64 and 128 bytes keep the 2 trips; they were
// not swept.
template <int RB>
constexpr uint32_t kPrefetchTrips = RB <= 32 ? 0u : 2u;
// Shared-table clean-up period: 128 trips = 98,304 pairs per CTA.  Config 3 with the 25 MB global table (H100 SXM,
// 700 W, 5-6 alternating runs, ms of k_combine): 14.19-14.22 with 128 trips, 14.31-14.32 with 256, 14.57 with 512,
// 14.74 with 1024; 128 trips with a threshold of 3 pairs instead of 2 took 14.52 (too many warm keys leave).
constexpr uint32_t kEpochTrips = 128;
__device__ __forceinline__ uint32_t ldv_u32(const uint32_t* p, uint64_t pol) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ldv_v4(const uint4* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.relaxed.gpu.global.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(pol)
               : "memory");
  return v;
}
__device__ __forceinline__ void red_add_u32(uint32_t* p, uint32_t v, uint64_t pol) {
  asm volatile("red.relaxed.gpu.global.add.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void red_add_u64(unsigned long long* p, unsigned long long v, uint64_t pol) {
  asm volatile("red.relaxed.gpu.global.add.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void stv_v4(uint4* p, const uint4& v, uint64_t pol) {
  asm volatile("st.relaxed.gpu.global.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w),
               "l"(pol)
               : "memory");
}

template <int RB>
__device__ __forceinline__ void load_rec_hint(const uint4* p, uint32_t* w, uint64_t pol) {
#pragma unroll
  for (int v = 0; v < Rec<RB>::kVec; v++) {
    uint4 x = ldg_stream_hint(p + v, pol);
    w[4 * v + 0] = x.x;
    w[4 * v + 1] = x.y;
    w[4 * v + 2] = x.z;
    w[4 * v + 3] = x.w;
  }
}

// ---- the global table --------------------------------------------------------------------------------------
// Layout: GtabLayout (mrhbm_kernels.h).  SHORT entries: open addressing with linear probing over BUCKETS of two
// entries, one 32-byte L2 sector each: a random L2 read costs per REQUEST, and a lane pair reads both halves of a
// bucket in one load instruction, so one sector request looks at two entries.  The entries of a bucket are claimed
// in order, so an empty first entry means an empty bucket.  A probe is never waited for: it is issued when 32 pairs
// have queued up and looked at when the next 32 have.
// String keys longer than 12 bytes (rare in word counts) go to the LONG entries of one record slot each behind the
// short ones, walked entry by entry by the whole warp (state first, then the key).
// A short key that finds no place within GtabLayout::kMaxProbes buckets raises ERRF_SKEW; from then on its table warp
// drops its remaining pairs, whose result the host discards.
constexpr int kGtabMaxLongProbes = 128;

// A pair on its way to the global table and a short entry share one 16-byte form: strings of up to 12 bytes
// {key word 0, 1, 2, u32 value}, u64 keys {key lo, key hi, u64 value}.  In the table the value word is the entry's
// state: 0 empty / kGtabLock being written / sum + 1.  A long entry is a record with the state in its value word.
template <typename State>
constexpr State kGtabLock = ~State(0);
template <int RB>
struct GtabEntry {
  using State = std::conditional_t<Rec<RB>::kU64, unsigned long long, uint32_t>;
  static __device__ __forceinline__ uint4 pack(uint32_t k0, uint32_t k1, uint32_t k2, State v) {
    if constexpr (Rec<RB>::kU64)
      return make_uint4(k0, k1, (uint32_t)v, (uint32_t)(v >> 32));
    else
      return make_uint4(k0, k1, k2, v);
  }
  static __device__ __forceinline__ State value(const uint4& x) {  // of a pair; of an entry: its state
    if constexpr (Rec<RB>::kU64)
      return (unsigned long long)x.z | ((unsigned long long)x.w << 32);
    else
      return x.w;
  }
  static __device__ __forceinline__ State* state(uint4* e) { return (State*)e + (Rec<RB>::kU64 ? 1 : 3); }
  static __device__ __forceinline__ bool same_key(const uint4& a, const uint4& b) {
    return a.x == b.x && a.y == b.y && (Rec<RB>::kU64 || a.z == b.z);
  }
};

// The update protocol of an entry's state word.  An entry is claimed with a CAS of its state from 0 to the lock,
// written (key + lock) with vector stores and published with an exchange of the state after a fence: a reader
// that sees a published state sees its key.  (A release store in place of fence + exchange measured the same on
// config 3, before and after the warp split of k_combine -- DESIGN §4.4 -- so the plain form stays.)
template <typename State>
__device__ __forceinline__ bool gtab_claim(State* st) {
  return atomicCAS(st, State(0), kGtabLock<State>) == State(0);
}
template <typename State>
__device__ __forceinline__ void gtab_publish(State* st, State v) {
  __threadfence();
  atomicExch(st, v + State(1));
}
// CHECKED (u32 states only): use the returned old value to catch a sum about to pass kMaxCombinedSum (otherwise
// the add is fire-and-forget and the caller has bounded the sums: pairs x largest value <= kMaxCombinedSum)
template <bool CHECKED, typename State>
__device__ __forceinline__ void gtab_add(State* st, State v, uint32_t* __restrict__ flags, uint64_t pol) {
  if (!v) return;
  if constexpr (CHECKED) {
    const State old = atomicAdd(st, v);
    if (old + v < old || old + v > kMaxCombinedSum) atomicOr(flags, (uint32_t)ERRF_OVERFLOW);
  } else if constexpr (sizeof(State) == 8) {
    red_add_u64(st, v, pol);
  } else {
    red_add_u32(st, v, pol);
  }
}

// the home bucket of a short key
template <int RB>
__device__ __forceinline__ uint32_t gtab_slot(const uint4& E, const GtabLayout& tab) {
  uint32_t g = (E.x ^ 0x9E3779B9u) * 0x85EBCA6Bu;
  g = (g ^ (g >> 15) ^ E.y) * 0x2C1B3C6Du;
  if (!Rec<RB>::kU64) g = (g ^ (g >> 13) ^ E.z) * 0x297A2D39u;
  g ^= g >> 16;
  g *= 0xC2B2AE35u;
  g ^= g >> 15;
  return tab.bucket(g);
}
// One probe of the short table: entry `e` as read into x.  Returns 0 = the pair is settled (added, or inserted into
// the empty entry), 1 = the entry holds another key (probe the next one), 2 = the entry is being written (look again).
template <int RB, bool CHECKED>
__device__ __forceinline__ int gtab_probe(uint4* e, const uint4& x, const uint4& E, uint32_t* __restrict__ flags, uint64_t pol) {
  using G = GtabEntry<RB>;
  using State = typename G::State;
  State* st_p = G::state(e);
  const State st = G::value(x), v = G::value(E);
  if (st == 0) {
    if (!gtab_claim(st_p)) return 2;
    stv_v4(e, G::pack(E.x, E.y, E.z, kGtabLock<State>), pol);
    gtab_publish(st_p, v);
    return 0;
  }
  if (st == kGtabLock<State>) return 2;
  if (!G::same_key(x, E)) return 1;
  gtab_add<CHECKED>(st_p, v, flags, pol);
  return 0;
}
// WARP-COLLECTIVE: string keys longer than 12 bytes, one record slot per entry, state first, then the key
template <int RB, bool CHECKED>
__device__ __forceinline__ void gtab_add_long(bool active, uint32_t* __restrict__ gtab, const GtabLayout& tab, const uint32_t* w,
                                              uint32_t v32, uint32_t* __restrict__ flags, uint64_t pol) {
  using R = Rec<RB>;
  constexpr int W = R::kWords, KW = R::kKeyWords;
  constexpr uint32_t kLock = kGtabLock<uint32_t>;
  uint32_t* ltab = gtab + tab.long_offset() / sizeof(uint32_t);
  uint32_t slot = tab.long_slot(slot_hash<KW>(w));
  bool ldone = !active;
#pragma unroll 1
  for (int probe = 0; probe < kGtabMaxLongProbes; probe++) {
    if (__all_sync(0xffffffffu, ldone)) break;
    if (!ldone) {
      uint32_t* e = ltab + (size_t)slot * W;
      uint32_t st = ldv_u32(e + KW, pol);
      if (st == 0) {
        if (gtab_claim(e + KW)) {
#pragma unroll
          for (int i = 0; i < R::kVec; i++)  // the last vector rewrites the lock word with itself
            stv_v4((uint4*)e + i, make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], 4 * i + 3 == KW ? kLock : w[4 * i + 3]), pol);
          gtab_publish(e + KW, v32);
          ldone = true;
        }
        st = kLock;
      }
      if (!ldone) {
        while (st == kLock) st = ldv_u32(e + KW, pol);
        bool eq = true;
#pragma unroll
        for (int i = 0; i < R::kVec; i++) {
          const uint4 y = ldv_v4((const uint4*)e + i, pol);
          eq = eq && y.x == w[4 * i] && y.y == w[4 * i + 1] && y.z == w[4 * i + 2] && (4 * i + 3 == KW || y.w == w[4 * i + 3]);
        }
        if (eq) {
          gtab_add<CHECKED>(e + KW, v32, flags, pol);
          ldone = true;
        }
      }
      slot = tab.long_next(slot);
    }
  }
  if (!ldone) atomicOr(flags, (uint32_t)ERRF_SKEW);
}

// The handoff from the stream warps to the table warps: one queue per table warp t, fed by the stream warps w with
// w % kCombineTableWarps == t.  A stream warp claims as many consecutive positions as it has entries with ONE shared
// atomic on the queue's tail, waits while they are not free yet (backpressure: the table warp has not yet taken what
// was there one lap ago -- nothing is ever dropped), writes the 16-byte entries and publishes each slot with its
// sequence word ((position + 1) << 1 | long key).  The table warp takes the published prefix at its head, up to 32
// slots at a time, and frees them by moving the head.  A pair with a key longer than 12 bytes travels as {its index,
// 0, 0, 0}: the table warp reloads the record for its walk.
struct CombineHandoff {
  uint4 e[kCombineTableWarps][kHandoffSlots];
  uint32_t seq[kCombineTableWarps][kHandoffSlots];
  uint32_t tail[kCombineTableWarps], head[kCombineTableWarps];
  uint32_t streams_done;  // stream warps that have handed off their last entry
};

// WARP-COLLECTIVE: the pairs lq[0 .. nl) (indices, nl <= 32) have keys longer than 12 bytes; each lane reloads
// its record and the warp walks the long entries of the global table for all of them at once
template <int RB, bool CHECKED>
__device__ __forceinline__ void walk_long_keys(const uint32_t* lq, uint32_t nl, const uint4* __restrict__ recs,
                                               uint32_t* __restrict__ gtab, const GtabLayout& tab, uint32_t* __restrict__ flags,
                                               const L2Policy& pol) {
  using R = Rec<RB>;
  uint32_t w[R::kWords];
#pragma unroll
  for (int k = 0; k < R::kWords; k++) w[k] = 0;
  const bool mine = (threadIdx.x & 31) < nl;
  if (mine) load_rec_hint<RB>(recs + (size_t)lq[threadIdx.x & 31] * R::kVec, w, pol.stream);
  gtab_add_long<RB, CHECKED>(mine, gtab, tab, w, (uint32_t)rec_value<RB>(w), flags, pol.keep);
  __syncwarp();
}

// One TABLE warp: drains handoff queue t into the global table until every stream warp is done and the queue is
// empty, then flushes what it still has in flight.
// Its entries queue up as 16-byte compact entries in a ring of 64 (with the number of the bucket probe they are at).
// When 32 are there the warp ISSUES their probes and takes the next entries from the handoff queue.  A probe reads
// the entry's whole bucket: in each of two load instructions lane pair (2i, 2i+1) reads the two halves of one
// bucket -- of lane 2i's entry in the first, of lane 2i+1's in the second -- so each instruction asks L2 for 16
// sectors.  The warp LOOKS at them when the next 32 are ready (or the queue is idle): a lane trades the half it holds
// of its partner's bucket for the half of its own with one shuffle and looks at the bucket's two entries in order.
// A match is added to with a fire-and-forget red, an empty entry is claimed; a bucket of other keys sends the entry
// on to the next bucket, an entry being written to the same bucket again (back into the ring).  Long keys are
// collected by index and walked 32 at a time.
template <int RB, bool CHECKED>
__device__ __forceinline__ void combine_table_warp(CombineHandoff& hq, uint32_t t, const uint4* __restrict__ recs,
                                                   uint32_t* __restrict__ gtab, const GtabLayout& tab, uint32_t* __restrict__ flags,
                                                   const L2Policy& pol) {
  using R = Rec<RB>;
  __shared__ uint4 queue[kCombineTableWarps][64];
  __shared__ uint8_t queue_probe[kCombineTableWarps][64];
  __shared__ uint32_t long_queue[kCombineTableWarps][32];
  static_assert(GtabLayout::kMaxProbes <= 256u, "the ring keeps bucket probes below the limit in 8 bits");
  const uint32_t lane = threadIdx.x & 31, odd = lane & 1u;
  uint4* q = queue[t];
  uint8_t* qp = queue_probe[t];
  uint32_t* lq = long_queue[t];
  uint32_t lq_n = 0;
  uint32_t q_tail = 0, q_pend = 0;  // ring: [.. in flight ..][.. q_pend pending ..] tail
  uint32_t fly_base = 0, fly_n = 0; // the batch in flight: fly_n entries from fly_base (0 = none)
  uint4 fx0, fx1;                   // ... this lane's halves (lane & 1) of the buckets of lanes 2i and 2i + 1
  bool full = false;                // (warp-uniform) this warp has found the table full
  uint4* const bkt = (uint4*)gtab;  // bucket b: entries 2b and 2b + 1
  auto append = [&](bool p, const uint4& E, uint32_t probe) {  // collective: the entries of the lanes with p go to the tail
    const uint32_t m = __ballot_sync(0xffffffffu, p);
    if (p) {
      const uint32_t at = (q_tail + __popc(m & ((1u << lane) - 1u))) & 63u;
      q[at] = E;
      qp[at] = (uint8_t)probe;
    }
    q_tail = (q_tail + __popc(m)) & 63u;
    q_pend += __popc(m);
    __syncwarp();
  };
  auto look = [&]() {  // collective: the batch in flight
    const uint4 send = odd ? fx0 : fx1, o = make_uint4(__shfl_xor_sync(0xffffffffu, send.x, 1), __shfl_xor_sync(0xffffffffu, send.y, 1),
                                                        __shfl_xor_sync(0xffffffffu, send.z, 1), __shfl_xor_sync(0xffffffffu, send.w, 1));
    const uint4 h0 = odd ? o : fx0, h1 = odd ? fx1 : o;  // this lane's bucket
    const bool mine = lane < fly_n;
    uint4 E = make_uint4(0, 0, 0, 0);
    uint32_t probe = 0;
    int r = 0;
    if (mine && !full) {
      E = q[(fly_base + lane) & 63u];
      probe = qp[(fly_base + lane) & 63u];
      uint4* e = bkt + 2u * tab.bucket_at(gtab_slot<RB>(E, tab), probe);
      r = gtab_probe<RB, CHECKED>(e, h0, E, flags, pol.keep);
      if (r == 1) r = gtab_probe<RB, CHECKED>(e + 1, h1, E, flags, pol.keep);
      if (r == 1 && ++probe >= GtabLayout::kMaxProbes) {
        atomicOr(flags, (uint32_t)ERRF_SKEW);  // table full: the host retries with a larger one and drops this result
        full = true;
        r = 0;
      }
    }
    full = __any_sync(0xffffffffu, full);
    fly_n = 0;
    __syncwarp();
    append(r != 0, E, probe);  // (never more than the batch just freed: the ring cannot overflow here)
  };
  auto issue = [&]() {  // collective: the oldest min(32, q_pend) pending entries
    fly_n = q_pend < 32u ? q_pend : 32u;
    fly_base = (q_tail - q_pend) & 63u;
    uint32_t b = 0;
    if (lane < fly_n) b = tab.bucket_at(gtab_slot<RB>(q[(fly_base + lane) & 63u], tab), qp[(fly_base + lane) & 63u]);
    const uint32_t b0 = __shfl_sync(0xffffffffu, b, lane & ~1u), b1 = __shfl_sync(0xffffffffu, b, lane | 1u);
    if ((lane & ~1u) < fly_n) fx0 = ldv_v4(bkt + 2u * b0 + odd, pol.keep);
    if ((lane | 1u) < fly_n) fx1 = ldv_v4(bkt + 2u * b1 + odd, pol.keep);
    q_pend -= fly_n;
  };
  auto push = [&](bool p, const uint4& E) {  // collective: new entries; makes room first, starts a batch when 32 wait
    const uint32_t k = __popc(__ballot_sync(0xffffffffu, p));
    while (fly_n + q_pend + k > 64) {  // (rare: the ring holds the batch in flight + what came back + what is new)
      if (fly_n) look();
      else issue();
    }
    append(p, E, 0u);
    if (q_pend >= 32) {
      if (fly_n) look();
      if (q_pend >= 32) issue();
    }
  };
  auto long_walk = [&]() {  // collective
    walk_long_keys<RB, CHECKED>(lq, lq_n, recs, gtab, tab, flags, pol);
    lq_n = 0;
  };
  const volatile uint32_t* seq = hq.seq[t];
  uint32_t head = 0;  // (hq.head[t] is this warp's to move)
  for (;;) {
    const bool last = *(volatile uint32_t*)&hq.streams_done == (uint32_t)kCombineStreamWarps;
    __threadfence_block();  // (a stream warp counts itself done after its last slot is published)
    const uint32_t at = head + lane, s = at % kHandoffSlots, sq = seq[s];
    const uint32_t ready = __ballot_sync(0xffffffffu, (sq & ~1u) == (at + 1u) << 1);
    const uint32_t k = ~ready ? __ffs(~ready) - 1u : 32u;  // the published prefix
    if (!k) {
      if (last) break;  // every stream warp is done and all it published is taken
      if (fly_n) look();  // the queue is idle: move the ring on
      else if (q_pend) issue();
      else __nanosleep(100);
      continue;
    }
    __threadfence_block();
    const bool mine = lane < k, lng = mine && (sq & 1u);
    const uint4 E = mine ? hq.e[t][s] : make_uint4(0, 0, 0, 0);
    __syncwarp();
    __threadfence_block();  // (the slots are read before they are freed)
    head += k;
    if (lane == 0) *(volatile uint32_t*)&hq.head[t] = head;
    if (!R::kU64) {
      const uint32_t ml = __ballot_sync(0xffffffffu, lng);
      if (ml) {
        if (lq_n + __popc(ml) > 32) long_walk();
        if (lng) lq[lq_n + __popc(ml & ((1u << lane) - 1u))] = E.x;
        lq_n += __popc(ml);
        __syncwarp();
      }
    }
    const bool p = mine && !lng;
    if (__any_sync(0xffffffffu, p)) push(p, E);
  }
  if (!R::kU64 && lq_n) long_walk();
  // drain: whatever is in flight or pending, batch by batch, until nothing comes back
  while (fly_n || q_pend) {
    if (fly_n) look();
    if (q_pend) issue();
  }
}

// flags[0] |= ERRF_*, flags[2] = max over the values seen (saturated to u32).
// vcap: largest value the shared table accepts -- chosen by the host so that one CTA's sum of such values cannot
// wrap 32 bits (pairs per CTA x vcap < 2^32), which keeps saturation tests out of the per-pair path.
// WARP ROLES.  The first kCombineStreamWarps warps STREAM the pairs: they load them, probe and fill the shared
// table and evict from it.  Every pair they cannot settle there, and every evicted entry, is handed off (see
// CombineHandoff) to one of the kCombineTableWarps TABLE warps, which alone probe, claim and add to the global table
// and walk the long keys.  So a stream warp never waits for an L2 round trip and its reads in flight are all
// stream reads.
template <int RB, bool CHECKED>
__global__ void __launch_bounds__(kCombineThreads, 1)
    k_combine(const uint4* __restrict__ recs, uint64_t n, uint32_t pf_trips, uint32_t vcap, uint32_t* __restrict__ gtab,
              GtabLayout layout, uint32_t* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using R = Rec<RB>;
  using G = GtabEntry<RB>;
  static_assert(!(CHECKED && R::kU64), "u64 keys keep u64 sums: their adds are never checked");
  const GtabLayout tab{RB, layout.nbuckets, layout.long_log};  // (RB a constant)
  constexpr int W = R::kWords, KW = R::kKeyWords;
  constexpr int KC = KW < 3 ? KW : 3;  // key words of a shared-table entry: only keys of up to 12 bytes live there
  // Shared table, ARRAY PER FIELD (32 lanes probing 32 random entries hit 32 random banks, not the four a record
  // stride allows): tag[e] = 0 empty / 1 being written / the key's 32-bit hash with bit 1 set; val[e] = u32 partial
  // sum; key[k][e] = key word k < KC.  A probe reads two neighbouring tags; only a tag hit touches the key words.
  // Longer keys (rare in a word count) bypass it: 20 bytes per entry instead of 36 buys 1.8 times the entries.
  // Every kEpochTrips trips the CTA stops at a barrier and evicts the entries that gathered less than two pairs
  // since they were admitted (into the global table, like a miss): the table is filled first come first served,
  // and without that the keys that happened to arrive first would keep out warmer keys that arrived later.
  // (compile-time sizes: table addresses become immediates -- the kernel is short of registers)
  constexpr uint32_t entries = (uint32_t)(kCombineSmem / (R::kU64 ? 16 : 20));  // tag + value + 2 (u64) or 3 key words
  uint32_t* tag = (uint32_t*)smem_raw;
  uint32_t* val = tag + entries;
  uint32_t* key = val + entries;
  __shared__ CombineHandoff hq;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const L2Policy pol = l2_policies();
  for (uint32_t i = tid; i < entries * (KC + 2); i += blockDim.x) tag[i] = 0;
  for (uint32_t i = tid; i < kCombineTableWarps * kHandoffSlots; i += blockDim.x) (&hq.seq[0][0])[i] = 0;
  if (tid < kCombineTableWarps) hq.tail[tid] = hq.head[tid] = 0;
  if (tid == 0) hq.streams_done = 0;
  __syncthreads();  // (the last barrier of the whole CTA: from here on the stream warps sync among themselves)
  if (warp >= (uint32_t)kCombineStreamWarps) {
    combine_table_warp<RB, CHECKED>(hq, warp - kCombineStreamWarps, recs, gtab, tab, flags, pol);
    return;
  }
  const uint32_t to = warp % kCombineTableWarps;  // the table warp this warp hands off to
  // (kStreamWalksLong<RB>) the indices of this warp's pairs with long keys, walked 32 at a time by this warp
  __shared__ uint32_t long_queue[kStreamWalksLong<RB> ? kCombineStreamWarps : 1][32];
  uint32_t* lq = long_queue[kStreamWalksLong<RB> ? warp : 0];
  uint32_t lq_n = 0;
  auto stream_sync = []() { asm volatile("bar.sync 1, %0;" ::"r"(kCombineStreamThreads) : "memory"); };
  auto handoff = [&](bool p, const uint4& E, bool lng) {  // collective: the entries of the lanes with p
    const uint32_t m = __ballot_sync(0xffffffffu, p), k = __popc(m);
    uint32_t base = 0;
    if (lane == 0) {
      base = atomicAdd(&hq.tail[to], k);
      while (base + k - *(volatile uint32_t*)&hq.head[to] > kHandoffSlots) __nanosleep(32);  // backpressure
    }
    base = __shfl_sync(0xffffffffu, base, 0);
    if (p) {
      const uint32_t at = base + __popc(m & ((1u << lane) - 1u)), s = at % kHandoffSlots;
      hq.e[to][s] = E;
      __threadfence_block();
      *(volatile uint32_t*)&hq.seq[to][s] = (at + 1u) << 1 | (uint32_t)lng;
    }
  };
  uint32_t vmax = 0;
  // (between two barriers of the stream warps) entries with a sum below `below` leave the shared table for the
  // global one
  auto evict = [&](uint32_t below) {
    const uint32_t e_round = (entries + 31) / 32 * 32;
    for (uint32_t e = tid; e < e_round; e += kCombineStreamThreads) {
      const bool out = e < entries && tag[e] > 1u && val[e] < below;
      uint4 E = make_uint4(0, 0, 0, 0);
      if (out) {
        E = G::pack(key[e], key[entries + e], KC > 2 ? key[2u * entries + e] : 0u, val[e]);
        tag[e] = 0;
      }
      if (__any_sync(0xffffffffu, out)) handoff(out, E, false);
    }
  };
  // every CTA streams ONE contiguous slice of the pairs, kCombineStreamThreads pairs per trip
  constexpr uint32_t T = kCombineStreamThreads;
  const uint64_t slice = ((n + gridDim.x - 1) / gridDim.x + 31) / 32 * 32;
  const uint64_t slice_lo = slice * blockIdx.x < n ? slice * blockIdx.x : n;
  const uint64_t slice_hi = slice_lo + slice < n ? slice_lo + slice : n;  // (this CTA's pairs: [slice_lo, slice_hi))
  const uint32_t ntrips = (uint32_t)((slice_hi - slice_lo + T - 1) / T);  // (the same for every stream thread: barriers inside)
  // the pair of the NEXT trip is requested before this one is processed (two trips ahead measured the same on
  // config 3).  Index arithmetic of the loop: running 64-bit pointers and 32-bit trip bounds (the per-trip 64-bit
  // index, bounds checks and prefetch address were a visible share of its instructions)
  const uint32_t npairs = (uint32_t)(slice_hi - slice_lo);                                  // pairs of this CTA (< 2^32)
  const uint32_t my_trips = tid < npairs ? (npairs - tid + T - 1) / T : 0u;  // trips in which this thread has a pair
  // the warp's 32 pairs of trip t + pf_trips lie inside the slice for t < pf_ok
  const uint32_t wbase = (tid & ~31u) + 32u;
  const uint32_t pf_full = npairs >= wbase ? (npairs - wbase) / T + 1u : 0u;      // trips whose 32 pairs are all there
  const uint32_t pf_ok = pf_trips && pf_full > pf_trips ? pf_full - pf_trips : 0u;
  const uint4* p_next = recs + (slice_lo + tid) * R::kVec;                                  // this thread's pair of the next trip
  const uint4* p_pf = recs + (slice_lo + (tid & ~31u) + (uint64_t)pf_trips * T) * R::kVec;  // the warp's prefetch target
  const size_t p_step = (size_t)T * R::kVec;
  uint32_t i32 = (uint32_t)slice_lo + tid;  // index of the pair in hand (all pairs of one shuffle: < 2^32)
  uint32_t wn[W];
  if (my_trips) load_rec_hint<RB>(p_next, wn, pol.stream);
  for (uint32_t trip = 0; trip < ntrips; trip++, i32 += T) {
    if (trip % kEpochTrips == kEpochTrips - 1) {
      stream_sync();
      evict(2u);
      stream_sync();
    }
    uint32_t w[W];
#pragma unroll
    for (int k = 0; k < W; k++) w[k] = wn[k];
    p_next += p_step;
    if (trip + 1 < my_trips) load_rec_hint<RB>(p_next, wn, pol.stream);
    // ... and (pf_trips > 0) the warp's 32 pairs of pf_trips trips ahead are pulled from DRAM into L2 by the bulk-copy engine:
    // one trip of work does not cover a DRAM access under load, an L2 hit it does.  (One 32 KB request per CTA by a
    // single thread instead of 1 KB per warp saves instructions but is slower: the warps of a CTA are not in step.)
    if (lane == 0 && trip < pf_ok) bulk_prefetch_l2(p_pf, 32u * RB, pol.stream);
    p_pf += p_step;
    bool need = trip < my_trips;
    const uint64_t v = need ? rec_value<RB>(w) : 0ull;
    vmax = max(vmax, (uint32_t)(v > 0xffffffffull ? 0xffffffffull : v));
    // Straight-line, predicated code: a probe loop that lanes leave at different trips falls apart into fragments
    // that do not reconverge inside it, and every fragment then waits for shared memory on its own.
    bool is_short = true;
    if (!R::kU64) {
#pragma unroll
      for (int k = 3; k < KW; k++) is_short = is_short && w[k] == 0;
    }
    if (need && is_short && v != 0 && v <= vcap) {  // (a zero would still have to create its key: left to the global table)
      const uint32_t h = slot_hash<KC>(w), tg = h | 2u;
      const uint32_t s0 = __umulhi(h, entries), s1 = s0 + 1 == entries ? 0u : s0 + 1;
      const uint32_t t0 = ((volatile uint32_t*)tag)[s0], t1 = ((volatile uint32_t*)tag)[s1];
      if (t0 == tg || t1 == tg) {
        const uint32_t sl = t0 == tg ? s0 : s1;
        uint32_t x[KC];
#pragma unroll
        for (int k = 0; k < KC; k++) x[k] = ((volatile uint32_t*)key)[(uint32_t)k * entries + sl];
        bool eq = true;
#pragma unroll
        for (int k = 0; k < KC; k++) eq = eq && x[k] == w[k];
        if (eq) {
          atomicAdd(val + sl, (uint32_t)v);
          need = false;
        }  // (same hash, other key: the pair goes to the global table, which is allowed to hold a key twice)
      } else if (t0 == 0 || t1 == 0) {  // claim the empty slot (the table fills early in the kernel's life; then rare)
        const uint32_t sl = t0 == 0 ? s0 : s1;
        if (atomicCAS(tag + sl, 0u, 1u) == 0u) {
#pragma unroll
          for (int k = 0; k < KC; k++) key[(uint32_t)k * entries + sl] = w[k];
          val[sl] = (uint32_t)v;
          __threadfence_block();
          atomicExch(tag + sl, tg);
          need = false;
        }
      }
    }
    // misses go to the table warps: a short key as its compact entry, a long string key by index (or, with
    // kStreamWalksLong, into this warp's own walk)
    if (!R::kU64 && need && v > kMaxCombinedSum) {  // (this test also keeps such values out of the long table)
      atomicOr(flags, (uint32_t)ERRF_OVERFLOW);
      need = false;
    }
    if constexpr (kStreamWalksLong<RB>) {
      const uint32_t ml = __ballot_sync(0xffffffffu, need && !is_short);
      if (ml) {
        if (lq_n + __popc(ml) > 32) {
          walk_long_keys<RB, CHECKED>(lq, lq_n, recs, gtab, tab, flags, pol);
          lq_n = 0;
        }
        if (need && !is_short) lq[lq_n + __popc(ml & ((1u << lane) - 1u))] = i32;
        lq_n += __popc(ml);
        __syncwarp();
        need = need && is_short;
      }
    }
    if (__any_sync(0xffffffffu, need)) handoff(need, is_short ? G::pack(w[0], w[1], w[2], v) : make_uint4(i32, 0, 0, 0), !is_short);
  }
  if (kStreamWalksLong<RB> && lq_n) walk_long_keys<RB, CHECKED>(lq, lq_n, recs, gtab, tab, flags, pol);
  stream_sync();
  evict(0xffffffffu);  // the shared table's entries take the same road as the misses
  __syncwarp();
  __threadfence_block();  // (this warp's slots are published before it counts itself done)
  if (lane == 0) atomicAdd(&hq.streams_done, 1u);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) vmax = max(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
  if (lane == 0 && vmax) atomicMax(flags + 2, vmax);
}

// one record per non-empty entry of the global table (short entries first, then the long ones), appended to out
template <int RB>
__global__ void __launch_bounds__(256) k_gtab_compact(const uint32_t* __restrict__ gtab, GtabLayout layout, uint4* __restrict__ out,
                                                      uint32_t* __restrict__ count) {
  using R = Rec<RB>;
  const GtabLayout tab{RB, layout.nbuckets, layout.long_log};  // (RB a constant)
  constexpr int W = R::kWords, KW = R::kKeyWords;
  const uint32_t nshort = tab.nshort(), lane = threadIdx.x & 31;
  const uint32_t* ltab = gtab + tab.long_offset() / sizeof(uint32_t);
  for (uint32_t base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < tab.records(); base += gridDim.x * blockDim.x) {
    const uint32_t s = base + lane;  // (nshort and nlong are multiples of 32: a warp never straddles the two tables)
    uint32_t w[W];
#pragma unroll
    for (int k = 0; k < W; k++) w[k] = 0;
    uint64_t st;  // the entry's state: sum + 1, 0 = empty
    if (s < nshort) {
      const uint4 x = ((const uint4*)gtab)[s];
      w[0] = x.x;
      w[1] = x.y;
      if (!R::kU64) w[2] = x.z;
      st = GtabEntry<RB>::value(x);
    } else {
      const uint4* e = (const uint4*)(ltab + (size_t)(s - nshort) * W);
#pragma unroll
      for (int i = 0; i < R::kVec; i++) {
        const uint4 x = e[i];
        w[4 * i] = x.x;
        w[4 * i + 1] = x.y;
        w[4 * i + 2] = x.z;
        w[4 * i + 3] = x.w;
      }
      st = rec_value<RB>(w);
    }
    const bool has = st != 0;
    st -= 1ull;
    if constexpr (R::kU64) {
      w[2] = (uint32_t)st;
      w[3] = (uint32_t)(st >> 32);
    } else {
      w[KW] = (uint32_t)st;
    }
    const uint32_t m = __ballot_sync(0xffffffffu, has);
    if (!m) continue;
    uint32_t pos = 0;
    if (lane == (uint32_t)(__ffs(m) - 1)) pos = atomicAdd(count, (uint32_t)__popc(m));
    pos = __shfl_sync(0xffffffffu, pos, __ffs(m) - 1) + __popc(m & ((1u << lane) - 1u));
    if (has) {
      uint4* d = out + (size_t)pos * R::kVec;
#pragma unroll
      for (int i = 0; i < R::kVec; i++) d[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
    }
  }
}

// pairs a rank reduces = the fill levels (clamped to the region capacity) of its regions in every rank's
// level-1 cursors; acc2[0] = all of them, acc2[1] = the ones that were already local (source == me)
__global__ void __launch_bounds__(256) k_region_totals(const uint32_t* __restrict__ counts, uint64_t zstride, uint32_t G,
                                                       uint32_t me, uint32_t first, uint32_t nreg, uint32_t shift,
                                                       uint32_t clamp, unsigned long long* __restrict__ acc2) {
  __shared__ unsigned long long s_tot[8], s_own[8];
  unsigned long long tot = 0, own = 0;
  for (uint64_t i = threadIdx.x; i < (uint64_t)nreg * G; i += blockDim.x) {
    const uint32_t z = (uint32_t)(i / nreg), r = (uint32_t)(i % nreg);
    uint32_t c = counts[(size_t)z * zstride + ((size_t)(first + r) << shift)];
    c = c < clamp ? c : clamp;
    tot += c;
    if (z == me) own += c;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    tot += __shfl_xor_sync(0xffffffffu, tot, o);
    own += __shfl_xor_sync(0xffffffffu, own, o);
  }
  if ((threadIdx.x & 31) == 0) {
    s_tot[threadIdx.x >> 5] = tot;
    s_own[threadIdx.x >> 5] = own;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    tot = own = 0;
    for (int w = 0; w < 8; w++) {
      tot += s_tot[w];
      own += s_own[w];
    }
    acc2[0] = tot;
    acc2[1] = own;
  }
}

// global per-bin totals from the all-gathered counts: this rank's bins go to tot[], and every
// rank counts the bins (of ALL ranks) above cap, so that all ranks take the same decision
__global__ void k_sum_src(const uint32_t* __restrict__ all, uint32_t world, uint32_t stride, uint32_t base,
                          uint32_t n, uint32_t* __restrict__ tot, uint32_t cap, uint32_t* __restrict__ nover) {
  for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < stride; b += gridDim.x * blockDim.x) {
    uint32_t t = 0;
    for (uint32_t s = 0; s < world; s++) t += all[(size_t)s * stride + b];
    if (b >= base && b < base + n) tot[b - base] = t;
    if (t > cap) atomicAdd(nover, 1u);
  }
}

// ============================================================================
// result gathering + parity properties
// ============================================================================
template <int RB>
__global__ void __launch_bounds__(256) k_compact(ShuffleBuffers b, uint32_t B, uint32_t* __restrict__ dkeys,
                                                 uint64_t* __restrict__ dsums) {
  constexpr int KW = Rec<RB>::kKeyWords;
  uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t* skeys = (const uint32_t*)b.out_keys;
  for (uint32_t bin = warp; bin < B; bin += nwarps) {
    uint32_t len = b.ucount[bin];
    uint64_t so = out_start(b, bin), d0 = b.uoff[bin];
    for (uint32_t i = lane; i < len * KW; i += 32) dkeys[d0 * KW + i] = skeys[so * KW + i];
    for (uint32_t i = lane; i < len; i += 32) dsums[d0 + i] = b.out_sums[so + i];
  }
}

__device__ __forceinline__ uint64_t warp_sum64(uint64_t v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

template <int RB>
__global__ void __launch_bounds__(256) k_checksum_in(const uint4* __restrict__ recs, uint64_t n,
                                                     unsigned long long* acc) {
  uint64_t a0 = 0, a1 = 0, a2 = 0, a3 = 0;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    uint32_t w[Rec<RB>::kWords];
    load_rec<RB>(recs + i * Rec<RB>::kVec, w);
    uint64_t f1, f2, v = rec_value<RB>(w);
    key_mix2<RB>(w, f1, f2);
    a0 += f1 * v;
    a1 += f2 * v;
    a2 += v;
    a3 += 1;
  }
  a0 = warp_sum64(a0);
  a1 = warp_sum64(a1);
  a2 = warp_sum64(a2);
  a3 = warp_sum64(a3);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(acc + 0, a0);
    atomicAdd(acc + 1, a1);
    atomicAdd(acc + 2, a2);
    atomicAdd(acc + 3, a3);
  }
}

template <int RB, typename BP = BinParams>
__global__ void __launch_bounds__(256) k_checksum_out(ShuffleBuffers b, uint32_t B, BP bp,
                                                      uint32_t bin_base, unsigned long long* acc) {
  constexpr int KW = Rec<RB>::kKeyWords;
  uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t* keys = (const uint32_t*)b.out_keys;
  uint64_t a0 = 0, a1 = 0, a2 = 0, a3 = 0, bad_order = 0, bad_part = 0;
  for (uint32_t bin = warp; bin < B; bin += nwarps) {
    uint32_t len = b.ucount[bin];
    uint64_t so = out_start(b, bin);
    for (uint32_t i = lane; i < len; i += 32) {
      uint32_t w[Rec<RB>::kWords], p[Rec<RB>::kWords];
#pragma unroll
      for (int k = 0; k < KW; k++) w[k] = keys[(so + i) * KW + k];
      uint64_t s = b.out_sums[so + i], f1, f2;
      key_mix2<RB>(w, f1, f2);
      a0 += f1 * s;
      a1 += f2 * s;
      a2 += s;
      a3 += 1;
      if (i > 0) {
#pragma unroll
        for (int k = 0; k < KW; k++) p[k] = keys[(so + i - 1) * KW + k];
        int oc = key_cmp<RB>(p, w);
        if (oc > 0 || (oc == 0 && !b.no_reduce)) bad_order++;
      }
      uint32_t pid;
      uint32_t mybin = bin_of<RB>(w, bp, &pid);
      if (mybin != bin + bin_base) bad_part++;
    }
  }
  a0 = warp_sum64(a0);
  a1 = warp_sum64(a1);
  a2 = warp_sum64(a2);
  a3 = warp_sum64(a3);
  bad_order = warp_sum64(bad_order);
  bad_part = warp_sum64(bad_part);
  if (lane == 0) {
    atomicAdd(acc + 0, a0);
    atomicAdd(acc + 1, a1);
    atomicAdd(acc + 2, a2);
    atomicAdd(acc + 3, a3);
    atomicAdd(acc + 4, bad_order);
    atomicAdd(acc + 5, bad_part);
  }
}

// ============================================================================
// launchers
// ============================================================================
static inline int stream_grid(uint64_t n, int threads, int ctas_per_sm) {
  uint64_t need = (n + threads - 1) / threads;
  uint64_t cap = (uint64_t)g_sm_count * ctas_per_sm;
  return (int)(need < cap ? (need ? need : 1) : cap);
}

cudaError_t kernels_configure() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) return e;
  g_sm_count = prop.multiProcessorCount;
#define CFG(KERNEL, RB, BYTES)                                                                           \
  e = cudaFuncSetAttribute(KERNEL<RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BYTES(RB));      \
  if (e != cudaSuccess) return e;
  CFG(k_sort_reduce, 32, sort_smem_bytes) CFG(k_sort_reduce, 64, sort_smem_bytes) CFG(k_sort_reduce, 128, sort_smem_bytes)
  CFG(k_big_bins, 16, big_smem_bytes) CFG(k_big_bins, 32, big_smem_bytes) CFG(k_big_bins, 64, big_smem_bytes)
  CFG(k_big_bins, 128, big_smem_bytes)
#undef CFG
#define CFGS(M, X)                                                                                                       \
  e = cudaFuncSetAttribute(k_sort_reduce_u64<M, X>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sort_smem_bytes(16)); \
  if (e != cudaSuccess) return e;
  CFGS(false, false) CFGS(false, true) CFGS(true, false) CFGS(true, true)
#undef CFGS
#define CFGC(RB, CH)                                                                                       \
  e = cudaFuncSetAttribute(k_combine<RB, CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, kCombineSmem);  \
  if (e != cudaSuccess) return e;
  CFGC(16, false) CFGC(32, false) CFGC(32, true) CFGC(64, false) CFGC(64, true) CFGC(128, false) CFGC(128, true)
#undef CFGC
#define CFGT1(RB, SPEC)                                                                                  \
  e = cudaFuncSetAttribute(k_split_tma<RB, SPEC>,                                                        \
                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tma_split_smem(RB));        \
  if (e != cudaSuccess) return e;
#define CFGT(RB) CFGT1(RB, 0) CFGT1(RB, 1) CFGT1(RB, 2) CFGT1(RB, 5) CFGT1(RB, 6) \
  CFGT1(RB, 8) CFGT1(RB, 9) CFGT1(RB, 10) CFGT1(RB, 13) CFGT1(RB, 14)
  CFGT(16) CFGT(32) CFGT(64) CFGT(128)
#undef CFGT
#undef CFGT1
  return cudaSuccess;
}

#define DISPATCH_RB(rb, CALL) \
  switch (rb) {               \
    case 16: { constexpr int RB = 16; CALL; } break;   \
    case 32: { constexpr int RB = 32; CALL; } break;   \
    case 64: { constexpr int RB = 64; CALL; } break;   \
    default: { constexpr int RB = 128; CALL; } break;  \
  }

int launch_gen_u64(void* dst, uint64_t seed, uint64_t start, uint64_t n, cudaStream_t s) {
  if (!n) return 0;
  k_gen_u64<<<stream_grid(n, 256, 8), 256, 0, s>>>((uint4*)dst, seed, start, n);
  return 1;
}
int launch_gen_zipf32(void* dst, uint64_t seed, uint64_t start, uint64_t n, const uint64_t* d_table,
                      uint64_t V, cudaStream_t s) {
  if (!n) return 0;
  k_gen_zipf32<<<stream_grid(n, 256, 8), 256, 0, s>>>((uint4*)dst, seed, start, n, d_table, V);
  return 1;
}
int launch_hist(int rb, const void* recs, uint64_t n, const RangeBinParams& bp, uint32_t* hist, cudaStream_t s) {
  if (!n) return 0;
  if (bp.partitioner == kPartRange)
    DISPATCH_RB(rb, (k_hist<RB, RangeBinParams><<<stream_grid(n, 256, 8), 256, 0, s>>>((const uint4*)recs, n, bp, hist)))
  else
    DISPATCH_RB(rb, (k_hist<RB><<<stream_grid(n, 256, 8), 256, 0, s>>>((const uint4*)recs, n, (const BinParams&)bp, hist)))
  return 1;
}
int launch_exscan(const uint32_t* in, uint32_t n, uint32_t* out_excl, uint32_t* out_copy, uint32_t* out_dense,
                  uint32_t cap, uint32_t* big_list, uint32_t* nbig, uint32_t* total, uint32_t shift,
                  cudaStream_t s, uint32_t* scratch) {
  const uint32_t nb = (n + 1023u) / 1024u;
  if (scratch && nb >= 4 && nb <= kScanScratchWords) {
    k_exscan_partials<<<nb, 1024, 0, s>>>(in, n, shift, scratch);
    k_exscan_apply<<<nb, 1024, 0, s>>>(in, n, out_excl, out_copy, out_dense, cap, big_list, nbig, total, shift, scratch);
    return 2;
  }
  k_exscan<<<1, 1024, 0, s>>>(in, n, out_excl, out_copy, out_dense, cap, big_list, nbig, total, shift);
  return 1;
}
int launch_tok_count(const unsigned char* text, uint64_t len, uint32_t* block_counts, cudaStream_t s) {
  if (!len) return 0;
  uint64_t nb = (len + 255) / 256;
  k_tok_count<<<(int)std::min<uint64_t>(nb, (uint64_t)g_sm_count * 16), 256, 0, s>>>(text, len, block_counts);
  return 1;
}
int launch_tok_emit(int rb, const unsigned char* text, uint64_t len, const uint32_t* block_off, void* recs,
                    uint32_t value, uint32_t* flags, cudaStream_t s) {
  if (!len || rb == 16) return 0;
  uint64_t nb = (len + 255) / 256;
  int grid = (int)std::min<uint64_t>(nb, (uint64_t)g_sm_count * 16);
  switch (rb) {
    case 32: k_tok_emit<32><<<grid, 256, 0, s>>>(text, len, block_off, (uint4*)recs, value, flags); break;
    case 64: k_tok_emit<64><<<grid, 256, 0, s>>>(text, len, block_off, (uint4*)recs, value, flags); break;
    default: k_tok_emit<128><<<grid, 256, 0, s>>>(text, len, block_off, (uint4*)recs, value, flags); break;
  }
  return 1;
}
int launch_kn_count(const unsigned char* text, uint64_t len, uint32_t* block_counts, cudaStream_t s) {
  if (!len) return 0;
  uint64_t nb = (len + 255) / 256;
  k_kn_count<<<(int)std::min<uint64_t>(nb, (uint64_t)g_sm_count * 16), 256, 0, s>>>(text, len, block_counts);
  return 1;
}
int launch_kn_emit(int rb, const unsigned char* text, uint64_t len, const uint32_t* block_off, const KnOut& o,
                   cudaStream_t s) {
  if (!len || rb == 16) return 0;
  uint64_t nb = (len + 255) / 256;
  int grid = (int)std::min<uint64_t>(nb, (uint64_t)g_sm_count * 16);
  switch (rb) {
    case 32: k_kn_emit<32><<<grid, 256, 0, s>>>(text, len, block_off, o); break;
    case 64: k_kn_emit<64><<<grid, 256, 0, s>>>(text, len, block_off, o); break;
    default: k_kn_emit<128><<<grid, 256, 0, s>>>(text, len, block_off, o); break;
  }
  return 1;
}
int launch_kn_patch(const void* fix, uint32_t n, unsigned char* vals, cudaStream_t s) {
  if (!n) return 0;
  k_kn_patch<<<(int)std::min<uint32_t>((n + 255) / 256, (uint32_t)g_sm_count * 4), 256, 0, s>>>((const ulonglong2*)fix, n, vals);
  return 1;
}
int launch_combine(const void* recs, uint64_t n, uint32_t* gtab, const GtabLayout& tab, uint32_t* flags, bool checked,
                   int sm_count, cudaStream_t s) {
  if (!n) return 0;
  const int rb = tab.rb;
  // the shared table only takes values whose per-CTA sum stays within kMaxCombinedSum
  const uint64_t per_cta = (n + sm_count - 1) / sm_count + kCombineThreads;
  const uint32_t vcap = (uint32_t)std::min<uint64_t>(0xffffull, kMaxCombinedSum / per_cta);
  if (checked) {  // (u64 keys keep u64 sums: never checked)
    DISPATCH_RB(rb, (k_combine<RB, !Rec<RB>::kU64><<<sm_count, kCombineThreads, kCombineSmem, s>>>((const uint4*)recs, n, kPrefetchTrips<RB>, vcap, gtab, tab, flags)));
  } else {
    DISPATCH_RB(rb, (k_combine<RB, false><<<sm_count, kCombineThreads, kCombineSmem, s>>>((const uint4*)recs, n, kPrefetchTrips<RB>, vcap, gtab, tab, flags)));
  }
  return 1;
}
int launch_gtab_compact(const uint32_t* gtab, const GtabLayout& tab, void* out, uint32_t* count, cudaStream_t s) {
  const int rb = tab.rb;
  const uint32_t slots = tab.records();
  int grid = (int)std::min<uint32_t>((slots + 255) / 256, (uint32_t)g_sm_count * 8);
  DISPATCH_RB(rb, (k_gtab_compact<RB><<<grid, 256, 0, s>>>(gtab, tab, (uint4*)out, count)));
  return 1;
}
int launch_sum_src(const uint32_t* all, uint32_t world, uint32_t stride, uint32_t base, uint32_t n,
                   uint32_t* tot, uint32_t cap, uint32_t* nover, cudaStream_t s) {
  if (!stride) return 0;
  k_sum_src<<<(stride + 255) / 256 < 1024 ? (stride + 255) / 256 : 1024, 256, 0, s>>>(all, world, stride, base, n, tot,
                                                                                      cap, nover);
  return 1;
}
int launch_region_totals(const uint32_t* counts, uint64_t zstride, uint32_t G, uint32_t me, uint32_t first, uint32_t nreg,
                         uint32_t shift, uint32_t clamp, uint64_t* acc2, cudaStream_t s) {
  k_region_totals<<<1, 256, 0, s>>>(counts, zstride, G, me, first, nreg, shift, clamp, (unsigned long long*)acc2);
  return 1;
}
int launch_exscan_rows(const uint32_t* all, uint32_t world, uint32_t stride, uint32_t base, uint32_t n, uint32_t* out,
                       uint32_t* totals, cudaStream_t s) {
  k_exscan_rows<<<world, 1024, 0, s>>>(all, stride, base, n, out, totals);
  return 1;
}
int launch_sample_u64(const void* recs, uint64_t n, uint32_t nsample, uint32_t* hist256, cudaStream_t s) {
  if (!n || !nsample) return 0;
  k_sample_u64<<<(nsample + 255) / 256 < 256 ? (nsample + 255) / 256 : 256, 256, 0, s>>>((const uint4*)recs, n, nsample, hist256);
  return 1;
}
int launch_sample_range_u64(const void* recs, uint64_t n, uint32_t nsample, const RangeBinParams& bp, uint32_t* hist256,
                            cudaStream_t s) {
  if (!n || !nsample) return 0;
  k_sample_range_u64<<<(nsample + 255) / 256 < 256 ? (nsample + 255) / 256 : 256, 256, 0, s>>>((const uint4*)recs, n, nsample, bp, hist256);
  return 1;
}
int launch_sample_keys(int rb, const void* recs, uint64_t n, uint32_t nsample, uint32_t* out, cudaStream_t s) {
  if (!n || !nsample) return 0;
  DISPATCH_RB(rb, (k_sample_keys<RB><<<stream_grid((uint64_t)nsample * Rec<RB>::kKeyWords, 256, 4), 256, 0, s>>>((const uint32_t*)recs, n, nsample, out)));
  return 1;
}
int launch_scatter(int rb, const void* recs, uint64_t n, const RangeBinParams& bp, uint32_t* cursor, void* mid,
                   cudaStream_t s) {
  if (!n) return 0;
  if (bp.partitioner == kPartRange)
    DISPATCH_RB(rb, (k_scatter<RB, RangeBinParams><<<stream_grid(n, 256, 8), 256, 0, s>>>((const uint4*)recs, n, bp, cursor, (uint4*)mid)))
  else
    DISPATCH_RB(rb, (k_scatter<RB><<<stream_grid(n, 256, 8), 256, 0, s>>>((const uint4*)recs, n, (const BinParams&)bp, cursor, (uint4*)mid)))
  return 1;
}
// level 1 (source -> coarse regions, possibly on peers) and level 2 (coarse regions -> fine bins) of the split,
// through the instantiation that has the launch-time facts folded in (k_split_tma's SPEC)
template <int RB>
static void launch_split_rb(dim3 grid, const SplitPlan& pl, uint32_t level, const void* src, uint64_t n,
                            const RangeBinParams& bp, cudaStream_t s) {
  const BinParams& hb = bp;  // the hash instances' parameter block
  const int spec = (pl.base_off ? 0 : (int)level | (pl.ndest > 1 ? 4 : 0)) | (bp.partitioner == kPartRange ? 8 : 0);
  const size_t smem = tma_split_smem(RB);
  const uint4* r = (const uint4*)src;
  switch (spec) {
    case 1: k_split_tma<RB, 1><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, hb); break;
    case 2: k_split_tma<RB, 2><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, hb); break;
    case 5: k_split_tma<RB, 5><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, hb); break;
    case 6: k_split_tma<RB, 6><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, hb); break;
    case 8: k_split_tma<RB, 8><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, bp); break;
    case 9: k_split_tma<RB, 9><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, bp); break;
    case 10: k_split_tma<RB, 10><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, bp); break;
    case 13: k_split_tma<RB, 13><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, bp); break;
    case 14: k_split_tma<RB, 14><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, bp); break;
    default: k_split_tma<RB, 0><<<grid, kTmaSplitThreads, smem, s>>>(pl, level, r, n, hb); break;
  }
}
int launch_split_l1(int rb, const void* recs, uint64_t n, const RangeBinParams& bp, const SplitPlan& pl, cudaStream_t s) {
  if (!n) return 0;
  DISPATCH_RB(rb, (launch_split_rb<RB>(dim3(2 * g_sm_count), pl, 1, recs, n, bp, s)));
  return 1;
}
int launch_split_l2(int rb, const RangeBinParams& bp, const SplitPlan& pl, cudaStream_t s) {
  const int ctas = 2 * g_sm_count;
  const uint32_t regions = pl.C1_local;
  if (!regions) return 0;
  const int x = split_l2_ctas_per_region(regions, pl.sub_stride, pl.ndest, rb, ctas);
  DISPATCH_RB(rb, (launch_split_rb<RB>(dim3(x, regions), pl, 2, nullptr, 0, bp, s)));
  return 1;
}
int launch_sort_reduce(int rb, const ShuffleBuffers& b, uint32_t B, uint32_t cap, int sm_count,
                       cudaStream_t s) {
  int grid = (int)(B < (uint32_t)(2 * sm_count) ? B : (uint32_t)(2 * sm_count));
  if (grid < 1) grid = 1;
  // u64 keys: the register-pipelined variant -- the key range of a bin from its index (key-ordered sub-bins) or from a
  // min / max over its records (hash sub-bins of clustered or sequential keys)
  if (rb == 16) {
    const bool multi = !(b.stride || b.nseg == 1), minmax = !(b.hint_S > 1);
    if (!multi && !minmax) k_sort_reduce_u64<false, false><<<grid, kSortThreads, sort_smem_bytes(16), s>>>(b, B, cap);
    if (!multi && minmax) k_sort_reduce_u64<false, true><<<grid, kSortThreads, sort_smem_bytes(16), s>>>(b, B, cap);
    if (multi && !minmax) k_sort_reduce_u64<true, false><<<grid, kSortThreads, sort_smem_bytes(16), s>>>(b, B, cap);
    if (multi && minmax) k_sort_reduce_u64<true, true><<<grid, kSortThreads, sort_smem_bytes(16), s>>>(b, B, cap);
    return 1;
  }
  switch (rb) {
    case 32: k_sort_reduce<32><<<grid, kSortThreads, sort_smem_bytes(32), s>>>(b, B, cap); break;
    case 64: k_sort_reduce<64><<<grid, kSortThreads, sort_smem_bytes(64), s>>>(b, B, cap); break;
    default: k_sort_reduce<128><<<grid, kSortThreads, sort_smem_bytes(128), s>>>(b, B, cap); break;
  }
  return 1;
}
int launch_big_bins(int rb, const ShuffleBuffers& b, uint32_t nbig, uint32_t cap, cudaStream_t s) {
  if (!nbig) return 0;
  DISPATCH_RB(rb, (k_big_bins<RB><<<nbig, kSortThreads, big_smem_bytes(RB), s>>>(b, cap)));
  return 1;
}
int launch_compact(int rb, const ShuffleBuffers& b, uint32_t B, void* dst_keys, uint64_t* dst_sums,
                   cudaStream_t s) {
  int grid = g_sm_count * 8;
  DISPATCH_RB(rb, (k_compact<RB><<<grid, 256, 0, s>>>(b, B, (uint32_t*)dst_keys, dst_sums)));
  return 1;
}
int launch_checksum_in(int rb, const void* recs, uint64_t n, uint64_t* acc4, cudaStream_t s) {
  if (!n) return 0;
  DISPATCH_RB(rb, (k_checksum_in<RB><<<stream_grid(n, 256, 8), 256, 0, s>>>((const uint4*)recs, n,
                                                                           (unsigned long long*)acc4)));
  return 1;
}
int launch_checksum_out(int rb, const ShuffleBuffers& b, uint32_t B, const RangeBinParams& bp, uint32_t bin_base,
                        uint64_t* acc6, cudaStream_t s) {
  int grid = g_sm_count * 8;
  if (bp.partitioner == kPartRange)
    DISPATCH_RB(rb, (k_checksum_out<RB, RangeBinParams><<<grid, 256, 0, s>>>(b, B, bp, bin_base, (unsigned long long*)acc6)))
  else
    DISPATCH_RB(rb, (k_checksum_out<RB><<<grid, 256, 0, s>>>(b, B, (const BinParams&)bp, bin_base, (unsigned long long*)acc6)))
  return 1;
}

}  // namespace mrhbm
