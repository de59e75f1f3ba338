// mrhbm_sort.cuh -- per-bin sort + segmented reduce inside one CTA's shared memory.
//
// Replaces, for one bin, keys_sorted (mapreduce/utils.lua:123-128), the heap k-way merge that
// concatenates the values of equal keys (utils.lua:206-271, heap.lua) and the reducer loop
// (job.lua:264-284) with the built-in sum.
//
// Fast path (counting_path): one counting pass over 2*capacity interpolated buckets of the
// 64-bit key prefix (about one record per bucket) moves the records into bucket order in a
// second buffer; every record then ranks itself among its few bucket mates by whole-key
// comparison and lands in its final sorted slot.  All later reads are sequential.
// General path: bitonic sort of (prefix digit | index) words, with whole-key LSD passes when
// equal digits hide different keys (heavy duplicates, clustered or long common prefixes).
#pragma once
#include "mrhbm_dev.cuh"
#include "mrhbm_kernels.h"

namespace mrhbm {

constexpr int kSortThreads = 512;
constexpr int kIdxBits = 12;  // kCapBytes/16 records at most
constexpr uint32_t kIdxMask = (1u << kIdxBits) - 1;
constexpr int kDigitBits = 64 - kIdxBits;
static_assert(kCapBytes / 16 <= (1 << kIdxBits), "index bits");

struct SortSmem {
  uint4* rec;     // cap records: the loaded bin, later the sorted bin
  uint4* rec2;    // cap records in bucket order (fast path) / permutations + flags (general path)
  uint32_t* cnt;  // 2*cap words: bucket counters -> offsets; general path: cap composite u64
  uint64_t* red;  // 80 words: process_loaded's min / max of the key prefixes
  uint16_t* heads;  // cap u16: head flags -> group numbers in sorted order (fast path)
};
__host__ __device__ inline size_t sort_smem_bytes(int rb) {
  size_t cap = kCapBytes / rb;
  return (size_t)kCapBytes * 2 + cap * 8 + 80 * 8 + cap * 2;
}
// k_big_bins: string keys carry the u64 values of the loaded chunk behind the carve (process_chunk_wide)
__host__ __device__ inline size_t big_smem_bytes(int rb) {
  return sort_smem_bytes(rb) + (rb == 16 ? 0 : (size_t)(kCapBytes / rb) * 8);
}
__device__ __forceinline__ SortSmem carve(unsigned char* base, int rb) {
  size_t cap = kCapBytes / rb;
  SortSmem s;
  s.rec = (uint4*)base;
  s.rec2 = (uint4*)(base + kCapBytes);
  s.cnt = (uint32_t*)(base + 2 * kCapBytes);
  s.red = (uint64_t*)(base + 2 * kCapBytes + cap * 8);
  s.heads = (uint16_t*)(s.red + 80);
  return s;
}

// ascending bitonic sort of comp[0..n2), n2 a power of two >= 64
__device__ __forceinline__ void bitonic_sort(uint64_t* comp, uint32_t n2) {
  const uint32_t tid = threadIdx.x, T = blockDim.x, half = n2 >> 1;
  for (uint32_t k = 2; k <= n2; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t t = tid; t < half; t += T) {
        uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // insert a 0 bit at log2(j)
        uint32_t l = i | j;
        uint64_t a = comp[i], b = comp[l];
        bool up = (i & k) == 0;
        if ((a > b) == up) {
          comp[i] = b;
          comp[l] = a;
        }
      }
      __syncthreads();
    }
  }
}

// in-place exclusive scan of a[0..n) by the whole CTA (thread t owns a[t*PER .. t*PER+PER)),
// PER * kSortThreads >= n required; returns the total
template <int PER, typename T_>
__device__ __forceinline__ uint32_t block_exscan(T_* a, uint32_t n) {
  const uint32_t tid = threadIdx.x;
  uint32_t v[PER];
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < PER; k++) {
    uint32_t i = tid * PER + k;
    v[k] = i < n ? (uint32_t)a[i] : 0u;
    s += v[k];
  }
  const CtaScan sc = cta_exscan<kSortThreads>(s);
  uint32_t run = sc.excl;
#pragma unroll
  for (int k = 0; k < PER; k++) {
    uint32_t i = tid * PER + k;
    if (i < n) a[i] = (T_)run;
    run += v[k];
  }
  __syncthreads();
  return sc.total;
}
// exclusive scan of a[0 .. 8*kSortThreads) in place, 8 consecutive words per thread; returns the total
__device__ __forceinline__ uint32_t block_exscan_u32x8(uint32_t* a) {
  const uint32_t tid = threadIdx.x;
  uint4 x = ((const uint4*)a)[2 * tid], y = ((const uint4*)a)[2 * tid + 1];
  const CtaScan sc = cta_exscan<kSortThreads>(x.x + x.y + x.z + x.w + y.x + y.y + y.z + y.w);
  uint32_t run = sc.excl;
  uint4 ox, oy;
  ox.x = run; run += x.x;
  ox.y = run; run += x.y;
  ox.z = run; run += x.z;
  ox.w = run; run += x.w;
  oy.x = run; run += y.x;
  oy.y = run; run += y.y;
  oy.z = run; run += y.z;
  oy.w = run;
  ((uint4*)a)[2 * tid] = ox;
  ((uint4*)a)[2 * tid + 1] = oy;
  __syncthreads();
  return sc.total;
}
// exclusive scan of the u16 flags a[0 .. 4*kSortThreads) in place (entries at index >= n count as 0)
__device__ __forceinline__ uint32_t block_exscan_u16x4(uint16_t* a, uint32_t n) {
  const uint32_t tid = threadIdx.x;
  uint2 x = ((const uint2*)a)[tid];
  uint32_t v0 = x.x & 0xffffu, v1 = x.x >> 16, v2 = x.y & 0xffffu, v3 = x.y >> 16;
  const uint32_t i0 = 4 * tid;
  v0 = i0 < n ? v0 : 0u;
  v1 = i0 + 1 < n ? v1 : 0u;
  v2 = i0 + 2 < n ? v2 : 0u;
  v3 = i0 + 3 < n ? v3 : 0u;
  const CtaScan sc = cta_exscan<kSortThreads>(v0 + v1 + v2 + v3);
  const uint32_t e0 = sc.excl, e1 = e0 + v0, e2 = e1 + v1, e3 = e2 + v2;
  ((uint2*)a)[tid] = make_uint2(e0 | (e1 << 16), e2 | (e3 << 16));
  __syncthreads();
  return sc.total;
}

// min of lo and max of hi over the CTA (kSortThreads threads), one barrier; the same reuse rule as cta_exscan
__device__ __forceinline__ void cta_minmax_u64(uint64_t& lo, uint64_t& hi) {
  constexpr uint32_t kWarps = kSortThreads / 32;
  __shared__ uint64_t s_mm[2][kWarps];  // per-warp min / max
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto warp_minmax = [&]() {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint64_t l2 = __shfl_xor_sync(0xffffffffu, lo, o), h2 = __shfl_xor_sync(0xffffffffu, hi, o);
      lo = l2 < lo ? l2 : lo;
      hi = h2 > hi ? h2 : hi;
    }
  };
  warp_minmax();
  if (lane == 0) {
    s_mm[0][warp] = lo;
    s_mm[1][warp] = hi;
  }
  __syncthreads();
  lo = lane < kWarps ? s_mm[0][lane] : ~0ull;
  hi = lane < kWarps ? s_mm[1][lane] : 0ull;
  warp_minmax();
}

// the source segments of `bin` in order (one per source rank after the all-to-all; one on a single GPU):
// seg(first, src, n) for each, `first` = the records of the bin in the segments before it
template <int RB, typename Seg>
__device__ __forceinline__ void for_each_segment(const ShuffleBuffers& b, uint32_t bin, Seg seg) {
  uint32_t first = 0;
  for (uint32_t s = 0; s < b.nseg; s++) {
    const uint32_t so = b.seg_off[s][bin], sc = b.seg_off[s][bin + 1] - so;
    seg(first, (const uint4*)b.src + (b.seg_base[s] + so) * Rec<RB>::kVec, sc);
    first += sc;
  }
}

// coalesced copy of nvec uint4 from global to shared memory, four independent loads in
// flight per thread (the load is latency bound otherwise)
__device__ __forceinline__ void load_bin(uint4* dst, const uint4* __restrict__ src, uint32_t nvec) {
  const uint32_t tid = threadIdx.x, T = blockDim.x;
  uint32_t v = tid;
  for (; v + 3 * T < nvec; v += 4 * T) {
    uint4 a = ldg_stream(src + v), b = ldg_stream(src + v + T), c = ldg_stream(src + v + 2 * T),
          d = ldg_stream(src + v + 3 * T);
    dst[v] = a;
    dst[v + T] = b;
    dst[v + 2 * T] = c;
    dst[v + 3 * T] = d;
  }
  for (; v < nvec; v += T) dst[v] = ldg_stream(src + v);
}

enum { MODE_FINAL = 0, MODE_PARTIAL = 1 };
struct ChunkOut {
  void* keys;      // FINAL: key slots; PARTIAL: AoS records
  uint64_t* sums;  // FINAL; PARTIAL with string keys: the u64 partial sums beside the records
  uint64_t base;   // element offset into the destination
  uint32_t no_reduce = 0;  // group-only mode: equal keys stay separate rows
  const uint64_t* wide = nullptr;  // WIDE: the loaded chunk's values, indexed by each record's value word
};

// The value of a loaded record.  WIDE (k_big_bins, string keys): a merge round's partial sums pass 2^32, so the
// record's u32 value word holds the index of its u64 value in out.wide instead.
template <int RB, bool WIDE>
__device__ __forceinline__ uint64_t chunk_value(const uint32_t* r, const ChunkOut& out) {
  if constexpr (WIDE)
    return out.wide[r[Rec<RB>::kKeyWords]];
  else
    return rec_value<RB>(r);
}

template <int RB, int MODE>
__device__ __forceinline__ void write_group(const ChunkOut& out, uint64_t o, const uint32_t* r, uint64_t s) {
  using R = Rec<RB>;
  if (MODE == MODE_FINAL) {
    if constexpr (R::kU64) {
      ((uint64_t*)out.keys)[o] = (uint64_t)r[0] | ((uint64_t)r[1] << 32);
    } else {
      uint32_t* d = (uint32_t*)out.keys + o * R::kKeyWords;
#pragma unroll
      for (int w = 0; w < R::kKeyWords; w++) d[w] = r[w];
    }
    out.sums[o] = s;
  } else {
    uint32_t* d = (uint32_t*)out.keys + o * R::kWords;
#pragma unroll
    for (int w = 0; w < R::kKeyWords; w++) d[w] = r[w];
    if constexpr (R::kU64) {
      d[2] = (uint32_t)s;
      d[3] = (uint32_t)(s >> 32);
    } else {
      out.sums[o] = s;  // (the record's value word is rewritten when the next round loads it)
    }
  }
}

// Shared epilogue: the bin is in ascending key order (position j holds record at(j)).  hs holds
// one u16 per position: on entry (HAVE_FLAGS) 1 for the first record of every key, else it is
// computed here.  An in-place scan turns the flags into group numbers (a position is a head iff
// the next number differs); each head sums its run and writes the group.
template <int RB, int MODE, bool HAVE_FLAGS, bool WIDE, typename At>
__device__ __forceinline__ uint32_t reduce_sorted(At at, uint32_t cnt, uint16_t* hs, const ChunkOut& out) {
  constexpr int CAP = kCapBytes / RB;
  constexpr int PER = (CAP + kSortThreads - 1) / kSortThreads;
  const uint32_t tid = threadIdx.x, T = blockDim.x;
  if (!HAVE_FLAGS) {
    for (uint32_t j = tid; j < cnt; j += T) {
      uint32_t head = 1;
      if (j > 0 && !out.no_reduce) head = !key_eq<RB>(at(j), at(j - 1));
      hs[j] = (uint16_t)head;
    }
    __syncthreads();
  }
  const uint32_t groups = block_exscan<PER>(hs, cnt);
  for (uint32_t j = tid; j < cnt; j += T) {
    uint32_t g = hs[j], gn = j + 1 < cnt ? hs[j + 1] : groups;
    if (gn == g) continue;  // not a head
    const uint32_t* r = at(j);
    uint64_t s = chunk_value<RB, WIDE>(r, out);
    for (uint32_t k = j + 1; k < cnt; k++) {  // the run: positions that do not start a group
      uint32_t a = hs[k], an = k + 1 < cnt ? hs[k + 1] : groups;
      if (an != a) break;
      s += chunk_value<RB, WIDE>(at(k), out);
    }
    write_group<RB, MODE>(out, out.base + g, r, s);
  }
  __syncthreads();
  return groups;
}

constexpr uint32_t kFixMax = 8;  // largest bucket the rank-among-mates step accepts
constexpr uint32_t kNoFastPath = 0xffffffffu;

template <int RB, int MODE, bool WIDE>
__device__ uint32_t counting_path(const SortSmem& sm, uint32_t cnt, uint64_t pmin, uint64_t pmax,
                                  const ChunkOut& out) {
  using R = Rec<RB>;
  constexpr uint32_t CAP = kCapBytes / RB;
  constexpr uint32_t NB = 2 * CAP;
  constexpr int ITEMS = (CAP + kSortThreads - 1) / kSortThreads;
  const uint32_t tid = threadIdx.x, T = blockDim.x;
  const uint32_t* recw = (const uint32_t*)sm.rec;
  const uint32_t* rec2w = (const uint32_t*)sm.rec2;
  uint32_t* bcnt = sm.cnt;
  uint16_t* heads = sm.heads;
  uint64_t range = pmax - pmin;
  // monotone map prefix -> [0, NB): drop just enough low bits of (prefix - pmin)
  int bits = range ? 64 - __clzll((long long)range) : 0;
  constexpr int kLogNB = 31 - __builtin_clz(NB);
  static_assert((1u << kLogNB) == NB, "NB must be a power of two");
  const int sh = bits > kLogNB ? bits - kLogNB : 0;
  auto bucket_of = [&](const uint32_t* r) -> uint32_t {
    return (uint32_t)((key_prefix64<RB>(r) - pmin) >> sh);
  };
  constexpr int ZPER = (NB + kSortThreads - 1) / kSortThreads;
#pragma unroll
  for (int k = 0; k < ZPER; k++)
    if (tid * ZPER + k < NB) bcnt[tid * ZPER + k] = 0;
  __syncthreads();
  uint32_t br[ITEMS];
  int over = 0;
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    uint32_t i = tid + k * T;
    br[k] = 0;
    if (i < cnt) {
      uint32_t b = bucket_of(recw + i * R::kWords);
      uint32_t r = atomicAdd(bcnt + b, 1u);
      br[k] = (b << 4) | (r & 15u);
      if (r >= kFixMax) over = 1;
    }
  }
  if (__syncthreads_or(over)) return kNoFastPath;
  block_exscan<ZPER>(bcnt, NB);  // bcnt[b] = first position of bucket b
  // records into bucket order
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    uint32_t i = tid + k * T;
    if (i < cnt) {
      uint32_t pos = bcnt[br[k] >> 4] + (br[k] & 15u);
#pragma unroll
      for (int v = 0; v < R::kVec; v++) sm.rec2[pos * R::kVec + v] = sm.rec[i * R::kVec + v];
    }
  }
  __syncthreads();
  // Every record ranks itself among its bucket mates: final sorted slot f = bucket start + rank,
  // "head" = first of its key (bucket order breaks ties), and a head sums its equals (equal keys
  // share a prefix, hence a bucket).  Only the head flags go back to shared memory, in sorted
  // order; the records are written to global memory straight from the bucket-ordered buffer.
  uint32_t fpos[ITEMS];
  uint64_t hsum[ITEMS];
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    uint32_t j = tid + k * T;
    fpos[k] = 0xffffffffu;
    hsum[k] = 0;
    if (j < cnt) {
      const uint32_t* r = rec2w + j * R::kWords;
      uint32_t b = bucket_of(r);
      uint32_t s = bcnt[b], e = (b + 1 < NB) ? bcnt[b + 1] : cnt;
      uint32_t rank = 0, head = 1;
      uint64_t sum = chunk_value<RB, WIDE>(r, out);
      if (e - s > 1) {  // most buckets hold one record
        for (uint32_t m = s; m < e; m++) {
          if (m == j) continue;
          const uint32_t* q = rec2w + m * R::kWords;
          int c = key_cmp<RB>(q, r);
          if (c < 0) {
            rank++;
          } else if (c == 0) {
            if (m < j) {
              rank++;
              if (!out.no_reduce) head = 0;  // an equal key sits earlier: not the first of its group
            } else if (!out.no_reduce) {
              sum += chunk_value<RB, WIDE>(q, out);
            }
          }
        }
      }
      heads[s + rank] = (uint16_t)head;
      fpos[k] = head ? s + rank : 0xffffffffu;
      hsum[k] = sum;
    }
  }
  __syncthreads();
  constexpr int PER = (CAP + kSortThreads - 1) / kSortThreads;
  const uint32_t groups = block_exscan<PER>(heads, cnt);  // heads[f] = groups before sorted slot f
#pragma unroll
  for (int k = 0; k < ITEMS; k++) {
    uint32_t j = tid + k * T;
    if (j < cnt && fpos[k] != 0xffffffffu)
      write_group<RB, MODE>(out, out.base + heads[fpos[k]], rec2w + j * R::kWords, hsum[k]);
  }
  __syncthreads();
  return groups;
}

// Sorts cnt (<= cap) records of one bin by key, sums the values of equal keys and writes
// the groups in ascending key order.  Returns the number of groups.
template <int RB, int MODE, bool WIDE = false>
__device__ uint32_t process_loaded(const SortSmem& sm, uint32_t cnt, const ChunkOut& out);

template <int RB, int MODE>
__device__ uint32_t process_chunk(const SortSmem& sm, const uint4* __restrict__ src, uint32_t cnt,
                                  const ChunkOut& out) {
  using R = Rec<RB>;
  // coalesced load of the bin
  for (uint32_t v = threadIdx.x; v < cnt * R::kVec; v += blockDim.x) sm.rec[v] = src[v];
  __syncthreads();
  return process_loaded<RB, MODE>(sm, cnt, out);
}

// k_big_bins, string keys: process_chunk with u64 values.  The chunk's values go to wide[] -- the records' own u32
// values (side == nullptr: the bin's first round) or the partial sums an earlier round left in side[0, cnt) -- and
// each record's value word becomes the index of its value there.  Every read of side[] happens before the barrier,
// so the chunk may write its groups over the range it was loaded from.
template <int RB, int MODE>
__device__ uint32_t process_chunk_wide(const SortSmem& sm, uint64_t* wide, const uint4* __restrict__ src,
                                       const uint64_t* side, uint32_t cnt, const ChunkOut& out) {
  using R = Rec<RB>;
  for (uint32_t v = threadIdx.x; v < cnt * R::kVec; v += blockDim.x) sm.rec[v] = src[v];
  __syncthreads();
  uint32_t* recw = (uint32_t*)sm.rec;
  for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) {
    uint32_t* r = recw + i * R::kWords;
    wide[i] = side ? side[i] : (uint64_t)r[R::kKeyWords];
    r[R::kKeyWords] = i;
  }
  __syncthreads();
  return process_loaded<RB, MODE, true>(sm, cnt, out);
}

// the bin's cnt records are in sm.rec (all threads have passed a barrier after the load)
template <int RB, int MODE, bool WIDE>
__device__ uint32_t process_loaded(const SortSmem& sm, uint32_t cnt, const ChunkOut& out) {
  using R = Rec<RB>;
  constexpr uint32_t CAP = kCapBytes / RB;
  const uint32_t tid = threadIdx.x, T = blockDim.x;
  const uint32_t* recw = (const uint32_t*)sm.rec;
  // range of the 64-bit key prefix
  uint64_t pmin = ~0ull, pmax = 0;
  for (uint32_t i = tid; i < cnt; i += T) {
    uint64_t p = key_prefix64<RB>(recw + i * R::kWords);
    pmin = p < pmin ? p : pmin;
    pmax = p > pmax ? p : pmax;
  }
  // (not cta_minmax_u64: inlined into k_sort_reduce_u64, its one-barrier form costs that kernel 32 more bytes of
  // spills in its hot loop)
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    uint64_t a = __shfl_xor_sync(0xffffffffu, pmin, d), b = __shfl_xor_sync(0xffffffffu, pmax, d);
    pmin = a < pmin ? a : pmin;
    pmax = b > pmax ? b : pmax;
  }
  if ((tid & 31) == 0) {
    sm.red[tid >> 5] = pmin;
    sm.red[32 + (tid >> 5)] = pmax;
  }
  __syncthreads();
  if (tid < 32) {
    pmin = tid < (T >> 5) ? sm.red[tid] : ~0ull;
    pmax = tid < (T >> 5) ? sm.red[32 + tid] : 0ull;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      uint64_t a = __shfl_xor_sync(0xffffffffu, pmin, d), b = __shfl_xor_sync(0xffffffffu, pmax, d);
      pmin = a < pmin ? a : pmin;
      pmax = b > pmax ? b : pmax;
    }
    if (tid == 0) {
      sm.red[64] = pmin;
      sm.red[65] = pmax;
    }
  }
  __syncthreads();
  pmin = sm.red[64];
  pmax = sm.red[65];
  __syncthreads();
  const uint32_t g = counting_path<RB, MODE, WIDE>(sm, cnt, pmin, pmax, out);
  if (g != kNoFastPath) return g;
  // general path: bitonic sort of (prefix digit | index) words, whole-key passes on ties
  uint64_t* comp = (uint64_t*)sm.cnt;
  uint16_t* perm = (uint16_t*)sm.rec2;
  uint16_t* other = perm + CAP;
  uint64_t range = pmax - pmin;
  int bits = range ? 64 - __clzll((long long)range) : 0;
  int drop = bits > kDigitBits ? bits - kDigitBits : 0;
  uint32_t n2 = 64;
  while (n2 < cnt) n2 <<= 1;
  for (uint32_t i = tid; i < n2; i += T) {
    uint64_t c = ~0ull;
    if (i < cnt) c = (((key_prefix64<RB>(recw + i * R::kWords) - pmin) >> drop) << kIdxBits) | i;
    comp[i] = c;
  }
  __syncthreads();
  bitonic_sort(comp, n2);
  int tie = 0;
  for (uint32_t j = tid; j < cnt; j += T) {
    uint64_t c = comp[j];
    perm[j] = (uint16_t)(c & kIdxMask);
    if (j > 0 && (R::kKeyWords > 2 || drop > 0)) {
      uint64_t p = comp[j - 1];
      if ((c >> kIdxBits) == (p >> kIdxBits) &&
          !key_eq<RB>(recw + (uint32_t)(c & kIdxMask) * R::kWords, recw + (uint32_t)(p & kIdxMask) * R::kWords))
        tie = 1;
    }
  }
  if (__syncthreads_or(tie)) {
    // LSD passes over kDigitBits-wide chunks of the whole key; the previous rank in the low
    // bits makes every pass stable
    constexpr int kKeyBits = R::kKeyWords * 32;
    constexpr int kChunks = (kKeyBits + kDigitBits - 1) / kDigitBits;
    for (int c = kChunks - 1; c >= 0; c--) {
      int bitpos = c * kDigitBits;
      int nb = kKeyBits - bitpos < kDigitBits ? kKeyBits - bitpos : kDigitBits;
      for (uint32_t j = tid; j < n2; j += T) {
        uint64_t w = ~0ull;
        if (j < cnt) w = (key_bits<RB>(recw + (uint32_t)perm[j] * R::kWords, bitpos, nb) << kIdxBits) | j;
        comp[j] = w;
      }
      __syncthreads();
      bitonic_sort(comp, n2);
      for (uint32_t j = tid; j < cnt; j += T) other[j] = perm[comp[j] & kIdxMask];
      __syncthreads();
      uint16_t* t = perm;
      perm = other;
      other = t;
    }
  }
  const uint16_t* pp = perm;
  auto at = [&](uint32_t j) -> const uint32_t* { return recw + (uint32_t)pp[j] * R::kWords; };
  return reduce_sorted<RB, MODE, false, WIDE>(at, cnt, other, out);
}

// string keys (u64 keys: k_sort_reduce_u64)
template <int RB>
__global__ void __launch_bounds__(kSortThreads, 2) k_sort_reduce(ShuffleBuffers b, uint32_t B, uint32_t cap) {
  static_assert(!Rec<RB>::kU64, "u64 keys are sorted by k_sort_reduce_u64");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ uint32_t s_bin;
  SortSmem sm = carve(smem_raw, RB);
  for (;;) {
    if (threadIdx.x == 0) s_bin = atomicAdd(b.counters + CNT_TICKET, 1u);
    __syncthreads();
    uint32_t bin = s_bin;
    __syncthreads();
    if (bin >= B) break;
    uint64_t off = bin_start(b, bin);
    uint32_t cnt = bin_count(b, bin);
    if (cnt > cap) continue;  // k_big_bins
    if (cnt == 0) {
      if (threadIdx.x == 0) b.ucount[bin] = 0;
      continue;
    }
    ChunkOut out{b.out_keys, b.out_sums, out_start(b, bin), b.no_reduce};
    if (b.stride) {
      load_bin(sm.rec, (const uint4*)b.src + off * Rec<RB>::kVec, cnt * Rec<RB>::kVec);
    } else {
      for_each_segment<RB>(b, bin, [&](uint32_t first, const uint4* src, uint32_t n) {
        load_bin(sm.rec + first * Rec<RB>::kVec, src, n * Rec<RB>::kVec);
      });
    }
    __syncthreads();
    uint32_t g = process_loaded<RB, MODE_FINAL>(sm, cnt, out);
    if (threadIdx.x == 0) b.ucount[bin] = g;
  }
}

// ---- u64 keys: the software-pipelined variant ----
//
// Same algorithm as counting_path, restructured around the two things the profile of the
// shared-memory path on u64 keys showed (most stall samples wait at barriers, then on the bin load): the records
// of a bin go from global memory into REGISTERS (4 x 16 B per thread), are counted from there and land
// directly in bucket order, and the loads of the CTA's next bin are issued right after that, so they
// fly while the current bin is ranked, scanned and written.
// Bins come from a ticket counter read ahead of time (below), so taking one adds no barrier; 7 barriers per bin
// instead of 14.

// MULTI: a bin is gathered from one segment per source rank (after the all-to-all); a small
// descriptor (cumulative counts + rebased segment addresses) is built by warp 0 one bin ahead.
// MINMAX: the bins are not key-ordered sub-bins (hash sub-bins of clustered / sequential keys, or one bin per partition):
// the range of a bin's keys is not known from its index, the CTA finds it with a min / max over the loaded records.
template <bool MULTI, bool MINMAX = false>
__global__ void __launch_bounds__(kSortThreads, 2) k_sort_reduce_u64(ShuffleBuffers b, uint32_t B, uint32_t cap) {
  constexpr int RB = 16;
  constexpr uint32_t CAP = kCapBytes / RB, NB = 2 * CAP, T = kSortThreads;
  constexpr int ITEMS = CAP / T;
  static_assert(ITEMS * T == CAP && NB == 8 * T && CAP == 4 * T, "tile shape");
  constexpr int kLogNB = 31 - __builtin_clz(NB);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SortSmem sm = carve(smem_raw, RB);
  const uint32_t tid = threadIdx.x;
  uint32_t* bcnt = sm.cnt;
  uint16_t* heads = sm.heads;
  const uint4* src = (const uint4*)b.src;
  const uint4 zero4 = make_uint4(0, 0, 0, 0);
  ((uint4*)bcnt)[2 * tid] = zero4;
  ((uint4*)bcnt)[2 * tid + 1] = zero4;
  __shared__ uint32_t s_cum[8];   // MULTI: records of the bin that come before segment s
  __shared__ uint64_t s_addr[8];  // MULTI: record i of the bin (in segment s) lives at src[s_addr[s] + i]
  const uint32_t lane = tid & 31, warp = tid >> 5, nseg = b.nseg;
  // warp 0: descriptor of bin `bn` from the per-source offsets (so, sn) each lane < nseg holds
  auto desc_store = [&](uint32_t so, uint32_t sn) {
    const uint32_t c = lane < nseg ? sn - so : 0u, incl = warp_inscan<8>(c);
    if (lane < nseg) {
      s_cum[lane] = incl - c;
      s_addr[lane] = b.seg_base[lane] + so - (incl - c);
    }
  };
  auto desc_load = [&](uint32_t bn, uint32_t& so, uint32_t& sn) {
    so = sn = 0;
    if (MULTI && warp == 0 && lane < nseg && bn < B) {
      so = b.seg_off[lane][bn];
      sn = b.seg_off[lane][bn + 1];
    }
  };
  auto rec_addr = [&](uint32_t i, uint64_t off1) -> const uint4* {
    if (!MULTI) return src + off1 + i;
    uint32_t sg = 0;
    while (sg + 1 < nseg && i >= s_cum[sg + 1]) sg++;
    return src + s_addr[sg] + i;
  };

  uint32_t bin = blockIdx.x;
  uint64_t off = 0;
  uint32_t cnt = 0;
  if (bin < B) {
    off = bin_start(b, bin);
    cnt = bin_count(b, bin);
  }
  // sub = mulhi(key, S): the keys of sub-bin `sub` lie in [sub * q, sub * q + q + S), q = floor(2^64 / S), so one
  // bucket shift serves every bin.  32-bit sort key of a record inside its bin: the top 32 significant bits of
  // key - sub * q (all of them when q + S has at most 32 bits).  Its top kLogNB bits are the bucket; two records of
  // one bucket tie on it with probability 2^-20 (or are real duplicates), and only then are the 64-bit keys compared.
  const uint32_t hint_S = MINMAX ? 1u : b.hint_S;
  const int bits_h = 64 - __clzll((long long)(b.hint_q + hint_S));
  const int sh0_h = bits_h > 32 ? bits_h - 32 : 0, sh1_h = (bits_h > kLogNB ? bits_h - kLogNB : 0) - sh0_h;
  uint32_t sub = bin % hint_S;
  // After its first bin (blockIdx.x) a CTA takes the next bin nobody has from a ticket counter: the CTAs do not run at
  // one speed (with equal static shares the first CTA ends well before the last).  Thread 0
  // fetches a ticket two bins ahead and publishes (bin, bin % S) one bin ahead, so neither the L2 round trip nor the
  // division is waited for.
  __shared__ uint32_t s_nbin[2], s_nsub[2];
  uint32_t* ticket = b.counters + 5;  // {next bin - gridDim.x, CTAs that have left}: zero at launch, zeroed again by the last CTA
  uint32_t tk = 0;
  if (tid == 0) {
    tk = gridDim.x + atomicAdd(ticket, 1u);
    s_nbin[0] = tk;
    s_nsub[0] = tk < B ? tk % hint_S : 0u;
    if (tk < B) tk = gridDim.x + atomicAdd(ticket, 1u);
  }
  uint4 rg[ITEMS];
  if (MULTI) {
    uint32_t so, sn;
    desc_load(bin, so, sn);
    if (warp == 0) desc_store(so, sn);
    __syncthreads();
  }
  if (cnt <= cap) {
#pragma unroll
    for (int k = 0; k < ITEMS; k++)
      if (tid + k * T < cnt) rg[k] = ldg_stream(rec_addr(tid + k * T, off));
  }
  __syncthreads();
  for (uint32_t it = 0; bin < B; it++) {
    // descriptor of the CTA's next bin: the loads are in flight until after the move
    const uint32_t nbin = s_nbin[it & 1], nsub = s_nsub[it & 1];
    if (tid == 0) {  // (read again by everybody at the top of the next iteration, behind at least one barrier)
      s_nbin[(it & 1) ^ 1] = tk;
      s_nsub[(it & 1) ^ 1] = tk < B ? tk % hint_S : 0u;
      if (tk < B) tk = gridDim.x + atomicAdd(ticket, 1u);
    }
    uint64_t noff = 0;
    uint32_t ncnt = 0;
    if (nbin < B) {
      noff = bin_start(b, nbin);
      ncnt = bin_count(b, nbin);
    }
    uint32_t d_so, d_sn;
    desc_load(nbin, d_so, d_sn);
    if (cnt == 0 || cnt > cap) {  // empty, or oversized (k_big_bins): nothing was loaded
      if (cnt == 0 && tid == 0) b.ucount[bin] = 0;
    } else {
      ChunkOut out{b.out_keys, b.out_sums, out_start(b, bin), b.no_reduce};
      uint64_t pmin = (uint64_t)sub * b.hint_q;
      int sh0 = sh0_h, sh1 = sh1_h;
      if (MINMAX) {
        uint64_t lo = ~0ull, hi = 0ull;
#pragma unroll
        for (int k = 0; k < ITEMS; k++)
          if (tid + k * T < cnt) {
            const uint64_t key = (uint64_t)rg[k].x | ((uint64_t)rg[k].y << 32);
            lo = key < lo ? key : lo;
            hi = key > hi ? key : hi;
          }
        cta_minmax_u64(lo, hi);
        pmin = lo;
        const uint64_t range = hi - lo;
        const int bits = range ? 64 - __clzll((long long)range) : 0;
        sh0 = bits > 32 ? bits - 32 : 0;
        sh1 = (bits > kLogNB ? bits - kLogNB : 0) - sh0;
      }
      uint32_t rpack = 0;  // 4 bits per item: arrival order inside the bucket
      int over = 0;
#pragma unroll
      for (int k = 0; k < ITEMS; k++) {
        if (tid + k * T < cnt) {
          const uint64_t key = (uint64_t)rg[k].x | ((uint64_t)rg[k].y << 32);
          const uint32_t kk = (uint32_t)((key - pmin) >> sh0);
          const uint32_t bk = (kk >> sh1) & (NB - 1);
          const uint32_t r = atomicAdd(bcnt + bk, 1u);
          rpack |= (r & 15u) << (4 * k);
          if (r >= kFixMax) over = 1;
        }
      }
      if (__syncthreads_or(over)) {
        // a bucket with more than kFixMax records (heavy duplicates / clustered keys): the general
        // kernel body on the same records
#pragma unroll
        for (int k = 0; k < ITEMS; k++)
          if (tid + k * T < cnt) sm.rec[tid + k * T] = rg[k];
        __syncthreads();
        uint32_t g = process_loaded<RB, MODE_FINAL>(sm, cnt, out);
        if (tid == 0) b.ucount[bin] = g;
        __syncthreads();
        ((uint4*)bcnt)[2 * tid] = zero4;
        ((uint4*)bcnt)[2 * tid + 1] = zero4;
      } else {
        block_exscan_u32x8(bcnt);  // bcnt[bk] = first position of bucket bk
        uint32_t* kk2 = (uint32_t*)sm.rec;  // bucket-ordered 32-bit sort keys (+ 4 sentinels)
#pragma unroll
        for (int k = 0; k < ITEMS; k++)
          if (tid + k * T < cnt) {
            const uint64_t key = (uint64_t)rg[k].x | ((uint64_t)rg[k].y << 32);
            const uint32_t kk = (uint32_t)((key - pmin) >> sh0);
            const uint32_t pos = bcnt[(kk >> sh1) & (NB - 1)] + ((rpack >> (4 * k)) & 15u);
            sm.rec2[pos] = rg[k];
            kk2[pos] = kk;
          }
        if (tid < 4) kk2[cnt + tid] = 0xffffffffu;  // what the four-slot window reads behind the last bucket
        if (MULTI && warp == 0) desc_store(d_so, d_sn);  // the current bin's loads were issued an iteration ago
        __syncthreads();
        // the registers are free: start loading the next bin
        if (ncnt <= cap) {
#pragma unroll
          for (int k = 0; k < ITEMS; k++)
            if (tid + k * T < ncnt) rg[k] = ldg_stream(rec_addr(tid + k * T, noff));
        }
        // every position of the bucket-ordered buffer ranks itself among its bucket mates: a four-slot window of
        // 32-bit keys from the bucket's start (later buckets and the sentinels compare greater)
        uint32_t fpos[ITEMS];  // sorted slot of a group's head, 0xffffffff: not a head
        int merged = 0;        // some record of the bin is not a head: the groups have to be counted
#pragma unroll
        for (int k = 0; k < ITEMS; k++) {
          const uint32_t j = tid + k * T;
          fpos[k] = 0xffffffffu;
          if (j < cnt) {
            const uint32_t mk = kk2[j];
            const uint32_t bk = (mk >> sh1) & (NB - 1);
            const uint32_t s0 = bcnt[bk], e0 = (bk + 1 < NB) ? bcnt[bk + 1] : cnt;
            const uint32_t k0 = kk2[s0], k1 = kk2[s0 + 1], k2 = kk2[s0 + 2], k3 = kk2[s0 + 3];
            uint32_t rank = (uint32_t)(k0 < mk) + (uint32_t)(k1 < mk) + (uint32_t)(k2 < mk) + (uint32_t)(k3 < mk);
            const uint32_t same = (uint32_t)(k0 == mk) + (uint32_t)(k1 == mk) + (uint32_t)(k2 == mk) + (uint32_t)(k3 == mk);
            uint32_t head = 1;
            if (same > 1 || e0 - s0 > 4) {  // a tie on the 32-bit key (real duplicates, mostly) or a long bucket: the exact walk
              const uint4 me = sm.rec2[j];
              const uint64_t key = (uint64_t)me.x | ((uint64_t)me.y << 32);
              uint64_t sum = (uint64_t)me.z | ((uint64_t)me.w << 32);
              rank = 0;
              for (uint32_t m = s0; m < e0; m++) {
                if (m == j) continue;
                const uint2 qk = *(const uint2*)(sm.rec2 + m);
                const uint64_t q = (uint64_t)qk.x | ((uint64_t)qk.y << 32);
                if (q < key) {
                  rank++;
                } else if (q == key) {
                  if (m < j) {
                    rank++;
                    if (!out.no_reduce) head = 0;
                  } else if (!out.no_reduce) {
                    const uint2 qv = *((const uint2*)(sm.rec2 + m) + 1);
                    sum += (uint64_t)qv.x | ((uint64_t)qv.y << 32);
                  }
                }
              }
              // the head of a group keeps the group's sum in its own value slot: nobody reads that slot (a walk only
              // reads the values of equal keys BEHIND its own position, and the head is the first of its keys)
              if (head && !out.no_reduce) *((uint2*)(sm.rec2 + j) + 1) = make_uint2((uint32_t)sum, (uint32_t)(sum >> 32));
              merged |= (int)(head == 0);
            }
            heads[s0 + rank] = (uint16_t)head;
            fpos[k] = head ? s0 + rank : 0xffffffffu;
          }
        }
        uint32_t groups = cnt;
        if (__syncthreads_or(merged)) {  // (unique keys: sorted slot = output slot, no scan)
          groups = block_exscan_u16x4(heads, cnt);  // heads[f] = groups before sorted slot f
#pragma unroll
          for (int k = 0; k < ITEMS; k++)
            if (fpos[k] != 0xffffffffu) fpos[k] = heads[fpos[k]];
        }
#pragma unroll
        for (int k = 0; k < ITEMS; k++) {
          if (fpos[k] != 0xffffffffu) {
            const uint64_t o = out.base + fpos[k];
            const uint4 me = sm.rec2[tid + k * T];
            ((uint64_t*)out.keys)[o] = (uint64_t)me.x | ((uint64_t)me.y << 32);
            out.sums[o] = (uint64_t)me.z | ((uint64_t)me.w << 32);
          }
        }
        ((uint4*)bcnt)[2 * tid] = zero4;
        ((uint4*)bcnt)[2 * tid + 1] = zero4;
        if (tid == 0) b.ucount[bin] = groups;
        bin = nbin;
        off = noff;
        cnt = ncnt;
        sub = nsub;
        __syncthreads();
        continue;
      }
    }
    // no prefetch happened on this path
    bin = nbin;
    off = noff;
    cnt = ncnt;
    sub = nsub;
    if (MULTI) {
      if (warp == 0) desc_store(d_so, d_sn);
      __syncthreads();
    }
    if (cnt <= cap) {
#pragma unroll
      for (int k = 0; k < ITEMS; k++)
        if (tid + k * T < cnt) rg[k] = ldg_stream(rec_addr(tid + k * T, off));
    }
    __syncthreads();
  }
  if (tid == 0 && atomicAdd(ticket + 1, 1u) == gridDim.x - 1) {  // the last CTA to leave: counters ready for the next launch
    ticket[0] = 0;
    ticket[1] = 0;
  }
}

// One CTA per oversized bin (hot keys): chunk-wise in-place reduce until the bin fits.  Sums are u64 on every round:
// u64 keys keep them in the record, string keys (a u32 value word) in the bin's own range of out_sums,
// [off, off + n), which no other bin writes and which the final round overwrites with the groups.
template <int RB>
__global__ void __launch_bounds__(kSortThreads, 2) k_big_bins(ShuffleBuffers b, uint32_t cap) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SortSmem sm = carve(smem_raw, RB);
  uint32_t bin = b.big_list[blockIdx.x];
  uint32_t off = (uint32_t)bin_start(b, bin), n = bin_count(b, bin);
  uint4* base = (uint4*)b.mid + (uint64_t)off * Rec<RB>::kVec;
  if (b.src != b.mid) {  // after an exchange: make the bin contiguous inside the (free) send buffer
    for_each_segment<RB>(b, bin, [&](uint32_t first, const uint4* src, uint32_t sc) {
      uint4* dst = base + (uint64_t)first * Rec<RB>::kVec;
      for (uint64_t v = threadIdx.x; v < (uint64_t)sc * Rec<RB>::kVec; v += blockDim.x) dst[v] = src[v];
    });
    __syncthreads();
  }
  if (b.no_reduce) {
    // group-only mode cannot shrink a bin (a key with more values than one CTA sorts): sort it
    // chunk by chunk; the bin becomes ceil(n / cap) ascending runs of cap rows, which the host
    // iterator merges (it knows the oversized bins from big_list).
    for (uint32_t c = 0; c < n; c += cap) {
      uint32_t m = n - c < cap ? n - c : cap;
      ChunkOut out{b.out_keys, b.out_sums, (uint64_t)off + c, 1u};
      process_chunk<RB, MODE_FINAL>(sm, base + (uint64_t)c * Rec<RB>::kVec, m, out);
    }
    if (threadIdx.x == 0) b.ucount[bin] = n;
    return;
  }
  uint64_t* side = b.out_sums + off;  // string keys: the partial sums of the records at base[0, n)
  uint64_t* wide = (uint64_t*)(smem_raw + sort_smem_bytes(RB));
  bool carried = false;               // ... once a merge round has written them
  while (n > cap) {
    uint32_t w = 0;
    for (uint32_t c = 0; c < n; c += cap) {
      uint32_t m = n - c < cap ? n - c : cap;
      ChunkOut out{base, side, w};
      out.wide = wide;
      // groups of a chunk never outnumber the records consumed so far: w + g <= c + m
      if constexpr (Rec<RB>::kU64)
        w += process_chunk<RB, MODE_PARTIAL>(sm, base + (uint64_t)c * Rec<RB>::kVec, m, out);
      else
        w += process_chunk_wide<RB, MODE_PARTIAL>(sm, wide, base + (uint64_t)c * Rec<RB>::kVec,
                                                  carried ? side + c : nullptr, m, out);
      __threadfence_block();
    }
    if (w == n) {  // nothing merged: more distinct keys than one CTA can sort
      if (threadIdx.x == 0) {
        atomicOr(b.counters + CNT_ERR, (uint32_t)ERRF_SKEW);
        b.ucount[bin] = 0;
      }
      return;
    }
    n = w;
    carried = true;
  }
  ChunkOut out{b.out_keys, b.out_sums, off, b.no_reduce};
  out.wide = wide;
  uint32_t g;
  if constexpr (Rec<RB>::kU64)
    g = process_chunk<RB, MODE_FINAL>(sm, base, n, out);
  else
    g = process_chunk_wide<RB, MODE_FINAL>(sm, wide, base, carried ? side : nullptr, n, out);
  if (threadIdx.x == 0) b.ucount[bin] = g;
}

}  // namespace mrhbm
