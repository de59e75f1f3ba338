// mrhbm_value_order.cu -- MRHBM_RED_DISTINCT: after the group-only sort (rows of a bin ascending by key, value ids in
// out_sums) every bin's rows are put in (key, value bytes) order.
//   k_value_order  one CTA per bin of at most `cap` rows (or per cap-row chunk of an oversized bin): the key groups
//                  are numbered with one CTA scan, each row caches its value's first 8 bytes big endian, and a bitonic
//                  sort in shared memory orders the rows by (group, prefix), comparing the rest of the bytes in the
//                  arena only when two prefixes tie.  Keys never move: a group keeps its rows, only their value ids
//                  are permuted.
//   k_value_merge  one CTA per oversized bin: its chunks, each ordered by k_value_order, are merged pairwise, pass
//                  after pass, between the output rows and a scratch of the same layout, into one ascending run.
// The shuffle dedupes across map jobs first (collect_sources), so no two rows of a bin compare equal.
#include <cstdint>

#include "mrhbm_dev.cuh"
#include "mrhbm_valbytes.cuh"

namespace mrhbm {

namespace {
constexpr int kOrderThreads = 256;
constexpr int kMergeThreads = 1024;
constexpr uint32_t kNoGroup = 0xffffffffu;  // the padding of the bitonic sort: after every row

template <int RB>
__device__ __forceinline__ void load_key(const uint32_t* keys, uint64_t row, uint32_t* k) {
#pragma unroll
  for (int i = 0; i < Rec<RB>::kKeyWords; i++) k[i] = keys[row * Rec<RB>::kKeyWords + i];
}

// row (group ga, prefix pa, id a) after row (gb, pb, b)
__device__ __forceinline__ bool after(uint32_t ga, uint64_t pa, uint64_t a, uint32_t gb, uint64_t pb, uint64_t b,
                                      const unsigned char* __restrict__ arena, const uint64_t* __restrict__ voff) {
  if (ga != gb) return ga > gb;
  if (pa != pb) return pa > pb;
  if (ga == kNoGroup) return false;
  return val_cmp(val_view(arena, voff, a), val_view(arena, voff, b), 2) > 0;
}
}  // namespace

// list == nullptr: CTA x orders bin x when it holds at most cap rows.  Else CTA (x, y) orders the chunks y, y + gridDim.y,
// ... of oversized bin list[x].
template <int RB>
__global__ void __launch_bounds__(kOrderThreads) k_value_order(ShuffleBuffers b, uint32_t cap, const uint32_t* list,
                                                               const unsigned char* __restrict__ arena,
                                                               const uint64_t* __restrict__ voff) {
  constexpr int kMax = kCapBytes / RB, kPer = kMax / kOrderThreads;
  __shared__ uint64_t s_pre[kMax], s_id[kMax];
  __shared__ uint32_t s_grp[kMax];
  const uint32_t bin = list ? list[blockIdx.x] : blockIdx.x;
  const uint32_t n = b.ucount[bin];
  if (list ? n <= cap : n > cap) return;
  const uint32_t* keys = (const uint32_t*)b.out_keys;
  const uint64_t o = out_start(b, bin);
  const uint32_t tid = threadIdx.x;
  for (uint64_t c0 = (uint64_t)blockIdx.y * cap; c0 < n; c0 += (uint64_t)gridDim.y * cap) {
    const uint32_t m = (uint32_t)min((uint64_t)cap, n - c0);
    const uint64_t base = o + c0;
    // group heads: thread t holds rows [t * kPer, (t + 1) * kPer)
    uint32_t head = 0;
    uint32_t prev[Rec<RB>::kKeyWords], cur[Rec<RB>::kKeyWords];
    if (tid * kPer < m && tid * kPer > 0) load_key<RB>(keys, base + tid * kPer - 1, prev);
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      const uint32_t i = tid * kPer + k;
      if (i < m) {
        load_key<RB>(keys, base + i, cur);
        if (i == 0 || !key_eq<RB>(cur, prev)) head |= 1u << k;
#pragma unroll
        for (int w = 0; w < Rec<RB>::kKeyWords; w++) prev[w] = cur[w];
      }
    }
    const CtaScan sc = cta_exscan<kOrderThreads>((uint32_t)__popc(head));
    if (sc.total == m) {  // every key has one row
      __syncthreads();
      continue;
    }
    uint32_t g = sc.excl;
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      const uint32_t i = tid * kPer + k;
      g += (head >> k) & 1u;
      if (i < m) {
        const uint64_t id = b.out_sums[base + i];
        s_id[i] = id;
        s_pre[i] = val_prefix(val_view(arena, voff, id));
        s_grp[i] = g;
      }
    }
    uint32_t np = 1;
    while (np < m) np <<= 1;
    for (uint32_t i = m + tid; i < np; i += kOrderThreads) {
      s_grp[i] = kNoGroup;
      s_pre[i] = 0;
    }
    __syncthreads();
    for (uint32_t k = 2; k <= np; k <<= 1)
      for (uint32_t j = k >> 1; j; j >>= 1) {
        for (uint32_t t = tid; t < np / 2; t += kOrderThreads) {
          const uint32_t lo = (t / j) * 2 * j + t % j, hi = lo + j;
          const bool up = (lo & k) == 0;
          if (after(s_grp[lo], s_pre[lo], s_id[lo], s_grp[hi], s_pre[hi], s_id[hi], arena, voff) == up) {
            const uint32_t tg = s_grp[lo];
            s_grp[lo] = s_grp[hi];
            s_grp[hi] = tg;
            const uint64_t tp = s_pre[lo];
            s_pre[lo] = s_pre[hi];
            s_pre[hi] = tp;
            const uint64_t ti = s_id[lo];
            s_id[lo] = s_id[hi];
            s_id[hi] = ti;
          }
        }
        __syncthreads();
      }
    for (uint32_t i = tid; i < m; i += kOrderThreads) b.out_sums[base + i] = s_id[i];
    __syncthreads();
  }
}

namespace {
template <int RB>
struct RowRef {
  const uint32_t* keys;
  const uint64_t* ids;
};
// row x of r before row y of q: by key, then by value bytes
template <int RB>
__device__ __forceinline__ bool row_less(const RowRef<RB>& r, uint64_t x, const RowRef<RB>& q, uint64_t y,
                                         const unsigned char* __restrict__ arena, const uint64_t* __restrict__ voff) {
  uint32_t a[Rec<RB>::kKeyWords], c[Rec<RB>::kKeyWords];
  load_key<RB>(r.keys, x, a);
  load_key<RB>(q.keys, y, c);
  const int kc = key_cmp<RB>(a, c);
  if (kc) return kc < 0;
  return val_cmp(val_view(arena, voff, r.ids[x]), val_view(arena, voff, q.ids[y])) < 0;
}
}  // namespace

// One CTA per oversized bin big_list[x]: its rows are cap-row chunks, each in (key, value) order; merge passes of width
// cap, 2 cap, ... alternate between the output rows and tmp (same row offsets), each thread taking an equal share of
// the pass's output positions through a merge-path search.  The result ends in the output rows.
template <int RB>
__global__ void __launch_bounds__(kMergeThreads) k_value_merge(ShuffleBuffers b, uint32_t cap,
                                                               const unsigned char* __restrict__ arena,
                                                               const uint64_t* __restrict__ voff, void* tmp_keys,
                                                               uint64_t* tmp_ids) {
  constexpr int KW = Rec<RB>::kKeyWords;
  const uint32_t bin = b.big_list[blockIdx.x];
  const uint64_t n = b.ucount[bin], o = out_start(b, bin);
  RowRef<RB> src{(const uint32_t*)b.out_keys + o * KW, b.out_sums + o};
  RowRef<RB> dst{(const uint32_t*)tmp_keys + o * KW, tmp_ids + o};
  const uint64_t per = (n + kMergeThreads - 1) / kMergeThreads;
  bool in_tmp = false;
  for (uint64_t w = cap; w < n; w <<= 1) {
    uint32_t* dk = (uint32_t*)dst.keys;
    uint64_t* di = (uint64_t*)dst.ids;
    const uint64_t k1 = min(n, (threadIdx.x + 1) * per);
    for (uint64_t k = threadIdx.x * per; k < k1;) {
      const uint64_t p0 = k / (2 * w) * (2 * w), la = min(w, n - p0), lb = min(w, n - p0 - la), d = k - p0;
      // i rows of run A and d - i of run B precede output position p0 + d
      uint64_t lo = d > lb ? d - lb : 0, hi = min(d, la);
      while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (row_less<RB>(src, p0 + mid, src, p0 + la + d - 1 - mid, arena, voff)) lo = mid + 1;
        else hi = mid;
      }
      uint64_t i = lo, j = d - lo;
      const uint64_t end = min(k1, p0 + la + lb);
      for (; k < end; k++) {
        const bool take_a = j >= lb || (i < la && row_less<RB>(src, p0 + i, src, p0 + la + j, arena, voff));
        const uint64_t from = take_a ? p0 + i++ : p0 + la + j++;
#pragma unroll
        for (int q = 0; q < KW; q++) dk[k * KW + q] = src.keys[from * KW + q];
        di[k] = src.ids[from];
      }
    }
    __syncthreads();
    const RowRef<RB> t = src;
    src = dst;
    dst = t;
    in_tmp = !in_tmp;
  }
  if (in_tmp) {
    uint32_t* ok = (uint32_t*)b.out_keys + o * KW;
    for (uint64_t v = threadIdx.x; v < n * KW; v += kMergeThreads) ok[v] = src.keys[v];
    for (uint64_t v = threadIdx.x; v < n; v += kMergeThreads) b.out_sums[o + v] = src.ids[v];
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

// Chunks of an oversized bin ordered by one CTA each, up to this many per bin at a time.
constexpr uint32_t kChunkCtas = 64;

int launch_value_order(int rb, const ShuffleBuffers& b, uint32_t nb, uint32_t nbig, uint32_t cap,
                       const unsigned char* arena, const uint64_t* voff, cudaStream_t s) {
  int n = 0;
  if (nb) {
    DISPATCH_RB(rb, (k_value_order<RB><<<nb, kOrderThreads, 0, s>>>(b, cap, nullptr, arena, voff)));
    n++;
  }
  if (nbig) {
    DISPATCH_RB(rb, (k_value_order<RB><<<dim3(nbig, kChunkCtas), kOrderThreads, 0, s>>>(b, cap, b.big_list, arena, voff)));
    n++;
  }
  return n;
}

int launch_value_merge(int rb, const ShuffleBuffers& b, uint32_t nbig, uint32_t cap, const unsigned char* arena,
                       const uint64_t* voff, void* tmp_keys, uint64_t* tmp_ids, cudaStream_t s) {
  if (!nbig) return 0;
  DISPATCH_RB(rb, (k_value_merge<RB><<<nbig, kMergeThreads, 0, s>>>(b, cap, arena, voff, tmp_keys, tmp_ids)));
  return 1;
}

}  // namespace mrhbm
