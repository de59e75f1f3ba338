// mrhbm_num_sum.cu -- MRHBM_RED_FSUM: after the group-only sort (rows of a bin ascending by key, value ids in out_sums)
// every key's values, Lua numbers (mrhbm_numsum.cuh), are summed exactly and rounded once, and the bin keeps one row
// per key whose out_sums holds the sum's double bits.
//   k_num_key_merge  oversized bins only: the cap-row chunks k_big_bins leaves, each ascending by key, merged into
//                  one key-ordered run, one launch per pass of doubling width, each bin's rows spread over many CTAs.
//   k_num_sum      one CTA per bin of at most `cap` rows (or per cap-row chunk of an oversized bin's run): the key groups are numbered with one CTA scan, a group of one or
//                  two values is added by one thread (IEEE addition of two doubles is their exact sum rounded once),
//                  a longer one by a warp into a shared-memory superaccumulator with 64-bit shared atomics.  A bin is
//                  compacted in place.  In an oversized bin a group that crosses a chunk edge leaves each chunk's
//                  part as a partial accumulator in HBM (NumScratch), and the other groups' sums land in their first
//                  row.
//   k_num_merge    one warp per chunk that starts such a group: its partial plus those of the chunks it runs into,
//                  rounded, into the group's first row.
//   k_num_compact  one CTA per oversized bin: its groups' first rows moved to the front, chunk after chunk.
#include <cstdint>
#include <utility>

#include "mrhbm_dev.cuh"
#include "mrhbm_numsum.cuh"
#include "mrhbm_valbytes.cuh"

namespace mrhbm {

namespace {
constexpr int kSumThreads = 256, kSumWarps = kSumThreads / 32, kMergeThreads = 256;
// a chunk's flags: its first rows continue a group of the chunk before (LEAD, their partial is at 2 slot), its last
// group starts in it and goes on (TAIL, at 2 slot + 1), or its rows are all one group that goes on (THROUGH)
enum : uint32_t { CHUNK_LEAD = 1, CHUNK_TAIL = 2, CHUNK_THROUGH = 4 };

template <int RB>
__device__ __forceinline__ void load_key(const uint32_t* keys, uint64_t row, uint32_t* k) {
#pragma unroll
  for (int i = 0; i < Rec<RB>::kKeyWords; i++) k[i] = keys[row * Rec<RB>::kKeyWords + i];
}

__device__ __forceinline__ void acc_add_shared(int64_t* w, uint64_t bits) {
  const NumTerm t = num_term(bits);
#pragma unroll
  for (int k = 0; k < 3; k++)
    if (t.d[k]) atomicAdd((unsigned long long*)&w[t.i + k], (unsigned long long)t.d[k]);
  if (t.flag) atomicOr((unsigned long long*)&w[kAccFlags], (unsigned long long)t.flag);
}
}  // namespace

// list == nullptr: CTA x sums bin x when it holds at most cap rows.  Else CTA (x, y) sums the chunks y, y + gridDim.y,
// ... of oversized bin list[x] (exact layout: rows are global row indices).
template <int RB>
__global__ void __launch_bounds__(kSumThreads) k_num_sum(ShuffleBuffers b, uint32_t cap, const uint32_t* list,
                                                         const unsigned char* __restrict__ arena,
                                                         const uint64_t* __restrict__ voff, NumScratch sc) {
  constexpr int KW = Rec<RB>::kKeyWords, kMax = kCapBytes / RB, kPer = kMax / kSumThreads;
  __shared__ uint64_t s_val[kMax];
  __shared__ uint32_t s_start[kMax + 1];
  __shared__ int64_t s_acc[kSumWarps][kAccWords];
  __shared__ uint32_t s_lead, s_tail;
  // An abandoned optimistic attempt (a full bin or region): a bin's count may cover slots no record was written to, so
  // their value ids are not to be followed.  The exact layout sums the pairs again.
  if (b.counters[CNT_ERR] & ERRF_CAPACITY) return;
  const uint32_t bin = list ? list[blockIdx.x] : blockIdx.x;
  const uint32_t n = b.ucount[bin];
  if (list ? n <= cap : n > cap) return;
  const uint32_t* keys = (const uint32_t*)b.out_keys;
  const uint64_t o = out_start(b, bin);
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint64_t c0 = (uint64_t)blockIdx.y * cap; c0 < n; c0 += (uint64_t)gridDim.y * cap) {
    const uint32_t m = (uint32_t)min((uint64_t)cap, n - c0);
    const uint64_t base = o + c0;
    uint32_t head = 0, bad = 0;
    uint32_t prev[KW], cur[KW];
    if (tid * kPer < m && (tid > 0 || c0 > 0)) load_key<RB>(keys, base + tid * kPer - 1, prev);
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      const uint32_t i = tid * kPer + k;
      if (i < m) {
        load_key<RB>(keys, base + i, cur);
        if ((i == 0 && c0 == 0) || !key_eq<RB>(cur, prev)) head |= 1u << k;
#pragma unroll
        for (int w = 0; w < KW; w++) prev[w] = cur[w];
        const ValView v = val_view(arena, voff, b.out_sums[base + i]);
        uint64_t bits = 0;
        if (v.len != kNumBytes || !num_decode_words(val_word(v, 0), val_word(v, 1), val_word(v, 2), &bits)) {
          bad = 1;
          bits = 0;
        }
        s_val[i] = bits;
      }
    }
    if (tid == 0) {
      s_lead = !(head & 1u);  // the chunk's first rows continue a group of the chunk before
      uint32_t t = 0;
      if (c0 + m < n) {  // ... and its last rows a group of the next one
        uint32_t a[KW], z[KW];
        load_key<RB>(keys, base + m - 1, a);
        load_key<RB>(keys, base + m, z);
        t = key_eq<RB>(a, z);
      }
      s_tail = t;
    }
    const CtaScan scan = cta_exscan<kSumThreads>((uint32_t)__popc(head));
    __syncthreads();
    const uint32_t lead = s_lead, G = scan.total + lead;
    {
      uint32_t g = scan.excl + lead;
#pragma unroll
      for (int k = 0; k < kPer; k++)
        if ((head >> k) & 1u) s_start[g++] = tid * kPer + k;
      if (tid == 0) {
        s_start[0] = 0;
        s_start[G] = m;
      }
    }
    __syncthreads();
    const bool tail_part = s_tail && !(G == 1 && lead);  // the last group starts here and goes on
    auto partial = [&](uint32_t g) { return (g == 0 && lead) || (g == G - 1 && tail_part); };
    // groups of one or two values: one thread each
    for (uint32_t g = tid; g < G; g += kSumThreads) {
      const uint32_t a = s_start[g], e = s_start[g + 1];
      if (e - a > 2 || partial(g)) continue;
      if (e - a == 2) {
        const double x = __dadd_rn(__longlong_as_double((long long)s_val[a]), __longlong_as_double((long long)s_val[a + 1]));
        s_val[a] = (uint64_t)__double_as_longlong(x);
        if (x != x) bad |= 2;
      }
    }
    // longer groups, and the parts of groups that cross a chunk edge: one warp each
    int64_t* acc = s_acc[warp];
    for (uint32_t g = warp; g < G; g += kSumWarps) {
      const uint32_t a = s_start[g], e = s_start[g + 1];
      const bool part = partial(g);
      if (e - a <= 2 && !part) continue;
      for (int k = lane; k < kAccWords; k += 32) acc[k] = 0;
      __syncwarp();
      for (uint32_t i = a + lane; i < e; i += 32) acc_add_shared(acc, s_val[i]);
      __syncwarp();
      if (part) {
        const uint64_t slot = num_slot(base, cap, c0 == 0);
        int64_t* dst = sc.acc + (2 * slot + (g == 0 && lead ? 0 : 1)) * kAccWords;
        for (int k = lane; k < kAccWords; k += 32) dst[k] = acc[k];
      } else if (lane == 0) {
        uint64_t bits;
        if (!acc_round(acc, &bits)) bad |= 2;
        s_val[a] = bits;
      }
      __syncwarp();
    }
    if (bad) atomicOr(b.counters + CNT_ERR, (bad & 1 ? (uint32_t)ERRF_NOTNUM : 0u) | (bad & 2 ? (uint32_t)ERRF_NAN : 0u));
    __syncthreads();
    if (!list) {  // the whole bin: its groups to the front, in place
      uint32_t gk[kPer][KW];
#pragma unroll
      for (int k = 0; k < kPer; k++) {
        const uint32_t g = tid + k * kSumThreads;
        if (g < G) load_key<RB>(keys, base + s_start[g], gk[k]);
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kPer; k++) {
        const uint32_t g = tid + k * kSumThreads;
        if (g < G) {
#pragma unroll
          for (int w = 0; w < KW; w++) ((uint32_t*)b.out_keys)[(base + g) * KW + w] = gk[k][w];
          b.out_sums[base + g] = s_val[s_start[g]];
        }
      }
      if (tid == 0) b.ucount[bin] = G;
    } else {  // a chunk of an oversized bin: each sum in its group's first row; k_num_merge and k_num_compact go on
      for (uint32_t g = tid; g < G; g += kSumThreads)
        if (!partial(g)) b.out_sums[base + s_start[g]] = s_val[s_start[g]];
      if (tid == 0) {
        const uint64_t slot = num_slot(base, cap, c0 == 0);
        sc.flags[slot] = (lead ? CHUNK_LEAD : 0u) | (tail_part ? CHUNK_TAIL : 0u) | (s_tail && G == 1 && lead ? CHUNK_THROUGH : 0u);
        if (tail_part) sc.head_row[slot] = (uint32_t)(base + s_start[G - 1]);
      }
    }
    __syncthreads();
  }
}

// One warp per chunk (y, y + gridDim.y, ... of oversized bin big_list[x]) whose last group starts in it and goes on:
// its partial, plus the leading partials of the chunks after it up to the one where the group ends, rounded into the
// group's first row.
__global__ void __launch_bounds__(32) k_num_merge(ShuffleBuffers b, uint32_t cap, NumScratch sc) {
  __shared__ int64_t acc[kAccWords];
  const uint32_t bin = b.big_list[blockIdx.x], lane = threadIdx.x;
  const uint64_t n = b.ucount[bin], o = out_start(b, bin);
  for (uint64_t c0 = (uint64_t)blockIdx.y * cap; c0 < n; c0 += (uint64_t)gridDim.y * cap) {
    const uint64_t slot = num_slot(o + c0, cap, c0 == 0);
    if (!(sc.flags[slot] & CHUNK_TAIL)) continue;
    const int64_t* t = sc.acc + (2 * slot + 1) * kAccWords;
    for (int k = lane; k < kAccWords; k += 32) acc[k] = t[k];
    for (uint64_t c1 = c0 + cap; c1 < n; c1 += cap) {
      const uint64_t s1 = num_slot(o + c1, cap, false);
      const uint32_t f = sc.flags[s1];
      if (!(f & CHUNK_LEAD)) break;
      const int64_t* l = sc.acc + 2 * s1 * kAccWords;
      for (int k = lane; k < kAccWords; k += 32) acc[k] = k == kAccFlags ? (acc[k] | l[k]) : acc[k] + l[k];
      if (!(f & CHUNK_THROUGH)) break;
    }
    __syncwarp();
    if (lane == 0) {
      uint64_t bits;
      if (!acc_round(acc, &bits)) atomicOr(b.counters + CNT_ERR, (uint32_t)ERRF_NAN);
      b.out_sums[sc.head_row[slot]] = bits;
    }
    __syncwarp();
  }
}

// One CTA per oversized bin big_list[x]: the first row of every group (key, sum) moved to the front of the bin, one
// chunk after the other (the rows written never reach the chunk being read); ucount[bin] becomes the group count.
template <int RB>
__global__ void __launch_bounds__(kSumThreads) k_num_compact(ShuffleBuffers b, uint32_t cap) {
  constexpr int KW = Rec<RB>::kKeyWords, kPer = kCapBytes / RB / kSumThreads;
  __shared__ uint32_t s_prev[KW];
  const uint32_t bin = b.big_list[blockIdx.x], tid = threadIdx.x;
  const uint32_t n = b.ucount[bin];
  const uint64_t o = out_start(b, bin);
  uint32_t* keys = (uint32_t*)b.out_keys;
  uint64_t done = 0;
  for (uint64_t c0 = 0; c0 < n; c0 += cap) {
    const uint32_t m = (uint32_t)min((uint64_t)cap, n - c0);
    const uint64_t base = o + c0;
    uint32_t head = 0, prev[KW], rk[kPer][KW];
    uint64_t rs[kPer];
    if (tid * kPer < m) {
      if (tid > 0) load_key<RB>(keys, base + tid * kPer - 1, prev);
      else
#pragma unroll
        for (int w = 0; w < KW; w++) prev[w] = s_prev[w];
    }
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      const uint32_t i = tid * kPer + k;
      if (i < m) {
        load_key<RB>(keys, base + i, rk[k]);
        if ((i == 0 && c0 == 0) || !key_eq<RB>(rk[k], prev)) head |= 1u << k;
#pragma unroll
        for (int w = 0; w < KW; w++) prev[w] = rk[k][w];
        rs[k] = b.out_sums[base + i];
      }
    }
    const CtaScan scan = cta_exscan<kSumThreads>((uint32_t)__popc(head));
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kPer; k++)
      if (tid * kPer + k == m - 1)  // the next chunk's first row compares with it (after the barrier below)
#pragma unroll
        for (int w = 0; w < KW; w++) s_prev[w] = rk[k][w];
    uint64_t d = o + done + scan.excl;
#pragma unroll
    for (int k = 0; k < kPer; k++)
      if ((head >> k) & 1u) {
#pragma unroll
        for (int w = 0; w < KW; w++) keys[d * KW + w] = rk[k][w];
        b.out_sums[d++] = rs[k];
      }
    done += scan.total;
    __syncthreads();
  }
  if (tid == 0) b.ucount[bin] = (uint32_t)done;
}

// One merge pass of width w over every oversized bin big_list[x]: runs [p0, p0 + w) and [p0 + w, p0 + 2 w) of the bin's
// rows (each ascending by key) merged from src into dst (row offsets as out_keys / out_sums), a bin of at most w rows
// copied.  The bin's output positions are split evenly over the gridDim.y CTAs of row x, each thread finding its start
// with a merge-path search, so a hot key's bin is merged by many CTAs at once.  Equal keys take the second run first:
// the order of a key's rows does not matter to its sum.
template <int RB>
__global__ void __launch_bounds__(kMergeThreads) k_num_key_merge(ShuffleBuffers b, uint64_t w, const uint32_t* sk,
                                                                 const uint64_t* si, uint32_t* dk, uint64_t* di) {
  constexpr int KW = Rec<RB>::kKeyWords;
  const uint32_t bin = b.big_list[blockIdx.x];
  const uint64_t n = b.ucount[bin], o = out_start(b, bin);
  const uint64_t threads = (uint64_t)gridDim.y * kMergeThreads, t = (uint64_t)blockIdx.y * kMergeThreads + threadIdx.x;
  const uint64_t per = (n + threads - 1) / threads, k0 = min(n, t * per), k1 = min(n, k0 + per);
  const uint32_t* src = sk + o * KW;
  const uint64_t* sid = si + o;
  uint32_t* dst = dk + o * KW;
  uint64_t* did = di + o;
  auto less = [&](uint64_t x, uint64_t y) {
    uint32_t a[KW], c[KW];
    load_key<RB>(src, x, a);
    load_key<RB>(src, y, c);
    return key_cmp<RB>(a, c) < 0;
  };
  for (uint64_t k = k0; k < k1;) {
    const uint64_t p0 = w >= n ? 0 : k / (2 * w) * (2 * w), la = min(w, n - p0), lb = min(w, n - p0 - la), d = k - p0;
    // i rows of run A and d - i of run B precede output position p0 + d
    uint64_t lo = d > lb ? d - lb : 0, hi = min(d, la);
    while (lo < hi) {
      const uint64_t mid = (lo + hi) >> 1;
      if (less(p0 + mid, p0 + la + d - 1 - mid)) lo = mid + 1;
      else hi = mid;
    }
    uint64_t i = lo, j = d - lo;
    const uint64_t end = min(k1, p0 + la + lb);
    for (; k < end; k++) {
      const bool take_a = j >= lb || (i < la && less(p0 + i, p0 + la + j));
      const uint64_t from = take_a ? p0 + i++ : p0 + la + j++;
#pragma unroll
      for (int q = 0; q < KW; q++) dst[k * KW + q] = src[from * KW + q];
      did[k] = sid[from];
    }
  }
}

// Compacted rows (ids[r]: the sum's double bits; COUNTS: an integer count below 2^53, so exact as a double) -> their
// encoded values: row r's 11 bytes at vals + 11 r, row_off[r] = 11 r (n + 1 entries), and ids[r] = r, the row's value id.
template <bool COUNTS>
__global__ void k_num_encode(uint64_t* ids, uint64_t n, unsigned char* vals, uint64_t* row_off) {
  for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r <= n; r += (uint64_t)gridDim.x * blockDim.x) {
    row_off[r] = kNumBytes * r;
    if (r < n) {
      const uint64_t x = ids[r];
      num_encode(COUNTS ? (uint64_t)__double_as_longlong((double)x) : x, vals + kNumBytes * r);
      ids[r] = r;
    }
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

// Chunks of an oversized bin summed by one CTA (merged by one warp) each, up to this many per bin at a time.
constexpr uint32_t kSumChunkCtas = 128;

int launch_num_sum(int rb, const ShuffleBuffers& b, uint32_t nb, uint32_t nbig, uint32_t cap, const unsigned char* arena,
                   const uint64_t* voff, const NumScratch& sc, cudaStream_t s) {
  int n = 0;
  if (nb) {
    DISPATCH_RB(rb, (k_num_sum<RB><<<nb, kSumThreads, 0, s>>>(b, cap, nullptr, arena, voff, sc)));
    n++;
  }
  if (nbig) {
    DISPATCH_RB(rb, (k_num_sum<RB><<<dim3(nbig, kSumChunkCtas), kSumThreads, 0, s>>>(b, cap, b.big_list, arena, voff, sc)));
    k_num_merge<<<dim3(nbig, kSumChunkCtas), 32, 0, s>>>(b, cap, sc);
    DISPATCH_RB(rb, (k_num_compact<RB><<<nbig, kSumThreads, 0, s>>>(b, cap)));
    n += 3;
  }
  return n;
}

// CTAs per oversized bin in each merge pass
constexpr uint32_t kMergeCtas = 32;

int launch_num_key_merge(int rb, const ShuffleBuffers& b, uint32_t nbig, uint32_t cap, uint64_t max_rows, void* tmp_keys,
                         uint64_t* tmp_ids, cudaStream_t s) {
  if (!nbig) return 0;
  int n = 0;
  uint32_t *ak = (uint32_t*)b.out_keys, *bk = (uint32_t*)tmp_keys;
  uint64_t *ai = b.out_sums, *bi = tmp_ids;
  bool in_tmp = false;
  const dim3 grid(nbig, kMergeCtas);
  for (uint64_t w = cap; w < max_rows; w <<= 1, n++) {
    DISPATCH_RB(rb, (k_num_key_merge<RB><<<grid, kMergeThreads, 0, s>>>(b, w, ak, ai, bk, bi)));
    std::swap(ak, bk);
    std::swap(ai, bi);
    in_tmp = !in_tmp;
  }
  if (in_tmp) {  // one more pass whose width covers every bin: a copy back into the output rows
    DISPATCH_RB(rb, (k_num_key_merge<RB><<<grid, kMergeThreads, 0, s>>>(b, ~0ull >> 1, ak, ai, bk, bi)));
    n++;
  }
  return n;
}

int launch_num_encode(uint64_t* ids, uint64_t n, unsigned char* vals, uint64_t* row_off, cudaStream_t s, bool counts) {
  const uint64_t blocks = (n + 256) / 256 < 4096 ? (n + 256) / 256 : 4096;
  if (counts)
    k_num_encode<true><<<(unsigned)blocks, 256, 0, s>>>(ids, n, vals, row_off);
  else
    k_num_encode<false><<<(unsigned)blocks, 256, 0, s>>>(ids, n, vals, row_off);
  return 1;
}

}  // namespace mrhbm
