// mrhbm_distinct.cu -- MRHBM_COMBINE_DISTINCT: at the commit of a map job on a byte-values ctx, the job's records are
// reduced to their distinct (key slot, value bytes) pairs, the first copy of each in pool order surviving.
//   k_distinct_mark     every record joins an open-addressing hash set of 16-byte entries {fingerprint, pool index of
//                       the first copy}: it claims an empty entry, or finds the entry of an equal pair and lowers its
//                       index to its own with atomicMin; it remembers the entry
//   k_distinct_count    a record survives when it is its entry's minimum; survivors per tile of kTile records
//   (launch_exscan of the tile counts)
//   k_distinct_scatter  the survivors, whole records in pool order, to a scratch buffer at their tile's offset (for
//                       MRHBM_RED_COUNT_DISTINCT with their value field set to 1)
// The caller copies each range's survivors back to the range's start.  Records move as they are: value ids, voff and
// the arena are not touched.
#include <cstdint>

#include "mrhbm_dev.cuh"
#include "mrhbm_job_tiles.cuh"
#include "mrhbm_valbytes.cuh"

namespace mrhbm {

namespace {
constexpr unsigned long long kEmpty = ~0ull;  // an entry's fingerprint and index before the claim (memset to 0xff)

// the record r (value id id, bytes v) against the record at q: equal key slots and equal value bytes
template <int RB>
__device__ __forceinline__ bool same_pair(const uint32_t* r, uint64_t id, const ValView& v, const uint32_t* __restrict__ q,
                                          const unsigned char* __restrict__ arena, const uint64_t* __restrict__ voff) {
  if (!key_eq<RB>(r, q)) return false;
  const uint64_t qid = rec_value<RB>(q);
  if (qid == id) return true;  // (the pairs of one tokeniser piece share their id)
  return val_eq(val_view(arena, voff, qid), v);
}

__device__ __forceinline__ bool survives(const DistinctRange* __restrict__ rg, uint32_t nr,
                                         const ulonglong2* __restrict__ tab, const uint32_t* __restrict__ slot_of,
                                         uint64_t* p) {
  uint64_t g;
  return tile_record(rg, nr, p, &g) && tab[slot_of[g]].y == *p;
}
}  // namespace

// Linear probing from fingerprint & mask.  An entry is claimed with atomicCAS on its fingerprint; its claimer stores
// its index right after, and a thread that meets the fingerprint waits for that index to compare against the pair it
// stands for.  A fingerprint shared by unequal pairs only costs a compare: the thread probes on.
template <int RB>
__global__ void __launch_bounds__(kDistinctTile) k_distinct_mark(const unsigned char* __restrict__ pool,
                                                                 const DistinctRange* __restrict__ rg, uint32_t nr,
                                                                 const unsigned char* __restrict__ arena,
                                                                 const uint64_t* __restrict__ voff, ulonglong2* tab,
                                                                 uint64_t mask, uint32_t* __restrict__ slot_of) {
  uint64_t p, g;
  if (!tile_record(rg, nr, &p, &g)) return;
  uint32_t r[Rec<RB>::kWords];
  load_record<RB>(pool, p, r);
  const uint64_t id = rec_value<RB>(r);
  const ValView v = val_view(arena, voff, id);
  const uint64_t fp = pair_fingerprint<RB>(r, v);
  for (uint64_t s = fp & mask;; s = (s + 1) & mask) {
    unsigned long long* e = (unsigned long long*)&tab[s];
    unsigned long long f = *(volatile unsigned long long*)e;
    if (f == kEmpty) {
      f = atomicCAS(e, kEmpty, (unsigned long long)fp);
      if (f == kEmpty) {
        atomicMin(e + 1, (unsigned long long)p);
        slot_of[g] = (uint32_t)s;
        return;
      }
    }
    if (f != fp) continue;
    unsigned long long q;
    while ((q = *(volatile unsigned long long*)(e + 1)) == kEmpty) {
    }
    if (same_pair<RB>(r, id, v, (const uint32_t*)(pool + q * RB), arena, voff)) {
      if (p < q) atomicMin(e + 1, (unsigned long long)p);  // (the index only falls: p > q cannot be the minimum)
      slot_of[g] = (uint32_t)s;
      return;
    }
  }
}

__global__ void __launch_bounds__(kDistinctTile) k_distinct_count(const DistinctRange* __restrict__ rg, uint32_t nr,
                                                                  const ulonglong2* __restrict__ tab,
                                                                  const uint32_t* __restrict__ slot_of,
                                                                  uint32_t* __restrict__ tile_cnt) {
  uint64_t p;
  const int n = __syncthreads_count(survives(rg, nr, tab, slot_of, &p));
  if (threadIdx.x == 0) tile_cnt[blockIdx.x] = (uint32_t)n;
}

// ONES (MRHBM_RED_COUNT_DISTINCT): every survivor's value field becomes 1, so the shuffle's integer sum of a key's
// rows is its count of distinct values; the existing callers keep the value ids.
template <int RB, bool ONES>
__global__ void __launch_bounds__(kDistinctTile) k_distinct_scatter(const unsigned char* __restrict__ pool,
                                                                    const DistinctRange* __restrict__ rg, uint32_t nr,
                                                                    const ulonglong2* __restrict__ tab,
                                                                    const uint32_t* __restrict__ slot_of,
                                                                    const uint32_t* __restrict__ tile_off,
                                                                    unsigned char* __restrict__ out) {
  uint64_t p = 0;
  const bool keep = survives(rg, nr, tab, slot_of, &p);
  const uint32_t rank = cta_exscan<kDistinctTile>(keep ? 1u : 0u).excl;
  if (!keep) return;
  const uint4* src = (const uint4*)(pool + p * RB);
  uint4* dst = (uint4*)(out + ((uint64_t)tile_off[blockIdx.x] + rank) * RB);
#pragma unroll
  for (int i = 0; i < Rec<RB>::kVec - (ONES ? 1 : 0); i++) dst[i] = __ldg(src + i);
  if constexpr (ONES) {  // the value field ends the record: the last vector's .z/.w for u64 keys, its .w for strings
    uint4 last = __ldg(src + Rec<RB>::kVec - 1);
    if constexpr (Rec<RB>::kU64) last.z = 1u;
    last.w = Rec<RB>::kU64 ? 0u : 1u;
    dst[Rec<RB>::kVec - 1] = last;
  }
}

int launch_distinct_mark(int rb, const void* pool, const DistinctRange* rg, uint32_t nr, uint32_t ntiles,
                         const unsigned char* arena, const uint64_t* voff, void* tab, uint64_t mask, uint32_t* slot_of,
                         cudaStream_t s) {
  if (!ntiles) return 0;
  const unsigned char* P = (const unsigned char*)pool;
  ulonglong2* T = (ulonglong2*)tab;
  switch (rb) {
    case 16: k_distinct_mark<16><<<ntiles, kDistinctTile, 0, s>>>(P, rg, nr, arena, voff, T, mask, slot_of); break;
    case 32: k_distinct_mark<32><<<ntiles, kDistinctTile, 0, s>>>(P, rg, nr, arena, voff, T, mask, slot_of); break;
    case 64: k_distinct_mark<64><<<ntiles, kDistinctTile, 0, s>>>(P, rg, nr, arena, voff, T, mask, slot_of); break;
    default: k_distinct_mark<128><<<ntiles, kDistinctTile, 0, s>>>(P, rg, nr, arena, voff, T, mask, slot_of); break;
  }
  return 1;
}

int launch_distinct_count(const DistinctRange* rg, uint32_t nr, uint32_t ntiles, const void* tab, const uint32_t* slot_of,
                          uint32_t* tile_cnt, cudaStream_t s) {
  if (!ntiles) return 0;
  k_distinct_count<<<ntiles, kDistinctTile, 0, s>>>(rg, nr, (const ulonglong2*)tab, slot_of, tile_cnt);
  return 1;
}

int launch_distinct_scatter(int rb, const void* pool, const DistinctRange* rg, uint32_t nr, uint32_t ntiles,
                            const void* tab, const uint32_t* slot_of, const uint32_t* tile_off, void* out, bool ones,
                            cudaStream_t s) {
  if (!ntiles) return 0;
  const unsigned char* P = (const unsigned char*)pool;
  const ulonglong2* T = (const ulonglong2*)tab;
  unsigned char* O = (unsigned char*)out;
#define SCATTER(RB)                                                                                                   \
  (ones ? k_distinct_scatter<RB, true><<<ntiles, kDistinctTile, 0, s>>>(P, rg, nr, T, slot_of, tile_off, O)            \
        : k_distinct_scatter<RB, false><<<ntiles, kDistinctTile, 0, s>>>(P, rg, nr, T, slot_of, tile_off, O))
  switch (rb) {
    case 16: SCATTER(16); break;
    case 32: SCATTER(32); break;
    case 64: SCATTER(64); break;
    default: SCATTER(128); break;
  }
#undef SCATTER
  return 1;
}

}  // namespace mrhbm
