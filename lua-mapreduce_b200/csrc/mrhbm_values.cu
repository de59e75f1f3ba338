// mrhbm_values.cu -- byte values (MRHBM_F_BYTE_VALUES): the map-side stamp of value ids (or of the offsets of a
// tokeniser piece's shared value) and, after the compaction of a group-only result, the per-row value lengths, their
// u64 exclusive scan and the gather of the value bytes from the arena into one buffer in row order.  The split, sort
// and compaction kernels carry the value id unchanged.
#include <cstdint>

#include "mrhbm_dev.cuh"

namespace mrhbm {

namespace {
constexpr int kScanThreads = 1024;
constexpr int kScanPer = (1 << kValTileLog) / kScanThreads;  // rows per thread of a scan tile
constexpr uint32_t kLaneBytes = 16;                          // values this short are copied by one lane each

int sm_count() {
  int dev = 0, n = 132;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    cudaGetLastError();
    n = 132;
  }
  return n;
}
}  // namespace

__global__ void __launch_bounds__(256) k_value_stamp(unsigned char* __restrict__ recs, int rb, uint64_t n, uint64_t first,
                                                     uint64_t* __restrict__ dvoff, uint64_t v0, uint64_t aoff) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += stride) {
    if (!recs) {  // one shared value (mrhbm_map_words_value), v0 its length
      dvoff[i] = i ? aoff + v0 : aoff;
      continue;
    }
    dvoff[i] = dvoff[i] - v0 + aoff;
    if (i == n) continue;
    if (rb == 16)
      *(uint64_t*)(recs + i * 16 + 8) = first + i;
    else
      *(uint32_t*)(recs + i * rb + rb - 4) = (uint32_t)(first + i);
  }
}

// pass 1: one CTA per tile of 2^kValTileLog rows, kScanPer consecutive rows per thread
__global__ void __launch_bounds__(kScanThreads) k_value_lengths(const uint64_t* __restrict__ ids, uint64_t n,
                                                                 const uint64_t* __restrict__ voff,
                                                                 uint64_t* __restrict__ row_off,
                                                                 uint64_t* __restrict__ tile_sum) {
  const uint64_t r0 = ((uint64_t)blockIdx.x << kValTileLog) + (uint64_t)threadIdx.x * kScanPer;
  uint64_t len[kScanPer], sum = 0;
#pragma unroll
  for (int k = 0; k < kScanPer; k++) {
    len[k] = 0;
    if (r0 + k < n) {
      const uint64_t id = ids[r0 + k];
      len[k] = voff[id + 1] - voff[id];
    }
    sum += len[k];
  }
  const CtaScanT<uint64_t> sc = cta_exscan<kScanThreads, uint64_t>(sum);
  uint64_t run = sc.excl;
#pragma unroll
  for (int k = 0; k < kScanPer; k++) {
    if (r0 + k < n) row_off[r0 + k] = run;
    run += len[k];
  }
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = sc.total;
}

// pass 2: one CTA, exclusive scan of the tile totals in place; the grand total goes to *total
__global__ void __launch_bounds__(kScanThreads) k_value_tiles(uint64_t* __restrict__ tile, uint64_t ntiles,
                                                               uint64_t* __restrict__ total) {
  const uint64_t per = (ntiles + kScanThreads - 1) / kScanThreads;
  const uint64_t b0 = threadIdx.x * per, b1 = b0 + per < ntiles ? b0 + per : ntiles;
  uint64_t s = 0;
  for (uint64_t i = b0; i < b1; i++) s += tile[i];
  const CtaScanT<uint64_t> sc = cta_exscan<kScanThreads, uint64_t>(s);
  uint64_t run = sc.excl;
  for (uint64_t i = b0; i < b1; i++) {
    const uint64_t c = tile[i];
    tile[i] = run;
    run += c;
  }
  if (threadIdx.x == 0) *total = sc.total;
}

// One warp copies len bytes: a byte head up to the destination's 16-byte boundary, then 16-byte vectors when the
// source is aligned alike, else aligned 4-byte words assembled from two source words, then a byte tail.
__device__ __forceinline__ void warp_copy(const unsigned char* __restrict__ src, unsigned char* __restrict__ dst,
                                          uint64_t len, uint32_t lane) {
  uint64_t head = (16 - ((uintptr_t)dst & 15)) & 15;
  if (head > len) head = len;
  if (lane < head) dst[lane] = src[lane];
  src += head;
  dst += head;
  len -= head;
  if (((uintptr_t)src & 15) == 0) {
    const uint64_t nv = len >> 4;
    for (uint64_t v = lane; v < nv; v += 32) ((uint4*)dst)[v] = __ldg((const uint4*)src + v);
    src += nv << 4;
    dst += nv << 4;
    len -= nv << 4;
  } else {
    const uint32_t sh = (uint32_t)((uintptr_t)src & 3);
    const uint32_t* sw = (const uint32_t*)(src - sh);
    const uint64_t nw = len >> 2;
    // (with sh > 0 the word after the last one still holds a byte of the value: no read past the value's words)
    for (uint64_t w = lane; w < nw; w += 32)
      ((uint32_t*)dst)[w] = sh ? __funnelshift_r(__ldg(sw + w), __ldg(sw + w + 1), 8 * sh) : __ldg(sw + w);
    src += nw << 2;
    dst += nw << 2;
    len -= nw << 2;
  }
  if (lane < len) dst[lane] = src[lane];
}

// pass 3: tiles of 32 rows per warp.  Each lane completes its row's offset; values of <= kLaneBytes are copied by
// their lane, values of <= kValChunk by the whole warp one after the other, longer ones are listed as pieces for
// k_value_pieces so that one long value does not serialise on one warp.
__global__ void __launch_bounds__(256) k_value_gather(const uint64_t* __restrict__ ids, uint64_t n,
                                                      const uint64_t* __restrict__ voff,
                                                      const unsigned char* __restrict__ arena,
                                                      uint64_t* __restrict__ row_off,
                                                      const uint64_t* __restrict__ tile_pre,
                                                      unsigned char* __restrict__ out, uint64_t* __restrict__ pieces,
                                                      unsigned long long* __restrict__ npieces) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t t = warp; t * 32 < n; t += nwarps) {
    const uint64_t r = t * 32 + lane;
    uint64_t s = 0, len = 0, d = 0;
    if (r < n) {
      const uint64_t id = ids[r];
      s = voff[id];
      len = voff[id + 1] - s;
      d = row_off[r] + tile_pre[r >> kValTileLog];
      row_off[r] = d;
      if (len <= kLaneBytes) {
        for (uint32_t k = 0; k < (uint32_t)len; k++) out[d + k] = arena[s + k];
      } else if (len > kValChunk) {
        const uint64_t np = (len + kValChunk - 1) / kValChunk;
        const uint64_t p0 = atomicAdd(npieces, (unsigned long long)np);
        for (uint64_t p = 0; p < np; p++) pieces[p0 + p] = (r << 32) | p;
      }
    }
    uint32_t mid = __ballot_sync(0xffffffffu, len > kLaneBytes && len <= kValChunk);
    while (mid) {
      const int j = __ffs(mid) - 1;
      mid &= mid - 1;
      const uint64_t sj = __shfl_sync(0xffffffffu, s, j), dj = __shfl_sync(0xffffffffu, d, j),
                     lj = __shfl_sync(0xffffffffu, len, j);
      warp_copy(arena + sj, out + dj, lj, lane);
    }
  }
}

// pass 4: one warp per piece {row << 32 | piece index} of a value longer than kValChunk
__global__ void __launch_bounds__(256) k_value_pieces(const uint64_t* __restrict__ ids, const uint64_t* __restrict__ voff,
                                                      const unsigned char* __restrict__ arena,
                                                      const uint64_t* __restrict__ row_off,
                                                      const uint64_t* __restrict__ pieces,
                                                      const unsigned long long* __restrict__ npieces,
                                                      unsigned char* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5, np = *npieces;
  for (uint64_t q = warp; q < np; q += nwarps) {
    const uint64_t e = pieces[q], r = e >> 32, p = e & 0xffffffffu, id = ids[r];
    const uint64_t s = voff[id], len = voff[id + 1] - s, o = p * kValChunk;
    const uint64_t l = len - o < kValChunk ? len - o : kValChunk;
    warp_copy(arena + s + o, out + row_off[r] + o, l, lane);
  }
}

int launch_value_stamp(int rb, void* recs, uint64_t n, uint64_t first, uint64_t* dvoff, uint64_t v0, uint64_t aoff,
                       cudaStream_t s) {
  const uint64_t blocks = (n + 1 + 255) / 256, cap = (uint64_t)sm_count() * 8;
  k_value_stamp<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, s>>>((unsigned char*)recs, rb, n, first, dvoff, v0, aoff);
  return 1;
}

int launch_value_scan(const uint64_t* ids, uint64_t n, const uint64_t* voff, uint64_t* row_off, uint64_t* tile_pre,
                      cudaStream_t s) {
  const uint64_t nt = val_tiles(n);
  if (nt) k_value_lengths<<<(unsigned)nt, kScanThreads, 0, s>>>(ids, n, voff, row_off, tile_pre);
  k_value_tiles<<<1, kScanThreads, 0, s>>>(tile_pre, nt, row_off + n);
  return nt ? 2 : 1;
}

int launch_value_gather(const uint64_t* ids, uint64_t n, const uint64_t* voff, const unsigned char* arena,
                        uint64_t* row_off, const uint64_t* tile_pre, unsigned char* out, uint64_t* pieces,
                        unsigned long long* npieces, cudaStream_t s) {
  if (!n) return 0;
  const int sms = sm_count();
  const uint64_t warps = (n + 31) / 32, cap = (uint64_t)sms * 64;  // 8 CTAs of 8 warps per SM
  const uint64_t grid = ((warps < cap ? warps : cap) + 7) / 8;
  k_value_gather<<<(unsigned)grid, 256, 0, s>>>(ids, n, voff, arena, row_off, tile_pre, out, pieces, npieces);
  k_value_pieces<<<sms * 8, 256, 0, s>>>(ids, voff, arena, row_off, pieces, npieces, out);
  return 2;
}

}  // namespace mrhbm
