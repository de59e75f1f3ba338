// mrhbm_dev.cuh -- device-side record model, key ordering, partitioners.
//
// Record layouts (little endian words), see include/mrhbm.h:
//   RB=16      : w[0..1] = u64 key, w[2..3] = u64 value (emitters store u32 value, zero pad;
//                in-place partial sums of the big-bin path use all 64 bits)
//   RB=32/64/128: w[0..KW) = key bytes zero padded (no NUL inside), w[KW] = u32 value
// Key order = the reference's keys_sorted / merge order (mapreduce/utils.lua:123-128,214):
// C-locale bytewise, shorter first == big-endian word compare of the zero padded slot;
// u64 keys are the reference's 8-byte big-endian strings (SURVEY A.4) == numeric order.
#pragma once
#include <cstdint>
#include <type_traits>
#include <cuda_runtime.h>

#include "mrhbm_kernels.h"

namespace mrhbm {

template <int RB>
struct Rec {
  static constexpr int kWords = RB / 4;
  static constexpr bool kU64 = (RB == 16);
  static constexpr int kKeyWords = kU64 ? 2 : kWords - 1;  // 32-bit words of key
  static constexpr int kKeyBytes = kKeyWords * 4;
  static constexpr int kVec = RB / 16;  // uint4 per record
};

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  return mix64(x + 0x9E3779B97F4A7C15ull);
}
__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// i-th most significant 32-bit word of the key, as an unsigned big-endian number
template <int RB>
__device__ __forceinline__ uint32_t be_word(const uint32_t* r, int i) {
  if constexpr (Rec<RB>::kU64) {
    return i == 0 ? r[1] : (i == 1 ? r[0] : 0u);
  } else {
    return i < Rec<RB>::kKeyWords ? bswap32(r[i]) : 0u;
  }
}
template <int RB>
__device__ __forceinline__ uint64_t key_prefix64(const uint32_t* r) {
  return ((uint64_t)be_word<RB>(r, 0) << 32) | be_word<RB>(r, 1);
}
// nbits (1..64; the LSD passes take kDigitBits = 52) of the key starting `bitpos` bits below the most significant bit
template <int RB>
__device__ __forceinline__ uint64_t key_bits(const uint32_t* r, int bitpos, int nbits) {
  int wi = bitpos >> 5, sh = bitpos & 31;
  uint64_t hi = ((uint64_t)be_word<RB>(r, wi) << 32) | be_word<RB>(r, wi + 1);
  uint64_t lo = (uint64_t)be_word<RB>(r, wi + 2) << 32;
  uint64_t win = sh ? ((hi << sh) | (lo >> (64 - sh))) : hi;
  return win >> (64 - nbits);
}
template <int RB>
__device__ __forceinline__ int key_cmp(const uint32_t* a, const uint32_t* b) {
  if constexpr (Rec<RB>::kU64) {
    uint64_t x = (uint64_t)a[0] | ((uint64_t)a[1] << 32), y = (uint64_t)b[0] | ((uint64_t)b[1] << 32);
    return (x > y) - (x < y);
  } else {
#pragma unroll
    for (int i = 0; i < Rec<RB>::kKeyWords; i++) {
      uint32_t x = be_word<RB>(a, i), y = be_word<RB>(b, i);
      if (x != y) return x < y ? -1 : 1;
    }
    return 0;
  }
}
template <int RB>
__device__ __forceinline__ bool key_eq(const uint32_t* a, const uint32_t* b) {
  bool e = true;
#pragma unroll
  for (int i = 0; i < Rec<RB>::kKeyWords; i++) e &= (a[i] == b[i]);
  return e;
}
template <int RB>
__device__ __forceinline__ uint64_t rec_value(const uint32_t* r) {
  if constexpr (Rec<RB>::kU64)
    return (uint64_t)r[2] | ((uint64_t)r[3] << 32);
  else
    return r[Rec<RB>::kKeyWords];
}

// ---- partitioners ---------------------------------------------------------
// examples/WordCount/partitionfn.lua:8-16 evaluated exactly as Lua 5.2 does, i.e. in IEEE
// doubles: h*16777619 reaches ~2^56, so the product is rounded to 53 significant bits
// (round-to-nearest-even) BEFORE "% 2^32".  Emulated with integers so no FP64 is issued.
// Only (h * 16777619 rounded to 53 bits) mod 2^32 is needed, and the rounding only touches the
// low `sh` bits, so everything is computed from the 32-bit halves of the product:
// sh = bitlen(product) - 53 = bitlen(high word) - 21.
__host__ __device__ __forceinline__ uint32_t fnv_lua_step(uint32_t h, uint32_t byte) {
  uint32_t lo = h * 16777619u;
#ifdef __CUDA_ARCH__
  uint32_t hi = __umulhi(h, 16777619u);
  int sh = 11 - __clz((int)hi);  // (32 - clz) - 21
#else
  uint32_t hi = (uint32_t)(((uint64_t)h * 16777619ull) >> 32);
  int sh = hi ? 11 - __builtin_clz(hi) : -21;
#endif
  if (sh > 0) {
    uint32_t half = 1u << (sh - 1), rem = lo & ((1u << sh) - 1u);
    uint32_t q = lo >> sh;  // bit 0 of q is bit sh of the product: the ties-to-even parity
    if (rem > half || (rem == half && (q & 1u))) q++;
    lo = q << sh;           // a carry out of bit 31 vanishes mod 2^32, as it must
  }
  return lo ^ byte;
}
// h over the key bytes (u64 keys: the 8 big-endian bytes; strings: up to the first NUL)
template <int RB>
__device__ __forceinline__ uint32_t fnv_lua_hash(const uint32_t* r) {
  uint32_t h = 2166136261u;
  if constexpr (Rec<RB>::kU64) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      uint32_t w = i < 4 ? r[1] : r[0];
      h = fnv_lua_step(h, (w >> (24 - 8 * (i & 3))) & 0xff);
    }
  } else {
    // The word loop is unrolled (the record lives in registers), the byte loop is NOT: fully unrolled,
    // 4 records x 28 bytes of fnv_lua_step overflowed the instruction cache (k_hist<32>
    // stalled on "no instruction").  Key bytes 0x00 / 0x01 are stored escaped (01 01 / 01 02,
    // mrhbm_emit_str); the reference's partitionfn sees the original bytes, so they are restored here.
    bool esc = false;
#pragma unroll
    for (int i = 0; i < Rec<RB>::kKeyWords; i++) {
      uint32_t w = r[i];
      if (w == 0) break;  // keys hold no NUL: a zero word is past the end (short keys leave early)
#pragma unroll 1
      do {
        const uint32_t b = w & 0xffu;
        if (esc) {
          h = fnv_lua_step(h, b - 1u);
          esc = false;
        } else if (b == 1u) {
          esc = true;
        } else {
          h = fnv_lua_step(h, b);
        }
        w >>= 8;
      } while (w);
      if ((r[i] >> 24) == 0) break;
    }
  }
  return h;
}
// 64-bit word hash over the little-endian u32 words of the key bytes while non-zero
// (length-exact for NUL-free keys, independent of the slot width): kWordHashSeed, word_hash_step per word, then
// word_hash_finish.  The host partitions keys longer than a slot with the same steps (mrhbm_keys.h).
constexpr uint64_t kWordHashSeed = 0x9E3779B97F4A7C15ull;
__host__ __device__ __forceinline__ uint64_t word_hash_step(uint64_t h, uint32_t w) {
  h = (h ^ w) * 0xBF58476D1CE4E5B9ull;
  return h ^ (h >> 29);
}
__host__ __device__ __forceinline__ uint64_t word_hash_finish(uint64_t h) {
  h ^= h >> 32;
  return h * 0x94D049BB133111EBull;
}
template <int RB>
__device__ __forceinline__ uint64_t word_hash(const uint32_t* r) {
  uint64_t h = kWordHashSeed;
#pragma unroll
  for (int i = 0; i < Rec<RB>::kKeyWords; i++) {
    uint32_t w;
    if constexpr (Rec<RB>::kU64)
      w = bswap32(i == 0 ? r[1] : r[0]);  // LE load of the 8 big-endian key bytes
    else
      w = r[i];
    if (w == 0) break;  // short keys leave early
    h = word_hash_step(h, w);
  }
  return word_hash_finish(h);
}

// floor(x * m / 2^64) for a 32-bit m: two 32x32 multiplies instead of the four of __umul64hi
__host__ __device__ __forceinline__ uint32_t mulhi_u64_u32(uint64_t x, uint32_t m) {
  const uint64_t lo = (uint64_t)(uint32_t)x * m, hi = (uint64_t)(uint32_t)(x >> 32) * m;
  return (uint32_t)((hi + (lo >> 32)) >> 32);
}

// MRHBM_PART_RANGE: pid = number of thresholds t_i <= slot(key).  Binary search over the 64-bit prefixes (read through
// the read-only cache: the first levels of the search are the same few words for every key), then, for string keys
// whose prefix ties with thresholds, a walk down over the tied ones with the full slot compare.
template <int RB>
__device__ __forceinline__ uint32_t range_pid(const uint32_t* r, const RangeBinParams& bp) {
  const uint64_t kp = key_prefix64<RB>(r);
  uint32_t pos = 0;
  for (uint32_t step = bp.spl_top; step; step >>= 1) {
    const uint32_t q = pos + step;
    if (q <= bp.spl_n && __ldg(bp.spl_pre + q - 1) <= kp) pos = q;
  }
  if constexpr (!Rec<RB>::kU64) {
    constexpr int KW = Rec<RB>::kKeyWords;
    while (pos > 0 && __ldg(bp.spl_pre + pos - 1) == kp) {
      const uint32_t* t = bp.spl_slot + (size_t)(pos - 1) * KW;
      int c = 0;
#pragma unroll
      for (int i = 2; i < KW; i++) {
        const uint32_t x = be_word<RB>(r, i), y = bswap32(__ldg(t + i));
        if (c == 0 && x != y) c = x < y ? -1 : 1;
      }
      if (c >= 0) break;  // key >= t_{pos-1}: so are all below it
      pos--;
    }
  }
  return pos;
}

// MRHBM_PART_RANGE, u64 keys: the position of key inside its partition [lo, lo + w) as a 64-bit fraction,
// floor((key - lo) * F / 2^64) with F = floor((2^128 - 1) / w) = {hi, lo64}: q * hi + mulhi(q, lo64).  Monotone in the
// key and < 2^64 (q < w); 128-bit F keeps it exact where floor(2^64 / w) alone would lose up to 1 / (2^64 / w).
__device__ __forceinline__ uint64_t range_pos(const RangeBinParams& bp, uint64_t key, uint32_t pid) {
  const uint64_t lo = pid ? __ldg(bp.spl_pre + pid - 1) : 0ull;
  const ulonglong2 f = __ldg(bp.spl_inv + pid);
  const uint64_t q = key - lo;
  return q * f.x + __umul64hi(q, f.y);
}

// partition id, owning rank and bin (= slot(pid)*S + sub) of a record held in registers / smem words
// WORLD: 0 = bp.world read at run time, 1 = one GPU, 2 = several (folded by the caller's template)
// BP = RangeBinParams: MRHBM_PART_RANGE, a compile-time variant (the hash instances do not carry its search).  Its
// sub-bins: u64 keys with bp.ordered = mulhi(range_pos, S), monotone in the key and < S, so that a partition is one
// ascending run; otherwise the word hash.
template <int RB, int WORLD = 0, typename BP = BinParams>
__device__ __forceinline__ uint32_t bin_of(const uint32_t* r, const BP& bp, uint32_t* pid_out,
                                           uint32_t* dest_out = nullptr) {
  constexpr bool RANGE = std::is_same<BP, RangeBinParams>::value;
  uint32_t pid;
  uint64_t h = 0;  // uniform 64-bit hash; feeds the hash sub-bin (only computed further when needed)
  const bool mul = bp.partitioner == 1u && Rec<RB>::kU64;
  if constexpr (RANGE) {
    pid = range_pid<RB>(r, bp);
  } else if (mul) {  // MULHASH
    uint64_t key = (uint64_t)r[0] | ((uint64_t)r[1] << 32);
    h = key * 0x9E3779B97F4A7C15ull;
    pid = mulhi_u64_u32(h, bp.P);
  } else if (bp.partitioner == 0u) {  // FNV_LUA
    pid = fnv_lua_hash<RB>(r) % bp.P;
  } else {  // WORDHASH
    h = word_hash<RB>(r);
    pid = mulhi_u64_u32(h, bp.P);
  }
  uint32_t sub = 0;
  if constexpr (RANGE) {
    if (bp.S > 1) {
      uint64_t src;
      if (Rec<RB>::kU64 && bp.ordered) {
        src = range_pos(bp, (uint64_t)r[0] | ((uint64_t)r[1] << 32), pid);
      } else {
        src = word_hash<RB>(r);
      }
      sub = mulhi_u64_u32(src, bp.S);
    }
  } else if (bp.S > 1) {
    uint64_t src;
    if (bp.ordered) {
      src = key_prefix64<RB>(r);
    } else if (bp.partitioner == 0u) {
      src = word_hash<RB>(r);
    } else {
      src = mix64(h * (uint64_t)bp.P + 0x632BE59BD9B4E019ull);  // independent of pid
    }
    sub = mulhi_u64_u32(src, bp.S);
  }
  if (pid_out) *pid_out = pid;
  // partition p is owned by rank p % world and sits in slot pbase[rank] + p / world
  uint32_t slot = pid, dest = 0;
  if (WORLD == 2 || (WORLD == 0 && bp.world > 1)) {
    uint32_t q;
    if (bp.wshift != 0xffffffffu) {  // power-of-two world: no integer division
      dest = pid & (bp.world - 1u);
      q = pid >> bp.wshift;
    } else {
      dest = pid % bp.world;
      q = pid / bp.world;
    }
    slot = bp.pbase[dest] + q;
  }
  if (dest_out) *dest_out = dest;
  return slot * bp.S + sub;
}

// checksum mixers over the whole key slot (input and result share the slot format)
template <int RB>
__device__ __forceinline__ void key_mix2(const uint32_t* r, uint64_t& f1, uint64_t& f2) {
  uint64_t a = 0x243F6A8885A308D3ull, b = 0x13198A2E03707344ull;
#pragma unroll
  for (int i = 0; i < Rec<RB>::kKeyWords; i++) {
    a = mix64(a ^ r[i]);
    b = (b ^ r[i]) * 0x9FB21C651E98DF25ull;
    b ^= b >> 28;
  }
  f1 = a;
  f2 = mix64(b);
}

// ---- streaming global access ------------------------------------------------
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ void stg_stream(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// ---- CTA-wide exclusive scan --------------------------------------------------
// inclusive prefix sum of v over the first WIDTH lanes of the warp (a power of two <= 32)
template <int WIDTH = 32, typename T = uint32_t>
__device__ __forceinline__ T warp_inscan(T v) {
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < WIDTH; d <<= 1) {
    const T t = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= (uint32_t)d) v += t;
  }
  return v;
}
template <typename T>
struct CtaScanT {
  T excl;   // sum of `mine` over the threads before this one
  T total;  // sum of `mine` over the CTA
};
using CtaScan = CtaScanT<uint32_t>;
// One value per thread, THREADS == blockDim.x threads, one barrier: every warp scans the warp totals itself.
// The warp totals live in static scratch that every call in the kernel shares: it may be written again only
// after a barrier that follows every read of it (a barrier after the call, before the next call).
// T: uint32_t (bin counts) or uint64_t (byte offsets of the value gather).
template <int THREADS, typename T = uint32_t>
__device__ __forceinline__ CtaScanT<T> cta_exscan(T mine) {
  constexpr int kWarps = THREADS / 32;
  __shared__ T s_warp[kWarps];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T incl = warp_inscan(mine);
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  const T w = lane < (uint32_t)kWarps ? s_warp[lane] : T(0), wi = warp_inscan<kWarps>(w);
  return {__shfl_sync(0xffffffffu, wi - w, warp) + incl - mine, __shfl_sync(0xffffffffu, wi, kWarps - 1)};
}

}  // namespace mrhbm
