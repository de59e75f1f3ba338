// mrhbm_valbytes.cuh -- a byte value (MRHBM_F_BYTE_VALUES) as the kernels read it: value id i has the bytes
// arena[voff[i] .. voff[i+1]), at any alignment of its first byte.  One definition for the distinct set's equality test
// (mrhbm_distinct.cu) and the distinct reducer's order (mrhbm_value_order.cu), host-callable so that
// tests/native/value_order_check.cu checks it against memcmp on the CPU.
#pragma once
#include <cstdint>

#include "mrhbm_kernels.h"  // MRHBM_HD

namespace mrhbm {

// A value's bytes as little-endian 32-bit words, whatever the alignment of its first byte in the arena: word i holds
// bytes 4i .. 4i+3, zero past the end.  Only aligned words that hold a byte of the value are read.
struct ValView {
  const uint32_t* w;
  uint32_t sh;
  uint64_t len;
};
MRHBM_HD inline ValView val_view(const unsigned char* arena, const uint64_t* voff, uint64_t id) {
  const uint64_t s = voff[id];
  ValView v;
  v.len = voff[id + 1] - s;
  v.sh = (uint32_t)(s & 3);
  v.w = (const uint32_t*)(arena + s - v.sh);
  return v;
}
MRHBM_HD inline uint32_t val_load(const uint32_t* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
MRHBM_HD inline uint32_t val_word(const ValView& v, uint64_t i) {
  uint32_t x = val_load(v.w + i);
  if (v.sh) {
    const uint32_t hi = 4 * (i + 1) < v.sh + v.len ? val_load(v.w + i + 1) : 0u;
#ifdef __CUDA_ARCH__
    x = __funnelshift_r(x, hi, 8 * v.sh);
#else
    x = (uint32_t)((((uint64_t)hi << 32) | x) >> (8 * v.sh));
#endif
  }
  const uint64_t rem = v.len - 4 * i;
  return rem < 4 ? x & ((1u << (8 * rem)) - 1) : x;
}
MRHBM_HD inline uint32_t val_bswap(uint32_t x) {
#ifdef __CUDA_ARCH__
  return __byte_perm(x, 0, 0x0123);
#else
  return __builtin_bswap32(x);
#endif
}
// The first 8 bytes as a big-endian number, zero padded: a < b as prefixes implies a < b as values.
MRHBM_HD inline uint64_t val_prefix(const ValView& v) {
  const uint64_t w0 = v.len ? val_bswap(val_word(v, 0)) : 0u, w1 = v.len > 4 ? val_bswap(val_word(v, 1)) : 0u;
  return (w0 << 32) | w1;
}
// Byte order (unsigned bytewise, a proper prefix first: memcmp over the shorter length, then the lengths), from word
// `from` on (the words before it are known equal).  Zero padding cannot decide: where one value has ended, the other's
// byte is >= 0, and equal words leave it to the lengths.
MRHBM_HD inline int val_cmp(const ValView& a, const ValView& b, uint64_t from = 0) {
  const uint64_t na = (a.len + 3) / 4, nb = (b.len + 3) / 4, n = na < nb ? na : nb;
  for (uint64_t i = from; i < n; i++) {
    const uint32_t x = val_word(a, i), y = val_word(b, i);
    if (x != y) return val_bswap(x) < val_bswap(y) ? -1 : 1;
  }
  return (a.len > b.len) - (a.len < b.len);
}
MRHBM_HD inline bool val_eq(const ValView& a, const ValView& b) {
  if (a.len != b.len) return false;
  const uint64_t nw = (a.len + 3) / 4;
  for (uint64_t i = 0; i < nw; i++)
    if (val_word(a, i) != val_word(b, i)) return false;
  return true;
}

}  // namespace mrhbm
