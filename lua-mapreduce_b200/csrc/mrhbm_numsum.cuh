// mrhbm_numsum.cuh -- MRHBM_RED_FSUM: a byte value as a Lua number, and the exact sum of many of them, rounded once.
// One definition for the kernels (mrhbm_num_sum.cu, and MRHBM_COMBINE_FSUM's split in mrhbm_num_combine.cu) and the
// host's long keys (mrhbm_api.cu), host-callable so that tests/native/num_sum_check.cu and fsum_split_check.cu check it
// against exact rational arithmetic on the CPU.
//
// Number encoding (include/mrhbm.h, mapreduce/tuple.py _enc_num, hbm.lua enc_num): 11 bytes, 0x10, then the IEEE
// double's bits u sign-folded (u | 2^63 for a sign bit of 0, ~u otherwise) as ten big-endian 7-bit groups, each OR 0x80
// (the first group holds bit 63 alone).
//
// The accumulator is a small superaccumulator (R. M. Neal, "Fast exact summation using small and large
// superaccumulators", 2015): a finite double is m * 2^(p - 1074) with an integer m < 2^53 and 0 <= p <= 2045, so
// m << (p & 31) lands in three 32-bit digits from digit p >> 5 on.  Digits are int64 and take each addend's signed
// 32-bit pieces without carrying, so fewer than 2^31 addends per digit cannot overflow; carries are propagated once,
// when the sum is rounded.  Infinities, NaN and "some value is not -0" are kept as flags in the last word.
#pragma once
#include <cstdint>
#include <cstring>

#include "mrhbm_kernels.h"  // MRHBM_HD

namespace mrhbm {

// (forced inline in the kernels: an out-of-line call spills its caller's registers to the stack)
#ifdef __CUDACC__
#define MRHBM_HDI __host__ __device__ __forceinline__
#else
#define MRHBM_HDI inline
#endif

constexpr int kNumBytes = 11;      // an encoded number
constexpr int kAccDigits = 67;     // 2^-1074 .. past 2^(1024 + 31): 67 x 32 bits
constexpr int kAccWords = 68;      // the digits and the flags word
constexpr int kAccFlags = 67;      // index of the flags word
enum : uint64_t { NUM_PINF = 1, NUM_NINF = 2, NUM_NAN = 4, NUM_NOT_NEG0 = 8 };
constexpr uint64_t kDblInf = 0x7ff0000000000000ull;

// The double's bits of an encoded number held in the little-endian words w0..w2 (bytes 0..11; byte 11 is ignored),
// or false when the 11 bytes are not a number encoding (a wrong tag, a group without bit 7, a first group above 1) or
// encode a NaN.
MRHBM_HDI bool num_decode_words(uint32_t w0, uint32_t w1, uint32_t w2, uint64_t* bits) {
  if ((w0 & 0xff) != 0x10) return false;
  uint64_t u = 0;
  bool ok = true;
  for (int k = 1; k < kNumBytes; k++) {
    const uint32_t w = k < 4 ? w0 : k < 8 ? w1 : w2;
    const uint32_t b = (w >> (8 * (k & 3))) & 0xff;
    ok &= (b & 0x80) != 0;
    u = (u << 7) | (b & 0x7f);
  }
  ok &= ((w0 >> 8) & 0x7f) <= 1;
  const uint64_t x = (u >> 63) ? (u & ~(1ull << 63)) : ~u;
  *bits = x;
  return ok && (x & ~(1ull << 63)) <= kDblInf;
}
MRHBM_HDI bool num_decode(const unsigned char* p, uint64_t len, uint64_t* bits) {
  if (len != kNumBytes) return false;
  uint32_t w[3] = {0, 0, 0};
  for (int k = 0; k < kNumBytes; k++) w[k >> 2] |= (uint32_t)p[k] << (8 * (k & 3));
  return num_decode_words(w[0], w[1], w[2], bits);
}
MRHBM_HDI void num_encode(uint64_t bits, unsigned char* out) {
  const uint64_t u = (bits >> 63) ? ~bits : (bits | (1ull << 63));
  out[0] = 0x10;
  for (int k = 0; k < 10; k++) out[1 + k] = (unsigned char)(0x80 | ((u >> (63 - 7 * k)) & 0x7f));
}

// What one double adds to an accumulator: d[0..2] to digits i .. i+2 and `flag` to the flags word.  Infinities and NaN
// only set their flag.
struct NumTerm {
  int i;
  int64_t d[3];
  uint64_t flag;
};
MRHBM_HDI NumTerm num_term(uint64_t bits) {
  NumTerm t{0, {0, 0, 0}, bits == (1ull << 63) ? 0ull : (uint64_t)NUM_NOT_NEG0};
  const uint32_t e = (uint32_t)(bits >> 52) & 0x7ff;
  const bool neg = bits >> 63;
  if (e == 0x7ff) {
    t.flag |= (bits & ((1ull << 52) - 1)) ? (uint64_t)NUM_NAN : neg ? (uint64_t)NUM_NINF : (uint64_t)NUM_PINF;
    return t;
  }
  const uint64_t m = (bits & ((1ull << 52) - 1)) | (e ? (1ull << 52) : 0);
  const uint32_t p = e ? e - 1 : 0, off = p & 31;
  const uint64_t lo = m << off, hi = off ? m >> (64 - off) : 0;
  t.i = (int)(p >> 5);
  t.d[0] = (int64_t)(lo & 0xffffffffu);
  t.d[1] = (int64_t)(lo >> 32);
  t.d[2] = (int64_t)hi;
  if (neg)
    for (int k = 0; k < 3; k++) t.d[k] = -t.d[k];
  return t;
}
MRHBM_HDI void acc_clear(int64_t* w) {
  for (int k = 0; k < kAccWords; k++) w[k] = 0;
}
// (host: the kernels add the same terms with shared-memory atomics)
MRHBM_HDI void acc_add(int64_t* w, uint64_t bits) {
  const NumTerm t = num_term(bits);
  for (int k = 0; k < 3; k++) w[t.i + k] += t.d[k];
  w[kAccFlags] |= (int64_t)t.flag;
}
MRHBM_HDI void acc_merge(int64_t* w, const int64_t* o) {
  for (int k = 0; k < kAccDigits; k++) w[k] += o[k];
  w[kAccFlags] |= o[kAccFlags];
}

namespace detail {
MRHBM_HDI void acc_carry(int64_t* w) {
#pragma unroll 1
  for (int k = 0; k + 1 < kAccDigits; k++) {
    const int64_t c = w[k] >> 32;  // floor: leaves the digit in [0, 2^32)
    w[k] -= c * 4294967296ll;
    w[k + 1] += c;
  }
}
MRHBM_HDI int clz32(uint32_t x) {
#ifdef __CUDA_ARCH__
  return __clz(x);
#else
  return __builtin_clz(x);
#endif
}
}  // namespace detail

// The accumulated sum rounded to the nearest double, ties to even, into *bits; the accumulator is consumed.  A sum
// whose magnitude rounds beyond DBL_MAX is +-inf; infinities of one sign give that infinity; an exact zero is +0
// unless every value was -0.  Returns false for a NaN (a NaN value, or +inf with -inf).
MRHBM_HDI bool acc_round(int64_t* w, uint64_t* bits) {
  const uint64_t f = (uint64_t)w[kAccFlags];
  if ((f & NUM_NAN) || ((f & NUM_PINF) && (f & NUM_NINF))) return false;
  if (f & (NUM_PINF | NUM_NINF)) {
    *bits = kDblInf | ((f & NUM_NINF) ? 1ull << 63 : 0);
    return true;
  }
  detail::acc_carry(w);
  uint64_t sign = 0;
  if (w[kAccDigits - 1] < 0) {  // negative: round the magnitude
    sign = 1ull << 63;
#pragma unroll 1
    for (int k = 0; k < kAccDigits; k++) w[k] = -w[k];
    detail::acc_carry(w);
  }
  int h = kAccDigits - 1;
  while (h >= 0 && w[h] == 0) h--;
  if (h < 0) {
    *bits = (f & NUM_NOT_NEG0) ? 0ull : 1ull << 63;
    return true;
  }
  const int L = 32 * h + 32 - detail::clz32((uint32_t)w[h]);  // bits of the integer M; the sum is M * 2^-1074
  if (L <= 53) {  // exact: the double whose bits are M is M * 2^-1074 (subnormal below 2^52)
    *bits = sign | ((uint64_t)(h ? w[1] : 0) << 32 | (uint64_t)w[0]);
    return true;
  }
  const int shift = L - 53, pos = shift - 1, idx = pos >> 5, off = pos & 31;
  const uint64_t lo = (uint64_t)w[idx] | ((uint64_t)w[idx + 1] << 32), hi = (uint64_t)w[idx + 2];
  const uint64_t x = (lo >> off) | (off ? hi << (64 - off) : 0);  // bits pos .. pos + 53 of M
  bool sticky = ((uint64_t)w[idx] & ((1ull << off) - 1)) != 0;
#pragma unroll 1
  for (int k = 0; k < idx; k++) sticky |= w[k] != 0;
  uint64_t mant = x >> 1;
  if ((x & 1) && (sticky || (mant & 1))) mant++;
  uint64_t b = ((uint64_t)shift << 52) + mant;  // mant's bit 52 (or its carry to 2^53) completes the exponent
  if (b >= kDblInf) b = kDblInf;
  *bits = sign | b;
  return true;
}

// MRHBM_COMBINE_FSUM: the greedy expansion of the accumulated sum S of a key's m values.  c1 = S rounded as acc_round
// rounds it, c(k+1) = (S - c1 - ... - ck) rounded the same way, until the remainder is 0; infinities of one sign and an
// exact zero give one term (acc_round's value).  Writes the terms' bits to out[0 ..] and returns their number; returns
// 0 when the key keeps its values as emitted (|S| rounds to +-inf, or more than `max` = m terms; out[0 .. max) may
// then hold anything) and -1 for a NaN (as acc_round).  The accumulator is consumed.
//
// After acc_round the accumulator holds |X| for the X it held, and the term is X rounded, so the remainder is
// sign(X) (|X| - |term|): subtracting |term| and tracking the sign keeps the whole split in the accumulator.
MRHBM_HDI int acc_split(int64_t* w, uint64_t* out, int max) {
  const uint64_t f = (uint64_t)w[kAccFlags];
  uint64_t c;
  if (!acc_round(w, &c)) return -1;
  if ((f & (NUM_PINF | NUM_NINF)) || (c << 1) == 0) {
    out[0] = c;
    return 1;
  }
  if ((c << 1) == kDblInf << 1) return 0;
  uint64_t sign = 0;  // the sign bit of the factor in remainder = factor x (the accumulator's value)
  int n = 0;
  do {
    if (n == max) return 0;
    out[n++] = c ^ sign;
    acc_add(w, c | 1ull << 63);  // minus |term|
    sign ^= c & 1ull << 63;
    acc_round(w, &c);
  } while ((c << 1) != 0);
  return n;
}

// The same split for a key of one or two finite or infinite values a, b (n = 1 or 2), in IEEE arithmetic: a + b
// rounded is c1, and where it does not overflow TwoSum's error term is the exact remainder, so it is c2 (when not 0).
// Returns as acc_split with max = n.
MRHBM_HDI int two_split(uint64_t a, uint64_t b, int n, uint64_t* out) {
  if (n == 1) {
    out[0] = a;
    return 1;
  }
#ifdef __CUDA_ARCH__
  const double x = __longlong_as_double((long long)a), y = __longlong_as_double((long long)b);
  const double s = __dadd_rn(x, y);
  const double bv = __dsub_rn(s, x), av = __dsub_rn(s, bv);
  const double e = __dadd_rn(__dsub_rn(x, av), __dsub_rn(y, bv));
  const uint64_t sb = (uint64_t)__double_as_longlong(s), eb = (uint64_t)__double_as_longlong(e);
#else
  double x, y;
  memcpy(&x, &a, 8);
  memcpy(&y, &b, 8);
  const volatile double s = x + y;  // (volatile: no reassociation or extended precision)
  const volatile double bv = s - x, av = s - bv;
  const volatile double e = (x - av) + (y - bv);
  uint64_t sb, eb;
  const double s_ = s, e_ = e;
  memcpy(&sb, &s_, 8);
  memcpy(&eb, &e_, 8);
#endif
  const bool ia = (a << 1) == kDblInf << 1, ib = (b << 1) == kDblInf << 1;
  if (ia || ib) {
    if (ia && ib && a != b) return -1;
    out[0] = ia ? a : b;
    return 1;
  }
  if ((sb << 1) == kDblInf << 1) return 0;
  out[0] = sb;
  if ((eb << 1) == 0) return 1;
  out[1] = eb;
  return 2;
}

}  // namespace mrhbm
