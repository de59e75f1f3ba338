// mrhbm_decimal.cuh -- mrhbm_map_key_numbers: a decimal number token to the nearest double, ties to even.  One
// definition of the grammar and of the conversion for the kernels (mrhbm_key_numbers.cu), the host's fall-back pieces
// and fix-ups (mrhbm_api.cu) and tests/native/decimal_parse_check.cu, which checks it against Python's float().
//
// Grammar (what Lua 5.2's tonumber takes through strtod, less hexadecimal): [+-]?(D+(\.D*)?|\.D+)([eE][+-]?D+)?
//
// Conversion: a token of at most 19 significant digits is w * 10^q with an integer w < 10^19.
//   - Clinger's fast path: w <= 2^53 and |q| <= 22 make w and 10^|q| exact doubles, so one IEEE multiply or divide
//     (round to nearest) is the answer.
//   - Otherwise Eisel-Lemire (D. Lemire, "Number parsing at a gigabyte per second", Software: Practice and Experience
//     51(8), 2021): w, normalised, times a 128-bit approximation of 5^q gives the 55 leading bits of the product; the
//     exponent follows from q * log2(10).  The table of approximations is computed here from exact integers
//     (dec_pow5_entry) and copied to the device once.
//   - Sent to the host (DEC_HOST), where std::from_chars rounds correctly: more than 19 significant digits, and the
//     algorithm's ambiguous case (the truncated product's low word all ones outside -27 <= q <= 55).
#pragma once
#include <cstdint>
#include <cstring>
#include <charconv>
#include <system_error>
#include <vector>

#include "mrhbm_numsum.cuh"  // MRHBM_HDI, kDblInf

namespace mrhbm {

constexpr int kPow5Min = -342, kPow5Max = 308;  // w * 10^q with w < 10^19 is 0 below, inf above
constexpr int kPow5Count = kPow5Max - kPow5Min + 1;
constexpr int kDecMaxDigits = 19;

enum { DEC_BAD = 0, DEC_EXACT = 1, DEC_HOST = 2 };

// What the grammar check learnt of a token: |value| = W * 10^e10, W the integer of its nd significant digits (first
// to last non-zero digit), of which w holds the first min(nd, 19).
struct DecScan {
  uint64_t w;
  int64_t e10;
  uint32_t nd;
  bool neg;
};

MRHBM_HDI bool dec_digit(unsigned char ch) { return ch >= '0' && ch <= '9'; }

// true when s[0 .. n) matches the grammar
MRHBM_HDI bool dec_scan(const unsigned char* s, uint64_t n, DecScan* d) {
  uint64_t i = 0, w = 0;
  int64_t pend = 0, dexp = 0, ex = 0;  // zeros not yet in w, digits after the point, the exponent part
  uint32_t nd = 0;
  d->neg = false;
  if (i < n && (s[i] == '+' || s[i] == '-')) d->neg = s[i++] == '-';
  uint64_t digits = 0;
  bool frac = false;
  for (; i < n; i++) {
    const unsigned char ch = s[i];
    if (ch == '.' && !frac) {
      frac = true;
      continue;
    }
    if (!dec_digit(ch)) break;
    digits++;
    if (frac) dexp--;
    if (ch == '0') {
      if (nd) pend++;  // (leading zeros are not significant)
      continue;
    }
    // a non-zero digit: the zeros before it become significant
    if (nd + pend + 1 <= (uint64_t)kDecMaxDigits) {
      for (int64_t k = 0; k < pend; k++) w *= 10;
      w = w * 10 + (ch - '0');
    }
    nd += (uint32_t)pend + 1;
    pend = 0;
  }
  if (!digits) return false;  // ".", "+", "", ".e1"
  if (i < n && (s[i] == 'e' || s[i] == 'E')) {
    i++;
    bool eneg = false;
    if (i < n && (s[i] == '+' || s[i] == '-')) eneg = s[i++] == '-';
    const uint64_t e0 = i;
    for (; i < n && dec_digit(s[i]); i++)
      if (ex < (1ll << 40)) ex = ex * 10 + (s[i] - '0');  // (saturated: far beyond every exponent that matters)
    if (i == e0) return false;  // "1e", "1e+"
    if (eneg) ex = -ex;
  }
  if (i != n) return false;
  d->w = w;
  d->nd = nd;
  d->e10 = pend + dexp + ex;
  return true;
}

// The 128-bit approximation of 5^q that Eisel-Lemire multiplies by, as {high, low} 64-bit words, from exact
// integers.  q >= 0: 5^q truncated to its leading 128 bits.  q < 0, with z the bit length of 5^-q:
// floor(2^(z + 127) / 5^-q) + 1 for q >= -27 (exact enough that the product decides halfway cases), else
// floor(2^(2z + 128) / 5^-q) + 1 truncated to its leading 128 bits.  Host only; the device gets a copy.
inline void dec_pow5_entry(int q, uint64_t* hi, uint64_t* lo) {
  using Big = std::vector<uint32_t>;  // little-endian 32-bit limbs
  auto bitlen = [](const Big& a) {
    for (size_t k = a.size(); k-- > 0;)
      if (a[k]) return (int)(32 * k + 32 - __builtin_clz(a[k]));
    return 0;
  };
  auto bit = [](const Big& a, int b) { return (size_t)(b >> 5) < a.size() ? (a[b >> 5] >> (b & 31)) & 1u : 0u; };
  auto top128 = [&](const Big& a, uint64_t* h, uint64_t* l) {  // the leading 128 bits, truncated
    const int L = bitlen(a);
    *h = *l = 0;
    for (int k = 0; k < 128; k++) {
      const int b = L - 1 - k;
      const uint64_t v = b >= 0 ? bit(a, b) : 0;
      if (k < 64) *h |= v << (63 - k);
      else *l |= v << (127 - k);
    }
  };
  Big p{1};
  for (int k = 0; k < (q < 0 ? -q : q); k++) {
    uint64_t carry = 0;
    for (uint32_t& limb : p) {
      const uint64_t x = (uint64_t)limb * 5 + carry;
      limb = (uint32_t)x;
      carry = x >> 32;
    }
    if (carry) p.push_back((uint32_t)carry);
  }
  if (q >= 0) {
    top128(p, hi, lo);
    return;
  }
  const int z = bitlen(p), b = q >= -27 ? z + 127 : 2 * z + 128;
  // floor(2^b / p) by shift and subtract, then + 1
  Big r(p.size() + 1, 0), quo((size_t)(b / 32 + 2), 0);
  auto ge = [](const Big& a, const Big& m) {  // a >= m (a has one limb more)
    for (size_t k = a.size(); k-- > 0;) {
      const uint32_t mk = k < m.size() ? m[k] : 0;
      if (a[k] != mk) return a[k] > mk;
    }
    return true;
  };
  for (int i = b; i >= 0; i--) {
    uint32_t carry = i == b;
    for (uint32_t& limb : r) {
      const uint32_t nc = limb >> 31;
      limb = (limb << 1) | carry;
      carry = nc;
    }
    if (ge(r, p)) {
      uint64_t borrow = 0;
      for (size_t k = 0; k < r.size(); k++) {
        const uint64_t sub = (uint64_t)(k < p.size() ? p[k] : 0) + borrow;
        borrow = (uint64_t)r[k] < sub;
        r[k] = (uint32_t)((uint64_t)r[k] - sub);
      }
      quo[i >> 5] |= 1u << (i & 31);
    }
  }
  for (uint32_t& limb : quo)
    if (++limb) break;
  top128(quo, hi, lo);
}
// the whole table, entry q at out[2 (q - kPow5Min)], out[2 (q - kPow5Min) + 1]
inline void dec_pow5_table(uint64_t* out) {
  for (int q = kPow5Min; q <= kPow5Max; q++) dec_pow5_entry(q, out + 2 * (q - kPow5Min), out + 2 * (q - kPow5Min) + 1);
}

namespace detail {
MRHBM_HDI uint64_t mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
MRHBM_HDI int clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
  return __clzll((long long)x);
#else
  return __builtin_clzll(x);
#endif
}
MRHBM_HDI uint64_t dbl_bits(double x) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(x);
#else
  uint64_t u;
  memcpy(&u, &x, 8);
  return u;
#endif
}
}  // namespace detail

// The double nearest a scanned token into *bits: DEC_EXACT, or DEC_HOST for the cases above.  pow5: dec_pow5_table.
MRHBM_HDI int dec_to_bits(const DecScan& d, const uint64_t* pow5, uint64_t* bits) {
  const uint64_t sign = d.neg ? 1ull << 63 : 0;
  if (d.nd == 0) {  // every digit 0, whatever the exponent
    *bits = sign;
    return DEC_EXACT;
  }
  if (d.nd > (uint32_t)kDecMaxDigits) return DEC_HOST;
  const int64_t q = d.e10;
  uint64_t w = d.w;
  if (w <= (1ull << 53) && q >= -22 && q <= 22) {
    double p = 1.0;
    for (int k = 0; k < (q < 0 ? -q : q); k++) p *= 10.0;  // exact: 10^22 < 2^53 * 2^22
#ifdef __CUDA_ARCH__
    const double x = q < 0 ? __ddiv_rn((double)w, p) : __dmul_rn((double)w, p);
#else
    const volatile double x = q < 0 ? (double)w / p : (double)w * p;
#endif
    *bits = sign | detail::dbl_bits(x);
    return DEC_EXACT;
  }
  if (q < kPow5Min) {  // w * 10^q < 10^-323 / 2: rounds to 0
    *bits = sign;
    return DEC_EXACT;
  }
  if (q > kPow5Max) {  // >= 10^309
    *bits = sign | kDblInf;
    return DEC_EXACT;
  }
  const int lz = detail::clz64(w);
  w <<= lz;
  const int idx = 2 * (int)(q - kPow5Min);
#ifdef __CUDA_ARCH__
  const uint64_t t_hi = __ldg((const unsigned long long*)pow5 + idx), t_lo = __ldg((const unsigned long long*)pow5 + idx + 1);
#else
  const uint64_t t_hi = pow5[idx], t_lo = pow5[idx + 1];
#endif
  // the product's leading 55 bits: 53 of the double, a rounding bit, and one that may be a leading zero
  uint64_t hi = detail::mulhi64(w, t_hi), lo = w * t_hi;
  constexpr uint64_t kMask = (1ull << 9) - 1;  // the 64 - 55 bits below them
  if ((hi & kMask) == kMask) {                  // they may carry: add the next 64 bits of the product
    const uint64_t s = detail::mulhi64(w, t_lo);
    lo += s;
    if (lo < s) hi++;
  }
  if (lo == ~0ull && (q < -27 || q > 55)) return DEC_HOST;
  const int upper = (int)(hi >> 63), shift = upper + 9;
  uint64_t mant = hi >> shift;
  // binary exponent + 1023: floor(q log2(10)) + 63 + upper - lz, with 217706 / 2^16 ~ log2(10)
  int p2 = (int)((217706 * (int32_t)q) >> 16) + 63 + upper - lz + 1023;
  if (p2 <= 0) {  // subnormal (no exact halfway case can have this few digits here)
    if (-p2 + 1 >= 64) {
      *bits = sign;
      return DEC_EXACT;
    }
    mant >>= -p2 + 1;
    mant += mant & 1;
    mant >>= 1;
    *bits = sign | mant;  // (mant == 2^52: the smallest normal)
    return DEC_EXACT;
  }
  // exactly halfway: round to even (only for -4 <= q <= 23 can w * 10^q be a halfway point of 55 bits)
  if (lo <= 1 && q >= -4 && q <= 23 && (mant & 3) == 1 && (mant << shift) == hi) mant &= ~1ull;
  mant += mant & 1;
  mant >>= 1;
  if (mant >= (2ull << 52)) {
    mant = 1ull << 52;
    p2++;
  }
  mant &= ~(1ull << 52);
  if (p2 >= 0x7ff) {
    *bits = sign | kDblInf;
    return DEC_EXACT;
  }
  *bits = sign | ((uint64_t)p2 << 52) | mant;
  return DEC_EXACT;
}

// The host's conversion of a token (fall-back pieces and DEC_HOST fix-ups): the grammar above, the value from
// std::from_chars, which rounds correctly in every case and reads no locale.  False when the token is malformed.
inline bool dec_parse_host(const unsigned char* s, uint64_t n, uint64_t* bits) {
  DecScan d;
  if (!dec_scan(s, n, &d)) return false;
  const uint64_t sign = d.neg ? 1ull << 63 : 0;
  if (d.nd == 0) {
    *bits = sign;
    return true;
  }
  const char* a = (const char*)s + (s[0] == '+' || s[0] == '-');
  double x = 0;
  const std::from_chars_result r = std::from_chars(a, (const char*)s + n, x, std::chars_format::general);
  if (r.ec == std::errc::result_out_of_range) {
    // beyond DBL_MAX or below half the smallest subnormal: the leading digit's decimal exponent tells which
    *bits = sign | (d.e10 + (int64_t)d.nd - 1 >= 0 ? kDblInf : 0);
    return true;
  }
  if (r.ec != std::errc() || r.ptr != (const char*)s + n) return false;
  *bits = sign | detail::dbl_bits(x);
  return true;
}

}  // namespace mrhbm
