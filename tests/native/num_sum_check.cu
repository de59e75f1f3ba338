// Host driver for tests/test_fsum_host.py: reads test cases from stdin and sums them with the shared number decoding
// and superaccumulator of MRHBM_RED_FSUM (csrc/mrhbm_numsum.cuh), as the host's long keys do.  Input: lines of
// "<n> <hex bits> ... [split]", a group of n doubles given as their IEEE bits; with "split" the values are added into
// two accumulators (even and odd positions) that are then merged, as a group that crosses a chunk is.  Each value goes
// through num_encode and num_decode first.  Output per line: the rounded sum's bits in hex, or "nan".  Also checks
// that malformed encodings are refused and prints "ok" or "FAIL" last.
#include <cinttypes>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "mrhbm_numsum.cuh"

using namespace mrhbm;

int main() {
  int fails = 0;
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    size_t n;
    in >> n;
    std::vector<uint64_t> v(n);
    for (auto& x : v) in >> std::hex >> x;
    std::string split;
    in >> split;
    int64_t a[kAccWords], b[kAccWords];
    acc_clear(a);
    acc_clear(b);
    for (size_t i = 0; i < n; i++) {
      unsigned char enc[kNumBytes];
      num_encode(v[i], enc);
      uint64_t bits = 0;
      if (!num_decode(enc, kNumBytes, &bits) || bits != v[i]) {
        if ((v[i] & ~(1ull << 63)) <= kDblInf) fails++;  // (a NaN is refused by design)
        std::printf("nan\n");
        goto next;
      }
      acc_add(split == "split" && (i & 1) ? b : a, bits);
    }
    acc_merge(a, b);
    {
      uint64_t r;
      if (acc_round(a, &r)) std::printf("%016" PRIx64 "\n", r);
      else std::printf("nan\n");
    }
  next:;
  }
  // malformed encodings: wrong tag, wrong length, a group without bit 7, a first group above 1
  unsigned char enc[kNumBytes + 1];
  uint64_t bits;
  num_encode(0x3ff0000000000000ull, enc);
  if (!num_decode(enc, kNumBytes, &bits) || bits != 0x3ff0000000000000ull) fails++;
  if (num_decode(enc, kNumBytes - 1, &bits) || num_decode(enc, kNumBytes + 1, &bits)) fails++;
  unsigned char e2[kNumBytes];
  std::memcpy(e2, enc, kNumBytes);
  e2[0] = 0x20;
  if (num_decode(e2, kNumBytes, &bits)) fails++;
  std::memcpy(e2, enc, kNumBytes);
  e2[5] &= 0x7f;
  if (num_decode(e2, kNumBytes, &bits)) fails++;
  std::memcpy(e2, enc, kNumBytes);
  e2[1] |= 0x02;
  if (num_decode(e2, kNumBytes, &bits)) fails++;
  std::printf(fails ? "FAIL\n" : "ok\n");
  return fails != 0;
}
