// Host driver for tests/test_gpu_distinct_reducer_paths.py: the distinct set's pair fingerprint (pair_fingerprint in
// csrc/mrhbm_job_tiles.cuh, the hash that places a (key slot, value bytes) pair in the set) for the tests' Python model
// to match.  Input: lines of "<record bytes> <value bytes in hex, or -> <hex u32 word> ..." (the key slot words of one
// record).  The value is placed in an arena at each of the four alignments of its first byte; the four fingerprints
// must agree.  Output per line: the fingerprint in hex.  Prints "ok" or "FAIL" last.
#include <cinttypes>
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "mrhbm_job_tiles.cuh"

using namespace mrhbm;

static uint64_t fp_of(int rb, const uint32_t* w, const ValView& v) {
  switch (rb) {
    case 16: return pair_fingerprint<16>(w, v);
    case 32: return pair_fingerprint<32>(w, v);
    case 64: return pair_fingerprint<64>(w, v);
    default: return pair_fingerprint<128>(w, v);
  }
}

int main() {
  int fails = 0;
  std::string line;
  while (std::getline(std::cin, line)) {
    if (line.empty()) continue;
    std::istringstream in(line);
    int rb;
    std::string hex;
    in >> rb >> hex;
    if (rb != 16 && rb != 32 && rb != 64 && rb != 128) {
      std::printf("bad record size %d\n", rb);
      fails++;
      continue;
    }
    std::string val;
    if (hex != "-")
      for (size_t i = 0; i + 1 < hex.size(); i += 2) val.push_back((char)std::stoi(hex.substr(i, 2), nullptr, 16));
    std::vector<uint32_t> w(32, 0);
    int n = 0;
    for (uint32_t x; n < 32 && in >> std::hex >> x;) w[n++] = x;
    uint64_t fp[4];
    for (uint32_t sh = 0; sh < 4; sh++) {
      // arena words past the value hold 0xa5 bytes: the fingerprint must not read them
      std::vector<uint32_t> arena((sh + val.size() + 8) / 4 + 2, 0xa5a5a5a5u);
      unsigned char* a = (unsigned char*)arena.data();
      for (size_t i = 0; i < val.size(); i++) a[sh + i] = (unsigned char)val[i];
      const uint64_t voff[2] = {sh, sh + val.size()};
      fp[sh] = fp_of(rb, w.data(), val_view(a, voff, 0));
    }
    if (fp[1] != fp[0] || fp[2] != fp[0] || fp[3] != fp[0]) {
      std::printf("alignments disagree: %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 "\n", fp[0], fp[1],
                  fp[2], fp[3]);
      fails++;
      continue;
    }
    std::printf("%016" PRIx64 "\n", fp[0]);
  }
  std::printf(fails ? "FAIL\n" : "ok\n");
  return fails != 0;
}
