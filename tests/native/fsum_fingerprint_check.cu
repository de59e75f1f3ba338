// Host driver for tests/test_gpu_fsum_combiner_paths.py: MRHBM_COMBINE_FSUM's key fingerprint (key_fingerprint in
// csrc/mrhbm_job_tiles.cuh, the hash that places a key in the commit's hash set) for the tests' Python model to match.
// Input: lines of "<record bytes> <hex u32 word> ..." (the key slot words of one record).  Output per line: the
// fingerprint in hex.  Prints "ok" or "FAIL" last.
#include <cinttypes>
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "mrhbm_job_tiles.cuh"

using namespace mrhbm;

int main() {
  int fails = 0;
  std::string line;
  while (std::getline(std::cin, line)) {
    if (line.empty()) continue;
    std::istringstream in(line);
    int rb;
    in >> rb;
    std::vector<uint32_t> w(32, 0);
    int n = 0;
    for (uint32_t x; n < 32 && in >> std::hex >> x;) w[n++] = x;
    uint64_t fp = 0;
    switch (rb) {
      case 16: fp = key_fingerprint<16>(w.data()); break;
      case 32: fp = key_fingerprint<32>(w.data()); break;
      case 64: fp = key_fingerprint<64>(w.data()); break;
      case 128: fp = key_fingerprint<128>(w.data()); break;
      default:
        std::printf("bad record size %d\n", rb);
        fails++;
        continue;
    }
    std::printf("%016" PRIx64 "\n", fp);
  }
  std::printf(fails ? "FAIL\n" : "ok\n");
  return fails != 0;
}
