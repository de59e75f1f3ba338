// Host driver for tests/test_gpu_fsum_reducer_paths.py: MRHBM_RED_FSUM's scratch slots (num_slot and num_slots in
// csrc/mrhbm_kernels.h, where the chunks of oversized bins keep their partial accumulators) for the tests' Python model
// to match.  Input: lines of "slot <first row> <cap> <first chunk 0/1>" or "slots <N> <cap>".  Output per line: the
// slot, or the slot count, in decimal.  Prints "ok" or "FAIL" last.
#include <cinttypes>
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

#include "mrhbm_kernels.h"

using namespace mrhbm;

int main() {
  int fails = 0;
  std::string line;
  while (std::getline(std::cin, line)) {
    if (line.empty()) continue;
    std::istringstream in(line);
    std::string what;
    uint64_t a = 0;
    uint32_t cap = 0, first = 0;
    in >> what >> a >> cap;
    if (what == "slot" && in >> first) {
      std::printf("%" PRIu64 "\n", num_slot(a, cap, first != 0));
    } else if (what == "slots") {
      std::printf("%" PRIu64 "\n", num_slots(a, cap));
    } else {
      std::printf("bad line: %s\n", line.c_str());
      fails++;
    }
  }
  std::printf(fails ? "FAIL\n" : "ok\n");
  return fails != 0;
}
