// Host driver for tests/test_fsum_combiner_host.py: reads groups of doubles from stdin and splits their exact sum with
// MRHBM_COMBINE_FSUM's greedy expansion (acc_split in csrc/mrhbm_numsum.cuh), as the host's long keys do.  Input:
// lines of "<n> <hex bits> ...".  Output per line: "nan", "keep" (the key keeps its values), or the terms' bits in hex.
// A group of one or two values is also split with two_split, the kernels' IEEE path, and must give the same answer.
// Prints "ok" or "FAIL" last.
#include <cinttypes>
#include <cstdio>
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
    int n;
    in >> n;
    std::vector<uint64_t> v(n), t(n + 1);
    int64_t a[kAccWords];
    acc_clear(a);
    for (auto& x : v) {
      in >> std::hex >> x;
      acc_add(a, x);
    }
    const int k = acc_split(a, t.data(), n);
    if (n <= 2) {
      uint64_t u[2];
      const int k2 = two_split(v[0], n == 2 ? v[1] : 0, n, u);
      bool same = k2 == k;
      for (int i = 0; same && i < k; i++) same = u[i] == t[i];
      if (!same) {
        std::printf("two_split differs\n");
        fails++;
        continue;
      }
    }
    if (k < 0) {
      std::printf("nan\n");
    } else if (k == 0) {
      std::printf("keep\n");
    } else {
      for (int i = 0; i < k; i++) std::printf(i ? " %016" PRIx64 : "%016" PRIx64, t[i]);
      std::printf("\n");
    }
  }
  std::printf(fails ? "FAIL\n" : "ok\n");
  return fails != 0;
}
