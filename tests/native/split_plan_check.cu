// Host driver for tests/test_split_plan.py: runs the split planner of csrc/mrhbm_split_plan.h on commands read from
// stdin, one per line, and prints one line per command.
//   P exact cap nmax ndest me Bl[0] .. Bl[ndest-1]  -> levels, then (levels > 0) F C1 C1_local sub_stride
//                                                     rbase[0..8] fbase[0..8]
//   X regions sub_stride ndest rb ctas              -> the level-2 CTAs per region
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

#include "mrhbm_split_plan.h"

using namespace mrhbm;

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op;
    in >> op;
    if (op == "P") {
      int exact = 0;
      uint32_t cap = 0, ndest = 0, me = 0;
      uint64_t nmax = 0, Bl[8] = {};
      in >> exact >> cap >> nmax >> ndest >> me;
      for (uint32_t d = 0; d < ndest; d++) in >> Bl[d];
      SplitPlan pl{};
      const int levels = plan_split(pl, Bl, ndest, me, cap, nmax, exact != 0);
      printf("%d", levels);
      if (levels) {
        printf(" %u %u %u %llu", pl.F, pl.C1, pl.C1_local, (unsigned long long)pl.sub_stride);
        for (int i = 0; i < 9; i++) printf(" %u", pl.rbase[i]);
        for (int i = 0; i < 9; i++) printf(" %u", pl.fbase[i]);
      }
      printf("\n");
    } else if (op == "X") {
      uint32_t regions = 0, ndest = 0;
      uint64_t sub_stride = 0;
      int rb = 0, ctas = 0;
      in >> regions >> sub_stride >> ndest >> rb >> ctas;
      printf("%d\n", split_l2_ctas_per_region(regions, sub_stride, ndest, rb, ctas));
    } else {
      printf("?\n");
    }
  }
  return 0;
}
