// Host driver for tests/test_pool_ledger_shrink.py: the commands of tests/native/pool_ledger_check.cu plus the two
// ledger operations of MRHBM_COMBINE_DISTINCT.  Runs the emit pool's ledger of csrc/mrhbm_pool.h on commands read from
// stdin, one per line, and prints one line per command: the command's own result (or "-"), then used, arena_used and
// the live ranges as off cnt off cnt ...
//   B                        -> byte values on (value ids are u32)
//   O                        -> new_owner
//   T n bytes                -> take: off aoff, or "refused" when the records do not fit
//   A owner job off cnt aoff -> add
//   C owner job              -> commit
//   X owner                  -> abort
//   M                        -> mark: its index
//   W index                  -> rewind to that mark
//   R                        -> reset
//   J                        -> open_job, "none" when no range is open
//   P owner                  -> open_ranges: off cnt off cnt ... ("none" when the owner has none)
//   S owner off cnt          -> shrink
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "mrhbm_pool.h"

using mrhbm::PoolLedger;

int main() {
  PoolLedger led;
  std::vector<PoolLedger::Mark> marks;
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, job;
    uint64_t a = 0, b = 0, c = 0, d = 0;
    in >> op;
    std::ostringstream out;
    if (op == "B") {
      led.byte_values = true;
      out << '-';
    } else if (op == "O") {
      out << led.new_owner();
    } else if (op == "T") {
      in >> a >> b;
      if (led.fits(a)) {
        const PoolLedger::Room r = led.take(a, b);
        out << r.off << ' ' << r.aoff;
      } else {
        out << "refused";
      }
    } else if (op == "A") {
      in >> a >> job >> b >> c >> d;
      led.add(a, job, b, c, d);
      out << '-';
    } else if (op == "C") {
      in >> a >> job;
      led.commit(a, job);
      out << '-';
    } else if (op == "X") {
      in >> a;
      led.abort(a);
      out << '-';
    } else if (op == "M") {
      marks.push_back(led.mark());
      out << marks.size() - 1;
    } else if (op == "W") {
      in >> a;
      led.rewind(marks.at(a));
      out << '-';
    } else if (op == "R") {
      led.reset();
      out << '-';
    } else if (op == "J") {
      const std::string* j = led.open_job();
      out << (j ? *j : "none");
    } else if (op == "P") {
      in >> a;
      const auto v = led.open_ranges(a);
      if (v.empty()) out << "none";
      for (size_t i = 0; i < v.size(); i++) out << (i ? " " : "") << v[i].first << ' ' << v[i].second;
    } else if (op == "S") {
      in >> a >> b >> c;
      led.shrink(a, b, c);
      out << '-';
    } else {
      out << '?';
    }
    out << " | " << led.used() << ' ' << led.arena_used();
    for (const auto& r : led.live()) out << ' ' << r.first << ' ' << r.second;
    std::cout << out.str() << '\n';
  }
  return 0;
}
