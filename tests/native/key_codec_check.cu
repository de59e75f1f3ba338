// Host driver for tests/test_key_codec.py: runs the key codec of csrc/mrhbm_keys.h on commands read from stdin,
// one per line, and prints one line per command.  Byte strings are hex, "-" for the empty string.
//   E key                   -> escaped esc_size unescape(escaped)
//   U esc                   -> unescape(esc)
//   O kb key...             -> the keys' slots stably sorted by slot_cmp (indices), then slot_key of every slot
//                              (kb = 8: u64 keys as 8 big-endian bytes; else keys that fit a slot)
//   L kb long key           -> sign of esc_cmp(long, the escaped key in key's slot), as the iterator merges them
//   T kb P spl...           -> range_table: fin, then the image
//   H part P n spl... key...-> host_partition of every key
#include <algorithm>
#include <cstdio>
#include <iostream>
#include <numeric>
#include <sstream>
#include <string>
#include <vector>

#include "mrhbm_keys.h"

using namespace mrhbm;
using Bytes = std::vector<unsigned char>;

static Bytes unhex(const std::string& s) {
  Bytes b;
  if (s == "-") return b;
  for (size_t i = 0; i + 1 < s.size(); i += 2) b.push_back((unsigned char)std::stoul(s.substr(i, 2), nullptr, 16));
  return b;
}
static std::string hex(const unsigned char* p, size_t n) {
  if (!n) return "-";
  std::string s;
  char buf[3];
  for (size_t i = 0; i < n; i++) {
    snprintf(buf, sizeof buf, "%02x", p[i]);
    s += buf;
  }
  return s;
}
static std::string hex(const Bytes& b) { return hex(b.data(), b.size()); }
static Bytes esc_of(const Bytes& k) {
  Bytes e(esc_size(k.data(), k.size()));
  escape(k.data(), k.size(), e.data());
  return e;
}
// the slot mrhbm_emit_str / mrhbm_emit_u64 store for a key
static Bytes slot_of(const Bytes& k, size_t kb) {
  Bytes s(kb, 0);
  if (kb == kU64SlotBytes) {
    const uint64_t v = be64_load(k.data());
    memcpy(s.data(), &v, 8);
  } else {
    const Bytes e = esc_of(k);
    memcpy(s.data(), e.data(), e.size());
  }
  return s;
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, tok;
    in >> op;
    std::vector<std::string> a;
    while (in >> tok) a.push_back(tok);
    std::ostringstream out;
    if (op == "E") {
      const Bytes k = unhex(a[0]), e = esc_of(k);
      Bytes u;
      unescape(e.data(), e.size(), u);
      out << hex(e) << ' ' << esc_size(k.data(), k.size()) << ' ' << hex(u);
    } else if (op == "U") {
      const Bytes e = unhex(a[0]);
      Bytes u;
      unescape(e.data(), e.size(), u);
      out << hex(u);
    } else if (op == "O") {
      const size_t kb = std::stoul(a[0]), n = a.size() - 1;
      std::vector<Bytes> slots;
      for (size_t i = 0; i < n; i++) slots.push_back(slot_of(unhex(a[i + 1]), kb));
      std::vector<size_t> idx(n);
      std::iota(idx.begin(), idx.end(), 0);
      std::stable_sort(idx.begin(), idx.end(),
                       [&](size_t x, size_t y) { return slot_cmp(slots[x].data(), slots[y].data(), kb) < 0; });
      for (size_t i : idx) out << i << ' ';
      Bytes k;
      for (const Bytes& s : slots) {
        slot_key(s.data(), kb, k);
        out << hex(k) << ' ';
      }
    } else if (op == "L") {
      const size_t kb = std::stoul(a[0]);
      const Bytes lesc = esc_of(unhex(a[1])), s = slot_of(unhex(a[2]), kb);
      out << esc_cmp(lesc.data(), lesc.size(), s.data(), slot_esc_len(s.data(), kb));
    } else if (op == "T") {
      const size_t kb = std::stoul(a[0]);
      const uint32_t P = (uint32_t)std::stoul(a[1]);
      std::vector<std::string> spl;
      for (size_t i = 2; i < a.size(); i++) {
        const Bytes b = unhex(a[i]);
        spl.emplace_back(b.begin(), b.end());
      }
      const RangeTable rt = range_table(spl, P, kb);
      out << rt.fin << ' ' << hex(rt.image);
    } else if (op == "H") {
      const uint32_t part = (uint32_t)std::stoul(a[0]), P = (uint32_t)std::stoul(a[1]);
      const size_t n = std::stoul(a[2]);
      std::vector<std::string> spl;
      for (size_t i = 0; i < n; i++) {
        const Bytes b = unhex(a[3 + i]);
        spl.emplace_back(b.begin(), b.end());
      }
      for (size_t i = 3 + n; i < a.size(); i++) {
        const Bytes e = esc_of(unhex(a[i]));
        out << host_partition(part, P, spl, std::string(e.begin(), e.end())) << ' ';
      }
    } else {
      out << "?";
    }
    std::cout << out.str() << '\n';
  }
  return 0;
}
