// Host driver for tests/test_value_order_host.py: checks the byte-value view and compare (csrc/mrhbm_valbytes.cuh)
// that the distinct set and the distinct reducer's ordering kernels share.  Every value is placed in an arena at each of
// the four alignments of its first byte; val_cmp must agree with memcmp over the shorter length, then the lengths,
// val_eq with equality of the bytes, and val_prefix with the first 8 bytes, big endian, zero padded.  Values: random
// ones, and adversarial ones (empty, zero bytes, proper prefixes, a difference in the last byte, past byte 8, past byte
// 4096, 0x80 / 0xff bytes that a signed compare gets wrong).  Prints one line per failed check, then "ok" or "FAIL".
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "mrhbm_valbytes.cuh"

using namespace mrhbm;

static int fails = 0;
#define CHECK(cond, ...)            \
  do {                              \
    if (!(cond)) {                  \
      if (++fails <= 20) {          \
        std::printf("%s: ", #cond); \
        std::printf(__VA_ARGS__);   \
        std::printf("\n");          \
      }                             \
    }                               \
  } while (0)

static int ref_cmp(const std::string& a, const std::string& b) {
  const size_t n = a.size() < b.size() ? a.size() : b.size();
  const int c = n ? std::memcmp(a.data(), b.data(), n) : 0;
  if (c) return c < 0 ? -1 : 1;
  return (a.size() > b.size()) - (a.size() < b.size());
}

int main() {
  std::mt19937_64 rng(17);
  auto rnd = [&](size_t n, int lo = 0, int hi = 255) {
    std::string s(n, '\0');
    std::uniform_int_distribution<int> d(lo, hi);
    for (auto& ch : s) ch = (char)d(rng);
    return s;
  };
  std::vector<std::string> vals = {"", std::string(1, '\0'), std::string(2, '\0'), "a", "ab", "abc", "abcd", "abcde",
                                    "abcdefgh", "abcdefghi", std::string("abcdefgh\0", 9), "abcdefgh\xff", "\x80",
                                    "\x7f", "\xff\xff\xff\xff\xff\xff\xff\xff\xff", "\x01"};
  const std::string big = rnd(5000);
  for (size_t at : {0ul, 3ul, 7ul, 8ul, 9ul, 4095ul, 4096ul, 4097ul, 4999ul}) {
    std::string v = big;
    v[at] = (char)(v[at] ^ 0x80);
    vals.push_back(v);
    vals.push_back(big.substr(0, at));
  }
  vals.push_back(big);
  for (int i = 0; i < 300; i++) vals.push_back(rnd(std::uniform_int_distribution<int>(0, 40)(rng), 0, i % 2 ? 3 : 255));
  for (int i = 0; i < 40; i++) {  // shared long prefixes, as file names have
    std::string v = "/data/corpus/file-" + rnd(i % 7, 'a', 'c');
    vals.push_back(v);
  }
  // four arenas: in arena s every value starts at an offset = s (mod 4), with a random gap before it
  for (uint32_t sh = 0; sh < 4; sh++) {
    std::vector<unsigned char> arena(64);
    std::vector<uint64_t> voff;
    for (const std::string& v : vals) {
      while (arena.size() % 4 != sh) arena.push_back(0xAA);
      voff.push_back(arena.size());
      arena.insert(arena.end(), v.begin(), v.end());
      voff.push_back(arena.size());
      for (int k = 0; k < 8; k++) arena.push_back(0x55);  // garbage after the value: must never be seen
    }
    arena.resize(arena.size() + 8, 0x55);
    // value i: id 2i, bytes arena[voff[2i], voff[2i+1])
    auto view = [&](size_t i) { return val_view(arena.data(), voff.data(), 2 * i); };
    for (size_t i = 0; i < vals.size(); i++) {
      const ValView a = view(i);
      CHECK(a.len == vals[i].size(), "value %zu length", i);
      std::string p8 = vals[i].substr(0, 8);
      p8.resize(8, '\0');
      uint64_t want = 0;
      for (unsigned char ch : p8) want = (want << 8) | ch;
      CHECK(val_prefix(a) == want, "value %zu prefix at alignment %u", i, sh);
      for (size_t j = 0; j < vals.size(); j++) {
        const ValView b = view(j);
        const int r = ref_cmp(vals[i], vals[j]), got = val_cmp(a, b);
        CHECK(got == r, "values %zu, %zu at alignment %u: %d, want %d", i, j, sh, got, r);
        CHECK(val_eq(a, b) == (vals[i] == vals[j]), "values %zu, %zu equal at alignment %u", i, j, sh);
        if (val_prefix(a) == val_prefix(b))
          CHECK(val_cmp(a, b, 2) == r, "values %zu, %zu from word 2 at alignment %u", i, j, sh);
        else
          CHECK((val_prefix(a) < val_prefix(b)) == (r < 0), "values %zu, %zu prefix order at alignment %u", i, j, sh);
      }
    }
  }
  std::printf("%s\n", fails ? "FAIL" : "ok");
  return fails ? 1 : 0;
}
