// Host driver for tests/test_gtab_layout.py: checks GtabLayout (csrc/mrhbm_kernels.h), the combiner's global table, at
// every size a shuffle can reach and for every record class.  Prints one line per failed check, then "ok" or "FAIL".
//   - every 32-bit hash maps to a bucket in range, the mapping is monotone and reaches every bucket;
//   - bucket probes wrap at the last bucket (not a power of two) and stay in range for every probe the kernel makes;
//   - long-entry slots stay in range and wrap;
//   - both parts fill whole warps of the compaction, the buckets are 32-byte aligned, and the bytes the compaction
//     reads (nshort 16-byte entries, then nlong records) are exactly bytes().
#include <cstdio>
#include <random>

#include "mrhbm_kernels.h"

using namespace mrhbm;

static int fails = 0;
#define CHECK(cond, ...)                          \
  do {                                            \
    if (!(cond)) {                                \
      if (++fails <= 20) {                        \
        std::printf("%s: ", #cond);               \
        std::printf(__VA_ARGS__);                 \
        std::printf("\n");                        \
      }                                           \
    }                                             \
  } while (0)

int main() {
  std::mt19937 rng(5);
  CHECK(GtabLayout::sized(32, 0).long_offset() == 25u << 20, "the default buckets are 25 MB");
  for (int rb : {16, 32, 64, 128}) {
    for (uint32_t grow = 0; grow <= GtabLayout::kMaxGrow; grow++) {
      const GtabLayout t = GtabLayout::sized(rb, grow);
      const uint32_t nb = t.nbuckets;
      CHECK(nb == GtabLayout::kBuckets << grow && t.long_log == GtabLayout::kLongLog + grow, "rb %d grow %u", rb, grow);
      CHECK(nb % 16 == 0 && t.nshort() == 2 * nb && t.nshort() % 32 == 0, "rb %d nb %u", rb, nb);
      CHECK(t.nlong() % 32 == 0 && t.nlong() == (rb == 16 ? 0u : 1u << t.long_log), "rb %d nlong %u", rb, t.nlong());
      CHECK(GtabLayout::kMaxProbes < nb, "nb %u", nb);
      // bytes the compaction reads: short entry s < nshort at 16 s, long entry l < nlong at long_offset + rb l
      const uint64_t short_end = (uint64_t)16 * t.nshort();
      const uint64_t long_end = t.long_offset() + (uint64_t)rb * t.nlong();
      CHECK(t.long_offset() == short_end && t.long_offset() % 32 == 0, "rb %d grow %u", rb, grow);
      CHECK(t.bytes() == long_end && t.records() == t.nshort() + t.nlong(), "rb %d grow %u", rb, grow);
      // hash -> bucket: the ends, then random hashes; monotone; bucket b is reached from the first hash above b/nb
      CHECK(t.bucket(0) == 0 && t.bucket(0xffffffffu) == nb - 1, "nb %u", nb);
      uint32_t prev_h = 0, prev_b = 0;
      for (int i = 0; i < 200000; i++) {
        const uint32_t h = prev_h + (rng() >> 10);
        if (h < prev_h) break;
        const uint32_t b = t.bucket(h);
        CHECK(b < nb && b >= prev_b, "h %u b %u nb %u", h, b, nb);
        prev_h = h, prev_b = b;
      }
      for (int i = 0; i < 1000; i++) {
        const uint32_t b = (uint32_t)(((uint64_t)rng() * nb) >> 32);
        const uint32_t h = (uint32_t)(((uint64_t)b << 32) / nb + (((uint64_t)b << 32) % nb != 0));
        CHECK(t.bucket(h) == b && (h == 0 || t.bucket(h - 1) == b - 1), "b %u h %u nb %u", b, h, nb);
      }
      // probes: bucket_at(home, p) == (home + p) mod nb, in range, wrapping at nb - 1
      CHECK(t.bucket_at(nb - 1, 1) == 0 && t.bucket_at(nb - 1, 0) == nb - 1, "nb %u", nb);
      for (uint32_t home : {0u, 1u, nb / 2, nb - GtabLayout::kMaxProbes, nb - 2, nb - 1}) {
        for (uint32_t p = 0; p < GtabLayout::kMaxProbes; p++) {
          const uint32_t b = t.bucket_at(home, p);
          CHECK(b < nb && b == (uint32_t)(((uint64_t)home + p) % nb), "home %u p %u nb %u", home, p, nb);
        }
      }
      if (t.nlong()) {
        CHECK(t.long_slot(0) == 0 && t.long_slot(0xffffffffu) == t.nlong() - 1, "nlong %u", t.nlong());
        CHECK(t.long_next(t.nlong() - 1) == 0 && t.long_next(0) == 1, "nlong %u", t.nlong());
        for (int i = 0; i < 1000; i++) CHECK(t.long_slot(rng()) < t.nlong(), "nlong %u", t.nlong());
      }
    }
  }
  std::printf(fails ? "FAIL\n" : "ok\n");
  return fails ? 1 : 0;
}
