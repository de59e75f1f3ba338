// Host check for tests/test_fsum_combiner_host.py: the ledger operation of MRHBM_COMBINE_FSUM (PoolLedger::replace_open
// in csrc/mrhbm_pool.h), in the three situations a commit can meet, with a reservation taken and added as
// mrhbm_map_commit does.  Prints each failed check and then "ok" or "FAIL".
#include <cstdio>
#include <string>
#include <utility>
#include <vector>

#include "mrhbm_pool.h"

using mrhbm::PoolLedger;
using Ranges = std::vector<std::pair<uint64_t, uint64_t>>;

static int fails = 0;
#define CHECK(cond)                                          \
  do {                                                       \
    if (!(cond)) {                                           \
      std::printf("line %d: %s\n", __LINE__, #cond);         \
      fails++;                                               \
    }                                                        \
  } while (0)

// the map's records: n pairs of v value bytes each at the tail, as stage_flush adds them
static void emit(PoolLedger& led, uint64_t owner, const std::string& job, uint64_t n, uint64_t v) {
  const PoolLedger::Room r = led.take(n, n * v);
  led.add(owner, job, r.off, n, r.aoff);
}
// the combine at commit: room for k survivors of 11 bytes each at the tail, then the owner's ranges replaced by it
static uint64_t combine(PoolLedger& led, uint64_t owner, const std::string& job, uint64_t k) {
  const PoolLedger::Room r = led.take(k, 11 * k);
  led.replace_open(owner, job, r.off, k, r.aoff);
  return r.off;
}

int main() {
  {  // a combined job replaced while its new range sits at the tail, and a later abort reaches it: the new range's
     // room and value bytes come back, the job's emptied original room does not
    PoolLedger led;
    led.byte_values = true;
    const uint64_t a = led.new_owner(), b = led.new_owner();
    emit(led, a, "j", 100, 11);
    emit(led, b, "j", 5, 11);  // the same job id again, on a second handle
    const uint64_t off = combine(led, a, "j", 7);
    CHECK(off == 105 && led.used() == 112 && led.arena_used() == 105 * 11 + 77);
    CHECK((led.open_ranges(a) == Ranges{{105, 7}}));
    led.commit(a, "j");
    CHECK((led.live() == Ranges{{105, 7}}));
    led.commit(b, "j");  // replace-by-job-id: the combined range dies at the tail
    CHECK((led.live() == Ranges{{100, 5}}));
    const uint64_t c = led.new_owner();
    emit(led, c, "k", 3, 11);
    led.abort(c);  // c's room, then the dead combined range's, come back; b's live range stops the walk
    CHECK(led.used() == 105 && led.arena_used() == 105 * 11 && (led.live() == Ranges{{100, 5}}));
    const uint64_t d = led.new_owner();
    emit(led, d, "k", 2, 11);  // the room is handed out again
    CHECK((led.open_ranges(d) == Ranges{{105, 2}}));
    led.commit(d, "k");
    led.commit(led.new_owner(), "j");  // (an owner without ranges replaces b's job: b's range dies)
    const uint64_t e = led.new_owner();
    emit(led, e, "z", 1, 11);
    led.abort(e);  // d's live range stops the walk
    CHECK(led.used() == 107 && (led.live() == Ranges{{105, 2}}));
  }
  {  // the combined job's own dead range at the tail, reached by an abort: the room down to the combined range's start
    PoolLedger led;
    led.byte_values = true;
    const uint64_t a = led.new_owner();
    emit(led, a, "j", 20, 11);
    combine(led, a, "j", 2);  // original room 0..20 emptied, new range 20..22
    const uint64_t b = led.new_owner();
    emit(led, b, "k", 3, 11);  // open behind it
    led.abort(a);  // a dies before commit: b is open at the tail, so nothing comes back
    CHECK(led.used() == 25);
    led.abort(b);  // b's room, then a's new range, come back; a's emptied original room does not
    CHECK(led.used() == 20 && led.arena_used() == 220 && led.live().empty());
    CHECK(led.open_job() == nullptr);
  }
  {  // several handles open and interleaved: only the committing owner's ranges are emptied and replaced
    PoolLedger led;
    led.byte_values = true;
    const uint64_t a = led.new_owner(), b = led.new_owner();
    emit(led, a, "ja", 10, 11);
    emit(led, b, "jb", 5, 11);
    emit(led, a, "ja", 10, 11);
    emit(led, b, "jb", 5, 11);
    const uint64_t off = combine(led, a, "ja", 4);
    CHECK(off == 30);
    CHECK((led.open_ranges(a) == Ranges{{30, 4}}));
    CHECK((led.open_ranges(b) == Ranges{{10, 5}, {25, 5}}));
    emit(led, b, "jb", 5, 11);  // b goes on behind a's new range: never joined to it
    CHECK((led.open_ranges(b) == Ranges{{10, 5}, {25, 5}, {34, 5}}));
    led.commit(a, "ja");
    CHECK((led.live() == Ranges{{30, 4}}));
    const uint64_t off2 = combine(led, b, "jb", 2);
    CHECK(off2 == 39);
    led.commit(b, "jb");
    CHECK((led.live() == Ranges{{30, 4}, {39, 2}}) && led.used() == 41);
    // a single handle whose open range ends at the tail: the new room is a range of its own, not a continuation
    PoolLedger l2;
    l2.byte_values = true;
    const uint64_t c = l2.new_owner();
    emit(l2, c, "j", 8, 11);
    combine(l2, c, "j", 1);
    CHECK((l2.open_ranges(c) == Ranges{{8, 1}}));
    l2.commit(c, "j");
    CHECK((l2.live() == Ranges{{8, 1}}));
  }
  {  // the pool grows during the commit: a mark taken before the combine's room rewinds it, and a combine after more
     // room than the first take (several flushes) keeps every original range emptied
    PoolLedger led;
    led.byte_values = true;
    const uint64_t a = led.new_owner();
    for (int k = 0; k < 5; k++) emit(led, a, "j", 1000, 11);  // one open range, grown flush by flush
    CHECK((led.open_ranges(a) == Ranges{{0, 5000}}));
    const PoolLedger::Mark mk = led.mark();
    led.take(9, 99);  // a failed combine: its room rewinds
    led.rewind(mk);
    CHECK(led.used() == 5000 && led.arena_used() == 55000 && (led.open_ranges(a) == Ranges{{0, 5000}}));
    combine(led, a, "j", 9);
    CHECK(led.used() == 5009 && led.arena_used() == 55099);
    led.commit(a, "j");
    CHECK((led.live() == Ranges{{5000, 9}}));
    // 2^32 - 1 pairs between resets: survivors count against it
    PoolLedger l2;
    l2.byte_values = true;
    const uint64_t b = l2.new_owner();
    emit(l2, b, "j", 0xffffffffull - 10, 0);
    CHECK(l2.fits(9) && !l2.fits(10));
  }
  std::printf(fails ? "FAIL\n" : "ok\n");
  return fails != 0;
}
