// mrhbm_pool.h -- the ledger of the HBM emit pool: which records belong to which map job, and how much of the pool
// and of the value arena is in use (no CUDA runtime calls, no ctx; the memory itself and its growth are the ctx's).
//
// The pool is filled from its tail.  A map handle (an owner) takes room, fills it and adds it as an open range of its
// job.  Commit makes the owner's open ranges the job's output and kills what an earlier commit of the same job id left
// (replace-by-job-id, mapreduce/job.lua:217-221); abort kills the owner's open ranges (worker.lua:120-127).  What the
// ledger keeps:
//   - ranges are in pool order and never overlap; every record below used() that no range covers is lost room, so
//     room that is taken is either added or rewound;
//   - MRHBM_F_BYTE_VALUES: a pair's value id is its pool index and values are appended to the arena in pool order,
//     so room in both is taken together (voff[used()] == arena_used() always) and goes back together: a range
//     remembers the arena offset of its first value.  The pairs of one tokeniser piece (mrhbm_map_words_value)
//     share the id of the piece's first pair, which holds the value; the other ids of the piece hold empty values;
//   - dead ranges at the tail give their room back when an abort finds them there; dead ranges with live or open
//     records behind them keep their room (records and value bytes) until reset();
//   - MRHBM_COMBINE_DISTINCT: shrink() keeps the first records of an open range (its distinct pairs, moved forward)
//     and leaves the rest as lost room until reset(): a kept pair's value id may point past the new end, to bytes
//     that must stay where they are.  A shrunk range that dies at the tail no longer ends at used(), so no abort
//     gives that room back.
//   - MRHBM_COMBINE_FSUM: replace_open() empties all of an owner's open ranges and makes room taken at the tail, which
//     holds the job's new pairs with values of their own, the owner's only open range with records.  The emptied
//     ranges' room is lost until reset(); the new range is like any other: it dies, and at the tail gives its room
//     back, as a whole.  An emptied range never ends at used() again (the new range lies behind it), so no abort
//     reaches past the new range into the job's original room.
#pragma once
#include <cassert>
#include <cstdint>
#include <string>
#include <utility>
#include <vector>

namespace mrhbm {

class PoolLedger {
 public:
  struct Mark {
    size_t ranges;
    uint64_t last_cnt, used, arena_used;
  };
  struct Room {
    uint64_t off, aoff;  // the first record, the first value byte
  };

  bool byte_values = false;  // value ids are u32 in string records: fewer than 2^32 - 1 pairs between resets

  uint64_t used() const { return used_; }
  uint64_t arena_used() const { return arena_used_; }
  uint64_t new_owner() { return ++owners_; }

  // rewind(mark()) undoes every take and add since the mark (no commit, shrink, abort or reset may lie between)
  Mark mark() const { return Mark{ranges_.size(), ranges_.empty() ? 0 : ranges_.back().cnt, used_, arena_used_}; }
  void rewind(const Mark& mk) {
    assert(mk.ranges <= ranges_.size() && mk.used <= used_ && mk.arena_used <= arena_used_);
    ranges_.erase(ranges_.begin() + (ptrdiff_t)mk.ranges, ranges_.end());
    if (mk.ranges) ranges_.back().cnt = mk.last_cnt;
    used_ = mk.used;
    arena_used_ = mk.arena_used;
  }

  bool fits(uint64_t n) const { return !byte_values || used_ + n < 0xffffffffull; }
  // n records and `bytes` value bytes at the tail; needs fits(n)
  Room take(uint64_t n, uint64_t bytes) {
    assert(fits(n));
    const Room r{used_, arena_used_};
    used_ += n;
    arena_used_ += bytes;
    return r;
  }
  // taken room becomes an open range of the owner's, one with the range it continues
  void add(uint64_t owner, const std::string& job, uint64_t off, uint64_t cnt, uint64_t aoff) {
    if (!ranges_.empty()) {
      Range& r = ranges_.back();
      if (r.owner == owner && r.state == OPEN && r.off + r.cnt == off) {
        r.cnt += cnt;
        return;
      }
    }
    ranges_.push_back(Range{off, cnt, job, OPEN, owner, aoff});
  }

  // the owner's open ranges that hold records, as (first, count), in pool order
  std::vector<std::pair<uint64_t, uint64_t>> open_ranges(uint64_t owner) const {
    std::vector<std::pair<uint64_t, uint64_t>> v;
    for (const Range& r : ranges_)
      if (r.owner == owner && r.state == OPEN && r.cnt) v.emplace_back(r.off, r.cnt);
    return v;
  }
  // the owner's open range of records that starts at off keeps its first cnt records (see the invariants above)
  void shrink(uint64_t owner, uint64_t off, uint64_t cnt) {
    for (Range& r : ranges_)
      if (r.owner == owner && r.state == OPEN && r.cnt && r.off == off) {
        assert(cnt <= r.cnt);
        r.cnt = cnt;
        return;
      }
    assert(!"shrink: no such open range");
  }
  // taken room [off, off + cnt) replaces all of the owner's open ranges: they keep no records, and the room becomes an
  // open range of the owner's of its own, never one with a range before it (see the invariants above)
  void replace_open(uint64_t owner, const std::string& job, uint64_t off, uint64_t cnt, uint64_t aoff) {
    assert(off + cnt == used_);
    for (Range& r : ranges_)
      if (r.owner == owner && r.state == OPEN) r.cnt = 0;
    ranges_.push_back(Range{off, cnt, job, OPEN, owner, aoff});
  }

  void commit(uint64_t owner, const std::string& job) {
    for (Range& r : ranges_)
      if (r.state == COMMITTED && r.job == job) r.state = DEAD;  // replace-by-job-id
    for (Range& r : ranges_)
      if (r.owner == owner && r.state == OPEN) r.state = COMMITTED;
  }
  // (the caller has waited for the copies into the owner's ranges: their room may be handed out again)
  void abort(uint64_t owner) {
    for (Range& r : ranges_)
      if (r.owner == owner && r.state == OPEN) r.state = DEAD;
    while (!ranges_.empty() && ranges_.back().state == DEAD && ranges_.back().off + ranges_.back().cnt == used_) {
      used_ = ranges_.back().off;
      arena_used_ = ranges_.back().aoff;
      ranges_.pop_back();
    }
  }
  void reset() {
    ranges_.clear();
    used_ = arena_used_ = 0;
  }

  // committed records as (first, count), adjacent ranges merged
  std::vector<std::pair<uint64_t, uint64_t>> live() const {
    std::vector<std::pair<uint64_t, uint64_t>> v;
    for (const Range& r : ranges_) {
      if (r.state != COMMITTED || !r.cnt) continue;
      if (!v.empty() && v.back().first + v.back().second == r.off)
        v.back().second += r.cnt;
      else
        v.emplace_back(r.off, r.cnt);
    }
    return v;
  }
  // the job of some range that is still open, or null
  const std::string* open_job() const {
    for (const Range& r : ranges_)
      if (r.state == OPEN) return &r.job;
    return nullptr;
  }

 private:
  enum { OPEN, COMMITTED, DEAD };
  struct Range {
    uint64_t off, cnt;
    std::string job;
    int state;
    uint64_t owner;  // map handle serial
    uint64_t aoff;   // the arena offset of the range's first value (its bytes follow in pool order)
  };
  std::vector<Range> ranges_;
  uint64_t used_ = 0, arena_used_ = 0, owners_ = 0;
};

}  // namespace mrhbm
