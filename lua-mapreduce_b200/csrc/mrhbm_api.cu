// mrhbm_api.cu -- host runtime behind the C ABI of include/mrhbm.h: HBM emit pool, map-job
// bookkeeping (commit = replace-by-job-id, abort = discard; mapreduce/job.lua:217-221,
// worker.lua:120-127), the shuffle driver, result iteration.  No CPU fallback anywhere.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <initializer_list>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "../../include/mrhbm.h"
#include "mrhbm_comm.h"
#include "mrhbm_decimal.cuh"
#include "mrhbm_kernels.h"
#include "mrhbm_dev.cuh"  // splitmix64
#include "mrhbm_keys.h"
#include "mrhbm_numsum.cuh"
#include "mrhbm_pool.h"
#include "mrhbm_split_plan.h"

using namespace mrhbm;

namespace {
constexpr uint32_t kErrfLongKeys = 0x80000000u;  // rides on the error-flag all-gather of a multi-GPU shuffle: this rank holds long keys
constexpr size_t kMaxLongKey = 1u << 20;  // bytes; longer keys are refused (MRHBM_E_KEY)
struct LongPair {
  std::string esc;  // the key as a record slot would hold it: 0x00 / 0x01 escaped (order preserving, see escape)
  uint64_t value;
  std::string bytes;  // MRHBM_F_BYTE_VALUES: the value
};
struct LongGroup {
  std::string esc;
  std::vector<uint64_t> values;  // built-in sum: one element
};

constexpr size_t kStageRecs = 1 << 16;
constexpr size_t kStageValBytes = 4u << 20;       // value bytes staged next to the records; a longer value goes alone
constexpr uint64_t kMaxValue = 1ull << 30;        // bytes; longer values are refused (MRHBM_E_INVAL)
enum { EV_START, EV_CSTART, EV_COMBINE, EV_HIST, EV_PLAN, EV_GATH, EV_SCATTER, EV_EXCH, EV_SORT, EV_BIG, EV_END, EV_PROBE, EV_N };
constexpr uint32_t kSampleKeys = 1u << 18;      // keys sampled to decide between key-ordered and hash sub-bins
}  // namespace

struct mrhbm_ctx {
  mrhbm_config cfg{};
  int dev = 0, rb = 16, kb = 8, sm_count = 132;
  cudaStream_t stream = nullptr;
  // HBM emit pool: committed + open map output, record granularity; led says what is in use and whose it is
  void* pool = nullptr;
  uint64_t pool_cap = 0;
  PoolLedger led;
  // MRHBM_F_BYTE_VALUES: a pair's value field holds its pool index (value id); value id i has the bytes
  // arena[voff[i] .. voff[i+1])
  bool bytevals = false;
  unsigned char* arena = nullptr;
  uint64_t arena_cap = 0;
  uint64_t* voff = nullptr;  // pool_cap + 1 entries
  // after the compaction: row r's value at cvals[row_off[r] .. row_off[r+1])
  unsigned char* cvals = nullptr;
  uint64_t *row_off = nullptr, *val_tile = nullptr, *val_pieces = nullptr;
  uint64_t cvals_cap = 0, row_cap = 0, tile_cap = 0, pieces_cap = 0, cvals_bytes = 0;
  std::vector<const std::string*> long_vals;  // values of the long-key groups (LongGroup::values index them)
  std::deque<std::string> long_sums;          // MRHBM_RED_FSUM / _COUNT_DISTINCT: the long-key groups' encoded results (long_vals point here)
  // Keys that do not fit a record slot (rare: the reference takes any key length, utils.lua:104-110) never reach the
  // device: their pairs wait on the host, per committed map job, are partitioned and grouped at the barrier (on several
  // GPUs after an all-gather) and merged into the reduce-side iteration at their place in the key order.
  std::map<std::string, std::vector<LongPair>> long_jobs;  // committed pairs by job id (commit = replace-by-id)
  std::vector<std::vector<LongGroup>> long_groups;         // after a shuffle: per owned partition, ascending escaped key
  uint64_t long_group_count = 0;
  bool any_long = false;  // several GPUs: some rank holds such pairs (learnt with the error flags every shuffle gathers anyway)
  // shuffle state
  ShuffleBuffers sb{};
  uint64_t B_cap = 0, mid_cap = 0, out_cap = 0;
  uint32_t B = 0, S = 1, ordered = 1, cap = 0, ctr_shift = 3;
  uint64_t ctr_cap = 0;
  ShuffleBuffers rv{};  // view the result accessors use (single GPU: == sb)
  // multi-GPU (one ctx per rank; partition p is owned by rank p % world)
  int world = 1, rank = 0;
  uint32_t Pl = 0, pbase[9] = {0}, bin_base = 0;
  uint64_t N_recv = 0;
  uint32_t *d_hd = nullptr, *d_hall = nullptr, *d_tot = nullptr, *d_outoff = nullptr, *d_segoff = nullptr;
  uint64_t hd_cap = 0, bl_cap = 0;
  void *recvbuf = nullptr, *bigbuf = nullptr;
  uint64_t recv_cap = 0, big_cap = 0;
  // coarse regions of the two-level split (optimistic layout).  On several GPUs every rank's buffer is exported
  // with cudaIpcGetMemHandle and mapped by its peers: level 2 of a region's owner pulls it from all of them.
  void* regions = nullptr;
  uint64_t regions_cap = 0;                   // records (the same on all ranks)
  void* peer_regions[8] = {nullptr};          // peer_regions[rank] == regions
  bool ipc_failed = false;                    // peer mapping unavailable: NCCL exchange (exact layout) instead
  uint32_t* d_l1all = nullptr;                // all ranks' level-1 fill levels
  uint64_t l1all_cap = 0;
  uint32_t *d_ipc = nullptr, *h_ipc = nullptr;  // 16 words per rank: the IPC handles
  uint32_t *d_sample = nullptr, *h_sample = nullptr;  // 256 buckets of the key sample
  // MRHBM_PART_RANGE: the installed splitters (original bytes; u64 keys: 8 big-endian bytes), a digest that the shuffle
  // compares across ranks, and their device form (RangeTable): prefixes, thresholds as key slots, per-partition inverse
  // widths in one allocation
  std::vector<std::string> spl;
  bool spl_set = false;
  uint64_t spl_digest = 0;
  void* d_spl = nullptr;
  uint32_t spl_fin = 0;  // finite thresholds (RangeBinParams::spl_n)
  uint64_t shuffle_spl_digest = 0;  // the splitters the last shuffle partitioned with (mrhbm_checksum_result)
  std::recursive_mutex mu;                    // entry points serialise per ctx
  uint32_t *d_small = nullptr, *h_small = nullptr;  // 64 words each
  bool no_optimistic = false;  // sticky: a fixed-capacity bin overflowed once (skewed keys)
  bool no_ordered = false;     // sticky: key-ordered sub-bins overflowed once (clustered keys)
  void* l1buf = nullptr;  // coarse regions of the two-level split
  uint64_t l1_cap = 0;
  // device tokeniser scratch (mrhbm_map_wordcount)
  unsigned char* d_tok_text[2] = {nullptr, nullptr};
  uint32_t *d_tok_cnt = nullptr, *d_tok_off = nullptr;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t tok_ev[2] = {nullptr, nullptr};
  // mrhbm_map_key_numbers: the power-of-five table of the decimal conversion and the fix-up list (kKnFixCap entries)
  uint64_t* d_pow5 = nullptr;
  void* d_kn_fix = nullptr;
  // map-side combiner: the global (L2 resident) hash table and the records compacted out of it
  void *comb = nullptr, *gtab = nullptr;
  uint64_t comb_cap = 0, gtab_cap = 0;  // records
  uint32_t gtab_grow = 0;               // doublings of the combiner's table beyond its L2-resident size (GtabLayout::sized)
  bool no_combine = false;              // sticky: more distinct keys than the largest table takes
  bool combine_checked = false;         // sticky: values large enough that u32 sums must be checked add by add
  // MRHBM_COMBINE_DISTINCT at commit: the hash set (kept across commits, grown by doubling), the entry of every record
  // of the job, the survivors before they are copied back, the job's ranges and its tile counts and offsets
  void *dd_tab = nullptr, *dd_out = nullptr, *dd_rg = nullptr;
  uint32_t *dd_slot = nullptr, *dd_tiles = nullptr;
  uint64_t dd_tab_cap = 0, dd_rec_cap = 0, dd_rg_cap = 0, dd_tiles_cap = 0;  // entries, records, ranges, tiles
  // MRHBM_COMBINE_FSUM at commit: the distinct combiner's hash set, entry of every record, ranges and tiles (dd_*), and
  // FsumScratch's per-entry words, values, big keys and their accumulators, and flag words
  uint32_t *fs_words = nullptr, *fs_big = nullptr, *fs_small = nullptr;
  uint64_t* fs_vals = nullptr;
  int64_t* fs_gacc = nullptr;
  uint64_t fs_words_cap = 0, fs_vals_cap = 0, fs_big_cap = 0;
  // MRHBM_RED_DISTINCT: the shuffle runs the same set over all committed pairs, and orders every bin's rows by value
  // bytes; the merge of an oversized bin's chunks alternates with these scratch rows (out_cap of them)
  bool red_distinct = false;
  void* vo_keys = nullptr;
  uint64_t* vo_ids = nullptr;
  uint64_t vo_cap = 0;
  // MRHBM_RED_FSUM: the shuffle sums every key's numbers (mrhbm_num_sum.cu); the partial accumulators of the groups
  // that cross a chunk of an oversized bin live here (ns_cap slots, see NumScratch)
  bool red_fsum = false;
  int64_t* ns_acc = nullptr;
  uint32_t *ns_flags = nullptr, *ns_head = nullptr;
  uint64_t ns_cap = 0;
  // MRHBM_RED_COUNT_DISTINCT: the distinct set's survivors carry the value 1 through the integer sum of MRHBM_RED_SUM;
  // the first result access encodes each key's count as a number (k_num_encode)
  bool red_count = false;
  uint64_t N = 0, groups = 0;
  bool shuffled = false;
  std::vector<uint32_t> h_bin_off, h_uoff;
  std::vector<uint32_t> h_big;  // group-only mode: oversized bins, each holding runs of `cap` rows
  void* ckeys = nullptr;
  uint64_t* csums = nullptr;
  uint64_t c_cap = 0;
  bool compacted = false;
  uint64_t* d_acc = nullptr;       // 8 x u64 scratch
  uint32_t* h_counters = nullptr;  // pinned, 8 x u32
  uint64_t* h_acc = nullptr;       // pinned, 8 x u64
  // zipf table cache
  uint64_t* d_table = nullptr;
  uint64_t d_table_V = 0, d_table_first = 0, d_table_last = 0;
  mrhbm_stats stats{};
  cudaEvent_t ev[EV_N]{};
  Comm* comm = nullptr;
  std::string err;
};

struct mrhbm_map {
  mrhbm_ctx* ctx;
  std::string job;
  std::vector<LongPair> long_pairs;  // keys longer than a record slot (host side, see mrhbm_ctx::long_jobs)
  uint64_t serial;
  unsigned char* stage[2] = {nullptr, nullptr};
  cudaEvent_t stage_ev[2] = {nullptr, nullptr};
  bool stage_busy[2] = {false, false};
  int cur = 0;
  size_t fill = 0;
  bool async_reads = false;  // pinned user memory still being read by the copy engine
  // MRHBM_F_BYTE_VALUES: the staged records' value bytes and their offsets (fill + 1 of them), pinned, double
  // buffered with the record stage
  unsigned char* vstage[2] = {nullptr, nullptr};
  uint64_t* vrel[2] = {nullptr, nullptr};
};

struct RunCursor {
  uint64_t pos, end;
};
struct mrhbm_iter {
  mrhbm_ctx* ctx;
  std::vector<uint64_t> valbuf;  // group-only mode: the values of the current key
  std::vector<unsigned char> unesc;  // the current key's original bytes (reserved: not null even for the empty key)
  std::vector<unsigned char> keys;
  std::vector<uint64_t> sums;
  std::vector<RunCursor> runs;
  std::vector<uint32_t> heap;  // the runs that still have rows, a binary min-heap on their current key (heap.lua:29-93)
  uint64_t base = 0;
  const std::vector<LongGroup>* longs = nullptr;  // the partition's long-key groups and the next one to hand out
  size_t long_pos = 0;
  bool sorted = true;
  size_t cur_run = 0;
  std::vector<uint64_t> rows;  // the rows of the current key (indices into keys / sums)
  // MRHBM_F_BYTE_VALUES: the partition's row offsets (rows + 1, relative to its first) and value bytes, and the
  // current group's values packed
  std::vector<uint64_t> roff;
  std::vector<unsigned char> vbytes;
  std::vector<unsigned char> vout;
  std::vector<uint64_t> vout_off;
};

namespace {

int fail(mrhbm_ctx* c, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code;
}
#define CU(c, expr)                                                                               \
  do {                                                                                            \
    cudaError_t e_ = (expr);                                                                      \
    if (e_ != cudaSuccess) {                                                                      \
      cudaGetLastError();                                                                         \
      return fail((c), e_ == cudaErrorMemoryAllocation ? MRHBM_E_NOMEM : MRHBM_E_CUDA,            \
                  "CUDA error %s at %s:%d: %s", cudaGetErrorName(e_), __FILE__, __LINE__,         \
                  cudaGetErrorString(e_));                                                        \
    }                                                                                             \
  } while (0)

// Every entry point that touches CUDA runs with the ctx's device current (a ctx may be driven from any
// thread, and several ctxs on different GPUs may share one thread) and holds the ctx lock: the handle is
// single-caller by contract (include/mrhbm.h), the lock turns a violation into serialisation instead of a race.
struct Entry {
  std::lock_guard<std::recursive_mutex> lk;
  int prev = -1;
  explicit Entry(mrhbm_ctx* c) : lk(c->mu) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != c->dev) cudaSetDevice(c->dev);
    else prev = -1;
  }
  ~Entry() {
    if (prev >= 0) cudaSetDevice(prev);
    cudaGetLastError();
  }
};

// a device buffer of `want` elements of `elem` bytes that keeps its first `keep` elements
int regrow(mrhbm_ctx* c, void** p, uint64_t want, uint64_t keep, size_t elem) {
  void* np = nullptr;
  CU(c, cudaMalloc(&np, want * elem));
  if (keep) CU(c, cudaMemcpyAsync(np, *p, keep * elem, cudaMemcpyDeviceToDevice, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  if (*p) CU(c, cudaFree(*p));
  *p = np;
  return 0;
}

// Room at the tail of the pool (and of the arena) between the moment it is taken and the moment it becomes a range of
// a map's output.  If its owner returns before add() -- a copy or a launch failed -- the ledger is rewound and the
// room is free again.
struct Reservation {
  PoolLedger* led = nullptr;  // set while the room is held
  PoolLedger::Mark mk{};
  uint64_t off = 0, aoff = 0, n = 0;
  ~Reservation() {
    if (led) led->rewind(mk);
  }
  void add(const mrhbm_map* m) {
    led->add(m->serial, m->job, off, n, aoff);
    led = nullptr;
  }
  // MRHBM_COMBINE_FSUM: the room replaces all of the map's open ranges
  void replace(const mrhbm_map* m) {
    led->replace_open(m->serial, m->job, off, n, aoff);
    led = nullptr;
  }
};

int stage_flush(mrhbm_map* m);

// r: room for n records straight in the pool and, with byte values, for the `bytes` bytes of their values in the arena
// (values follow pool order).  With `behind`, the room lies behind what that map has staged (emission order).  The
// caller fills the room and then adds it.
int reserve(mrhbm_ctx* c, mrhbm_map* behind, uint64_t n, uint64_t bytes, Reservation& r) {
  int rc = behind ? stage_flush(behind) : 0;
  if (rc) return rc;
  PoolLedger& led = c->led;
  if (!led.fits(n)) return fail(c, MRHBM_E_INVAL, "byte values: 2^32 pairs emitted since the last reset");
  if (led.used() + n > c->pool_cap) {
    uint64_t want = std::max<uint64_t>(led.used() + n, c->pool_cap * 2);
    want = std::max<uint64_t>(want, 1 << 16);
    rc = regrow(c, &c->pool, want, led.used(), (size_t)c->rb);
    if (!rc && c->bytevals) rc = regrow(c, (void**)&c->voff, want + 1, c->voff ? led.used() + 1 : 0, sizeof(uint64_t));
    if (rc) return rc;
    c->pool_cap = want;
  }
  if (led.arena_used() + bytes > c->arena_cap) {
    uint64_t want = std::max<uint64_t>(led.arena_used() + bytes, c->arena_cap * 2);
    want = std::max<uint64_t>(want, 1 << 20);
    rc = regrow(c, (void**)&c->arena, want, led.arena_used(), 1);
    if (rc) return rc;
    c->arena_cap = want;
  }
  r.mk = led.mark();
  const PoolLedger::Room room = led.take(n, bytes);
  r.led = &led;
  r.off = room.off;
  r.aoff = room.aoff;
  r.n = n;
  return 0;
}

// MRHBM_F_BYTE_VALUES: the value id into a record
void put_value_id(unsigned char* rec, int rb, int kb, uint64_t id) {
  if (rb == 16)
    memcpy(rec + 8, &id, 8);
  else {
    const uint32_t id32 = (uint32_t)id;
    memcpy(rec + kb, &id32, 4);
  }
}

int stage_flush(mrhbm_map* m) {
  mrhbm_ctx* c = m->ctx;
  if (!m->fill) return 0;
  const uint64_t bytes = c->bytevals ? m->vrel[m->cur][m->fill] : 0;
  Reservation r;
  int rc = reserve(c, nullptr, m->fill, bytes, r);
  if (rc) return rc;
  if (c->bytevals) {
    // the staged records get their value ids, the staged offsets become arena offsets
    for (size_t i = 0; i < m->fill; i++) put_value_id(m->stage[m->cur] + i * c->rb, c->rb, c->kb, r.off + i);
    for (size_t i = 0; i <= m->fill; i++) m->vrel[m->cur][i] += r.aoff;
    if (bytes) CU(c, cudaMemcpyAsync(c->arena + r.aoff, m->vstage[m->cur], bytes, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(c->voff + r.off, m->vrel[m->cur], (m->fill + 1) * 8, cudaMemcpyHostToDevice, c->stream));
  }
  CU(c, cudaMemcpyAsync((char*)c->pool + r.off * c->rb, m->stage[m->cur], m->fill * c->rb, cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaEventRecord(m->stage_ev[m->cur], c->stream));
  m->stage_busy[m->cur] = true;
  r.add(m);
  m->fill = 0;
  m->cur ^= 1;
  if (m->stage_busy[m->cur]) {
    CU(c, cudaEventSynchronize(m->stage_ev[m->cur]));
    m->stage_busy[m->cur] = false;
  }
  return 0;
}

int stage_slot(mrhbm_map* m, unsigned char** slot) {
  mrhbm_ctx* c = m->ctx;
  if (!m->stage[0]) {
    for (int i = 0; i < 2; i++) {
      CU(c, cudaHostAlloc((void**)&m->stage[i], kStageRecs * c->rb, cudaHostAllocDefault));
      CU(c, cudaEventCreateWithFlags(&m->stage_ev[i], cudaEventDisableTiming));
      if (c->bytevals) {
        CU(c, cudaHostAlloc((void**)&m->vstage[i], kStageValBytes, cudaHostAllocDefault));
        CU(c, cudaHostAlloc((void**)&m->vrel[i], (kStageRecs + 1) * sizeof(uint64_t), cudaHostAllocDefault));
      }
    }
  }
  if (m->fill == kStageRecs) {
    int rc = stage_flush(m);
    if (rc) return rc;
  }
  *slot = m->stage[m->cur] + m->fill * c->rb;
  m->fill++;
  return 0;
}

int check_value(mrhbm_ctx* c, const void* val, size_t vlen) {
  if (vlen > kMaxValue) return fail(c, MRHBM_E_INVAL, "value of %zu bytes (limit %llu)", vlen, (unsigned long long)kMaxValue);
  if (vlen && !val) return fail(c, MRHBM_E_INVAL, "null value");
  return 0;
}

// MRHBM_F_BYTE_VALUES: one pair, its key written into the record slot by key_to_slot, its value staged next to it.  A
// value larger than the value stage goes to the device on its own, behind what is staged.
template <class F>
int stage_value_pair(mrhbm_map* m, const void* val, size_t vlen, F key_to_slot) {
  mrhbm_ctx* c = m->ctx;
  int rc = check_value(c, val, vlen);
  if (rc) return rc;
  if (vlen > kStageValBytes) {
    Reservation r;
    rc = reserve(c, m, 1, vlen, r);
    if (rc) return rc;
    unsigned char rec[128];
    key_to_slot(rec);
    put_value_id(rec, c->rb, c->kb, r.off);
    const uint64_t vo[2] = {r.aoff, r.aoff + vlen};
    CU(c, cudaMemcpyAsync(c->arena + r.aoff, val, vlen, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(c->voff + r.off, vo, sizeof vo, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync((char*)c->pool + r.off * c->rb, rec, c->rb, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));  // (the caller's value may be pinned memory: copied before return)
    r.add(m);
    return MRHBM_OK;
  }
  if (m->stage[0] && m->fill && m->vrel[m->cur][m->fill] + vlen > kStageValBytes) {
    rc = stage_flush(m);
    if (rc) return rc;
  }
  unsigned char* slot;
  rc = stage_slot(m, &slot);
  if (rc) return rc;
  const size_t i = m->fill - 1;
  if (i == 0) m->vrel[m->cur][0] = 0;
  key_to_slot(slot);
  if (vlen) memcpy(m->vstage[m->cur] + m->vrel[m->cur][i], val, vlen);
  m->vrel[m->cur][i + 1] = m->vrel[m->cur][i] + vlen;
  return MRHBM_OK;
}

int refuse_int_values(mrhbm_ctx* c) {
  return fail(c, MRHBM_E_INVAL, "the ctx carries byte values (MRHBM_F_BYTE_VALUES): use the *_value calls");
}
int refuse_byte_values(mrhbm_ctx* c) {
  return fail(c, MRHBM_E_INVAL, "byte values need a ctx with MRHBM_F_BYTE_VALUES");
}

// A key whose escaped form (elen bytes) does not fit a record slot stays on the host, escaped like a slot would hold
// it, with its value or value bytes (see mrhbm_ctx::long_jobs).
int long_pair(mrhbm_map* m, const unsigned char* k, size_t klen, size_t elen, uint64_t value, const void* val, size_t vlen) {
  mrhbm_ctx* c = m->ctx;
  if (klen > kMaxLongKey) return fail(c, MRHBM_E_KEY, "key of %zu bytes (limit %zu)", klen, (size_t)kMaxLongKey);
  int rc = check_value(c, val, vlen);
  if (rc) return rc;
  LongPair lp;
  lp.esc.resize(elen);
  escape(k, klen, (unsigned char*)&lp.esc[0]);
  lp.value = value;
  if (vlen) lp.bytes.assign((const char*)val, vlen);
  m->long_pairs.push_back(std::move(lp));
  return MRHBM_OK;
}

// a host pointer that the copy engine reads in place: a copy from it is still running when the call returns
bool is_pinned(const void* p) {
  cudaPointerAttributes at{};
  const bool pinned = p && cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeHost;
  cudaGetLastError();
  return pinned;
}

void map_release(mrhbm_map* m) {
  for (int i = 0; i < 2; i++) {
    if (m->stage_busy[i]) cudaEventSynchronize(m->stage_ev[i]);
    if (m->stage_ev[i]) cudaEventDestroy(m->stage_ev[i]);
    if (m->stage[i]) cudaFreeHost(m->stage[i]);
    if (m->vstage[i]) cudaFreeHost(m->vstage[i]);
    if (m->vrel[i]) cudaFreeHost(m->vrel[i]);
  }
  delete m;
}

void invalidate(mrhbm_ctx* c) {
  c->shuffled = false;
  c->compacted = false;
  c->long_groups.clear();
  c->long_group_count = 0;
  c->long_vals.clear();
  c->long_sums.clear();
}

struct DevBuf {
  void** p;
  size_t elem;  // bytes per element
};
// Grows device buffers that share one capacity to at least `need` elements each; their contents are not kept.  When
// they hold fewer, they are freed and `alloc` >= need elements (the caller's headroom) are allocated: *cap = alloc.
int grow(mrhbm_ctx* c, uint64_t* cap, uint64_t need, uint64_t alloc, std::initializer_list<DevBuf> bufs) {
  if (need <= *cap) return 0;
  *cap = 0;
  for (const DevBuf& b : bufs) {
    if (*b.p) CU(c, cudaFree(*b.p));
    *b.p = nullptr;
  }
  for (const DevBuf& b : bufs) CU(c, cudaMalloc(b.p, alloc * b.elem));
  *cap = alloc;
  return 0;
}

// at least `need` records, and at least one
int ensure_records(mrhbm_ctx* c, void** buf, uint64_t* cap, uint64_t need) {
  need = std::max<uint64_t>(need, 1);
  return grow(c, cap, need, need, {{buf, (size_t)c->rb}});
}

// the sorted output: keys and sums of at least `need` rows, and at least one
int ensure_out(mrhbm_ctx* c, uint64_t need) {
  need = std::max<uint64_t>(need, 1);
  return grow(c, &c->out_cap, need, need, {{&c->sb.out_keys, (size_t)c->kb}, {(void**)&c->sb.out_sums, sizeof(uint64_t)}});
}

// per-bin arrays (offsets, group counts, spread-out atomic counters) for B bins
int ensure_small_arrays(mrhbm_ctx* c, uint64_t B) {
  int rc = grow(c, &c->B_cap, B + 1, B + 1 + (B >> 2),
                {{(void**)&c->sb.bin_off, 4}, {(void**)&c->sb.ucount, 4}, {(void**)&c->sb.uoff, 4}, {(void**)&c->sb.big_list, 4}});
  if (rc) return rc;
  rc = grow(c, &c->ctr_cap, B << c->ctr_shift, (B + (B >> 2) + 1) << c->ctr_shift,  // spread-out atomic counters
            {{(void**)&c->sb.hist, 4}, {(void**)&c->sb.cursor, 4}});
  if (rc) return rc;
  if (!c->sb.counters) CU(c, cudaMalloc((void**)&c->sb.counters, 8 * sizeof(uint32_t)));
  return 0;
}

int ensure_buffers(mrhbm_ctx* c, uint64_t B, uint64_t N) {
  int rc = ensure_small_arrays(c, B);
  if (!rc) rc = ensure_records(c, &c->sb.mid, &c->mid_cap, N);
  return rc ? rc : ensure_out(c, N);
}

int ensure_compact(mrhbm_ctx* c) {
  if (!c->shuffled) return fail(c, MRHBM_E_INVAL, "no shuffle result (call mrhbm_shuffle first)");
  if (c->compacted) return 0;
  const uint64_t need = std::max<uint64_t>(c->groups, 1);
  int rc = grow(c, &c->c_cap, need, need, {{&c->ckeys, (size_t)c->kb}, {(void**)&c->csums, sizeof(uint64_t)}});
  if (rc) return rc;
  launch_compact(c->rb, c->rv, c->B, c->ckeys, c->csums, c->stream);
  CU(c, cudaGetLastError());
  if (c->red_fsum || c->red_count) {
    // every row's sum (double bits; MRHBM_RED_COUNT_DISTINCT: its integer count) is in csums: its 11-byte number at
    // cvals[11 r ..), and the row index as its id
    const uint64_t n = c->groups;
    rc = grow(c, &c->row_cap, n + 1, n + 1, {{(void**)&c->row_off, sizeof(uint64_t)}});
    if (!rc) rc = grow(c, &c->cvals_cap, kNumBytes * n + 1, kNumBytes * n + 1, {{(void**)&c->cvals, 1}});
    if (rc) return rc;
    launch_num_encode(c->csums, n, c->cvals, c->row_off, c->stream, c->red_count);
    CU(c, cudaGetLastError());
    c->cvals_bytes = kNumBytes * n;
  } else if (c->bytevals) {
    // the value id of every row is in csums: lengths, their offsets, then the bytes in row order
    const uint64_t n = c->groups, nt = val_tiles(n);
    rc = grow(c, &c->row_cap, n + 1, n + 1, {{(void**)&c->row_off, sizeof(uint64_t)}});
    if (!rc) rc = grow(c, &c->tile_cap, nt + 1, nt + 1, {{(void**)&c->val_tile, sizeof(uint64_t)}});
    if (rc) return rc;
    launch_value_scan(c->csums, n, c->voff, c->row_off, c->val_tile, c->stream);
    CU(c, cudaGetLastError());
    CU(c, cudaMemcpyAsync(c->h_acc, c->row_off + n, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    const uint64_t total = c->h_acc[0];
    rc = grow(c, &c->cvals_cap, total + 1, total + 1, {{(void**)&c->cvals, 1}});
    if (!rc) rc = grow(c, &c->pieces_cap, val_chunks_cap(total) + 1, val_chunks_cap(total) + 1, {{(void**)&c->val_pieces, sizeof(uint64_t)}});
    if (rc) return rc;
    CU(c, cudaMemsetAsync(c->d_acc, 0, 8, c->stream));
    launch_value_gather(c->csums, n, c->voff, c->arena, c->row_off, c->val_tile, c->cvals, c->val_pieces,
                        (unsigned long long*)c->d_acc, c->stream);
    CU(c, cudaGetLastError());
    c->cvals_bytes = total;
  }
  CU(c, cudaStreamSynchronize(c->stream));
  c->compacted = true;
  return 0;
}

// The distinct set over the pool ranges `ranges` (first, count; none empty): k_distinct_mark, k_distinct_count and the
// scan of the tile counts (mrhbm_distinct.cu), then, when some pair repeats, k_distinct_scatter of the first copy of
// each distinct (key slot, value bytes) pair, in pool order, to dd_out.  off[t] receives the survivors before tile t
// (off.back(): all of them); rg the ranges as the kernels saw them (rg[k].tbase: the first tile of range k).
// `what` names the caller in the error of a set larger than it takes; *launches (optional) += kernels launched.
// ones (MRHBM_RED_COUNT_DISTINCT): the survivors always go to dd_out, repeats or not, with their value field set to 1.
int distinct_set(mrhbm_ctx* c, const std::vector<std::pair<uint64_t, uint64_t>>& ranges, const char* what,
                 std::vector<DistinctRange>& rg, std::vector<uint32_t>& off, uint32_t* launches = nullptr,
                 bool ones = false) {
  cudaStream_t s = c->stream;
  rg.clear();
  uint64_t n = 0, nt = 0;
  for (const auto& r : ranges) {
    rg.push_back(DistinctRange{r.first, n, (uint32_t)nt, 0});
    n += r.second;
    nt += (r.second + kDistinctTile - 1) / kDistinctTile;
  }
  rg.push_back(DistinctRange{0, n, (uint32_t)nt, 0});
  off.assign(nt + 1, 0);
  const uint32_t nr = (uint32_t)rg.size() - 1;
  if (n > (1ull << 31)) return fail(c, MRHBM_E_INVAL, "%s: %llu pairs (limit 2^31)", what, (unsigned long long)n);
  if (!n) return 0;
  uint64_t T = 1024;
  while (T < 2 * n) T <<= 1;
  int rc = grow(c, &c->dd_tab_cap, T, std::max(T, 2 * c->dd_tab_cap), {{&c->dd_tab, 16}});
  if (!rc) rc = grow(c, &c->dd_rec_cap, n, n, {{(void**)&c->dd_slot, 4}, {&c->dd_out, (size_t)c->rb}});
  if (!rc) rc = grow(c, &c->dd_rg_cap, nr + 1, nr + 1, {{&c->dd_rg, sizeof(DistinctRange)}});
  if (!rc) rc = grow(c, &c->dd_tiles_cap, 2 * (nt + 1), 2 * (nt + 1), {{(void**)&c->dd_tiles, 4}});
  if (rc) return rc;
  uint32_t *tile_cnt = c->dd_tiles, *tile_off = c->dd_tiles + nt + 1;
  const DistinctRange* drg = (const DistinctRange*)c->dd_rg;
  CU(c, cudaMemsetAsync(c->dd_tab, 0xff, T * 16, s));
  CU(c, cudaMemcpyAsync(c->dd_rg, rg.data(), rg.size() * sizeof(DistinctRange), cudaMemcpyHostToDevice, s));
  uint32_t k = launch_distinct_mark(c->rb, c->pool, drg, nr, (uint32_t)nt, c->arena, c->voff, c->dd_tab, T - 1, c->dd_slot, s);
  k += launch_distinct_count(drg, nr, (uint32_t)nt, c->dd_tab, c->dd_slot, tile_cnt, s);
  k += launch_exscan(tile_cnt, (uint32_t)nt, tile_off, nullptr, nullptr, 0xffffffffu, nullptr, nullptr, nullptr, 0, s,
                     c->d_small + 64);
  CU(c, cudaGetLastError());
  CU(c, cudaMemcpyAsync(off.data(), tile_off, (nt + 1) * 4, cudaMemcpyDeviceToHost, s));
  CU(c, cudaStreamSynchronize(s));
  if (off[nt] < n || ones) {
    k += launch_distinct_scatter(c->rb, c->pool, drg, nr, (uint32_t)nt, c->dd_tab, c->dd_slot, tile_off, c->dd_out, ones, s);
    CU(c, cudaGetLastError());
  }
  if (launches) *launches += k;
  return 0;
}

// MRHBM_COMBINE_DISTINCT, at commit: the map's open ranges are reduced to their distinct (key slot, value bytes) pairs
// in place, the first copy of each in pool order surviving (distinct_set), and its long-key pairs to their distinct
// (key, value bytes) pairs.  kept receives every open range as (first, survivors); the caller shrinks the ranges in
// the ledger once the whole commit has succeeded.
int distinct_pairs(mrhbm_map* m, std::vector<std::pair<uint64_t, uint64_t>>& kept) {
  mrhbm_ctx* c = m->ctx;
  kept = c->led.open_ranges(m->serial);
  std::vector<DistinctRange> rg;
  std::vector<uint32_t> off;
  int rc = distinct_set(c, kept, "distinct combiner: a map job", rg, off);
  if (rc) return rc;
  if (off.back() < rg.back().vbase) {
    for (size_t k = 0; k < kept.size(); k++) {
      const uint64_t a = off[rg[k].tbase], b = off[rg[k + 1].tbase];
      if (b - a < kept[k].second && b > a)
        CU(c, cudaMemcpyAsync((char*)c->pool + kept[k].first * c->rb, (char*)c->dd_out + a * c->rb, (b - a) * c->rb,
                              cudaMemcpyDeviceToDevice, c->stream));
      kept[k].second = b - a;
    }
    CU(c, cudaStreamSynchronize(c->stream));
  }
  std::set<std::pair<std::string, std::string>> seen;
  std::vector<LongPair> longs;
  for (LongPair& lp : m->long_pairs)
    if (seen.emplace(lp.esc, lp.bytes).second) longs.push_back(std::move(lp));
  m->long_pairs.swap(longs);
  return 0;
}

// MRHBM_COMBINE_FSUM, for keys longer than a record slot: the pairs of each key (by their bytes, in the order of its
// first pair) replaced by acc_split's terms, or kept as emitted
int fsum_long_pairs(mrhbm_ctx* c, std::vector<LongPair>& pairs) {
  std::map<std::string, std::vector<size_t>> by_key;
  std::vector<const std::string*> order;
  for (size_t i = 0; i < pairs.size(); i++) {
    auto it = by_key.emplace(pairs[i].esc, std::vector<size_t>()).first;
    if (it->second.empty()) order.push_back(&it->first);
    it->second.push_back(i);
  }
  std::vector<LongPair> out;
  for (const std::string* k : order) {
    const std::vector<size_t>& idx = by_key[*k];
    int64_t acc[kAccWords];
    acc_clear(acc);
    for (size_t i : idx) {
      uint64_t bits;
      const std::string& b = pairs[i].bytes;
      if (!num_decode((const unsigned char*)b.data(), b.size(), &bits))
        return fail(c, MRHBM_E_INVAL, "combiner MRHBM_COMBINE_FSUM: a value of a long key is not a number");
      acc_add(acc, bits);
    }
    std::vector<uint64_t> terms(idx.size());
    const int n = acc_split(acc, terms.data(), (int)idx.size());
    if (n < 0) return fail(c, MRHBM_E_INVAL, "combiner MRHBM_COMBINE_FSUM: a long key has +inf and -inf among its values");
    if (n == 0) {
      for (size_t i : idx) out.push_back(pairs[i]);
      continue;
    }
    for (int t = 0; t < n; t++) {
      std::string enc(kNumBytes, '\0');
      num_encode(terms[t], (unsigned char*)&enc[0]);
      out.push_back(LongPair{*k, 0, std::move(enc)});
    }
  }
  pairs.swap(out);
  return 0;
}

// MRHBM_COMBINE_FSUM, at commit: the map's pairs replaced by each key's terms (launch_fsum_split), as new pairs at the
// tail of the pool in the order of their keys' first pairs, each with its own value; the keys that keep their values
// are then placed in pool order by the host (only when some key does).  The map's open ranges are replaced by the new
// room once everything has succeeded; a failure rewinds the room.  One host synchronisation, plus the pool's growth
// and the kept keys' placement when they happen.
int fsum_pairs(mrhbm_map* m) {
  mrhbm_ctx* c = m->ctx;
  cudaStream_t s = c->stream;
  const std::vector<std::pair<uint64_t, uint64_t>> ranges = c->led.open_ranges(m->serial);
  std::vector<DistinctRange> rg;
  uint64_t n = 0, nt = 0;
  for (const auto& r : ranges) {
    rg.push_back(DistinctRange{r.first, n, (uint32_t)nt, 0});
    n += r.second;
    nt += (r.second + kDistinctTile - 1) / kDistinctTile;
  }
  rg.push_back(DistinctRange{0, n, (uint32_t)nt, 0});
  const uint32_t nr = (uint32_t)rg.size() - 1;
  if (n >= (1ull << 31))  // (each accumulator digit takes fewer than 2^31 addends; counts are u32)
    return fail(c, MRHBM_E_INVAL, "combiner MRHBM_COMBINE_FSUM: a map job of %llu pairs (limit 2^31)", (unsigned long long)n);
  std::vector<LongPair> longs = m->long_pairs;
  int rc = fsum_long_pairs(c, longs);
  if (rc) return rc;
  if (n) {
    uint64_t T = 1024;
    while (T < 2 * n) T <<= 1;
    const uint64_t nbig = n / kFsumWarpValues + 1;
    rc = grow(c, &c->dd_tab_cap, T, std::max(T, 2 * c->dd_tab_cap), {{&c->dd_tab, 16}});
    if (!rc) rc = grow(c, &c->dd_rec_cap, n, n, {{(void**)&c->dd_slot, 4}, {&c->dd_out, (size_t)c->rb}});
    if (!rc) rc = grow(c, &c->dd_rg_cap, nr + 1, nr + 1, {{&c->dd_rg, sizeof(DistinctRange)}});
    if (!rc) rc = grow(c, &c->dd_tiles_cap, 2 * (nt + 1), 2 * (nt + 1), {{(void**)&c->dd_tiles, 4}});
    if (!rc) rc = grow(c, &c->fs_words_cap, 4 * T, 4 * T, {{(void**)&c->fs_words, 4}});
    if (!rc) rc = grow(c, &c->fs_vals_cap, 2 * n, 2 * n, {{(void**)&c->fs_vals, 8}});
    if (!rc) rc = grow(c, &c->fs_big_cap, nbig, nbig, {{(void**)&c->fs_big, 4}, {(void**)&c->fs_gacc, kAccWords * 8}});
    if (!rc && !c->fs_small) CU(c, cudaMalloc((void**)&c->fs_small, 4 * sizeof(uint32_t)));
    if (rc) return rc;
    FsumScratch fs{c->dd_tab, T - 1, c->dd_slot, c->fs_words, c->fs_big, c->fs_small, c->fs_vals, c->fs_vals + n, c->fs_gacc};
    uint32_t *tile_cnt = c->dd_tiles, *tile_off = c->dd_tiles + nt + 1;
    const DistinctRange* drg = (const DistinctRange*)c->dd_rg;
    CU(c, cudaMemsetAsync(c->dd_tab, 0xff, T * 16, s));
    CU(c, cudaMemsetAsync(c->fs_words, 0, T * 4, s));
    CU(c, cudaMemsetAsync(c->fs_small, 0, 4 * sizeof(uint32_t), s));
    CU(c, cudaMemsetAsync(c->fs_gacc, 0, nbig * kAccWords * 8, s));
    CU(c, cudaMemcpyAsync(c->dd_rg, rg.data(), rg.size() * sizeof(DistinctRange), cudaMemcpyHostToDevice, s));
    launch_fsum_split(c->rb, c->pool, drg, nr, (uint32_t)nt, n, c->arena, c->voff, fs, tile_cnt, c->sm_count, s);
    launch_exscan(tile_cnt, (uint32_t)nt, tile_off, nullptr, nullptr, 0xffffffffu, nullptr, nullptr, nullptr, 0, s,
                  c->d_small + 64);
    CU(c, cudaGetLastError());
    CU(c, cudaMemcpyAsync(c->h_counters, c->fs_small, 4, cudaMemcpyDeviceToHost, s));
    CU(c, cudaMemcpyAsync(c->h_counters + 1, tile_off + nt, 4, cudaMemcpyDeviceToHost, s));
    CU(c, cudaStreamSynchronize(s));
    const uint32_t flags = c->h_counters[0];
    const uint64_t total = c->h_counters[1];
    if (flags & ERRF_NOTNUM)
      return fail(c, MRHBM_E_INVAL, "combiner MRHBM_COMBINE_FSUM: a value is not a number (11-byte encoding, tag 0x10)");
    if (flags & ERRF_NAN)
      return fail(c, MRHBM_E_INVAL, "combiner MRHBM_COMBINE_FSUM: a key has +inf and -inf among its values");
    Reservation r;
    rc = reserve(c, nullptr, total, kNumBytes * total, r);
    if (rc) return rc;
    launch_fsum_write(c->rb, c->pool, drg, nr, (uint32_t)nt, fs, tile_off, r.off, r.aoff, c->voff, c->arena, s);
    CU(c, cudaGetLastError());
    if (flags & kFsumKeep) {
      // the kept keys' pairs in pool order, each after the key's first new pair (the cursor words of its entry)
      std::vector<uint32_t> slot_of(n), nterm(T), first(T);
      CU(c, cudaMemcpyAsync(slot_of.data(), c->dd_slot, n * 4, cudaMemcpyDeviceToHost, s));
      CU(c, cudaMemcpyAsync(nterm.data(), c->fs_words + 3 * T, T * 4, cudaMemcpyDeviceToHost, s));
      CU(c, cudaMemcpyAsync(first.data(), c->fs_words + 2 * T, T * 4, cudaMemcpyDeviceToHost, s));
      CU(c, cudaStreamSynchronize(s));
      std::vector<uint64_t> cp;
      for (size_t k = 0; k < ranges.size(); k++)
        for (uint64_t j = 0; j < ranges[k].second; j++) {
          const uint64_t g = rg[k].vbase + j;
          const uint32_t e = slot_of[g];
          if (!(nterm[e] & kFsumKeep)) continue;
          cp.insert(cp.end(), {(uint64_t)first[e]++, ranges[k].first + j, g});
        }
      uint64_t* d_cp = nullptr;
      CU(c, cudaMalloc((void**)&d_cp, cp.size() * 8));
      cudaError_t e = cudaMemcpyAsync(d_cp, cp.data(), cp.size() * 8, cudaMemcpyHostToDevice, s);
      if (e == cudaSuccess) {
        launch_fsum_copy(c->rb, c->pool, d_cp, cp.size() / 3, fs, r.off, r.aoff, c->voff, c->arena, s);
        e = cudaGetLastError();
      }
      if (e == cudaSuccess) e = cudaStreamSynchronize(s);
      cudaFree(d_cp);
      if (e != cudaSuccess) return fail(c, MRHBM_E_CUDA, "combiner MRHBM_COMBINE_FSUM: %s", cudaGetErrorString(e));
    }
    r.replace(m);
  }
  m->long_pairs.swap(longs);
  return 0;
}

float ev_ms(mrhbm_ctx* c, int a, int b) {
  float ms = 0;
  if (cudaEventElapsedTime(&ms, c->ev[a], c->ev[b]) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return ms;
}

int install_splitters(mrhbm_ctx* c, std::vector<std::string>&& spl);  // (with the shuffle, below)

}  // namespace

extern "C" {

int mrhbm_abi_version(void) { return MRHBM_ABI_VERSION; }

int mrhbm_init(const mrhbm_config* cfg, mrhbm_ctx** out) {
  if (!cfg || !out || cfg->struct_size != sizeof(mrhbm_config)) return MRHBM_E_INVAL;
  *out = nullptr;
  mrhbm_ctx* c = new mrhbm_ctx();
  *out = c;  // returned even on failure so that the caller can read last_error, then destroy
  c->cfg = *cfg;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(c, MRHBM_E_NODEVICE, "no CUDA device (%s): mrhbm has no CPU path",
                e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
  }
  int dev = cfg->device;
  if (dev < 0) CU(c, cudaGetDevice(&dev));
  if (dev >= ndev) return fail(c, MRHBM_E_INVAL, "device %d out of range (%d devices)", dev, ndev);
  CU(c, cudaSetDevice(dev));
  cudaDeviceProp prop;
  CU(c, cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0)
    return fail(c, MRHBM_E_NODEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", dev,
                prop.major, prop.minor);
  c->dev = dev;
  c->sm_count = prop.multiProcessorCount;
  if (cfg->num_partitions == 0) return fail(c, MRHBM_E_INVAL, "num_partitions must be >= 1");
  if (cfg->key_kind == MRHBM_KEY_U64) {
    c->rb = 16;
    c->kb = 8;
    if (cfg->partitioner > MRHBM_PART_RANGE) return fail(c, MRHBM_E_INVAL, "unknown partitioner");
  } else if (cfg->key_kind == MRHBM_KEY_STR) {
    uint32_t m = cfg->max_key_bytes ? cfg->max_key_bytes : 27;
    if (m <= 27) c->rb = 32;
    else if (m <= 59) c->rb = 64;
    else if (m <= 123) c->rb = 128;
    else return fail(c, MRHBM_E_KEY, "max_key_bytes %u exceeds the largest record class (123)", m);
    c->kb = c->rb - 4;
    if (cfg->partitioner != MRHBM_PART_FNV_LUA && cfg->partitioner != MRHBM_PART_WORDHASH && cfg->partitioner != MRHBM_PART_RANGE)
      return fail(c, MRHBM_E_INVAL, "string keys need partitioner FNV_LUA, WORDHASH or RANGE");
  } else
    return fail(c, MRHBM_E_INVAL, "unknown key_kind %u", cfg->key_kind);
  if (cfg->reducer > MRHBM_RED_COUNT_DISTINCT) return fail(c, MRHBM_E_INVAL, "unknown reducer %u", cfg->reducer);
  if (cfg->combiner > MRHBM_COMBINE_FSUM) return fail(c, MRHBM_E_INVAL, "unknown combiner %u", cfg->combiner);
  if (cfg->combiner == MRHBM_COMBINE_FSUM && (!(cfg->flags & MRHBM_F_BYTE_VALUES) || cfg->reducer != MRHBM_RED_FSUM))
    return fail(c, MRHBM_E_INVAL, "combiner MRHBM_COMBINE_FSUM needs byte values (MRHBM_F_BYTE_VALUES) and reducer MRHBM_RED_FSUM");
  if (cfg->combiner == MRHBM_COMBINE_DISTINCT && !(cfg->flags & MRHBM_F_BYTE_VALUES))
    return fail(c, MRHBM_E_INVAL, "combiner MRHBM_COMBINE_DISTINCT needs byte values (MRHBM_F_BYTE_VALUES)");
  if (cfg->reducer == MRHBM_RED_NONE && cfg->combiner == MRHBM_COMBINE_REDUCER) return fail(c, MRHBM_E_INVAL, "a general reducer cannot be combined on the device (combiner must be 0)");
  if (cfg->reducer == MRHBM_RED_DISTINCT && !(cfg->flags & MRHBM_F_BYTE_VALUES))
    return fail(c, MRHBM_E_INVAL, "reducer MRHBM_RED_DISTINCT needs byte values (MRHBM_F_BYTE_VALUES)");
  if (cfg->reducer == MRHBM_RED_FSUM && (!(cfg->flags & MRHBM_F_BYTE_VALUES) ||
                                         (cfg->combiner != MRHBM_COMBINE_NONE && cfg->combiner != MRHBM_COMBINE_FSUM)))
    return fail(c, MRHBM_E_INVAL, "reducer MRHBM_RED_FSUM needs byte values (MRHBM_F_BYTE_VALUES) and combiner MRHBM_COMBINE_NONE or MRHBM_COMBINE_FSUM");
  if (cfg->reducer == MRHBM_RED_COUNT_DISTINCT && (!(cfg->flags & MRHBM_F_BYTE_VALUES) ||
                                                   (cfg->combiner != MRHBM_COMBINE_NONE && cfg->combiner != MRHBM_COMBINE_DISTINCT)))
    return fail(c, MRHBM_E_INVAL, "reducer MRHBM_RED_COUNT_DISTINCT needs byte values (MRHBM_F_BYTE_VALUES) and combiner MRHBM_COMBINE_NONE or MRHBM_COMBINE_DISTINCT");
  if ((cfg->flags & MRHBM_F_BYTE_VALUES) && (cfg->reducer == MRHBM_RED_SUM || cfg->combiner == MRHBM_COMBINE_REDUCER))
    return fail(c, MRHBM_E_INVAL, "byte values (MRHBM_F_BYTE_VALUES) need reducer MRHBM_RED_NONE, MRHBM_RED_DISTINCT, MRHBM_RED_FSUM or MRHBM_RED_COUNT_DISTINCT and combiner 0 or MRHBM_COMBINE_DISTINCT");
  c->bytevals = c->led.byte_values = (cfg->flags & MRHBM_F_BYTE_VALUES) != 0;
  c->red_distinct = cfg->reducer == MRHBM_RED_DISTINCT;
  c->red_fsum = cfg->reducer == MRHBM_RED_FSUM;
  c->red_count = cfg->reducer == MRHBM_RED_COUNT_DISTINCT;
  // (MRHBM_RED_COUNT_DISTINCT sums a 1 per distinct pair: the sort reduces as for MRHBM_RED_SUM)
  c->sb.no_reduce = cfg->reducer != MRHBM_RED_SUM && !c->red_count;
  CU(c, cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  if (cfg->partitioner == MRHBM_PART_RANGE && cfg->num_partitions == 1) {  // one key range, no splitters: its table now
    int rc = install_splitters(c, {});
    if (rc) return rc;
  }
  for (int i = 0; i < EV_N; i++) CU(c, cudaEventCreate(&c->ev[i]));
  CU(c, kernels_configure());
  CU(c, cudaMalloc((void**)&c->d_acc, 8 * sizeof(uint64_t)));
  CU(c, cudaHostAlloc((void**)&c->h_counters, 8 * sizeof(uint32_t), cudaHostAllocDefault));
  CU(c, cudaHostAlloc((void**)&c->h_acc, 8 * sizeof(uint64_t), cudaHostAllocDefault));
  CU(c, cudaMalloc((void**)&c->d_small, (64 + kScanScratchWords) * sizeof(uint32_t)));  // [64..): scan scratch
  CU(c, cudaHostAlloc((void**)&c->h_small, 64 * sizeof(uint32_t), cudaHostAllocDefault));
  c->Pl = cfg->num_partitions;
  for (int r = 1; r <= 8; r++) c->pbase[r] = cfg->num_partitions;
  c->cap = (cfg->flags & MRHBM_F_SMALL_BINS) ? 96 : cap_records(c->rb);
  CU(c, cudaMalloc((void**)&c->d_sample, 256 * sizeof(uint32_t)));
  CU(c, cudaHostAlloc((void**)&c->h_sample, 256 * sizeof(uint32_t), cudaHostAllocDefault));
  if (cfg->reserve_pairs) {  // capacity only: the room goes straight back
    Reservation r;
    int rc = reserve(c, nullptr, cfg->reserve_pairs, 0, r);
    if (rc) return rc;
  }
  return MRHBM_OK;
}

void mrhbm_destroy(mrhbm_ctx* c) {
  if (!c) return;
  int prev = -1;
  if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
  if (c->stream) cudaSetDevice(c->dev);
  if (c->stream) cudaStreamSynchronize(c->stream);
  for (int r = 0; r < 8; r++)
    if (c->world > 1 && r != c->rank && c->peer_regions[r]) cudaIpcCloseMemHandle(c->peer_regions[r]);
  if (c->d_ipc) cudaFree(c->d_ipc);
  if (c->h_ipc) cudaFreeHost(c->h_ipc);
  if (c->h_sample) cudaFreeHost(c->h_sample);
  if (c->comm) comm_destroy(c->comm);
  void* frees[] = {c->pool,        c->sb.hist,     c->sb.bin_off, c->sb.cursor,   c->sb.ucount, c->sb.uoff,
                   c->sb.big_list, c->sb.counters, c->sb.mid,     c->sb.out_keys, c->sb.out_sums, c->ckeys,
                   c->csums,       c->d_acc,       c->d_table,    c->d_hd,        c->d_hall,    c->d_tot,
                   c->d_outoff,    c->d_segoff,    c->recvbuf,    c->bigbuf,      c->d_small,   c->comb,
                   c->gtab,        c->l1buf,       c->regions,    c->d_l1all,     c->d_sample,   c->d_tok_text[0],
                   c->d_tok_text[1], c->d_tok_cnt, c->d_tok_off, c->d_spl,     c->arena,       c->voff,
                   c->cvals,       c->row_off,     c->val_tile,   c->val_pieces, c->dd_tab,     c->dd_out,
                   c->dd_rg,       c->dd_slot,     c->dd_tiles,   c->vo_keys,    c->vo_ids,
                   c->ns_acc,      c->ns_flags,    c->ns_head,    c->fs_words,   c->fs_big,     c->fs_small,
                   c->fs_vals,     c->fs_gacc,     c->d_pow5,     c->d_kn_fix};
  for (void* p : frees)
    if (p) cudaFree(p);
  if (c->h_counters) cudaFreeHost(c->h_counters);
  if (c->h_acc) cudaFreeHost(c->h_acc);
  if (c->h_small) cudaFreeHost(c->h_small);
  for (int i = 0; i < EV_N; i++)
    if (c->ev[i]) cudaEventDestroy(c->ev[i]);
  for (int i = 0; i < 2; i++)
    if (c->tok_ev[i]) cudaEventDestroy(c->tok_ev[i]);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->stream) cudaStreamDestroy(c->stream);
  if (prev >= 0) cudaSetDevice(prev);
  cudaGetLastError();
  delete c;
}

const char* mrhbm_last_error(const mrhbm_ctx* c) { return c ? c->err.c_str() : "null ctx"; }
uint32_t mrhbm_record_bytes(const mrhbm_ctx* c) { return c ? (uint32_t)c->rb : 0; }

void* mrhbm_host_alloc(mrhbm_ctx* c, size_t bytes) {
  void* p = nullptr;
  Entry g(c);
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    if (c) c->err = "cudaHostAlloc failed";
    return nullptr;
  }
  return p;
}
void mrhbm_host_free(mrhbm_ctx*, void* p) {
  if (p) cudaFreeHost(p);
}

// ---------------------------------------------------------------------------
// map side
// ---------------------------------------------------------------------------
int mrhbm_map_begin(mrhbm_ctx* c, const char* job, mrhbm_map** out) {
  if (!c || !job || !out) return MRHBM_E_INVAL;
  Entry g(c);
  if (!c->stream) return fail(c, MRHBM_E_INVAL, "ctx failed to initialise");
  mrhbm_map* m = new mrhbm_map();
  m->ctx = c;
  m->job = job;
  m->serial = c->led.new_owner();
  *out = m;
  return MRHBM_OK;
}

int mrhbm_emit_str(mrhbm_map* m, const void* key, size_t klen, uint32_t value) {
  if (!m) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (c->cfg.key_kind != MRHBM_KEY_STR) return fail(c, MRHBM_E_INVAL, "ctx holds u64 keys");
  if (c->bytevals) return refuse_int_values(c);
  // (keys are stored escaped, see escape)
  const unsigned char* k = (const unsigned char*)key;
  const size_t elen = esc_size(k, klen);
  if (elen >= (size_t)c->kb) return long_pair(m, k, klen, elen, value, nullptr, 0);
  unsigned char* slot;
  int rc = stage_slot(m, &slot);
  if (rc) return rc;
  escape(k, klen, slot);
  memset(slot + elen, 0, c->kb - elen);
  memcpy(slot + c->kb, &value, 4);
  return MRHBM_OK;
}

int mrhbm_emit_u64(mrhbm_map* m, uint64_t key, uint64_t value) {
  if (!m) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (c->cfg.key_kind != MRHBM_KEY_U64) return fail(c, MRHBM_E_INVAL, "ctx holds string keys");
  if (c->bytevals) return refuse_int_values(c);
  unsigned char* slot;
  int rc = stage_slot(m, &slot);
  if (rc) return rc;
  memcpy(slot, &key, 8);
  memcpy(slot + 8, &value, 8);
  return MRHBM_OK;
}

int mrhbm_emit_str_value(mrhbm_map* m, const void* key, size_t klen, const void* val, size_t vlen) {
  if (!m || (!key && klen)) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (!c->bytevals) return refuse_byte_values(c);
  if (c->cfg.key_kind != MRHBM_KEY_STR) return fail(c, MRHBM_E_INVAL, "ctx holds u64 keys");
  const unsigned char* k = (const unsigned char*)key;
  const size_t elen = esc_size(k, klen);
  if (elen >= (size_t)c->kb) return long_pair(m, k, klen, elen, 0, val, vlen);
  return stage_value_pair(m, val, vlen, [&](unsigned char* slot) {
    escape(k, klen, slot);
    memset(slot + elen, 0, c->kb - elen);
  });
}

int mrhbm_emit_u64_value(mrhbm_map* m, uint64_t key, const void* val, size_t vlen) {
  if (!m) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (!c->bytevals) return refuse_byte_values(c);
  if (c->cfg.key_kind != MRHBM_KEY_U64) return fail(c, MRHBM_E_INVAL, "ctx holds string keys");
  return stage_value_pair(m, val, vlen, [&](unsigned char* slot) { memcpy(slot, &key, 8); });
}

int mrhbm_emit_batch_values(mrhbm_map* m, const void* recs, size_t n, const void* vals, const uint64_t* voff) {
  if (!m || (n && (!recs || !voff))) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (!c->bytevals) return refuse_byte_values(c);
  if (!n) return MRHBM_OK;
  for (size_t i = 0; i < n; i++)
    if (voff[i + 1] < voff[i] || voff[i + 1] - voff[i] > kMaxValue)
      return fail(c, MRHBM_E_INVAL, "value %zu: offsets %llu .. %llu (non-decreasing, at most %llu bytes apart)", i,
                  (unsigned long long)voff[i], (unsigned long long)voff[i + 1], (unsigned long long)kMaxValue);
  const uint64_t bytes = voff[n] - voff[0];
  if (bytes && !vals) return fail(c, MRHBM_E_INVAL, "null values");
  Reservation r;
  int rc = reserve(c, m, n, bytes, r);
  if (rc) return rc;
  const bool pinned = is_pinned(recs) || is_pinned(vals) || is_pinned(voff);
  CU(c, cudaMemcpyAsync((char*)c->pool + r.off * c->rb, recs, n * c->rb, cudaMemcpyHostToDevice, c->stream));
  if (bytes) CU(c, cudaMemcpyAsync(c->arena + r.aoff, (const char*)vals + voff[0], bytes, cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemcpyAsync(c->voff + r.off, voff, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
  launch_value_stamp(c->rb, (char*)c->pool + r.off * c->rb, n, r.off, c->voff + r.off, voff[0], r.aoff, c->stream);
  CU(c, cudaGetLastError());
  if (pinned) m->async_reads = true;  // pageable sources are fully staged before the call returns
  r.add(m);
  return MRHBM_OK;
}

int mrhbm_emit_batch(mrhbm_map* m, const void* recs, size_t n) {
  if (!m || (!recs && n)) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (c->bytevals) return refuse_int_values(c);
  if (!n) return MRHBM_OK;
  Reservation r;
  int rc = reserve(c, m, n, 0, r);
  if (rc) return rc;
  const bool pinned = is_pinned(recs);
  CU(c, cudaMemcpyAsync((char*)c->pool + r.off * c->rb, recs, n * c->rb, cudaMemcpyHostToDevice, c->stream));
  if (pinned) m->async_reads = true;  // pageable sources are fully staged before the call returns
  r.add(m);
  return MRHBM_OK;
}

int mrhbm_emit_device(mrhbm_map* m, const void* drecs, size_t n) {
  if (!m || (!drecs && n)) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (c->bytevals) return refuse_int_values(c);
  if (!n) return MRHBM_OK;
  Reservation r;
  int rc = reserve(c, m, n, 0, r);
  if (rc) return rc;
  CU(c, cudaMemcpyAsync((char*)c->pool + r.off * c->rb, drecs, n * c->rb, cudaMemcpyDeviceToDevice, c->stream));
  r.add(m);
  return MRHBM_OK;
}

int mrhbm_map_gen_u64(mrhbm_map* m, uint64_t seed, uint64_t start, uint64_t n) {
  if (!m) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (c->rb != 16) return fail(c, MRHBM_E_INVAL, "gen_u64 needs a u64-key ctx");
  if (c->bytevals) return refuse_int_values(c);
  Reservation r;
  int rc = reserve(c, m, n, 0, r);
  if (rc) return rc;
  launch_gen_u64((char*)c->pool + r.off * c->rb, seed, start, n, c->stream);
  CU(c, cudaGetLastError());
  r.add(m);
  return MRHBM_OK;
}

int mrhbm_map_gen_zipf(mrhbm_map* m, uint64_t seed, uint64_t start, uint64_t n, const uint64_t* table,
                       uint64_t V) {
  if (!m || !table || !V) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (c->rb != 32) return fail(c, MRHBM_E_INVAL, "gen_zipf needs 32-byte string records (max_key_bytes <= 27)");
  if (c->bytevals) return refuse_int_values(c);
  if (!c->d_table || c->d_table_V != V || c->d_table_first != table[0] || c->d_table_last != table[V - 1]) {
    if (c->d_table) CU(c, cudaFree(c->d_table));
    c->d_table = nullptr;
    CU(c, cudaMalloc((void**)&c->d_table, V * sizeof(uint64_t)));
    CU(c, cudaMemcpyAsync(c->d_table, table, V * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    c->d_table_V = V;
    c->d_table_first = table[0];
    c->d_table_last = table[V - 1];
  }
  Reservation r;
  int rc = reserve(c, m, n, 0, r);
  if (rc) return rc;
  launch_gen_zipf32((char*)c->pool + r.off * c->rb, seed, start, n, c->d_table, V, c->stream);
  CU(c, cudaGetLastError());
  r.add(m);
  return MRHBM_OK;
}

}  // extern "C"

namespace {

constexpr size_t kTokPiece = 64u << 20;  // bytes of text per device piece
inline bool is_space(unsigned char ch) { return ch == ' ' || (ch >= 9 && ch <= 13); }

// The piece driver of the device mapfns over text (the caller has checked the ctx and the arguments).  The text is
// handled in pieces of <= kTokPiece bytes through two device buffers: the upload of piece k+1 (copy stream) runs while
// piece k is counted, scanned and emitted (ctx stream).  The scratch (text x 2, per-256-byte-block counts and offsets)
// lives with the ctx.  Job says where a piece may end -- after white space, or with Job::kLines after '\n' -- and
// handles one piece: job.device(...) on the device, which may leave it to job.host(...) on the host (a key that does
// not fit the record class, say).  A failure of either emits nothing of the call.
template <class Job>
int map_pieces(mrhbm_map* m, const unsigned char* t, size_t len, Job& job, uint64_t* count) {
  mrhbm_ctx* c = m->ctx;
  if (!len) return MRHBM_OK;
  int rc = stage_flush(m);
  if (rc) return rc;
  if (!c->d_tok_text[0]) {
    const uint64_t tcap = kTokPiece + 4096, bcap = tok_blocks(tcap) + 1;
    cudaError_t ea = cudaMalloc((void**)&c->d_tok_text[0], tcap);
    if (ea == cudaSuccess) ea = cudaMalloc((void**)&c->d_tok_text[1], tcap);
    if (ea == cudaSuccess) ea = cudaMalloc((void**)&c->d_tok_cnt, bcap * 4);
    if (ea == cudaSuccess) ea = cudaMalloc((void**)&c->d_tok_off, (bcap + 1) * 4);
    if (ea == cudaSuccess) ea = cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking);
    for (int i = 0; i < 2 && ea == cudaSuccess; i++) ea = cudaEventCreateWithFlags(&c->tok_ev[i], cudaEventDisableTiming);
    if (ea != cudaSuccess) {
      cudaGetLastError();
      return fail(c, MRHBM_E_NOMEM, "%s: %s", job.what, cudaGetErrorString(ea));
    }
  }
  // undo information: a piece that fails emits NOTHING of this call
  const PoolLedger::Mark mark0 = c->led.mark();
  const size_t long0 = m->long_pairs.size();
  auto piece_end = [&](size_t p) -> size_t {  // end of the piece that starts at p: <= kTokPiece bytes
    size_t e = std::min(len, p + kTokPiece);
    if (e < len) {
      size_t q = e;
      if constexpr (Job::kLines) {  // cut after the last '\n'; p itself when the line is longer than a piece
        while (q > p && t[q - 1] != '\n') q--;
        return q;
      }
      while (q > p && !is_space(t[q - 1])) q--;
      if (q > p) e = q;  // (no white space in 64 MB: one giant "word", the length check below refuses it)
    }
    return e;
  };
  auto long_line = [&](size_t p) {
    return fail(c, MRHBM_E_INVAL, "%s: the line at byte %zu is longer than a piece (%zu bytes)", job.what, p, kTokPiece);
  };
  cudaError_t e = cudaSuccess;
  uint64_t total_pairs = 0;
  size_t p = 0, pe = piece_end(0);
  if (pe == 0) return long_line(0);
  int k = 0;
  e = cudaMemcpyAsync(c->d_tok_text[0], t, pe, cudaMemcpyHostToDevice, c->copy_stream);
  if (e == cudaSuccess) e = cudaEventRecord(c->tok_ev[0], c->copy_stream);
  while (e == cudaSuccess && rc == 0 && p < len) {
    const size_t n = pe - p, pn = pe, pne = pe < len ? piece_end(pe) : pe;
    if (pne == pn && pn < len) {
      rc = long_line(pn);
      break;
    }
    unsigned char* d_text = c->d_tok_text[k & 1];
    if (pn < len) {  // next piece's upload: its buffer was last read by piece k-1, whose kernels are behind a sync
      e = cudaMemcpyAsync(c->d_tok_text[(k + 1) & 1], t + pn, pne - pn, cudaMemcpyHostToDevice, c->copy_stream);
      if (e == cudaSuccess) e = cudaEventRecord(c->tok_ev[(k + 1) & 1], c->copy_stream);
      if (e != cudaSuccess) break;
    }
    if ((e = cudaStreamWaitEvent(c->stream, c->tok_ev[k & 1], 0)) != cudaSuccess) break;
    bool on_host = false;
    uint64_t pairs = 0;
    e = job.device(d_text, p, n, rc, on_host, pairs);
    if (e != cudaSuccess || rc) break;
    if (on_host && (rc = job.host(p, pn, pairs)) != 0) break;
    total_pairs += pairs;
    p = pn;
    pe = pne;
    k++;
  }
  if (e != cudaSuccess || rc) {
    cudaStreamSynchronize(c->copy_stream);  // an upload may still be reading the caller's text
    cudaStreamSynchronize(c->stream);
    c->led.rewind(mark0);
    m->long_pairs.resize(long0);  // (pairs of a piece that was handled on the host)
    m->fill = 0;                  // the staging buffer was empty when the call began (stage_flush above)
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(c, MRHBM_E_CUDA, "%s: %s", job.what, cudaGetErrorString(e));
    }
    return rc;
  }
  if (count) *count = total_pairs;
  return MRHBM_OK;
}

// mrhbm_map_wordcount and mrhbm_map_words_value: every maximal run of non-space bytes of the text becomes the pair
// (word, 1), or on a byte-values ctx (word, val[0 .. vlen)).  With byte values the value bytes go to the arena once per
// device piece and every pair of the piece carries the value id of the piece's first pair (see PoolLedger).
struct WordsJob {
  static constexpr bool kLines = false;
  mrhbm_map* m;
  const unsigned char* t;
  const void* val;
  size_t vlen;
  const char* what;

  cudaError_t device(const unsigned char* d_text, size_t, size_t n, int& rc, bool& on_host, uint64_t& pairs) {
    mrhbm_ctx* c = m->ctx;
    cudaError_t e;
    uint32_t* flagw = c->d_small + 1;
    const uint64_t nb = tok_blocks(n);
    launch_tok_count(d_text, n, c->d_tok_cnt, c->stream);
    launch_exscan(c->d_tok_cnt, (uint32_t)nb, c->d_tok_off, nullptr, nullptr, 0xffffffffu, nullptr, nullptr, c->d_small, 0, c->stream,
                  c->d_small + 64);
    if ((e = cudaMemcpyAsync(c->h_small, c->d_small, 4, cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess) return e;
    const uint64_t total = c->h_small[0];
    if (!total) return cudaSuccess;
    Reservation r;
    rc = reserve(c, nullptr, total, c->bytevals ? vlen : 0, r);
    if (rc) return cudaSuccess;
    uint32_t value = 1;
    if (c->bytevals) {  // one copy of the value; ids r.off + 1 .. r.off + total - 1 get empty values
      if (vlen && (e = cudaMemcpyAsync(c->arena + r.aoff, val, vlen, cudaMemcpyHostToDevice, c->stream)) != cudaSuccess)
        return e;
      launch_value_stamp(c->rb, nullptr, total, 0, c->voff + r.off, vlen, r.aoff, c->stream);
      value = (uint32_t)r.off;
    }
    if ((e = cudaMemsetAsync(flagw, 0, 4, c->stream)) != cudaSuccess) return e;
    launch_tok_emit(c->rb, d_text, n, c->d_tok_off, (char*)c->pool + r.off * c->rb, value, flagw, c->stream);
    if ((e = cudaMemcpyAsync(c->h_small + 1, flagw, 4, cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess) return e;
    if (c->h_small[1] & ERRF_KEYLEN) {  // the piece's records are dropped again (r rewinds)
      on_host = true;
      return cudaSuccess;
    }
    r.add(m);
    pairs = total;
    return cudaSuccess;
  }
  // a word of this piece does not fit the key slot (a URL in a corpus): the piece is tokenised on the host -- words
  // that fit are staged like emit_str / emit_str_value pairs, the long ones go to the host-side store of long keys.
  // Rare by assumption: 64 MB take a fraction of a second here.
  int host(size_t p, size_t pn, uint64_t& pairs) {
    mrhbm_ctx* c = m->ctx;
    int rc = 0;
    uint64_t words_here = 0;
    for (size_t a = p; a < pn && rc == 0;) {
      while (a < pn && is_space(t[a])) a++;
      size_t b = a;
      while (b < pn && !is_space(t[b])) b++;
      if (b > a) {
        rc = c->bytevals ? mrhbm_emit_str_value(m, t + a, b - a, val, vlen) : mrhbm_emit_str(m, t + a, b - a, 1u);
        words_here++;
      }
      a = b;
    }
    if (!rc) pairs = words_here;
    return rc;
  }
};

// mrhbm_map_key_numbers: every line "key number" becomes the pair (key, the number's 11 bytes), each pair with a value
// of its own.  A device piece reserves one record and 11 value bytes per line; the kernel writes the records, voff and
// the values, and lists the tokens the device does not round (mrhbm_decimal.cuh), which the host then rounds and
// patches.  A key longer than the record class, or more such tokens than the list holds, leaves the piece to the host.
constexpr uint32_t kKnFixCap = 1u << 16;
struct KeyNumbersJob {
  static constexpr bool kLines = true;
  mrhbm_map* m;
  const unsigned char* t;
  const char* what = "key_numbers";

  int bad_line(size_t at) {
    return fail(m->ctx, MRHBM_E_INVAL, "key_numbers: the line at byte %zu is not \"key number\" (a decimal number)", at);
  }
  cudaError_t device(const unsigned char* d_text, size_t p, size_t n, int& rc, bool& on_host, uint64_t& pairs) {
    mrhbm_ctx* c = m->ctx;
    cudaError_t e;
    uint32_t* flags = c->d_small + 1;  // [0] ERRF_*, [1] the first malformed line's offset, [2] fix-ups
    const uint64_t nb = tok_blocks(n);
    launch_kn_count(d_text, n, c->d_tok_cnt, c->stream);
    launch_exscan(c->d_tok_cnt, (uint32_t)nb, c->d_tok_off, nullptr, nullptr, 0xffffffffu, nullptr, nullptr, c->d_small, 0, c->stream,
                  c->d_small + 64);
    if ((e = cudaMemcpyAsync(c->h_small, c->d_small, 4, cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess) return e;
    const uint64_t total = c->h_small[0];
    if (!total) return cudaSuccess;
    Reservation r;
    rc = reserve(c, nullptr, total, total * kNumBytes, r);
    if (rc) return cudaSuccess;
    if ((e = cudaMemsetAsync(flags, 0, 12, c->stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(flags + 1, 0xff, 4, c->stream)) != cudaSuccess) return e;
    const KnOut o{(uint4*)((char*)c->pool + r.off * c->rb), c->arena + r.aoff, c->voff + r.off, r.off, r.aoff,
                  c->d_pow5, (uint4*)c->d_kn_fix, kKnFixCap, flags};
    launch_kn_emit(c->rb, d_text, n, c->d_tok_off, o, c->stream);
    if ((e = cudaMemcpyAsync(c->h_small + 1, flags, 12, cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess) return e;
    const uint32_t ef = c->h_small[1], nfix = c->h_small[3];
    if (ef & ERRF_LINE) {
      rc = bad_line(p + c->h_small[2]);
      return cudaSuccess;
    }
    if ((ef & ERRF_KEYLEN) || nfix > kKnFixCap) {  // the piece's records are dropped again (r rewinds)
      on_host = true;
      return cudaSuccess;
    }
    if (nfix) {
      std::vector<uint4> fx(nfix);
      if ((e = cudaMemcpyAsync(fx.data(), c->d_kn_fix, nfix * sizeof(uint4), cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess)
        return e;
      if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess) return e;
      std::vector<ulonglong2> patch(nfix);
      for (uint32_t i = 0; i < nfix; i++) {
        uint64_t bits = 0;
        dec_parse_host(t + p + fx[i].y, fx[i].z, &bits);  // (the kernel has checked the grammar)
        patch[i] = make_ulonglong2(fx[i].x, bits);
      }
      // (pageable: staged before the call returns)
      if ((e = cudaMemcpyAsync(c->d_kn_fix, patch.data(), nfix * sizeof(ulonglong2), cudaMemcpyHostToDevice, c->stream)) !=
          cudaSuccess)
        return e;
      launch_kn_patch(c->d_kn_fix, nfix, c->arena + r.aoff, c->stream);
    }
    r.add(m);
    pairs = total;
    return cudaSuccess;
  }
  // the same lines on the host, the same grammar, values from std::from_chars, pairs through mrhbm_emit_str_value
  // (long keys to the host-side store); flushed at the end so that the next device piece's records follow them
  int host(size_t p, size_t pn, uint64_t& pairs) {
    uint64_t here = 0;
    for (size_t a = p; a < pn;) {
      size_t eol = a;
      while (eol < pn && t[eol] != '\n') eol++;
      size_t f[4], nf = 0, i = a;  // the first two fields' bounds
      bool extra = false;
      while (i < eol) {
        while (i < eol && is_space(t[i])) i++;
        if (i == eol) break;
        const size_t b = i;
        while (i < eol && !is_space(t[i])) i++;
        if (nf == 4) {
          extra = true;
          break;
        }
        f[nf++] = b;
        f[nf++] = i;
      }
      if (nf) {
        uint64_t bits = 0;
        if (extra || nf != 4 || !dec_parse_host(t + f[2], f[3] - f[2], &bits)) return bad_line(a);
        unsigned char enc[kNumBytes];
        num_encode(bits, enc);
        const int rc = mrhbm_emit_str_value(m, t + f[0], f[1] - f[0], enc, kNumBytes);
        if (rc) return rc;
        here++;
      }
      a = eol + 1;
    }
    const int rc = stage_flush(m);
    if (!rc) pairs = here;
    return rc;
  }
};

}  // namespace

extern "C" {

int mrhbm_map_wordcount(mrhbm_map* m, const void* text, size_t len, uint64_t* words) {
  if (!m || (!text && len)) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (words) *words = 0;
  if (c->cfg.key_kind != MRHBM_KEY_STR) return fail(c, MRHBM_E_INVAL, "wordcount needs a string-key ctx");
  if (c->bytevals) return refuse_int_values(c);
  WordsJob job{m, (const unsigned char*)text, nullptr, 0, "wordcount"};
  return map_pieces(m, (const unsigned char*)text, len, job, words);
}

int mrhbm_map_words_value(mrhbm_map* m, const void* text, size_t len, const void* val, size_t vlen, uint64_t* words) {
  if (!m || (!text && len)) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (words) *words = 0;
  if (!c->bytevals) return refuse_byte_values(c);
  if (c->cfg.key_kind != MRHBM_KEY_STR) return fail(c, MRHBM_E_INVAL, "words_value needs a string-key ctx");
  int rc = check_value(c, val, vlen);
  if (rc) return rc;
  WordsJob job{m, (const unsigned char*)text, val, vlen, "words_value"};
  return map_pieces(m, (const unsigned char*)text, len, job, words);
}

int mrhbm_map_key_numbers(mrhbm_map* m, const void* text, size_t len, uint64_t* lines) {
  if (!m || (!text && len)) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  if (lines) *lines = 0;
  if (!c->bytevals) return refuse_byte_values(c);
  if (c->cfg.key_kind != MRHBM_KEY_STR) return fail(c, MRHBM_E_INVAL, "key_numbers needs a string-key ctx");
  if (!c->d_pow5) {
    static const std::vector<uint64_t> pow5 = [] {  // (computed once per process)
      std::vector<uint64_t> v(2 * kPow5Count);
      dec_pow5_table(v.data());
      return v;
    }();
    cudaError_t ea = cudaMalloc((void**)&c->d_pow5, pow5.size() * sizeof(uint64_t));
    if (ea == cudaSuccess) ea = cudaMalloc(&c->d_kn_fix, kKnFixCap * sizeof(uint4));
    if (ea == cudaSuccess)
      ea = cudaMemcpy(c->d_pow5, pow5.data(), pow5.size() * sizeof(uint64_t), cudaMemcpyHostToDevice);
    if (ea != cudaSuccess) {
      cudaGetLastError();
      if (c->d_pow5) cudaFree(c->d_pow5);
      if (c->d_kn_fix) cudaFree(c->d_kn_fix);
      c->d_pow5 = nullptr;
      c->d_kn_fix = nullptr;
      return fail(c, MRHBM_E_NOMEM, "key_numbers: %s", cudaGetErrorString(ea));
    }
  }
  KeyNumbersJob job{m, (const unsigned char*)text};
  return map_pieces(m, (const unsigned char*)text, len, job, lines);
}

// ---- synthetic word-count text (SURVEY App. B), host side: the input of the end-to-end word-count measurements
namespace {
// (splitmix64: mrhbm_dev.cuh)
inline int synth_rank_to_key(uint64_t rank, char* out) {  // bijective base 26 prefix + hashed upper-case suffix
  char tmp[16];
  int n = 0, o = 0;
  for (uint64_t r = rank; r > 0; r /= 26) {
    r -= 1;
    tmp[n++] = (char)('a' + (r % 26));
  }
  while (n > 0) out[o++] = tmp[--n];
  const uint64_t h = splitmix64(rank ^ 0xA5A5A5A5A5A5A5A5ull);
  unsigned l = (unsigned)(h % 8);
  if (((h >> 8) % 64) == 0) l = 8 + (unsigned)((h >> 16) % 15);
  for (unsigned j = 0; j < l; j++) out[o++] = (char)('A' + (splitmix64(h + j) % 26));
  return o;
}
inline uint64_t synth_zipf_rank(const uint64_t* T, uint64_t V, uint64_t u) {
  uint64_t lo = 0, hi = V;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (T[mid] < u) lo = mid + 1;
    else hi = mid;
  }
  return lo + 1 > V ? V : lo + 1;
}
}  // namespace

int mrhbm_synth_zipf_text(uint64_t seed, uint64_t first, uint64_t n, uint32_t words_per_line, const uint64_t* table,
                          uint64_t V, void* out, size_t cap, size_t* len, int threads) {
  if (!table || !V || !len || !words_per_line || (!out && cap)) return MRHBM_E_INVAL;
  threads = std::max(1, std::min(threads, 256));
  const uint64_t lines = (n + words_per_line - 1) / words_per_line;
  std::vector<uint64_t> bytes((size_t)threads + 1, 0);
  auto span = [&](int t, uint64_t* l0, uint64_t* l1) {
    *l0 = lines / threads * t;
    *l1 = t + 1 == threads ? lines : lines / threads * (t + 1);
  };
  auto run = [&](int t, char* dst) -> uint64_t {  // dst == nullptr: only measure
    uint64_t l0, l1, total = 0;
    span(t, &l0, &l1);
    char key[32];
    for (uint64_t l = l0; l < l1; l++) {
      const uint64_t w0 = l * words_per_line, w1 = std::min<uint64_t>(n, w0 + words_per_line);
      for (uint64_t w = w0; w < w1; w++) {
        const uint64_t u = splitmix64(seed + (1ull << 41) + first + w);
        const int kl = synth_rank_to_key(synth_zipf_rank(table, V, u), key);
        if (dst) {
          memcpy(dst + total, key, (size_t)kl);
          dst[total + kl] = w + 1 == w1 ? '\n' : ' ';
        }
        total += (uint64_t)kl + 1;
      }
    }
    return total;
  };
  {
    std::vector<std::thread> th;
    for (int t = 0; t < threads; t++) th.emplace_back([&, t] { bytes[(size_t)t + 1] = run(t, nullptr); });
    for (auto& x : th) x.join();
  }
  for (int t = 0; t < threads; t++) bytes[(size_t)t + 1] += bytes[(size_t)t];
  *len = (size_t)bytes[(size_t)threads];
  if (*len > cap) return MRHBM_E_INVAL;
  std::vector<std::thread> th;
  for (int t = 0; t < threads; t++) th.emplace_back([&, t] { run(t, (char*)out + bytes[(size_t)t]); });
  for (auto& x : th) x.join();
  return MRHBM_OK;
}

int mrhbm_pool_read(mrhbm_ctx* c, uint64_t first, uint64_t n, void* host_out) {
  if (!c || (!host_out && n)) return MRHBM_E_INVAL;
  Entry g(c);
  uint64_t skip = first, done = 0;
  for (auto& r : c->led.live()) {
    if (done == n) break;
    if (skip >= r.second) {
      skip -= r.second;
      continue;
    }
    uint64_t take = std::min<uint64_t>(n - done, r.second - skip);
    CU(c, cudaMemcpyAsync((char*)host_out + done * c->rb, (char*)c->pool + (r.first + skip) * c->rb, take * c->rb,
                          cudaMemcpyDeviceToHost, c->stream));
    done += take;
    skip = 0;
  }
  CU(c, cudaStreamSynchronize(c->stream));
  if (done != n) return fail(c, MRHBM_E_INVAL, "pool_read: only %llu of %llu pairs committed", (unsigned long long)done, (unsigned long long)n);
  return MRHBM_OK;
}

int mrhbm_map_commit(mrhbm_map* m) {
  if (!m) return MRHBM_E_INVAL;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  int rc = stage_flush(m);
  if (rc == 0 && m->async_reads) {
    cudaError_t e = cudaStreamSynchronize(c->stream);  // caller may reuse its pinned buffers now
    if (e != cudaSuccess) rc = fail(c, MRHBM_E_CUDA, "commit: %s", cudaGetErrorString(e));
  }
  std::vector<std::pair<uint64_t, uint64_t>> kept;
  if (rc == 0 && c->cfg.combiner == MRHBM_COMBINE_DISTINCT) rc = distinct_pairs(m, kept);
  if (rc == 0 && c->cfg.combiner == MRHBM_COMBINE_FSUM) rc = fsum_pairs(m);
  if (rc) {
    mrhbm_map_abort(m);
    return rc;
  }
  for (const auto& r : kept) c->led.shrink(m->serial, r.first, r.second);
  c->led.commit(m->serial, m->job);
  c->long_jobs.erase(m->job);  // replace-by-job-id on the host side too
  if (!m->long_pairs.empty()) c->long_jobs[m->job] = std::move(m->long_pairs);
  invalidate(c);
  map_release(m);
  return MRHBM_OK;
}

void mrhbm_map_abort(mrhbm_map* m) {
  if (!m) return;
  mrhbm_ctx* c = m->ctx;
  Entry g(c);
  cudaStreamSynchronize(c->stream);  // (copies into the room that goes back)
  c->led.abort(m->serial);
  map_release(m);
}

int mrhbm_reset(mrhbm_ctx* c) {
  if (!c) return MRHBM_E_INVAL;
  Entry g(c);
  c->led.reset();
  c->long_jobs.clear();
  invalidate(c);
  return MRHBM_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------
// shuffle
// ---------------------------------------------------------------------------
namespace {

// The sort may take a bin's key range from its index only for the global key-ordered sub-bins (sub = mulhi(key, S));
// the range partitioner's sub-bins are relative to their partition: min / max.
void set_range_hint(const mrhbm_ctx* c, ShuffleBuffers& b, uint32_t S, uint32_t ordered) {
  b.hint_S = (ordered && S > 1 && c->cfg.partitioner != MRHBM_PART_RANGE) ? S : 0;
  b.hint_q = S > 1 ? (uint64_t)(((unsigned __int128)1 << 64) / S) : 0;
}

RangeBinParams make_bp(const mrhbm_ctx* c, uint32_t S, uint32_t ordered) {
  RangeBinParams bp{};
  bp.P = c->cfg.num_partitions;
  bp.S = S;
  bp.partitioner = c->cfg.partitioner;
  bp.ordered = ordered;
  bp.ctr_shift = c->ctr_shift;
  bp.world = (uint32_t)c->world;
  bp.wshift = 0xffffffffu;
  for (uint32_t k = 0; k < 4; k++)
    if ((1u << k) == bp.world) bp.wshift = k;
  for (int r = 0; r <= 8; r++) bp.pbase[r] = c->pbase[r];
  if (c->cfg.partitioner == MRHBM_PART_RANGE && c->d_spl) {
    const uint32_t n = (uint32_t)c->spl.size();
    bp.spl_inv = (const ulonglong2*)c->d_spl;  // (first: 16-byte aligned)
    bp.spl_pre = (const unsigned long long*)(bp.spl_inv + bp.P);
    bp.spl_slot = (const uint32_t*)(bp.spl_pre + n);
    bp.spl_n = c->spl_fin;
    bp.spl_top = bp.spl_n ? 1u : 0u;
    while (bp.spl_top && bp.spl_top * 2 <= bp.spl_n) bp.spl_top *= 2;
  }
  return bp;
}

// The range partitioner's splitters must be the same on every rank: each shuffle's first all-gather carries two words
// of their digest (all ones: none installed).  Fails on all ranks alike.
uint32_t spl_word(const mrhbm_ctx* c, int i) {
  return c->spl_set ? (uint32_t)(c->spl_digest >> (32 * i)) : 0xffffffffu;
}
int check_splitters(mrhbm_ctx* c, const uint32_t* all, int k, int first) {
  bool ok = c->spl_set;
  for (int r = 0; r < c->world; r++)
    ok = ok && all[r * k + first] == spl_word(c, 0) && all[r * k + first + 1] == spl_word(c, 1);
  if (!ok)
    return fail(c, MRHBM_E_INVAL, c->spl_set ? "the ranks hold different splitters (mrhbm_set_splitters)"
                                             : "MRHBM_PART_RANGE needs splitters: call mrhbm_set_splitters or mrhbm_sample_splitters");
  return 0;
}

// all ranks: k <= 4 words from every rank (host values in, all[rank * k + i] out); synchronises the stream
int gather_words(mrhbm_ctx* c, const uint32_t* mine, int k, uint32_t* all) {
  if (c->world == 1) {
    for (int i = 0; i < k; i++) all[i] = mine[i];
    return 0;
  }
  for (int i = 0; i < k; i++) c->h_small[i] = mine[i];
  CU(c, cudaMemcpyAsync(c->d_small, c->h_small, 4 * k, cudaMemcpyHostToDevice, c->stream));
  int rc = comm_allgather_u32(c->comm, c->d_small, c->d_small + 16, (size_t)k, c->stream, &c->err);
  if (rc) return rc;
  CU(c, cudaMemcpyAsync(c->h_small + 16, c->d_small + 16, 4 * (size_t)k * c->world, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < k * c->world; i++) all[i] = c->h_small[16 + i];
  return 0;
}

// The region buffer of the two-level split.  One GPU: a plain allocation.  Several GPUs: COLLECTIVE -- every
// rank calls it with the same `need`; all buffers grow together and their IPC handles are re-exchanged, so that
// level 2 of every rank can pull its regions from every peer.  *shared_ok = false (on all ranks alike) when peer
// mapping is unavailable on any rank.
int ensure_regions(mrhbm_ctx* c, uint64_t need, bool* shared_ok) {
  *shared_ok = true;
  if (c->world == 1) return ensure_records(c, &c->regions, &c->regions_cap, need);
  if (c->ipc_failed) {
    *shared_ok = false;
    return 0;
  }
  if (need <= c->regions_cap) return 0;
  const int G = c->world, me = c->rank;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  CU(c, cudaStreamSynchronize(c->stream));
  for (int r = 0; r < G; r++) {
    if (r != me && c->peer_regions[r]) cudaIpcCloseMemHandle(c->peer_regions[r]);
    c->peer_regions[r] = nullptr;
  }
  cudaGetLastError();
  uint32_t flag = 0, flags[8];
  int rc = gather_words(c, &flag, 1, flags);  // every rank has unmapped its peers before anybody frees
  if (rc) return rc;
  rc = grow(c, &c->regions_cap, need, need + need / 8 + 1024, {{&c->regions, (size_t)c->rb}});
  if (rc) return rc;
  bool ok = true;
  cudaIpcMemHandle_t h;
  memset(&h, 0, sizeof h);
  if (cudaIpcGetMemHandle(&h, c->regions) != cudaSuccess) {
    cudaGetLastError();
    ok = false;
  }
  memcpy(c->h_ipc, &h, 64);
  CU(c, cudaMemcpyAsync(c->d_ipc, c->h_ipc, 64, cudaMemcpyHostToDevice, c->stream));
  rc = comm_allgather_u32(c->comm, c->d_ipc, c->d_ipc + 16, 16, c->stream, &c->err);
  if (rc) return rc;
  CU(c, cudaMemcpyAsync(c->h_ipc + 16, c->d_ipc + 16, 64 * (size_t)G, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  flag = ok ? 0u : 1u;
  rc = gather_words(c, &flag, 1, flags);  // a rank that could not export: nobody opens anything
  if (rc) return rc;
  for (int r = 0; r < G; r++) ok = ok && flags[r] == 0;
  if (ok) {
    for (int r = 0; r < G; r++) {
      if (r == me) {
        c->peer_regions[r] = c->regions;
        continue;
      }
      cudaIpcMemHandle_t hr;
      memcpy(&hr, c->h_ipc + 16 + 16 * r, 64);
      if (cudaIpcOpenMemHandle(&c->peer_regions[r], hr, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        cudaGetLastError();
        c->peer_regions[r] = nullptr;
        ok = false;
      }
    }
    flag = ok ? 0u : 1u;
    rc = gather_words(c, &flag, 1, flags);
    if (rc) return rc;
    for (int r = 0; r < G; r++) ok = ok && flags[r] == 0;
  }
  if (!ok) {
    for (int r = 0; r < G; r++) {
      if (r != me && c->peer_regions[r]) cudaIpcCloseMemHandle(c->peer_regions[r]);
      c->peer_regions[r] = nullptr;
    }
    cudaGetLastError();
    c->ipc_failed = true;
    *shared_ok = false;
  }
  return 0;
}

int ensure_multi_buffers(mrhbm_ctx* c, uint64_t B, uint64_t Bl) {
  const size_t G = (size_t)c->world;
  int rc = grow(c, &c->hd_cap, B, B + (B >> 2) + 1, {{(void**)&c->d_hd, 4}, {(void**)&c->d_hall, 4 * G}});
  if (rc) return rc;
  return grow(c, &c->bl_cap, Bl + 1, Bl + (Bl >> 2) + 2,
              {{(void**)&c->d_tot, 4}, {(void**)&c->d_outoff, 4}, {(void**)&c->d_segoff, 4 * G}});
}

struct Src {
  const char* p;
  uint64_t n;
};

// The pairs the shuffle partitions: the committed pool ranges, or -- with a combiner declared
// (job.lua:92-96,198-202) and enough pairs to pay for it -- one record per distinct key of this rank's pairs
// with their sum (shared-memory table per SM + one L2-resident global table, see k_combine).  A rank-local
// decision: the stages that follow only see "the pairs this rank contributes".  The combiner never fails a
// shuffle: when a string key's sum does not fit the u32 value of a combined record (or one value is too large
// for the table's state word), this shuffle hands on the raw pairs instead.  MRHBM_RED_DISTINCT: the first copy of
// each distinct (key slot, value bytes) pair over all committed pairs (distinct_set), in the set's scratch; the pool
// and the ledger stay as they are.  MRHBM_RED_COUNT_DISTINCT: the same pairs, always in the scratch and each with the
// value 1 (pool values are value ids, never summed).  EV_START .. EV_CSTART.
int collect_sources(mrhbm_ctx* c, std::vector<Src>& srcs, uint64_t* N, mrhbm_stats& st) {
  srcs.clear();
  uint64_t n = 0;
  std::vector<std::pair<uint64_t, uint64_t>> live;
  for (auto& r : c->led.live()) {
    srcs.push_back(Src{(const char*)c->pool + r.first * c->rb, r.second});
    if (r.second) live.push_back(r);
    n += r.second;
  }
  *N = n;
  if (c->red_distinct || c->red_count) {
    std::vector<DistinctRange> rg;
    std::vector<uint32_t> off;
    int rc = distinct_set(c, live, c->red_count ? "count-distinct reducer: a shuffle of" : "distinct reducer: a shuffle of",
                          rg, off, &st.launches, c->red_count);
    if (rc || (off.back() == n && !c->red_count)) return rc;
    srcs.assign(1, Src{(const char*)c->dd_out, off.back()});
    *N = off.back();
    return 0;
  }
  if (c->cfg.combiner != MRHBM_COMBINE_REDUCER || c->no_combine || n < (1u << 20)) return 0;
  cudaStream_t s = c->stream;
  bool checked = c->combine_checked;
  for (;;) {
    const GtabLayout tab = GtabLayout::sized(c->rb, c->gtab_grow);
    const uint64_t tab_bytes = tab.bytes();
    int rc = ensure_records(c, &c->gtab, &c->gtab_cap, (tab_bytes + c->rb - 1) / c->rb);
    if (rc) return rc;
    rc = ensure_records(c, &c->comb, &c->comb_cap, tab.records());
    if (rc) return rc;
    CU(c, cudaMemsetAsync(c->gtab, 0, tab_bytes, s));
    CU(c, cudaMemsetAsync(c->d_small, 0, 3 * sizeof(uint32_t), s));  // [0] flags, [1] records out, [2] largest value
    for (auto& sr : srcs)
      st.launches += launch_combine(sr.p, sr.n, (uint32_t*)c->gtab, tab, c->d_small, checked, c->sm_count, s);
    st.launches += launch_gtab_compact((const uint32_t*)c->gtab, tab, c->comb, c->d_small + 1, s);
    CU(c, cudaGetLastError());
    CU(c, cudaMemcpyAsync(c->h_small, c->d_small, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CU(c, cudaStreamSynchronize(s));
    const uint32_t ef = c->h_small[0];
    if (ef & ERRF_OVERFLOW) return 0;  // not sticky: the next shuffle's sums may fit again
    if (ef & ERRF_SKEW) {  // the table filled up: more distinct keys than it takes
      if (c->gtab_grow < GtabLayout::kMaxGrow) {
        c->gtab_grow++;
        continue;
      }
      c->no_combine = true;  // the partition / sort / reduce stages take the raw pairs
      return 0;
    }
    if (!checked && c->rb != 16 && (uint64_t)c->h_small[2] * n > kMaxCombinedSum) {
      // the fire-and-forget adds could have wrapped a u32 sum unnoticed: again, with checked adds (sticky)
      checked = c->combine_checked = true;
      continue;
    }
    srcs.clear();
    srcs.push_back(Src{(const char*)c->comb, c->h_small[1]});
    *N = c->h_small[1];
    return 0;
  }
}

uint32_t pick_sub_bins(const mrhbm_ctx* c, uint64_t n_total, uint32_t copies = 1) {
  // mean bin = capacity of one CTA's shared-memory sort minus 6 sigma of a Poisson fill.  `copies`: records arrive in
  // clumps of up to that many with one key (every rank's combiner emits each key once: a bin then holds Poisson-many
  // KEYS times `copies` records, its sigma is sqrt(copies) times wider -- a 6-sigma-of-records capacity lets
  // enough bins of the combined Zipf stream on 8 GPUs overflow to send every shuffle to the exact layout)
  uint64_t target = (uint64_t)std::max(1.0, (double)c->cap - 6.0 * std::sqrt((double)c->cap * (double)copies));
  uint64_t P = c->cfg.num_partitions;
  return (uint32_t)std::max<uint64_t>(1, (n_total + P * target - 1) / (P * target));
}

// The sub-bins of the exact layout's next attempt after a bin held more distinct keys than one CTA sorts (ERRF_SKEW):
// twice as many.  Hash partitions are balanced, so that is enough; a key range may hold almost every key (splitters
// inside a narrow key range), so the range partitioner sizes S at once from its fullest partition, whose records the
// bin offsets of this attempt (h_bin_off, nb local bins of S per partition) already count: enough sub-bins that it
// fills them to the mean pick_sub_bins aims at.  COLLECTIVE on several GPUs (the fullest partition of the job).
// 0: more bins than the layout addresses.
int next_sub_bins(mrhbm_ctx* c, uint32_t S, uint64_t nb, uint64_t* S_next) {
  const uint64_t P = c->cfg.num_partitions;
  uint64_t want = 2ull * S;
  if (c->cfg.partitioner == MRHBM_PART_RANGE) {
    uint32_t mx = 0;
    for (uint64_t b = 0; b + S <= nb; b += S) mx = std::max(mx, c->h_bin_off[b + S] - c->h_bin_off[b]);
    uint32_t all[8];
    int rc = gather_words(c, &mx, 1, all);
    if (rc) return rc;
    for (int r = 0; r < c->world; r++) mx = std::max(mx, all[r]);
    const double target = std::max(1.0, (double)c->cap - 6.0 * std::sqrt((double)c->cap));
    while ((double)mx / (double)want > target && P * want < (1ull << 31)) want *= 2;
  }
  *S_next = P * want < (1ull << 31) ? want : 0;
  return 0;
}

// The error flags of an attempt, OR-ed over all ranks: every rank must take the same branch.  The all-gather also
// tells every rank whether any rank holds long keys (c->any_long).  One GPU: *ef stays as it is.
int agree_flags(mrhbm_ctx* c, uint32_t* ef) {
  if (c->world > 1) {
    const uint32_t mine = *ef | (c->long_jobs.empty() ? 0u : kErrfLongKeys);
    uint32_t all[8];
    int rc = gather_words(c, &mine, 1, all);
    if (rc) return rc;
    for (int r = 0; r < c->world; r++) *ef |= all[r];
    c->any_long = (*ef & kErrfLongKeys) != 0;
    *ef &= ~kErrfLongKeys;
  }
  return 0;
}

// Exact layout (bin offsets in sb.bin_off after k_hist + k_exscan): the records of `live` go to their B bins in sb.mid
// (on several GPUs: the destination-major send buffer), through the two-level coalesced split when there are enough
// bins (claims relative to bin_off), else the direct scatter.
int exact_split(mrhbm_ctx* c, const std::vector<Src>& live, const RangeBinParams& bp, uint64_t B, uint64_t N, mrhbm_stats& st) {
  cudaStream_t s = c->stream;
  SplitPlan pl{};
  if (plan_split(pl, &B, 1, 0, c->cap, 0, true)) {
    int rc = ensure_records(c, &c->l1buf, &c->l1_cap, N);
    if (rc) return rc;
    // relative fill levels: coarse levels live in hist (dead after the scan), fine levels in cursor
    CU(c, cudaMemsetAsync(c->sb.hist, 0, ((uint64_t)pl.C1 << c->ctr_shift) * sizeof(uint32_t), s));
    CU(c, cudaMemsetAsync(c->sb.cursor, 0, (B << c->ctr_shift) * sizeof(uint32_t), s));
    pl.cursor1 = c->sb.hist;
    pl.cursor = c->sb.cursor;
    pl.ctr_shift = bp.ctr_shift;
    pl.l1 = c->l1buf;
    pl.mid = c->sb.mid;
    pl.err_flags = c->sb.counters + CNT_ERR;
    pl.base_off = c->sb.bin_off;
    for (auto& r : live) st.launches += launch_split_l1(c->rb, r.p, r.n, bp, pl, s);
    st.launches += launch_split_l2(c->rb, bp, pl, s);
  } else {
    for (auto& r : live) st.launches += launch_scatter(c->rb, r.p, r.n, bp, c->sb.cursor, c->sb.mid, s);
  }
  return 0;
}

// MRHBM_RED_DISTINCT, after the sort of the nb bins of view v and k_big_bins: every bin's rows in (key, value bytes)
// order, an oversized bin (nbig of them) as one run (mrhbm_value_order.cu).  Inside ms_bigbins.
int order_values(mrhbm_ctx* c, const ShuffleBuffers& v, uint64_t nb, uint32_t nbig, mrhbm_stats& st) {
  st.launches += launch_value_order(c->rb, v, (uint32_t)nb, nbig, c->cap, c->arena, c->voff, c->stream);
  if (nbig) {
    int rc = grow(c, &c->vo_cap, c->out_cap, c->out_cap, {{&c->vo_keys, (size_t)c->kb}, {(void**)&c->vo_ids, sizeof(uint64_t)}});
    if (rc) return rc;
    st.launches += launch_value_merge(c->rb, v, nbig, c->cap, c->arena, c->voff, c->vo_keys, c->vo_ids, c->stream);
  }
  CU(c, cudaGetLastError());
  return 0;
}

// MRHBM_RED_FSUM, after the sort of the nb bins of view v and k_big_bins: an oversized bin's chunks merged into one run
// by key (k_num_key_merge, many CTAs per bin), then every bin reduced to one row per key holding its values' exact sum, rounded
// (mrhbm_num_sum.cu).  Inside ms_bigbins; a value that is not a number or a NaN sum is flagged in counters[CNT_ERR].
int sum_values(mrhbm_ctx* c, const ShuffleBuffers& v, uint64_t nb, uint32_t nbig, mrhbm_stats& st) {
  if (nbig) {  // (exact layout: rows [0, out_cap))
    int rc = grow(c, &c->vo_cap, c->out_cap, c->out_cap, {{&c->vo_keys, (size_t)c->kb}, {(void**)&c->vo_ids, sizeof(uint64_t)}});
    const uint64_t slots = num_slots(c->out_cap, c->cap);
    if (!rc) rc = grow(c, &c->ns_cap, slots, slots, {{(void**)&c->ns_acc, 2 * kAccWords * sizeof(int64_t)},
                                                     {(void**)&c->ns_flags, 4}, {(void**)&c->ns_head, 4}});
    if (rc) return rc;
    st.launches += launch_num_key_merge(c->rb, v, nbig, c->cap, c->out_cap, c->vo_keys, c->vo_ids, c->stream);
  }
  const NumScratch sc{c->ns_acc, c->ns_flags, c->ns_head};
  st.launches += launch_num_sum(c->rb, v, (uint32_t)nb, nbig, c->cap, c->arena, c->voff, sc, c->stream);
  CU(c, cudaGetLastError());
  return 0;
}

// Exact layout, after the sort of the nb bins of view v (nbig of them oversized): k_big_bins, the group offsets, and
// the bin offsets (v.bin_off), group offsets and counters read back.  EV_BIG, EV_END; synchronises the stream.
int exact_tail(mrhbm_ctx* c, const ShuffleBuffers& v, uint64_t nb, uint32_t nbig, mrhbm_stats& st) {
  cudaStream_t s = c->stream;
  st.launches += launch_big_bins(c->rb, v, nbig, c->cap, s);
  if (c->red_distinct || c->red_fsum) {
    int rc = c->red_distinct ? order_values(c, v, nb, nbig, st) : sum_values(c, v, nb, nbig, st);
    if (rc) return rc;
  }
  CU(c, cudaEventRecord(c->ev[EV_BIG], s));
  c->h_big.clear();
  if (c->sb.no_reduce && !c->red_distinct && !c->red_fsum && nbig) {  // group-only mode: the iterator merges the runs of an oversized bin
    c->h_big.resize(nbig);
    CU(c, cudaMemcpyAsync(c->h_big.data(), c->sb.big_list, nbig * 4, cudaMemcpyDeviceToHost, s));
  }
  st.launches += launch_exscan(c->sb.ucount, (uint32_t)nb, c->sb.uoff, nullptr, nullptr, 0xffffffffu, nullptr, nullptr,
                               c->sb.counters + CNT_TOTAL, 0, s, c->d_small + 64);
  c->h_bin_off.resize(nb + 1);
  c->h_uoff.resize(nb + 1);
  CU(c, cudaMemcpyAsync(c->h_bin_off.data(), v.bin_off, (nb + 1) * 4, cudaMemcpyDeviceToHost, s));
  CU(c, cudaMemcpyAsync(c->h_uoff.data(), c->sb.uoff, (nb + 1) * 4, cudaMemcpyDeviceToHost, s));
  CU(c, cudaMemcpyAsync(c->h_counters, c->sb.counters, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CU(c, cudaEventRecord(c->ev[EV_END], s));
  CU(c, cudaGetLastError());
  CU(c, cudaStreamSynchronize(s));
  return 0;
}

// View v over Bl local bins (the first is global bin bin_base) becomes the result the accessors read, and the stats
// are filled in.  Which events bound the exchange and the scatter depends on the path: the caller times them.
int publish(mrhbm_ctx* c, const ShuffleBuffers& v, uint64_t Bl, uint32_t S, uint32_t ordered, uint64_t N_in,
            uint64_t N_recv, uint32_t bin_base, uint32_t nbig, mrhbm_stats& st, float ms_exchange, float ms_scatter) {
  c->rv = v;
  c->B = (uint32_t)Bl;
  c->S = S;
  c->ordered = ordered;
  c->N = N_in;
  c->N_recv = N_recv;
  c->bin_base = bin_base;
  c->groups = c->h_uoff[Bl];
  c->shuffled = true;
  c->compacted = false;
  c->shuffle_spl_digest = c->spl_digest;
  st.bins = (uint32_t)Bl;
  st.sub_bins = S;
  st.big_bins = nbig;
  st.groups = c->groups;
  st.ms_total = ev_ms(c, EV_START, EV_END);
  st.ms_combine = ev_ms(c, EV_START, EV_CSTART);
  st.ms_hist = ev_ms(c, EV_COMBINE, EV_HIST);
  st.ms_plan = ev_ms(c, EV_HIST, EV_PLAN);
  st.ms_exchange = ms_exchange;
  st.ms_scatter = ms_scatter;
  st.ms_sort_reduce = ev_ms(c, EV_EXCH, EV_SORT);
  st.ms_bigbins = ev_ms(c, EV_SORT, EV_BIG);
  st.ms_setup = ev_ms(c, EV_CSTART, EV_COMBINE);
  st.ms_finish = ev_ms(c, EV_BIG, EV_END);
  c->stats = st;
  return MRHBM_OK;
}

// ---- the default path: optimistic fixed-capacity layout, no histogram pass, any number of GPUs --------
//
//   level 1  k_split_tma   committed pairs -> coarse regions (this rank's region buffer, all regions of the job)
//   [G > 1]  all-gather of the level-1 fill levels (a few KB): counts for the peers + the barrier that orders
//            every rank's level 1 before anybody's level 2
//   level 2  k_split_tma   the owner of a region pulls it from every rank's region buffer (NVLink bulk copies
//            into shared memory, overlapped with the split of the previous tile) -> fine bins
//   sort     k_sort_reduce_u64 / k_sort_reduce on local bins
// Every bin and region has a fixed capacity (mean + slack); the claim cursor doubles as the count.  A full one
// sets ERRF_CAPACITY, nothing is lost (the input stays in the pool) and the exact layout below takes over, for
// good on this ctx.  Returns 0 with *done = true, 0 with *done = false (fall back), or an error.
int shuffle_fast(mrhbm_ctx* c, std::vector<Src>& live, uint64_t N, uint64_t N_in, mrhbm_stats& st, bool* done) {
  *done = false;
  const int G = c->world, me = c->rank;
  const uint32_t P = c->cfg.num_partitions;
  cudaStream_t s = c->stream;
  int rc = 0;
  // ---- would key-ordered sub-bins be balanced?  sample the keys before anything moves
  const bool want_ordered = c->cfg.key_kind == MRHBM_KEY_U64 && !(c->cfg.flags & MRHBM_F_FORCE_RUNS) && !c->no_ordered;
  const bool range = c->cfg.partitioner == MRHBM_PART_RANGE;
  uint32_t nonuniform = 0;
  if (want_ordered && N >= 4096 && (!range || c->spl_set)) {
    CU(c, cudaMemsetAsync(c->d_sample, 0, 256 * sizeof(uint32_t), s));
    uint64_t total = 0;
    const RangeBinParams sbp = make_bp(c, 1, 1);
    for (auto& r : live) {
      uint32_t ns = (uint32_t)std::min<uint64_t>(r.n, (uint64_t)((double)kSampleKeys * (double)r.n / (double)N) + 1);
      if (range)  // the position of the keys inside their partitions
        st.launches += launch_sample_range_u64(r.p, r.n, ns, sbp, c->d_sample, s);
      else
        st.launches += launch_sample_u64(r.p, r.n, ns, c->d_sample, s);
      total += ns;
    }
    CU(c, cudaMemcpyAsync(c->h_sample, c->d_sample, 256 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CU(c, cudaStreamSynchronize(s));
    uint32_t mx = 0;
    for (int i = 0; i < 256; i++) mx = std::max(mx, c->h_sample[i]);
    const double mean = (double)total / 256.0;
    nonuniform = (double)mx > mean * 1.08 + 5.0 * std::sqrt(mean) + 2.0;
  }
  // ---- job-wide facts.  On several GPUs this all-gather is also the barrier that keeps a rank from refilling
  // its region buffer while a peer's level 2 of the previous shuffle may still read it.
  // (range partitioner: two more words, the splitter digest)
  const int k = range ? 4 : 2;
  uint32_t mine[4] = {(uint32_t)N, nonuniform, spl_word(c, 0), spl_word(c, 1)}, all[32];
  rc = gather_words(c, mine, k, all);
  if (rc) return rc;
  if (range && (rc = check_splitters(c, all, k, 2))) return rc;
  uint64_t Nglobal = 0, Nmax = 0;
  for (int r = 0; r < G; r++) {
    Nglobal += all[k * r];
    Nmax = std::max<uint64_t>(Nmax, all[k * r]);
    nonuniform |= all[k * r + 1];
  }
  if (Nglobal == 0) return 0;  // nothing to do here: the exact path handles the empty shuffle
  const uint32_t S = pick_sub_bins(c, Nglobal, c->cfg.combiner == MRHBM_COMBINE_REDUCER && G > 1 ? (uint32_t)G : 1u);
  const uint64_t B = (uint64_t)P * S;
  if (B >= (1ull << 31)) return 0;
  const uint32_t ordered = (want_ordered && !nonuniform) || S == 1;
  uint64_t Bl_of[8];
  for (int r = 0; r < G; r++) Bl_of[r] = (uint64_t)(c->pbase[r + 1] - c->pbase[r]) * S;
  const uint64_t Bl = Bl_of[me];
  const uint32_t bin_stride = c->cap;  // slots per fine bin: what one CTA sorts in shared memory
  // ---- levels.  One GPU, few bins: level 1 goes straight into the fine bins.
  SplitPlan pl{};
  const int levels = plan_split(pl, Bl_of, (uint32_t)G, (uint32_t)me, bin_stride, Nmax, false);
  if (!levels) return 0;  // more bins than two levels reach: exact path
  const bool single_level = levels == 1;
  // ---- buffers
  rc = ensure_small_arrays(c, std::max<uint64_t>(Bl, pl.C1));
  if (rc) return rc;
  // k_split_tma addresses destination slots with 32 bits, and lets the records of a run that does not fit (the
  // attempt is abandoned then) land at the start of the run's region: one tile of slack behind the last region
  const uint64_t tile_slack = kSplitTileBytes / c->rb;
  if (Bl * bin_stride + tile_slack >= (1ull << 32) || (uint64_t)pl.C1 * pl.sub_stride + tile_slack >= (1ull << 32)) return 0;
  rc = ensure_records(c, &c->sb.mid, &c->mid_cap, Bl * bin_stride + tile_slack);
  if (rc) return rc;
  rc = ensure_out(c, Bl * (uint64_t)c->cap);
  if (rc) return rc;
  if (!single_level) {
    bool shared_ok = true;
    rc = ensure_regions(c, (uint64_t)pl.C1 * pl.sub_stride + tile_slack, &shared_ok);
    if (rc) return rc;
    if (!shared_ok) {  // peer mapping unavailable (decided by all ranks together): NCCL exchange instead
      c->no_optimistic = true;
      return 0;
    }
    if (G > 1) {
      const uint64_t words = ((uint64_t)pl.C1 << c->ctr_shift) * G;
      rc = grow(c, &c->l1all_cap, words, words + words / 4, {{(void**)&c->d_l1all, sizeof(uint32_t)}});
      if (rc) return rc;
    }
  }
  pl.cursor1 = c->sb.hist;
  pl.cursor = c->sb.cursor;
  pl.ctr_shift = c->ctr_shift;
  pl.l1 = single_level ? c->sb.mid : c->regions;
  pl.mid = c->sb.mid;
  pl.err_flags = c->sb.counters + CNT_ERR;
  pl.ticket = c->sb.counters + 5;  // (words 5 and 6 of the 8 counters cleared below)
  pl.base_off = nullptr;
  for (int r = 0; r < 8; r++) pl.peer[r] = (unsigned long long)(uintptr_t)(G == 1 ? (r == 0 ? c->regions : nullptr) : c->peer_regions[r]);
  pl.l1_counts = G == 1 ? c->sb.hist : c->d_l1all;
  pl.l1_zstride = G == 1 ? 0 : ((uint64_t)pl.C1 << c->ctr_shift);
  const RangeBinParams bp = make_bp(c, S, ordered);
  st.attempts++;
  CU(c, cudaMemsetAsync(c->sb.hist, 0, (((uint64_t)pl.C1) << c->ctr_shift) * sizeof(uint32_t), s));
  if (!single_level) CU(c, cudaMemsetAsync(c->sb.cursor, 0, (std::max<uint64_t>(Bl, 1) << c->ctr_shift) * sizeof(uint32_t), s));
  CU(c, cudaMemsetAsync(c->sb.counters, 0, 8 * sizeof(uint32_t), s));
  CU(c, cudaEventRecord(c->ev[EV_COMBINE], s));
  CU(c, cudaEventRecord(c->ev[EV_HIST], s));
  for (auto& r : live) st.launches += launch_split_l1(c->rb, r.p, r.n, bp, pl, s);
  CU(c, cudaEventRecord(c->ev[EV_PLAN], s));
  if (G > 1) {
    rc = comm_allgather_u32(c->comm, c->sb.hist, c->d_l1all, (size_t)pl.C1 << c->ctr_shift, s, &c->err);
    if (rc) return rc;
  }
  CU(c, cudaEventRecord(c->ev[EV_GATH], s));
  if (!single_level) st.launches += launch_split_l2(c->rb, bp, pl, s);
  CU(c, cudaEventRecord(c->ev[EV_SCATTER], s));
  CU(c, cudaEventRecord(c->ev[EV_EXCH], s));
  c->sb.src = c->sb.mid;
  c->sb.nseg = 1;
  c->sb.stride = bin_stride;
  c->sb.out_stride = c->cap;
  c->sb.ctr_shift = c->ctr_shift;
  // single level: the level-1 cursors ARE the fine fill levels
  uint32_t* fine_cursor = single_level ? c->sb.hist : c->sb.cursor;
  ShuffleBuffers v = c->sb;
  v.cursor = fine_cursor;
  set_range_hint(c, v, S, ordered);
  if (Bl) st.launches += launch_sort_reduce(c->rb, v, (uint32_t)Bl, c->cap, c->sm_count, s);
  CU(c, cudaEventRecord(c->ev[EV_SORT], s));
  if (c->red_distinct && (rc = order_values(c, v, Bl, 0, st))) return rc;
  if (c->red_fsum && (rc = sum_values(c, v, Bl, 0, st))) return rc;
  CU(c, cudaEventRecord(c->ev[EV_BIG], s));
  c->h_uoff.assign(Bl + 1, 0);
  if (Bl) {
    st.launches += launch_exscan(c->sb.ucount, (uint32_t)Bl, c->sb.uoff, nullptr, nullptr, 0xffffffffu, nullptr, nullptr,
                                 c->sb.counters + CNT_TOTAL, 0, s, c->d_small + 64);
    CU(c, cudaMemcpyAsync(c->h_uoff.data(), c->sb.uoff, (Bl + 1) * 4, cudaMemcpyDeviceToHost, s));
  }
  // pairs this rank reduced (and how many of them came from peers)
  st.launches += launch_region_totals(pl.l1_counts, pl.l1_zstride, (uint32_t)G, (uint32_t)me, pl.rbase[me], pl.C1_local,
                                      c->ctr_shift, (uint32_t)std::min<uint64_t>(single_level ? bin_stride : pl.sub_stride, 0xffffffffull),
                                      c->d_acc, s);
  CU(c, cudaMemcpyAsync(c->h_acc, c->d_acc, 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  CU(c, cudaMemcpyAsync(c->h_counters, c->sb.counters, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CU(c, cudaEventRecord(c->ev[EV_END], s));
  CU(c, cudaGetLastError());
  CU(c, cudaStreamSynchronize(s));
  uint32_t ef = c->h_counters[CNT_ERR];
  rc = agree_flags(c, &ef);  // (several GPUs: also, nobody leaves while a peer still reads its regions)
  if (rc) return rc;
  if (ef & ERRF_CAPACITY) {  // skewed keys: the exact layout from now on
    c->sb.stride = 0;
    c->no_optimistic = true;
    if ((ordered && S > 1) || nonuniform) c->no_ordered = true;  // key-ordered sub-bins overflowed, or would
    return 0;
  }
  c->h_big.clear();
  c->sb.stride = 0;
  st.bytes_exchanged = (c->h_acc[0] - c->h_acc[1]) * (uint64_t)c->rb;
  *done = true;
  // plan = level 1, exchange = the fill-level all-gather (waits for the slowest rank's level 1), scatter = level 2
  // (on several GPUs: including the NVLink pulls)
  return publish(c, v, Bl, S, ordered, N_in, c->h_acc[0], c->pbase[me] * S, 0, st, ev_ms(c, EV_PLAN, EV_GATH),
                 ev_ms(c, EV_GATH, EV_SCATTER));
}

// ---- one GPU, exact layout: hist -> scan -> scatter -> sort+reduce (skewed keys, oversized bins) ---------
int shuffle_single_exact(mrhbm_ctx* c, std::vector<Src>& live, uint64_t N, uint64_t N_in, mrhbm_stats& st) {
  const uint32_t P = c->cfg.num_partitions;
  int rc = 0;
  uint32_t nbig = 0, ordered = 1;
  cudaStream_t s = c->stream;
  uint64_t B = 0;
  uint32_t S = pick_sub_bins(c, N);
  bool skip_ordered = c->no_ordered;
  // A bin that holds more distinct keys than one CTA sorts (ERRF_SKEW) is retried with
  // twice the sub-bins: distinct keys spread, hot keys keep collapsing in k_big_bins.
  for (int widen = 0;; widen++) {
    B = (uint64_t)P * S;
    if (B >= (1ull << 31)) return fail(c, MRHBM_E_INVAL, "too many bins");
    rc = ensure_buffers(c, B, N);
    if (rc) return rc;
    ordered = ((c->cfg.key_kind == MRHBM_KEY_U64 && !(c->cfg.flags & MRHBM_F_FORCE_RUNS) && widen == 0 && !skip_ordered) || S == 1);
    c->sb.stride = 0;
    for (;;) {
      st.attempts++;
      RangeBinParams bp = make_bp(c, S, ordered);
      CU(c, cudaMemsetAsync(c->sb.hist, 0, (B << c->ctr_shift) * sizeof(uint32_t), s));
      CU(c, cudaMemsetAsync(c->sb.counters, 0, 8 * sizeof(uint32_t), s));
      CU(c, cudaEventRecord(c->ev[EV_COMBINE], s));
      for (auto& r : live) st.launches += launch_hist(c->rb, r.p, r.n, bp, c->sb.hist, s);
      CU(c, cudaEventRecord(c->ev[EV_HIST], s));
      st.launches += launch_exscan(c->sb.hist, (uint32_t)B, c->sb.bin_off, c->sb.cursor, nullptr, c->cap, c->sb.big_list,
                                   c->sb.counters + CNT_NBIG, c->sb.counters + CNT_TOTAL, c->ctr_shift, s, c->d_small + 64);
      CU(c, cudaMemcpyAsync(c->h_counters, c->sb.counters, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
      CU(c, cudaEventRecord(c->ev[EV_PROBE], s));
      CU(c, cudaEventRecord(c->ev[EV_PLAN], s));
      rc = exact_split(c, live, bp, B, N, st);
      if (rc) return rc;
      CU(c, cudaEventRecord(c->ev[EV_SCATTER], s));
      CU(c, cudaEventRecord(c->ev[EV_EXCH], s));
      c->sb.src = c->sb.mid;
      c->sb.nseg = 1;
      c->sb.seg_off[0] = c->sb.bin_off;
      c->sb.seg_base[0] = 0;
      set_range_hint(c, c->sb, S, ordered);
      st.launches += launch_sort_reduce(c->rb, c->sb, (uint32_t)B, c->cap, c->sm_count, s);
      CU(c, cudaEventRecord(c->ev[EV_SORT], s));
      CU(c, cudaGetLastError());
      CU(c, cudaEventSynchronize(c->ev[EV_PROBE]));  // overlaps with scatter / sort on the device
      nbig = c->h_counters[CNT_NBIG];
      if (nbig && ordered && S > 1) {
        // key-ordered sub-bins are unbalanced for this key distribution: redo with hash sub-bins
        ordered = 0;
        c->no_ordered = true;
        continue;
      }
      break;
    }
    rc = exact_tail(c, c->sb, B, nbig, st);
    if (rc) return rc;
    uint32_t ef = c->h_counters[CNT_ERR];
    rc = agree_flags(c, &ef);
    if (rc) return rc;
    if (ef & ERRF_SKEW) {
      uint64_t S_next = 0;
      if (widen < 4 && (rc = next_sub_bins(c, S, B, &S_next))) return rc;
      if (S_next) {
        S = (uint32_t)S_next;
        continue;
      }
      return fail(c, MRHBM_E_SKEW, "a bin holds more distinct keys than one SM can sort (%u oversized bins)", nbig);
    }
    break;
  }
  return publish(c, c->sb, B, S, ordered, N_in, N, 0, nbig, st, 0.f, ev_ms(c, EV_PLAN, EV_SCATTER));
}

// ---- several GPUs, exact layout: hist -> all-gather counts -> scatter (destination-major) -> NCCL all-to-all
//      -> sort+reduce of the owned partitions, each bin gathered from one segment per source
int shuffle_multi_exact(mrhbm_ctx* c, std::vector<Src>& live, uint64_t N, uint64_t N_in, mrhbm_stats& st) {
  const int G = c->world, me = c->rank;
  const uint32_t P = c->cfg.num_partitions;
  // (range partitioner: two more words, the splitter digest)
  const bool range = c->cfg.partitioner == MRHBM_PART_RANGE;
  const int k = range ? 3 : 1;
  const uint32_t mine[3] = {(uint32_t)N, spl_word(c, 0), spl_word(c, 1)};
  uint32_t all[24];
  int rc = gather_words(c, mine, k, all);
  if (rc) return rc;
  if (range && (rc = check_splitters(c, all, k, 1))) return rc;
  uint64_t Nglobal = 0;
  for (int r = 0; r < G; r++) Nglobal += all[k * r];
  uint32_t S = pick_sub_bins(c, Nglobal);
  uint32_t nbig = 0, ordered = 1;
  cudaStream_t s = c->stream;
  uint64_t B = 0, Bl = 0, total_recv = 0;
  uint64_t send_off[9], send_cnt[8], recv_off[9], recv_cnt[8];
  ShuffleBuffers v{};
  for (int widen = 0;; widen++) {
    B = (uint64_t)P * S;
    Bl = (uint64_t)c->Pl * S;
    const uint32_t bin_base = c->pbase[me] * S;
    if (B >= (1ull << 31)) return fail(c, MRHBM_E_INVAL, "too many bins");
    rc = ensure_buffers(c, B, N);
    if (rc) return rc;
    rc = ensure_multi_buffers(c, B, Bl);
    if (rc) return rc;
    ordered = ((c->cfg.key_kind == MRHBM_KEY_U64 && !(c->cfg.flags & MRHBM_F_FORCE_RUNS) && widen == 0 && !c->no_ordered) || S == 1);
    c->sb.stride = 0;
    for (;;) {
      st.attempts++;
      RangeBinParams bp = make_bp(c, S, ordered);
      CU(c, cudaMemsetAsync(c->sb.hist, 0, (B << c->ctr_shift) * sizeof(uint32_t), s));
      CU(c, cudaMemsetAsync(c->sb.counters, 0, 8 * sizeof(uint32_t), s));
      CU(c, cudaEventRecord(c->ev[EV_COMBINE], s));
      for (auto& r : live) st.launches += launch_hist(c->rb, r.p, r.n, bp, c->sb.hist, s);
      CU(c, cudaEventRecord(c->ev[EV_HIST], s));
      // send layout (destination-major bins) + dense counts for the all-gather
      st.launches += launch_exscan(c->sb.hist, (uint32_t)B, c->sb.bin_off, c->sb.cursor, c->d_hd, 0xffffffffu, nullptr,
                                   nullptr, nullptr, c->ctr_shift, s, c->d_small + 64);
      rc = comm_allgather_u32(c->comm, c->d_hd, c->d_hall, B, s, &c->err);
      if (rc) return rc;
      // receive layout: per owned bin the total and the per-source offsets
      st.launches += launch_sum_src(c->d_hall, G, (uint32_t)B, bin_base, (uint32_t)Bl, c->d_tot, c->cap,
                                    c->sb.counters + CNT_GBIG, s);
      st.launches += launch_exscan(c->d_tot, (uint32_t)Bl, c->d_outoff, nullptr, nullptr, c->cap, c->sb.big_list,
                                   c->sb.counters + CNT_NBIG, c->sb.counters + CNT_TOTAL, 0, s, c->d_small + 64);
      st.launches += launch_exscan_rows(c->d_hall, G, (uint32_t)B, bin_base, (uint32_t)Bl, c->d_segoff, c->d_small + 32, s);
      for (int d = 0; d <= G; d++)
        CU(c, cudaMemcpyAsync(c->h_small + 48 + d, c->sb.bin_off + (uint64_t)c->pbase[d] * S, 4, cudaMemcpyDeviceToHost, s));
      CU(c, cudaMemcpyAsync(c->h_small + 32, c->d_small + 32, 4 * G, cudaMemcpyDeviceToHost, s));
      CU(c, cudaMemcpyAsync(c->h_counters, c->sb.counters, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
      CU(c, cudaEventRecord(c->ev[EV_PLAN], s));
      rc = exact_split(c, live, bp, B, N, st);  // into the send buffer
      if (rc) return rc;
      CU(c, cudaEventRecord(c->ev[EV_SCATTER], s));
      CU(c, cudaGetLastError());
      CU(c, cudaStreamSynchronize(s));
      nbig = c->h_counters[CNT_NBIG];
      total_recv = c->h_counters[CNT_TOTAL];
      // every rank counted the oversized bins of ALL ranks from the same all-gathered counts:
      // the decision is identical everywhere without another collective
      bool redo = c->h_counters[CNT_GBIG] && ordered && S > 1;
      if (redo) {
        ordered = 0;
        continue;
      }
      break;
    }
    send_off[0] = 0;
    recv_off[0] = 0;
    st.bytes_exchanged = 0;
    for (int d = 0; d < G; d++) {
      send_off[d] = (uint64_t)c->h_small[48 + d] * c->rb;
      send_cnt[d] = (uint64_t)(c->h_small[48 + d + 1] - c->h_small[48 + d]) * c->rb;
      recv_cnt[d] = (uint64_t)c->h_small[32 + d] * c->rb;
      recv_off[d + 1] = recv_off[d] + recv_cnt[d];
      if (d != me) st.bytes_exchanged += send_cnt[d];
    }
    rc = ensure_records(c, &c->recvbuf, &c->recv_cap, total_recv);
    if (rc) return rc;
    rc = ensure_out(c, total_recv);
    if (rc) return rc;
    if (nbig) {
      rc = ensure_records(c, &c->bigbuf, &c->big_cap, total_recv);
      if (rc) return rc;
    }
    // one grouped send/recv over NVLink replaces the GridFS / scp store-and-forward.  The rank's own
    // share never moves: the sort kernels read that segment in place from the send buffer.
    uint64_t net_send[8], net_recv[8];
    for (int d = 0; d < G; d++) {
      net_send[d] = d == me ? 0 : send_cnt[d];
      net_recv[d] = d == me ? 0 : recv_cnt[d];
    }
    rc = comm_alltoallv(c->comm, c->sb.mid, send_off, net_send, c->recvbuf, recv_off, net_recv, s, &c->err);
    if (rc) return rc;
    CU(c, cudaEventRecord(c->ev[EV_EXCH], s));
    v = c->sb;
    v.stride = 0;
    v.bin_off = c->d_outoff;
    v.src = c->recvbuf;
    v.mid = nbig ? c->bigbuf : c->recvbuf;
    v.nseg = (uint32_t)G;
    set_range_hint(c, v, S, ordered);
    for (int r = 0; r < G; r++) {
      v.seg_off[r] = c->d_segoff + (uint64_t)r * (Bl + 1);
      v.seg_base[r] = recv_off[r] / c->rb;
    }
    {
      // own segment: record offset of (send buffer + send_off[me]) relative to v.src, possibly "negative"
      // (two's complement; the kernels add it to the source pointer with 64-bit wrap-around).  Both
      // buffers come from cudaMalloc (>= 256-byte aligned), so the difference is a multiple of rb.
      const int64_t delta = (int64_t)((const char*)c->sb.mid - (const char*)c->recvbuf) + (int64_t)send_off[me];
      v.seg_base[me] = (uint64_t)(delta / (int64_t)c->rb);
    }
    st.launches += launch_sort_reduce(c->rb, v, (uint32_t)Bl, c->cap, c->sm_count, s);
    CU(c, cudaEventRecord(c->ev[EV_SORT], s));
    rc = exact_tail(c, v, Bl, nbig, st);
    if (rc) return rc;
    uint32_t ef = c->h_counters[CNT_ERR];
    rc = agree_flags(c, &ef);
    if (rc) return rc;
    if (ef & ERRF_SKEW) {
      uint64_t S_next = 0;
      if (widen < 4 && (rc = next_sub_bins(c, S, Bl, &S_next))) return rc;
      if (S_next) {
        S = (uint32_t)S_next;
        continue;
      }
      return fail(c, MRHBM_E_SKEW, "a bin holds more distinct keys than one SM can sort");
    }
    break;
  }
  return publish(c, v, Bl, S, ordered, N_in, total_recv, c->pbase[me] * S, nbig, st, ev_ms(c, EV_SCATTER, EV_EXCH),
                 ev_ms(c, EV_PLAN, EV_SCATTER));
}

// partition p -> local slot on this rank, or -1 when another rank owns it
inline int64_t slot_of(const mrhbm_ctx* c, uint32_t p) {
  return (p % (uint32_t)c->world) == (uint32_t)c->rank ? (int64_t)(p / (uint32_t)c->world) : -1;
}

}  // namespace

namespace {
// ---- the range partitioner's splitters ------------------------------------------------------------------------
// Checks the splitters (original bytes) and installs them with their device form (range_table, mrhbm_keys.h)
int install_splitters(mrhbm_ctx* c, std::vector<std::string>&& spl) {
  const uint32_t P = c->cfg.num_partitions;
  if (spl.size() != (size_t)P - 1)
    return fail(c, MRHBM_E_INVAL, "%u partitions need %u splitters, got %zu", P, P - 1, spl.size());
  const bool u64 = c->cfg.key_kind == MRHBM_KEY_U64;
  for (size_t i = 0; i < spl.size(); i++) {
    if (u64 && spl[i].size() != 8) return fail(c, MRHBM_E_INVAL, "u64 splitter %zu has %zu bytes (8 big-endian bytes)", i, spl[i].size());
    if (i && spl[i] < spl[i - 1]) return fail(c, MRHBM_E_INVAL, "splitters must be non-decreasing (splitter %zu < splitter %zu)", i, i - 1);
  }
  const RangeTable rt = range_table(spl, P, (size_t)c->kb);  // (never empty: P >= 1)
  if (c->d_spl) CU(c, cudaFree(c->d_spl));
  c->d_spl = nullptr;
  c->spl_set = false;
  CU(c, cudaMalloc(&c->d_spl, rt.image.size()));
  CU(c, cudaMemcpyAsync(c->d_spl, rt.image.data(), rt.image.size(), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  // digest (FNV-1a over the lengths and bytes): compared across ranks by the shuffle
  uint64_t d = 0xcbf29ce484222325ull;
  auto mixb = [&](unsigned char x) { d = (d ^ x) * 0x100000001b3ull; };
  for (const std::string& sp : spl) {
    for (int b = 0; b < 8; b++) mixb((unsigned char)(sp.size() >> (8 * b)));
    for (unsigned char x : sp) mixb(x);
  }
  c->spl = std::move(spl);
  c->spl_fin = rt.fin;
  c->spl_digest = d == ~0ull ? 0 : d;  // (all ones marks "none installed")
  c->spl_set = true;
  return MRHBM_OK;
}

int build_long_groups(mrhbm_ctx* c) {
  c->long_groups.clear();
  c->long_group_count = 0;
  c->long_vals.clear();
  c->long_sums.clear();
  const int G = c->world;
  // this rank's committed long pairs as one blob: {u32 key bytes, u64 value, key bytes padded to 4}*
  // (byte values, one GPU only: the value travels as its index in long_vals)
  std::vector<uint32_t> blob;
  for (auto& job : c->long_jobs)
    for (const LongPair& lp : job.second) {
      const size_t w0 = blob.size(), kw = (lp.esc.size() + 3) / 4;
      blob.resize(w0 + 3 + kw, 0u);
      blob[w0] = (uint32_t)lp.esc.size();
      uint64_t v = lp.value;
      if (c->bytevals) {
        v = c->long_vals.size();
        c->long_vals.push_back(&lp.bytes);
      }
      memcpy(&blob[w0 + 1], &v, 8);
      memcpy(&blob[w0 + 3], lp.esc.data(), lp.esc.size());
    }
  std::vector<uint32_t> all_blobs;
  std::vector<uint32_t> sizes(G, 0u);
  if (G == 1) {
    if (blob.empty()) return MRHBM_OK;
    sizes[0] = (uint32_t)blob.size();
    all_blobs.swap(blob);
  } else {  // COLLECTIVE, entered by all ranks or none (any_long travelled with the shuffle's error flags): sizes first,
            // then the blobs padded to the largest
    if (!c->any_long) return MRHBM_OK;
    if (blob.size() >= (1u << 28)) return fail(c, MRHBM_E_NOMEM, "more than 1 GB of long keys on one rank");
    const uint32_t words = (uint32_t)blob.size();
    int rc = gather_words(c, &words, 1, sizes.data());
    if (rc) return rc;
    uint32_t mx = 0;
    for (int r = 0; r < G; r++) mx = std::max(mx, sizes[r]);
    if (!mx) return MRHBM_OK;
    uint32_t *d_send = nullptr, *d_recv = nullptr;
    CU(c, cudaMalloc((void**)&d_send, (size_t)mx * 4));
    cudaError_t e = cudaMalloc((void**)&d_recv, (size_t)mx * 4 * G);
    if (e != cudaSuccess) {
      cudaFree(d_send);
      cudaGetLastError();
      return fail(c, MRHBM_E_NOMEM, "long keys: %s", cudaGetErrorString(e));
    }
    blob.resize(mx, 0u);
    all_blobs.resize((size_t)mx * G);
    e = cudaMemcpyAsync(d_send, blob.data(), (size_t)mx * 4, cudaMemcpyHostToDevice, c->stream);
    int rc2 = e == cudaSuccess ? comm_allgather_u32(c->comm, d_send, d_recv, mx, c->stream, &c->err) : 0;
    if (e == cudaSuccess && !rc2) e = cudaMemcpyAsync(all_blobs.data(), d_recv, (size_t)mx * 4 * G, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess && !rc2) e = cudaStreamSynchronize(c->stream);
    cudaFree(d_send);
    cudaFree(d_recv);
    if (rc2) return rc2;
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(c, MRHBM_E_CUDA, "long keys: %s", cudaGetErrorString(e));
    }
    // compact: rank r's blob starts at r * mx and holds sizes[r] words
    std::vector<uint32_t> packed;
    for (int r = 0; r < G; r++) packed.insert(packed.end(), all_blobs.begin() + (size_t)r * mx, all_blobs.begin() + (size_t)r * mx + sizes[r]);
    all_blobs.swap(packed);
  }
  // group the pairs of the partitions this rank owns (partition p lives on rank p % G, slot p / G)
  std::vector<std::map<std::string, std::vector<uint64_t>>> acc(c->Pl);
  const bool sum = !c->sb.no_reduce && !c->red_count;  // (count distinct: the value indices, counted below)
  for (size_t w = 0; w + 3 <= all_blobs.size();) {
    const uint32_t klen = all_blobs[w];
    uint64_t v;
    memcpy(&v, &all_blobs[w + 1], 8);
    std::string esc((const char*)&all_blobs[w + 3], klen);
    w += 3 + (klen + 3) / 4;
    const uint32_t pid = host_partition(c->cfg.partitioner, c->cfg.num_partitions, c->spl, esc);
    if ((int)(pid % (uint32_t)G) != c->rank) continue;
    const uint32_t slot = pid / (uint32_t)G;
    if (slot >= c->Pl) continue;
    std::vector<uint64_t>& vals = acc[slot][esc];
    if (sum && !vals.empty())
      vals[0] += v;
    else
      vals.push_back(v);
  }
  c->long_groups.resize(c->Pl);
  for (uint32_t sl = 0; sl < c->Pl; sl++)
    for (auto& kv : acc[sl]) {  // std::map iterates in ascending bytewise key order (unsigned char_traits compare)
      if (c->red_fsum) {  // the key's values summed with the kernels' accumulator, into one encoded number
        int64_t sum[kAccWords];
        acc_clear(sum);
        for (uint64_t i : kv.second) {
          uint64_t bits;
          const std::string& b = *c->long_vals[i];
          if (!num_decode((const unsigned char*)b.data(), b.size(), &bits))
            return fail(c, MRHBM_E_INVAL, "reducer MRHBM_RED_FSUM: a value of a long key is not a number");
          acc_add(sum, bits);
        }
        uint64_t bits;
        if (!acc_round(sum, &bits)) return fail(c, MRHBM_E_INVAL, "reducer MRHBM_RED_FSUM: a long key's sum is NaN (+inf and -inf)");
        std::string& e = c->long_sums.emplace_back(kNumBytes, '\0');
        num_encode(bits, (unsigned char*)&e[0]);
        kv.second.assign(1, c->long_vals.size());
        c->long_vals.push_back(&e);
      }
      if (c->red_count) {  // the number of the key's distinct value bytes, encoded as the device encodes it
        std::set<std::string> seen;
        for (uint64_t i : kv.second) seen.insert(*c->long_vals[i]);
        const double n = (double)seen.size();
        uint64_t bits;
        memcpy(&bits, &n, 8);
        std::string& e = c->long_sums.emplace_back(kNumBytes, '\0');
        num_encode(bits, (unsigned char*)&e[0]);
        kv.second.assign(1, c->long_vals.size());
        c->long_vals.push_back(&e);
      }
      if (c->red_distinct) {  // the key's distinct values, ascending by their bytes (std::string compares unsigned)
        std::vector<uint64_t>& vals = kv.second;
        auto bytes = [c](uint64_t i) -> const std::string& { return *c->long_vals[i]; };
        std::sort(vals.begin(), vals.end(), [&](uint64_t a, uint64_t b) { return bytes(a) < bytes(b); });
        vals.erase(std::unique(vals.begin(), vals.end(), [&](uint64_t a, uint64_t b) { return bytes(a) == bytes(b); }),
                   vals.end());
      }
      c->long_groups[sl].push_back(LongGroup{kv.first, std::move(kv.second)});
      c->long_group_count++;
    }
  return MRHBM_OK;
}

// After the device part of a shuffle: MRHBM_RED_FSUM's error flags (read back with the counters at its end), then the
// long keys.  A shuffle that fails here leaves no result.
int finish_shuffle(mrhbm_ctx* c) {
  int rc = 0;
  const uint32_t ef = c->red_fsum ? c->h_counters[CNT_ERR] : 0u;
  if (ef & ERRF_NOTNUM)
    rc = fail(c, MRHBM_E_INVAL, "reducer MRHBM_RED_FSUM: a value is not a number (11-byte encoding, tag 0x10)");
  else if (ef & ERRF_NAN)
    rc = fail(c, MRHBM_E_INVAL, "reducer MRHBM_RED_FSUM: a key's sum is NaN (+inf and -inf among its values)");
  else
    rc = build_long_groups(c);
  if (rc) invalidate(c);
  return rc;
}
}  // namespace

extern "C" {

int mrhbm_shuffle(mrhbm_ctx* c) {
  if (!c || !c->stream) return MRHBM_E_INVAL;
  Entry g(c);
  if (const std::string* job = c->led.open_job()) return fail(c, MRHBM_E_INVAL, "map job '%s' is still open", job->c_str());
  invalidate(c);
  uint64_t N_in = 0, N = 0;
  for (auto& r : c->led.live()) N_in += r.second;
  if (N_in >= 0xfffffff0ull) return fail(c, MRHBM_E_INVAL, "more than 2^32 pairs on one GPU (%llu)", (unsigned long long)N_in);
  if (c->red_fsum && N_in >= (1ull << 31))  // (each accumulator digit takes fewer than 2^31 addends)
    return fail(c, MRHBM_E_INVAL, "reducer MRHBM_RED_FSUM: a shuffle of %llu pairs (limit 2^31)", (unsigned long long)N_in);
  if (c->red_count && N_in >= (1ull << 31))  // (the distinct set's limit; every count is then exact in a double)
    return fail(c, MRHBM_E_INVAL, "reducer MRHBM_RED_COUNT_DISTINCT: a shuffle of %llu pairs (limit 2^31)", (unsigned long long)N_in);
  if (c->cfg.partitioner == MRHBM_PART_RANGE && c->world == 1 && !c->spl_set)  // (several GPUs: at the first all-gather)
    return fail(c, MRHBM_E_INVAL, "MRHBM_PART_RANGE needs splitters: call mrhbm_set_splitters or mrhbm_sample_splitters");
  mrhbm_stats st{};
  st.pairs = N_in;
  std::vector<Src> live;
  CU(c, cudaEventRecord(c->ev[EV_START], c->stream));
  int rc = collect_sources(c, live, &N, st);
  if (rc) return rc;
  CU(c, cudaEventRecord(c->ev[EV_CSTART], c->stream));
  if (!c->no_optimistic && !(c->cfg.flags & MRHBM_F_NO_OPTIMISTIC)) {
    bool done = false;
    rc = shuffle_fast(c, live, N, N_in, st, &done);
    if (rc) return rc;
    if (done) return finish_shuffle(c);
  }
  rc = c->world > 1 ? shuffle_multi_exact(c, live, N, N_in, st) : shuffle_single_exact(c, live, N, N_in, st);
  return rc ? rc : finish_shuffle(c);
}

int mrhbm_set_splitters(mrhbm_ctx* c, const void* keys, const uint64_t* off, size_t n) {
  if (!c || (n && (!keys || !off))) return MRHBM_E_INVAL;
  Entry g(c);
  if (c->cfg.partitioner != MRHBM_PART_RANGE) return fail(c, MRHBM_E_INVAL, "splitters need partitioner MRHBM_PART_RANGE");
  std::vector<std::string> spl(n);
  for (size_t i = 0; i < n; i++) {
    if (off[i + 1] < off[i]) return fail(c, MRHBM_E_INVAL, "splitter offsets must be non-decreasing");
    spl[i].assign((const char*)keys + off[i], off[i + 1] - off[i]);
  }
  return install_splitters(c, std::move(spl));
}

int mrhbm_sample_splitters(mrhbm_ctx* c, void* keys, size_t cap, uint64_t* off, size_t* need) {
  if (!c || !need) return MRHBM_E_INVAL;
  Entry g(c);
  if (c->cfg.partitioner != MRHBM_PART_RANGE) return fail(c, MRHBM_E_INVAL, "splitters need partitioner MRHBM_PART_RANGE");
  const int G = c->world, me = c->rank;
  const uint32_t P = c->cfg.num_partitions, KW = (uint32_t)c->kb / 4;
  const auto live = c->led.live();
  uint64_t N = 0;
  for (auto& r : live) N += r.second;
  // every rank's share of the sample follows its committed pairs (the same arithmetic on every rank)
  const uint32_t n32 = (uint32_t)std::min<uint64_t>(N, 0xffffffffull);
  uint32_t all[8];
  int rc = gather_words(c, &n32, 1, all);
  if (rc) return rc;
  uint64_t Ntot = 0;
  for (int r = 0; r < G; r++) Ntot += all[r];
  if (!Ntot) return fail(c, MRHBM_E_INVAL, "no committed pairs to sample splitters from");
  uint64_t m[8], mmax = 0, mtot = 0;
  for (int r = 0; r < G; r++) {
    m[r] = Ntot <= kSampleKeys ? all[r] : (uint64_t)(((unsigned __int128)kSampleKeys * all[r]) / Ntot);
    mmax = std::max(mmax, m[r]);
    mtot += m[r];
  }
  if (!mtot) return fail(c, MRHBM_E_INVAL, "no committed pairs to sample splitters from");
  const size_t words = (size_t)std::max<uint64_t>(mmax, 1) * KW;
  uint32_t* d_buf = nullptr;
  CU(c, cudaMalloc((void**)&d_buf, words * 4 * (G + 1)));
  uint32_t* d_recv = d_buf + words;
  std::vector<uint32_t> h((size_t)words * G);
  cudaError_t e = cudaMemsetAsync(d_buf, 0, words * 4, c->stream);
  // evenly spaced over this rank's committed ranges, m[me] keys in all
  uint64_t before = 0, taken = 0;
  for (auto& r : live) {
    const uint64_t upto = (uint64_t)(((unsigned __int128)m[me] * (before + r.second)) / N);
    launch_sample_keys(c->rb, (const char*)c->pool + r.first * c->rb, r.second, (uint32_t)(upto - taken), d_buf + taken * KW, c->stream);
    taken = upto;
    before += r.second;
  }
  if (e == cudaSuccess) e = cudaGetLastError();
  int rc2 = 0;
  if (e == cudaSuccess) {
    if (G > 1)
      rc2 = comm_allgather_u32(c->comm, d_buf, d_recv, words, c->stream, &c->err);
    else
      e = cudaMemcpyAsync(d_recv, d_buf, words * 4, cudaMemcpyDeviceToDevice, c->stream);
  }
  if (e == cudaSuccess && !rc2) e = cudaMemcpyAsync(h.data(), d_recv, words * 4 * G, cudaMemcpyDeviceToHost, c->stream);
  if (e == cudaSuccess && !rc2) e = cudaStreamSynchronize(c->stream);
  cudaFree(d_buf);
  if (rc2) return rc2;
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(c, MRHBM_E_CUDA, "splitter sample: %s", cudaGetErrorString(e));
  }
  // the sample in key order
  std::vector<const unsigned char*> smp;
  smp.reserve(mtot);
  for (int r = 0; r < G; r++)
    for (uint64_t i = 0; i < m[r]; i++) smp.push_back((const unsigned char*)(h.data() + (size_t)r * words + i * KW));
  const size_t kb = (size_t)c->kb;
  std::sort(smp.begin(), smp.end(), [kb](const unsigned char* a, const unsigned char* b) { return slot_cmp(a, b, kb) < 0; });
  std::vector<std::string> spl(P - 1);
  std::vector<unsigned char> raw;
  for (uint32_t i = 1; i < P; i++) {
    slot_key(smp[(size_t)(((unsigned __int128)i * mtot) / P)], kb, raw);
    spl[i - 1].assign(raw.begin(), raw.end());
  }
  size_t total = 0;
  for (auto& sp : spl) total += sp.size();
  *need = total;
  rc = install_splitters(c, std::move(spl));
  if (rc) return rc;
  if (keys && cap < total) return fail(c, MRHBM_E_INVAL, "the splitters need %zu bytes, the buffer holds %zu", total, cap);
  size_t o = 0;
  for (size_t i = 0; i < c->spl.size(); i++) {
    if (off) off[i] = o;
    if (keys) memcpy((char*)keys + o, c->spl[i].data(), c->spl[i].size());
    o += c->spl[i].size();
  }
  if (off) off[c->spl.size()] = o;
  return MRHBM_OK;
}

int mrhbm_stats_get(mrhbm_ctx* c, mrhbm_stats* out) {
  if (!c || !out) return MRHBM_E_INVAL;
  Entry g(c);
  *out = c->stats;
  return MRHBM_OK;
}

int mrhbm_partitions(mrhbm_ctx* c, uint32_t* ids, size_t cap, size_t* n) {
  if (!c || !n) return MRHBM_E_INVAL;
  Entry g(c);
  if (!c->shuffled) return fail(c, MRHBM_E_INVAL, "no shuffle result (call mrhbm_shuffle first)");
  size_t k = 0;
  for (uint32_t i = 0; i < c->Pl; i++) {
    const bool longs = i < c->long_groups.size() && !c->long_groups[i].empty();
    if (c->h_uoff[(uint64_t)(i + 1) * c->S] > c->h_uoff[(uint64_t)i * c->S] || longs) {
      if (ids && k < cap) ids[k] = (uint32_t)c->rank + i * (uint32_t)c->world;
      k++;
    }
  }
  *n = k;
  return MRHBM_OK;
}

int mrhbm_result_info_get(mrhbm_ctx* c, mrhbm_result_info* info) {
  if (!c || !info) return MRHBM_E_INVAL;
  Entry g(c);
  if (!c->shuffled) return fail(c, MRHBM_E_INVAL, "no shuffle result (call mrhbm_shuffle first)");
  size_t np = 0;
  mrhbm_partitions(c, nullptr, 0, &np);
  info->pairs_in = c->N;
  info->pairs_recv = c->N_recv;
  info->groups = c->groups;
  info->key_bytes = (uint32_t)c->kb;
  info->sorted = (c->ordered || c->S == 1) ? 1 : 0;
  info->runs_per_partition = c->S;
  info->partitions_nonempty = (uint32_t)np;
  return MRHBM_OK;
}

int mrhbm_result_copy(mrhbm_ctx* c, void* keys, uint64_t* sums, uint64_t* part_off) {
  if (!c) return MRHBM_E_INVAL;
  Entry g(c);
  if (c->bytevals && sums) return fail(c, MRHBM_E_INVAL, "byte values: result_copy takes sums = NULL (see mrhbm_result_values)");
  int rc = ensure_compact(c);
  if (rc) return rc;
  if (c->long_group_count)
    return fail(c, MRHBM_E_KEY, "%llu groups have keys longer than the %d-byte slots of mrhbm_result_copy: iterate with mrhbm_groups_*",
                (unsigned long long)c->long_group_count, c->kb);
  if (keys && c->groups) CU(c, cudaMemcpyAsync(keys, c->ckeys, c->groups * c->kb, cudaMemcpyDeviceToHost, c->stream));
  if (sums && c->groups) CU(c, cudaMemcpyAsync(sums, c->csums, c->groups * 8, cudaMemcpyDeviceToHost, c->stream));
  if (part_off)
    for (uint32_t p = 0; p <= c->cfg.num_partitions; p++) {
      // groups of the owned partitions with id < p (other ranks' partitions are empty ranges here)
      uint64_t slots = p <= (uint32_t)c->rank ? 0 : ((uint64_t)p - c->rank + c->world - 1) / c->world;
      part_off[p] = c->h_uoff[std::min<uint64_t>(slots, c->Pl) * c->S];
    }
  CU(c, cudaStreamSynchronize(c->stream));
  return MRHBM_OK;
}

int mrhbm_result_values(mrhbm_ctx* c, void* vals, size_t cap, uint64_t* row_off, size_t* need) {
  if (!c || !need || (vals && !row_off)) return MRHBM_E_INVAL;
  Entry g(c);
  if (!c->bytevals) return refuse_byte_values(c);
  int rc = ensure_compact(c);
  if (rc) return rc;
  if (c->long_group_count)
    return fail(c, MRHBM_E_KEY, "%llu groups have keys longer than the %d-byte slots of mrhbm_result_copy: iterate with mrhbm_groups_*",
                (unsigned long long)c->long_group_count, c->kb);
  *need = (size_t)c->cvals_bytes;
  if (!vals) return MRHBM_OK;
  if (cap < c->cvals_bytes) return fail(c, MRHBM_E_INVAL, "the values need %llu bytes, the buffer holds %zu", (unsigned long long)c->cvals_bytes, cap);
  if (c->cvals_bytes) CU(c, cudaMemcpyAsync(vals, c->cvals, c->cvals_bytes, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(row_off, c->row_off, (c->groups + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return MRHBM_OK;
}

int mrhbm_checksum_input(mrhbm_ctx* c, uint64_t in[4]) {
  if (!c || !in) return MRHBM_E_INVAL;
  Entry g(c);
  CU(c, cudaMemsetAsync(c->d_acc, 0, 8 * sizeof(uint64_t), c->stream));
  for (auto& r : c->led.live()) launch_checksum_in(c->rb, (char*)c->pool + r.first * c->rb, r.second, c->d_acc, c->stream);
  CU(c, cudaGetLastError());
  CU(c, cudaMemcpyAsync(c->h_acc, c->d_acc, 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  memcpy(in, c->h_acc, 4 * sizeof(uint64_t));
  return MRHBM_OK;
}

int mrhbm_checksum_result(mrhbm_ctx* c, uint64_t out[6]) {
  if (!c || !out) return MRHBM_E_INVAL;
  Entry g(c);
  if (!c->shuffled) return fail(c, MRHBM_E_INVAL, "no shuffle result (call mrhbm_shuffle first)");
  if (c->cfg.partitioner == MRHBM_PART_RANGE && c->spl_digest != c->shuffle_spl_digest)
    return fail(c, MRHBM_E_INVAL, "the splitters changed after the shuffle: its partitions cannot be checked against them");
  CU(c, cudaMemsetAsync(c->d_acc, 0, 8 * sizeof(uint64_t), c->stream));
  launch_checksum_out(c->rb, c->rv, c->B, make_bp(c, c->S, c->ordered), c->bin_base, c->d_acc, c->stream);
  CU(c, cudaGetLastError());
  CU(c, cudaMemcpyAsync(c->h_acc, c->d_acc, 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  memcpy(out, c->h_acc, 6 * sizeof(uint64_t));
  return MRHBM_OK;
}

// ---------------------------------------------------------------------------
// reduce side iteration
// ---------------------------------------------------------------------------
// k-way merge of the partition's ascending runs (utils.lua:206-271 merges spill files the same way): a binary heap of
// run indices ordered by the key each run stands on (ties: lower run first)
static inline bool run_less(const mrhbm_iter* it, uint32_t a, uint32_t b) {
  const mrhbm_ctx* c = it->ctx;
  const int x = slot_cmp(&it->keys[it->runs[a].pos * c->kb], &it->keys[it->runs[b].pos * c->kb], c->kb);
  return x < 0 || (x == 0 && a < b);
}
static inline void heap_sift_down(mrhbm_iter* it, size_t i) {
  std::vector<uint32_t>& h = it->heap;
  const size_t n = h.size();
  for (;;) {
    const size_t l = 2 * i + 1, r = l + 1;
    size_t m = i;
    if (l < n && run_less(it, h[l], h[m])) m = l;
    if (r < n && run_less(it, h[r], h[m])) m = r;
    if (m == i) return;
    std::swap(h[i], h[m]);
    i = m;
  }
}
// the run at the top moved on (or ran dry): restore the heap
static inline void heap_fix_top(mrhbm_iter* it) {
  std::vector<uint32_t>& h = it->heap;
  if (it->runs[h[0]].pos >= it->runs[h[0]].end) {
    h[0] = h.back();
    h.pop_back();
  }
  if (!h.empty()) heap_sift_down(it, 0);
}

int mrhbm_groups_open(mrhbm_ctx* c, uint32_t part, mrhbm_iter** out) {
  if (!c || !out) return MRHBM_E_INVAL;
  Entry g(c);
  if (part >= c->cfg.num_partitions) return fail(c, MRHBM_E_INVAL, "partition %u out of range", part);
  int rc = ensure_compact(c);
  if (rc) return rc;
  int64_t slot = slot_of(c, part);
  if (slot < 0) return fail(c, MRHBM_E_INVAL, "partition %u is owned by rank %u", part, part % (uint32_t)c->world);
  mrhbm_iter* it = new mrhbm_iter();
  it->ctx = c;
  it->unesc.reserve(c->kb);
  uint64_t b0 = (uint64_t)slot * c->S;
  uint64_t lo = c->h_uoff[b0], hi = c->h_uoff[b0 + c->S];
  it->base = lo;
  it->keys.resize((hi - lo) * c->kb);
  it->sums.resize(hi - lo);
  if (hi > lo) {
    cudaError_t e = cudaMemcpyAsync(it->keys.data(), (char*)c->ckeys + lo * c->kb, (hi - lo) * c->kb, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(it->sums.data(), c->csums + lo, (hi - lo) * 8, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess && c->bytevals) {  // the partition's row offsets, then its value bytes
      it->roff.resize(hi - lo + 1);
      e = cudaMemcpyAsync(it->roff.data(), c->row_off + lo, (hi - lo + 1) * 8, cudaMemcpyDeviceToHost, c->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
      if (e == cudaSuccess) {
        const uint64_t v0 = it->roff[0], nb = it->roff[hi - lo] - v0;
        for (uint64_t& o : it->roff) o -= v0;
        it->vbytes.resize(nb);
        if (nb) e = cudaMemcpyAsync(it->vbytes.data(), c->cvals + v0, nb, cudaMemcpyDeviceToHost, c->stream);
      }
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) {
      delete it;
      cudaGetLastError();
      return fail(c, MRHBM_E_CUDA, "groups_open: %s", cudaGetErrorString(e));
    }
  }
  if ((uint64_t)slot < c->long_groups.size() && !c->long_groups[(size_t)slot].empty()) it->longs = &c->long_groups[(size_t)slot];
  it->sorted = (c->ordered || c->S == 1) && c->h_big.empty();
  if (it->sorted) {
    it->runs.push_back(RunCursor{0, hi - lo});
  } else {
    for (uint32_t r = 0; r < c->S; r++) {
      uint64_t a = c->h_uoff[b0 + r] - lo, b = c->h_uoff[b0 + r + 1] - lo;
      if (b <= a) continue;
      bool big = std::find(c->h_big.begin(), c->h_big.end(), (uint32_t)(b0 + r)) != c->h_big.end();
      if (!big) {
        it->runs.push_back(RunCursor{a, b});
      } else {  // group-only mode: an oversized bin is a sequence of ascending runs of cap rows
        for (uint64_t q = a; q < b; q += c->cap) it->runs.push_back(RunCursor{q, std::min<uint64_t>(q + c->cap, b)});
      }
    }
  }
  for (uint32_t r = 0; r < it->runs.size(); r++)
    if (it->runs[r].pos < it->runs[r].end) it->heap.push_back(r);
  for (size_t i = it->heap.size() / 2; i-- > 0;) heap_sift_down(it, i);
  *out = it;
  return MRHBM_OK;
}

// The next group of the iteration into it->unesc (its original key bytes) and either *lg (a key longer than a slot)
// or it->rows (its device rows).  1 = one group, 0 = end.
static int next_group(mrhbm_iter* it, const LongGroup** lg) {
  mrhbm_ctx* c = it->ctx;
  *lg = nullptr;
  // k-way merge over the ascending runs of the partition (a single run when sorted): the smallest key is on top
  const int best = it->heap.empty() ? -1 : (int)it->heap[0];
  if (it->longs && it->long_pos < it->longs->size()) {
    // a key longer than a slot comes next when it sorts before the smallest device key
    const LongGroup& g = (*it->longs)[it->long_pos];
    bool take = best < 0;
    if (!take) {
      const unsigned char* dk = &it->keys[it->runs[best].pos * c->kb];
      take = esc_cmp((const unsigned char*)g.esc.data(), g.esc.size(), dk, slot_esc_len(dk, c->kb)) < 0;
    }
    if (take) {
      it->long_pos++;
      unescape(g.esc.data(), g.esc.size(), it->unesc);
      *lg = &g;
      return 1;
    }
  }
  if (best < 0) return 0;
  uint64_t i = it->runs[best].pos++;
  const unsigned char* k = &it->keys[i * c->kb];
  it->rows.clear();
  it->rows.push_back(i);
  if (c->sb.no_reduce) {
    // every row of this key: adjacent in its run, and -- for an oversized bin -- at the head of
    // sibling runs too
    for (;;) {  // the run on top, then whichever run comes to the top with the same key
      RunCursor& rc = it->runs[it->heap[0]];
      while (rc.pos < rc.end && slot_cmp(&it->keys[rc.pos * c->kb], k, c->kb) == 0) it->rows.push_back(rc.pos++);
      heap_fix_top(it);
      if (it->heap.empty()) break;
      const RunCursor& top = it->runs[it->heap[0]];
      if (slot_cmp(&it->keys[top.pos * c->kb], k, c->kb) != 0) break;
    }
  } else {
    heap_fix_top(it);
  }
  slot_key(k, c->kb, it->unesc);
  return 1;
}

int mrhbm_groups_next(mrhbm_iter* it, const void** key, size_t* klen, const uint64_t** values, size_t* nvalues) {
  if (!it || !key || !klen || !values || !nvalues) return MRHBM_E_INVAL;
  mrhbm_ctx* c = it->ctx;
  if (c->bytevals) return fail(c, MRHBM_E_INVAL, "the ctx carries byte values (MRHBM_F_BYTE_VALUES): use mrhbm_groups_next_values");
  const LongGroup* lg;
  const int r = next_group(it, &lg);
  if (r <= 0) return r;
  *key = it->unesc.data();
  *klen = it->unesc.size();
  if (lg) {
    *values = lg->values.data();
    *nvalues = lg->values.size();
  } else if (c->cfg.reducer == MRHBM_RED_NONE) {
    it->valbuf.clear();
    for (uint64_t row : it->rows) it->valbuf.push_back(it->sums[row]);
    *values = it->valbuf.data();
    *nvalues = it->valbuf.size();
  } else {
    *values = &it->sums[it->rows[0]];
    *nvalues = 1;
  }
  return 1;
}

int mrhbm_groups_next_values(mrhbm_iter* it, const void** key, size_t* klen, const void** vals, const uint64_t** voff,
                             size_t* nvalues) {
  if (!it || !key || !klen || !vals || !voff || !nvalues) return MRHBM_E_INVAL;
  mrhbm_ctx* c = it->ctx;
  if (!c->bytevals) return refuse_byte_values(c);
  const LongGroup* lg;
  const int r = next_group(it, &lg);
  if (r <= 0) return r;
  it->vout.clear();
  it->vout_off.assign(1, 0);
  auto add = [&](const unsigned char* p, uint64_t n) {
    it->vout.insert(it->vout.end(), p, p + n);
    it->vout_off.push_back(it->vout.size());
  };
  if (lg) {
    for (uint64_t v : lg->values) add((const unsigned char*)c->long_vals[v]->data(), c->long_vals[v]->size());
  } else {
    for (uint64_t row : it->rows) add(it->vbytes.data() + it->roff[row], it->roff[row + 1] - it->roff[row]);
  }
  it->vout.reserve(1);  // (a valid pointer for a group of empty values)
  *key = it->unesc.data();
  *klen = it->unesc.size();
  *vals = it->vout.data();
  *voff = it->vout_off.data();
  *nvalues = it->vout_off.size() - 1;
  return 1;
}

void mrhbm_groups_close(mrhbm_iter* it) { delete it; }

// ---------------------------------------------------------------------------
// multi-GPU
// ---------------------------------------------------------------------------
int mrhbm_comm_unique_id(mrhbm_ctx* c, void* id) {
  if (!c || !id) return MRHBM_E_INVAL;
  return comm_unique_id(id, &c->err);
}
int mrhbm_comm_init(mrhbm_ctx* c, const void* id, int rank, int world) {
  if (!c || !id || world < 1 || rank < 0 || rank >= world) return MRHBM_E_INVAL;
  Entry g(c);
  // (before any communicator exists: the value ids are pool indices of this rank only)
  if (c->bytevals && world > 1) return fail(c, MRHBM_E_INVAL, "byte values (MRHBM_F_BYTE_VALUES) run on one GPU");
  if (world > 8) return fail(c, MRHBM_E_INVAL, "at most 8 ranks (one NVSwitch box)");
  if (c->world != 1) return fail(c, MRHBM_E_INVAL, "communicator already initialised");
  if (world == 1) return MRHBM_OK;
  int rc = comm_create(&c->comm, id, rank, world, c->dev, &c->err);
  if (rc) return rc;
  c->world = world;
  c->rank = rank;
  const uint32_t P = c->cfg.num_partitions;
  c->pbase[0] = 0;
  for (int r = 0; r < 8; r++) {
    uint32_t owned = r < world && (uint32_t)r < P ? (P - (uint32_t)r + (uint32_t)world - 1) / (uint32_t)world : 0;
    c->pbase[r + 1] = c->pbase[r] + owned;
  }
  c->Pl = c->pbase[rank + 1] - c->pbase[rank];
  CU(c, cudaMalloc((void**)&c->d_ipc, 16 * 9 * sizeof(uint32_t)));
  CU(c, cudaHostAlloc((void**)&c->h_ipc, 16 * 9 * sizeof(uint32_t), cudaHostAllocDefault));
  invalidate(c);
  return MRHBM_OK;
}

}  // extern "C"
