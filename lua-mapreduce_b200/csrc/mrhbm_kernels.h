// mrhbm_kernels.h -- host-callable launchers of the sm_90a kernels (internal, C++).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace mrhbm {

#ifdef __CUDACC__
#define MRHBM_HD __host__ __device__
#else
#define MRHBM_HD
#endif

struct BinParams {
  uint32_t P;            // partitions
  uint32_t S;            // sub-bins per partition
  uint32_t partitioner;  // MRHBM_PART_*
  uint32_t ordered;      // 1: sub-bin = top key bits (partition becomes one ascending run)
                         // 0: sub-bin = further hash bits (partition = S ascending runs)
  uint32_t ctr_shift;    // hist / cursor counters live at index bin << ctr_shift: the L2
                         // atomic unit serialises per 32 B sector, so counters are spread out
  // multi-GPU: partition p is owned by rank p % world and sits in slot pbase[p % world] + p / world,
  // so that the bins of one destination rank are contiguous (its all-to-all send region)
  uint32_t world;        // 1 = single GPU (slot == p)
  uint32_t wshift;       // log2(world) when world is a power of two, else 0xffffffff
  uint32_t pbase[9];
};
// MRHBM_PART_RANGE: the kernel instances compiled for it take this larger block (the hash instances keep BinParams, so
// their parameter layout and code do not change).  The spl_n finite thresholds t_i, ascending, with
// key >= splitter i  <=>  slot(key) >= t_i as big-endian numbers (see range_table in mrhbm_keys.h).
struct RangeBinParams : BinParams {
  const unsigned long long* spl_pre;  // [spl_n] the first 8 bytes of t_i, big endian (u64 keys: the splitter itself)
  const uint32_t* spl_slot;           // [spl_n * key words] t_i as a zero-padded key slot (strings only)
  const ulonglong2* spl_inv;          // [P] u64 keys: floor((2^128 - 1) / width of partition p) as {high, low} 64
                                      // bits, 0 when the partition is empty (see range_pos)
  uint32_t spl_n;                     // finite thresholds (splitters above every slot key are left out)
  uint32_t spl_top;                   // largest power of two <= spl_n (0 when spl_n = 0)
};
constexpr uint32_t kPartRange = 3;  // MRHBM_PART_RANGE

MRHBM_HD inline uint32_t partition_slot(const BinParams& bp, uint32_t pid) {
  return bp.world > 1 ? bp.pbase[pid % bp.world] + pid / bp.world : pid;
}

constexpr int kSplitTileBytes = 40 * 1024;  // bytes of records k_split_tma partitions in shared memory at a time
constexpr uint32_t kSplitMaxBins = 1024;    // bins one level of k_split_tma distinguishes
constexpr int kCapBytes = 32 * 1024;  // record bytes one CTA sorts in shared memory (2 CTAs per SM)
inline uint32_t cap_records(int rb) { return (uint32_t)(kCapBytes / rb); }

struct ShuffleBuffers {
  // all device pointers
  uint32_t* hist;      // [B]
  uint32_t* bin_off;   // [B+1] exclusive scan of hist
  uint32_t* cursor;    // [B]   scatter cursors (start = bin_off)
  uint32_t* ucount;    // [B]   groups per bin after sort+reduce
  uint32_t* uoff;      // [B+1] exclusive scan of ucount
  uint32_t* big_list;  // [B]   bins larger than cap
  uint32_t* counters;  // [8]: 0 = nbig, 1 = ticket, 2 = error flags, 3 = total
  void* mid;           // scattered records, N * RB
  void* out_keys;      // N * key_bytes (runs at bin_off)
  uint64_t* out_sums;  // N
  // Where the records of bin b live: nseg segments, segment s holds
  // seg_off[s][b+1]-seg_off[s][b] records at src + (seg_base[s] + seg_off[s][b]) records.
  // Single GPU: one segment == the scattered buffer (seg_off[0] = bin_off).  After the
  // all-to-all: one segment per source rank inside the receive buffer.
  const void* src;
  uint32_t nseg;
  const uint32_t* seg_off[8];
  uint64_t seg_base[8];
  // Optimistic single-pass layout (no histogram pass): bin b owns the fixed slots
  // [b*stride, (b+1)*stride) of mid / out and its fill level is its scatter cursor.
  uint32_t stride;     // 0 = exact layout through bin_off
  uint32_t out_stride; // optimistic layout: the groups of bin b start at out slot b * out_stride (<= stride: a
                       // duplicate-heavy bin holds many records but at most one CTA's worth of distinct keys)
  uint32_t ctr_shift;  // cursor[b << ctr_shift]
  // key-ordered sub-bins of u64 keys (sub = mulhi(key, S)): lets the sort kernel skip the
  // min/max pass.  hint_S = 0: unknown.
  uint32_t hint_S;
  uint64_t hint_q;     // floor(2^64 / S)
  uint32_t no_reduce;  // MRHBM_RED_NONE: every pair is its own output row (sorted, grouped on the host)
};
MRHBM_HD inline uint64_t bin_start(const ShuffleBuffers& b, uint32_t bin) {
  return b.stride ? (uint64_t)bin * b.stride : (uint64_t)b.bin_off[bin];
}
MRHBM_HD inline uint64_t out_start(const ShuffleBuffers& b, uint32_t bin) {
  return b.stride ? (uint64_t)bin * b.out_stride : (uint64_t)b.bin_off[bin];
}
MRHBM_HD inline uint32_t bin_count(const ShuffleBuffers& b, uint32_t bin) {
  if (b.stride) {
    uint32_t c = b.cursor[(size_t)bin << b.ctr_shift];
    return c < b.stride ? c : b.stride;
  }
  return b.bin_off[bin + 1] - b.bin_off[bin];
}
enum { CNT_NBIG = 0, CNT_TICKET = 1, CNT_ERR = 2, CNT_TOTAL = 3, CNT_GBIG = 4 };
// ERRF_NOTNUM / ERRF_NAN (MRHBM_RED_FSUM): a value that is not a number encoding, a key whose sum is NaN
// ERRF_LINE (mrhbm_map_key_numbers): a line that is not "key number"
enum { ERRF_SKEW = 1, ERRF_OVERFLOW = 2, ERRF_CAPACITY = 4, ERRF_KEYLEN = 8, ERRF_NOTNUM = 16, ERRF_NAN = 32, ERRF_LINE = 64 };

// every launcher returns the number of kernels it launched
int launch_gen_u64(void* dst, uint64_t seed, uint64_t start, uint64_t n, cudaStream_t s);
int launch_gen_zipf32(void* dst, uint64_t seed, uint64_t start, uint64_t n, const uint64_t* d_table,
                      uint64_t V, cudaStream_t s);
int launch_hist(int rb, const void* recs, uint64_t n, const RangeBinParams& bp, uint32_t* hist, cudaStream_t s);
// exclusive scan of in[i << shift], i < n: out_excl[n+1]; optional copies: out_copy[i << shift] (scatter
// cursors), out_dense[i] (the counts, densely packed), entries > cap appended to big_list
// scratch: kScanScratchWords words for the multi-CTA variant (nullptr: single CTA)
constexpr uint32_t kScanScratchWords = 4096;
int launch_exscan(const uint32_t* in, uint32_t n, uint32_t* out_excl, uint32_t* out_copy,
                  uint32_t* out_dense, uint32_t cap, uint32_t* big_list, uint32_t* nbig, uint32_t* total,
                  uint32_t shift, cudaStream_t s, uint32_t* scratch = nullptr);
// histogram of the top 8 key bits of `nsample` evenly spaced u64 records (hist256 += counts)
int launch_sample_u64(const void* recs, uint64_t n, uint32_t nsample, uint32_t* hist256, cudaStream_t s);
// MRHBM_PART_RANGE, u64 keys: the same sample, histogram of the top 8 bits of each key's position inside its partition
int launch_sample_range_u64(const void* recs, uint64_t n, uint32_t nsample, const RangeBinParams& bp, uint32_t* hist256,
                            cudaStream_t s);
// key slots (kKeyWords words each) of `nsample` evenly spaced records to out (splitter sampling)
int launch_sample_keys(int rb, const void* recs, uint64_t n, uint32_t nsample, uint32_t* out, cudaStream_t s);
int launch_scatter(int rb, const void* recs, uint64_t n, const RangeBinParams& bp, uint32_t* cursor, void* mid,
                   cudaStream_t s);
// device-side tokeniser: word starts per 256-byte block, then (after an exclusive scan of the
// block counts) one record (word, value) per word; *flags gets ERRF_KEYLEN when a word exceeds the key slot
int launch_tok_count(const unsigned char* text, uint64_t len, uint32_t* block_counts, cudaStream_t s);
int launch_tok_emit(int rb, const unsigned char* text, uint64_t len, const uint32_t* block_off, void* recs,
                    uint32_t value, uint32_t* flags, cudaStream_t s);
inline uint64_t tok_blocks(uint64_t len) { return (len + 255) / 256; }
// device-side key-number mapfn: first fields of lines per 256-byte block, then (after the same exclusive scan) one
// record (key, value id first + i) and one 11-byte number per line.  flags[0] |= ERRF_KEYLEN for a key that exceeds
// the key slot, ERRF_LINE for a malformed line, flags[1] = min over malformed lines of their start, flags[2] = the
// tokens the host must round (the first fix_cap of them in fix[]: {pair index, token offset, token length, 0})
struct KnOut {
  uint4* recs;           // the piece's records
  unsigned char* vals;   // arena + aoff: the piece's values, 11 bytes each
  uint64_t* voff;        // voff + first
  uint64_t first, aoff;  // the piece's first pool index and arena offset
  const uint64_t* pow5;  // dec_pow5_table
  uint4* fix;
  uint32_t fix_cap;
  uint32_t* flags;
};
int launch_kn_count(const unsigned char* text, uint64_t len, uint32_t* block_counts, cudaStream_t s);
int launch_kn_emit(int rb, const unsigned char* text, uint64_t len, const uint32_t* block_off, const KnOut& o,
                   cudaStream_t s);
// fix[i] = {pair index, double bits}: the number's 11 bytes at vals + 11 * pair index
int launch_kn_patch(const void* fix, uint32_t n, unsigned char* vals, cudaStream_t s);
// The map-side combiner's global table for records of rb bytes: `nbuckets` buckets of one 32-byte L2 sector each,
// two 16-byte short entries per bucket, then, for string records only, 2^long_log long entries of one record each.
// A short key probes buckets linearly from bucket(hash), wrapping at nbuckets (not a power of two: the table is
// sized to the keys).  The compaction emits at most one record per entry.
struct GtabLayout {
  int rb;
  uint32_t nbuckets;  // a multiple of 16, so that short and long entries each fill whole warps of the compaction
  uint32_t long_log;
  // The size a shuffle starts at, and after `grow` tables that filled up (each doubles both parts).  25 MB of
  // buckets: 1.64 M short entries, load 0.64 on config 3's 1.05 M keys.  On config 3 (H100 SXM, 700 W) k_combine
  // took 14.72 ms with 20 MB (load 0.8: longer chains), 14.38-14.43 from 23 to 28 MB, 14.59 with 32 MB and 16.03
  // with 48 MB (the table no longer stays in L2 beside the pair stream; DESIGN §4.4).  2^15 long entries: keys of
  // more than 12 bytes are 0.64 % of config 3's pairs, ~16 K distinct keys.
  static constexpr uint32_t kBuckets = 819200, kLongLog = 15, kMaxGrow = 6;
  // Bucket probes of a short key before the table counts as full (and grows).  In a CPU model of linear probing with
  // uniform hashes over 819,200 two-entry buckets, no key moved more than 132 buckets from its home at load 0.8,
  // 239 at 0.85 and 560 at 0.9: a table below 0.8 never reports full, one above 0.9 does.  Fuller tables cost more
  // than a retry: at load 0.92, 2^24 pairs over 1.5 M keys took k_combine 2.64 ms against 1.46 ms with the earlier
  // 32 MB table (DESIGN §4.4).
  static constexpr uint32_t kMaxProbes = 256;
  static MRHBM_HD GtabLayout sized(int rb, uint32_t grow) { return GtabLayout{rb, kBuckets << grow, kLongLog + grow}; }
  MRHBM_HD uint32_t nshort() const { return 2u * nbuckets; }
  MRHBM_HD uint32_t nlong() const { return rb == 16 ? 0u : 1u << long_log; }
  MRHBM_HD uint64_t long_offset() const { return (uint64_t)32 * nbuckets; }  // bytes
  MRHBM_HD uint64_t bytes() const { return long_offset() + (uint64_t)rb * nlong(); }
  MRHBM_HD uint32_t records() const { return nshort() + nlong(); }
  // the home bucket of a 32-bit key hash (its top bits, scaled to nbuckets), and the bucket `probe` steps after it
  // (probe < nbuckets)
  MRHBM_HD uint32_t bucket(uint32_t h) const { return (uint32_t)(((uint64_t)h * nbuckets) >> 32); }
  MRHBM_HD uint32_t bucket_at(uint32_t home, uint32_t probe) const {
    const uint32_t b = home + probe;
    return b >= nbuckets ? b - nbuckets : b;
  }
  // the home entry of a long key's 32-bit hash, and the entry after e
  MRHBM_HD uint32_t long_slot(uint32_t h) const { return h >> (32 - long_log); }
  MRHBM_HD uint32_t long_next(uint32_t e) const { return (e + 1) & (nlong() - 1u); }
};
// Largest sum (and so largest value) a combined string record carries in its u32 value: the table keeps sum + 1,
// and all ones marks an entry being written.
constexpr uint32_t kMaxCombinedSum = 0xffffffefu;
// map-side combine of one committed range into the global table gtab (tab.bytes(), 32-byte aligned, zeroed by the
// caller); flags[0] |= ERRF_SKEW when the table is full, ERRF_OVERFLOW when a u32 sum would pass kMaxCombinedSum
// (checked mode only: unchecked adds are fire-and-forget and the caller verifies afterwards that pairs x flags[2],
// the largest value seen, stays within it)
int launch_combine(const void* recs, uint64_t n, uint32_t* gtab, const GtabLayout& tab, uint32_t* flags, bool checked,
                   int sm_count, cudaStream_t s);
// one record per non-empty table entry appended to out; *count (zeroed by the caller) += entries
int launch_gtab_compact(const uint32_t* gtab, const GtabLayout& tab, void* out, uint32_t* count, cudaStream_t s);
// tot[b] = sum over s < world of all[s * stride + base + b], b < n; *nover += bins (of all `stride`
// bins) whose global total exceeds cap
int launch_sum_src(const uint32_t* all, uint32_t world, uint32_t stride, uint32_t base, uint32_t n,
                   uint32_t* tot, uint32_t cap, uint32_t* nover, cudaStream_t s);
// row r < world: out[r*(n+1) ..] = exclusive scan of all[r*stride + base ..+n), totals[r] = its sum
// acc2[0] = sum over source ranks z < G and regions r in [first, first+nreg) of min(counts[z*zstride + (r << shift)], clamp),
// acc2[1] = the z == me part of it
int launch_region_totals(const uint32_t* counts, uint64_t zstride, uint32_t G, uint32_t me, uint32_t first, uint32_t nreg,
                         uint32_t shift, uint32_t clamp, uint64_t* acc2, cudaStream_t s);
int launch_exscan_rows(const uint32_t* all, uint32_t world, uint32_t stride, uint32_t base, uint32_t n,
                       uint32_t* out, uint32_t* totals, cudaStream_t s);
// Two-level coalesced split, as the host plans it and k_split_tma reads it: the kernel takes this block as it is,
// with the level and (level 1) its source records, and derives each level's destination, stride, cursor and
// capacity from it.  Optimistic layout (base_off == nullptr): level 1 sends every record to the coarse region of
// its bin inside this rank's region buffer l1 (all C1 regions of the job, sub_stride slots each); level 2 of the
// rank that owns region y pulls it from every rank's buffer (peer[z], NVLink) and splits it into fine bins of `cap`
// slots in mid.  C1 == B, F == 1 on one GPU with few bins = single level straight into mid.
// Exact layout (base_off = bin offsets after k_hist + k_exscan): both levels write absolute slots into ONE
// destination (on several GPUs the destination-major send buffer): ndest = 1, me = 0.
struct SplitPlan {
  uint32_t B;                 // fine bins (of the whole job)
  uint32_t F;                 // fine bins per coarse region (power of two)
  uint32_t C1;                // coarse regions of the whole job (bins level 1 distinguishes, <= kSplitMaxBins)
  uint32_t C1_local;          // regions this rank owns (level 2 splits these)
  uint32_t cap;               // slots per fine bin (optimistic)
  uint64_t sub_stride;        // slots per coarse region in a rank's region buffer (exact layout: F * cap, what the
                              // level-2 grid is sized by)
  uint32_t* cursor1;          // level-1 fill levels, [C1 << ctr_shift]
  uint32_t* cursor;           // fine fill levels, [B_local << ctr_shift]
  void* l1;                   // this rank's region buffer: C1 * sub_stride records
  void* mid;                  // fine bins
  uint32_t* err_flags;
  const uint32_t* base_off;
  uint32_t ndest, me;         // ranks, this rank (1, 0 on a single GPU)
  unsigned long long peer[8]; // byte address of every rank's region buffer as mapped into this process
  // rank d owns the coarse regions [rbase[d], rbase[d+1]) = its fine bins [fbase[d], fbase[d+1]) in blocks of F
  uint32_t rbase[9], fbase[9];
  const uint32_t* l1_counts;  // level 2: fill of region r on rank z at l1_counts[z * l1_zstride + (r << ctr_shift)]
  uint64_t l1_zstride;
  uint32_t ctr_shift;         // spacing of the fill levels above (BinParams::ctr_shift)
  uint32_t* ticket;          // two zeroed words: level 1 hands out its tiles from a counter (the kernel zeroes them again)
};
int launch_split_l1(int rb, const void* recs, uint64_t n, const RangeBinParams& bp, const SplitPlan& pl, cudaStream_t s);
int launch_split_l2(int rb, const RangeBinParams& bp, const SplitPlan& pl, cudaStream_t s);
int launch_sort_reduce(int rb, const ShuffleBuffers& b, uint32_t B, uint32_t cap, int sm_count,
                       cudaStream_t s);
int launch_big_bins(int rb, const ShuffleBuffers& b, uint32_t nbig, uint32_t cap, cudaStream_t s);
int launch_compact(int rb, const ShuffleBuffers& b, uint32_t B, void* dst_keys, uint64_t* dst_sums,
                   cudaStream_t s);
int launch_checksum_in(int rb, const void* recs, uint64_t n, uint64_t* acc4, cudaStream_t s);
int launch_checksum_out(int rb, const ShuffleBuffers& b, uint32_t B, const RangeBinParams& bp, uint32_t bin_base,
                        uint64_t* acc6, cudaStream_t s);
cudaError_t kernels_configure();  // opt-in shared memory sizes; call once per device

// ---- byte values (MRHBM_F_BYTE_VALUES, mrhbm_values.cu) ----
// A pair's value field holds its value id (its pool index); value id i has the bytes arena[voff[i] .. voff[i+1]).
// Rows of the value gather per scan tile (the first pass scans each tile, the second the tile totals).
constexpr uint32_t kValTileLog = 13;
// Values longer than this are copied in pieces of this size, one warp per piece, after the row gather.
constexpr uint32_t kValChunk = 4096;
inline uint64_t val_tiles(uint64_t rows) { return (rows + (1u << kValTileLog) - 1) >> kValTileLog; }
// most pieces of the values longer than kValChunk that `bytes` value bytes can hold
inline uint64_t val_chunks_cap(uint64_t bytes) { return 2 * (bytes / kValChunk) + 1; }
// records [0, n) of the rb-byte records at recs get value id first + i; dvoff[i] (i <= n, the caller's offsets as
// copied) becomes dvoff[i] - v0 + aoff, an offset into the arena.  recs == nullptr: the n pairs of a tokeniser piece
// share one value of v0 bytes at aoff: dvoff[0] = aoff and dvoff[1 .. n] = aoff + v0 (first is unused)
int launch_value_stamp(int rb, void* recs, uint64_t n, uint64_t first, uint64_t* dvoff, uint64_t v0, uint64_t aoff,
                       cudaStream_t s);
// row_off[r] for rows r < n whose value id is ids[r]: value bytes of the rows before r inside its scan tile;
// tile_pre[t] (val_tiles(n) + 1 entries) the bytes before tile t, row_off[n] the total.  The gather completes row_off.
int launch_value_scan(const uint64_t* ids, uint64_t n, const uint64_t* voff, uint64_t* row_off, uint64_t* tile_pre,
                      cudaStream_t s);
// copies every row's value bytes from the arena to out at its row offset (row_off is final afterwards); pieces is
// scratch of val_chunks_cap(total) entries, npieces one zeroed word
int launch_value_gather(const uint64_t* ids, uint64_t n, const uint64_t* voff, const unsigned char* arena,
                        uint64_t* row_off, const uint64_t* tile_pre, unsigned char* out, uint64_t* pieces,
                        unsigned long long* npieces, cudaStream_t s);

// ---- MRHBM_COMBINE_DISTINCT (mrhbm_distinct.cu) ----
// One map job's records: range k holds pool records [off, off + rg[k+1].vbase - vbase), which are the job's records
// [vbase, ...) and its tiles of kDistinctTile records [tbase, rg[k+1].tbase).  nr ranges, none empty, then one entry
// {0, total records, total tiles}.
struct DistinctRange {
  uint64_t off, vbase;
  uint32_t tbase, pad;
};
constexpr uint32_t kDistinctTile = 256;
// every record into the hash set tab (mask + 1 16-byte entries, a power of two >= 2 x the job's records, memset to
// 0xff by the caller); slot_of[g] receives the entry of the job's record g
int launch_distinct_mark(int rb, const void* pool, const DistinctRange* rg, uint32_t nr, uint32_t ntiles,
                         const unsigned char* arena, const uint64_t* voff, void* tab, uint64_t mask, uint32_t* slot_of,
                         cudaStream_t s);
// tile_cnt[t] = the records of tile t that are the first copy of their pair
int launch_distinct_count(const DistinctRange* rg, uint32_t nr, uint32_t ntiles, const void* tab, const uint32_t* slot_of,
                          uint32_t* tile_cnt, cudaStream_t s);
// those records, in pool order, to out: tile t's at out[tile_off[t] ..) (tile_off: the exclusive scan of tile_cnt);
// ones: with their value field set to 1 (MRHBM_RED_COUNT_DISTINCT), else as they are
int launch_distinct_scatter(int rb, const void* pool, const DistinctRange* rg, uint32_t nr, uint32_t ntiles,
                            const void* tab, const uint32_t* slot_of, const uint32_t* tile_off, void* out, bool ones,
                            cudaStream_t s);

// ---- MRHBM_RED_DISTINCT (mrhbm_value_order.cu) ----
// Every bin's rows (ucount[bin] of them at out_start, sorted by key, value ids in out_sums) in (key, value bytes)
// order: the nb bins of at most cap rows, and the cap-row chunks of the nbig oversized bins of big_list
int launch_value_order(int rb, const ShuffleBuffers& b, uint32_t nb, uint32_t nbig, uint32_t cap,
                       const unsigned char* arena, const uint64_t* voff, cudaStream_t s);
// then each oversized bin's chunks merged into one run; tmp_keys / tmp_ids: scratch rows laid out as out_keys / out_sums
int launch_value_merge(int rb, const ShuffleBuffers& b, uint32_t nbig, uint32_t cap, const unsigned char* arena,
                       const uint64_t* voff, void* tmp_keys, uint64_t* tmp_ids, cudaStream_t s);

// ---- MRHBM_RED_FSUM (mrhbm_num_sum.cu) ----
// Oversized bins (exact layout, rows [0, N)): the partial accumulators of the groups that cross the edge of a cap-row
// chunk.  The chunk that starts at row r is slot num_slot(r, ...): no two chunks of oversized bins share a slot (chunks
// of one bin lie cap rows apart; a bin's first chunk and another bin's later chunk differ in parity), so 2 ceil(N / cap)
// + 2 slots take every chunk.  Slot s: acc[2 s] (the chunk's leading part of a group), acc[2 s + 1] (its trailing
// group), kAccWords each (mrhbm_numsum.cuh); flags[s]; head_row[s]: the trailing group's first row.
struct NumScratch {
  int64_t* acc;
  uint32_t* flags;
  uint32_t* head_row;
};
MRHBM_HD inline uint64_t num_slot(uint64_t first_row, uint32_t cap, bool first_chunk) {
  return 2 * (first_row / cap) + (first_chunk ? 1 : 0);
}
inline uint64_t num_slots(uint64_t N, uint32_t cap) { return 2 * ((N + cap - 1) / cap) + 2; }
// The cap-row chunks of each of the nbig oversized bins of big_list (ascending by key, as k_big_bins leaves them)
// merged by key into one run, pass after pass of doubling width up to max_rows (at least every such bin's rows), each
// pass spread over many CTAs per bin; tmp_keys / tmp_ids: scratch rows laid out as out_keys / out_sums.  The run ends in
// the output rows.
int launch_num_key_merge(int rb, const ShuffleBuffers& b, uint32_t nbig, uint32_t cap, uint64_t max_rows, void* tmp_keys,
                         uint64_t* tmp_ids, cudaStream_t s);
// Every bin's rows (ucount[bin] of them at out_start, sorted by key, value ids in out_sums; the nbig oversized bins of
// big_list merged into one run each) become one row per key, out_sums its values' exact sum rounded to a double (bits),
// ucount[bin] the keys.  ERRF_NOTNUM / ERRF_NAN in counters[CNT_ERR].
int launch_num_sum(int rb, const ShuffleBuffers& b, uint32_t nb, uint32_t nbig, uint32_t cap, const unsigned char* arena,
                   const uint64_t* voff, const NumScratch& sc, cudaStream_t s);
// compacted rows whose ids hold double bits -> row r's encoded number at vals[11 r ..), row_off[r] = 11 r (n + 1
// entries), ids[r] = r
// counts: the ids hold integer counts instead (MRHBM_RED_COUNT_DISTINCT), each encoded as the number (double) it is
int launch_num_encode(uint64_t* ids, uint64_t n, unsigned char* vals, uint64_t* row_off, cudaStream_t s,
                      bool counts = false);

// ---- MRHBM_COMBINE_FSUM (mrhbm_num_combine.cu) ----
// One map job's records (DistinctRange, as the distinct combiner takes them) grouped by key slot and each key's numbers
// split into the greedy expansion of their exact sum (acc_split, mrhbm_numsum.cuh).  Scratch, all sized by the caller:
//   tab      mask + 1 16-byte entries {fingerprint, smallest pool index of the key}, memset to 0xff
//   slot_of  the entry of each of the job's n records; vbits: their values' double bits
//   words    4 (mask + 1) words: the entries' counts (zeroed), rooms in vals, cursors, terms (see kFsumKeep)
//   vals     n: each key's values, then its terms, in a room of its own
//   big      n / kFsumWarpValues + 1 keys longer than a warp takes; gacc: an accumulator for each (zeroed)
//   small    4 zeroed words: flags (ERRF_NOTNUM, ERRF_NAN, kFsumKeep), the rooms' bump, the number of big keys
constexpr uint32_t kFsumWarpValues = 4096;
constexpr uint32_t kFsumKeep = 1u << 31;  // in a key's term count and in the flags: the key keeps its values
struct FsumScratch {
  void* tab;
  uint64_t mask;
  uint32_t *slot_of, *words, *big, *small;
  uint64_t *vbits, *vals;
  int64_t* gacc;
};
// The sums and terms of every key, and tile_cnt[t] = the new pairs of the keys whose first pair lies in tile t
int launch_fsum_split(int rb, const void* pool, const DistinctRange* rg, uint32_t nr, uint32_t ntiles, uint64_t n,
                      const unsigned char* arena, const uint64_t* voff, const FsumScratch& fs, uint32_t* tile_cnt,
                      int sm_count, cudaStream_t s);
// The new pairs (tile_off: the exclusive scan of tile_cnt) at pool records first + i with value id first + i, voff
// entries from aoff on (11 bytes each, voff[first + total] included) and their encoded values in the arena.  A key
// that keeps its values is left to launch_fsum_copy: the words' cursor of its entry receives its first new pair.
int launch_fsum_write(int rb, void* pool, const DistinctRange* rg, uint32_t nr, uint32_t ntiles, const FsumScratch& fs,
                      const uint32_t* tile_off, uint64_t first, uint64_t aoff, uint64_t* voff, unsigned char* arena,
                      cudaStream_t s);
// The kept values: cp[3 i .. 3 i + 2] = {new pair's index after first, its record's pool index, its job index}
int launch_fsum_copy(int rb, void* pool, const uint64_t* cp, uint64_t m, const FsumScratch& fs, uint64_t first,
                     uint64_t aoff, uint64_t* voff, unsigned char* arena, cudaStream_t s);

}  // namespace mrhbm
