/*
 * mrhbm.h -- C ABI of the H100-native shuffle / sort / reduce core ("storage = hbm").
 *
 * This is the drop-in boundary for lua-mapreduce's map-side emit buffer and
 * reduce-side group-by.  Each entry point names the reference interface it
 * replaces (file:line in pakozm/lua-mapreduce @ 767321e).  The library is plain
 * C ABI: pointers and sizes only, no C++/torch types, no exception or CUDA
 * sticky error crosses it.  Every function that returns int returns >= 0 on
 * success and a negative MRHBM_E_* on failure; the message is available from
 * mrhbm_last_error() (luamongo's `nil, "<msg>"` convention,
 * external/luamongo/mongo_gridfilebuilder.cpp:64-69).
 *
 * Threading: a ctx and everything created from it is single-caller (the
 * reference's concurrency model is one single-threaded Lua worker process per
 * ctx, mapreduce/worker.lua:42-105).  One ctx drives one GPU; a multi-GPU job
 * is one ctx per rank joined by mrhbm_comm_init().
 *
 * There is NO CPU fallback: mrhbm_init() fails if no sm_90 device (H100) is
 * usable.
 */
#ifndef MRHBM_H
#define MRHBM_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define MRHBM_ABI_VERSION 2

enum { /* error codes */
  MRHBM_OK = 0,
  MRHBM_E_INVAL = -1,     /* bad argument / bad state */
  MRHBM_E_CUDA = -2,      /* CUDA runtime error (message has the CUDA string) */
  MRHBM_E_NOMEM = -3,     /* host or device allocation failed */
  MRHBM_E_KEY = -4,       /* key does not fit: a fixed-width record or result slot, a word of the device tokeniser, > 1 MB */
  MRHBM_E_SKEW = -5,      /* a bin holds more distinct keys than one SM can sort (see DESIGN.md) */
  MRHBM_E_OVERFLOW = -6,  /* reserved, no longer returned: sums are u64 on every path, exact up to 2^53 */
  MRHBM_E_NCCL = -7,      /* NCCL missing or failed */
  MRHBM_E_NODEVICE = -8   /* no usable sm_90 GPU: there is no CPU path */
};

enum { MRHBM_KEY_U64 = 0, MRHBM_KEY_STR = 1 };

/* built-in partitionfn (the user's Lua partitionfn, mapreduce/job.lua:203-207, is a
 * pure key -> integer function; these are the ones the device evaluates) */
enum {
  MRHBM_PART_FNV_LUA = 0,  /* examples/WordCount/partitionfn.lua:8-16, bit-exact incl. the
                              double-precision rounding; pid = h % num_partitions */
  MRHBM_PART_MULHASH = 1,  /* u64 keys: mulhi(key * 0x9E3779B97F4A7C15, P) (SURVEY 8d cfg 4) */
  MRHBM_PART_WORDHASH = 2, /* string keys: 64-bit word hash, mulhi(h, P) */
  /* u64 and string keys: key ranges.  num_partitions-1 non-decreasing splitters s_0 <= ... <= s_{P-2}
     (duplicates allowed: they leave partitions empty); pid(key) = |{ i : s_i <= key }| (a key equal to a splitter
     goes to the upper side).  Order is the library's key order: strings C-locale bytewise on the original bytes, a
     proper prefix first; u64 keys numeric (= their 8 big-endian bytes).  A string splitter is any byte string (it may
     be longer than the record class and hold 0x00 / 0x01); a u64 splitter is exactly 8 big-endian bytes.  With
     P = 1 there are no splitters.  Partition k then holds the k-th slice of the key space, so the partitions read in
     order 0 .. P-1 give every key in one global ascending order.  Set with mrhbm_set_splitters or
     mrhbm_sample_splitters before the shuffle; a shuffle without them fails with MRHBM_E_INVAL. */
  MRHBM_PART_RANGE = 3
};
/* built-in reducefn/combinerfn (examples/WordCount/reducefn.lua:1-15: integer sum,
 * associative + commutative + idempotent flags set) */
enum {
  MRHBM_RED_SUM = 0,
  /* general (non-built-in) Lua reducefn, job.lua:264-284: the device only partitions, sorts and
   * groups; mrhbm_groups_next hands out every value of a key (order unspecified, like the
   * reference's heap-pop order among equal keys) and the host calls reducefn per group.
   * Needs combiner = 0.  mrhbm_result_copy then returns one row per pair (keys repeat).  A key may
   * carry any number of values, on one GPU or several: a bin larger than one shared-memory sort is
   * sorted run by run on its owner and the iterator merges the runs. */
  MRHBM_RED_NONE = 1,
  /* MRHBM_F_BYTE_VALUES only, with combiner MRHBM_COMBINE_NONE or MRHBM_COMBINE_DISTINCT (any other combination fails
   * mrhbm_init with MRHBM_E_INVAL; one GPU, as byte values are): the reducefn "each key's distinct values, ascending",
   * an inverted index's, computed on the device -- no host reducefn runs.  After mrhbm_shuffle the result holds exactly
   * one row per distinct (key, value bytes) pair over all committed pairs of all map jobs: keys compare as everywhere
   * else, values by their bytes, never by their value id (two emits of the same bytes under different ids are one row;
   * the empty value is a value like any other).  Which of several equal pairs gives the row its value id is
   * unspecified.  Inside each run rows ascend by (key, value bytes), values in the key order's sense: unsigned
   * bytewise, a proper prefix first.  So mrhbm_groups_next_values gives every group, long keys included, its distinct
   * values ascending; mrhbm_result_copy / mrhbm_result_values rows follow info.sorted (with sorted = 1 a partition's
   * rows ascend by (key, value) as a whole), and an oversized bin is one run, not several.  mrhbm_result_info: pairs_in
   * = committed pairs, pairs_recv = distinct pairs the shuffle carried, groups = rows.  mrhbm_checksum_result's
   * out[3..5] keep their meaning; in[0..2] == out[0..2] does not hold (duplicates are gone and a row's value id may be
   * another copy's).  The ordering kernels are timed in mrhbm_stats.ms_bigbins, the dedupe in ms_combine, both inside
   * ms_total.  Limits: fewer than 2^31 committed pairs per shuffle (else MRHBM_E_INVAL).  Extra device memory: the
   * distinct set of MRHBM_COMBINE_DISTINCT sized for all committed pairs (16 bytes x a power of two >= 2 x pairs, plus
   * 4 + record bytes per pair), and, in a shuffle with a bin of more rows than one shared-memory sort takes, key slot +
   * 8 bytes per result row of scratch. */
  MRHBM_RED_DISTINCT = 2,
  /* MRHBM_F_BYTE_VALUES only, with combiner MRHBM_COMBINE_NONE (any other combination fails mrhbm_init with
   * MRHBM_E_INVAL; one GPU, as byte values are): the reducefn "count = count + v" over Lua numbers (weighted word
   * counts, PageRank contributions, loss totals), computed on the device -- no host reducefn runs.  Every value must be
   * a number as the bindings encode it (mapreduce/tuple.py _enc_num with key=False, hbm.lua enc_num): 11 bytes, 0x10,
   * then the IEEE double's bits u sign-folded (u | 2^63 when the sign bit is 0, ~u when it is 1) as ten big-endian
   * 7-bit groups of u (the first holding bit 63 alone), each OR 0x80.  A value that is not such an encoding, or that
   * encodes a NaN, fails mrhbm_shuffle with MRHBM_E_INVAL and leaves no result (Lua's arithmetic on a non-number
   * breaks the reduce job).  After mrhbm_shuffle there is exactly one row per key; its value is the key's values
   * summed exactly and rounded once to the nearest double, ties to even: float(sum(Fraction(v) for v in values)) in
   * Python.  A sum whose magnitude rounds beyond DBL_MAX is +-inf; infinities of one sign give that infinity; +inf and
   * -inf on one key fail mrhbm_shuffle with MRHBM_E_INVAL (Lua would make a NaN, which the reference's "%.14g" spill
   * cannot load back); an exact zero is +0 unless every value is -0, then -0.  The result does not depend on emission
   * order, map jobs, bins or runs, and is bit-identical for every MRHBM_F_* layout flag.  Where the reference's own
   * left-to-right double sum is exact (integers whose partial sums stay below 2^53, say) the two are equal, so an
   * integer word count gives what MRHBM_RED_SUM gives.  Reading the result: mrhbm_groups_next_values gives every
   * group, long keys included, its one value in the encoding above; mrhbm_result_values gives one value per
   * mrhbm_result_copy row, and the row's value field is the row index.  mrhbm_result_info: pairs_in = committed pairs,
   * pairs_recv = pairs the shuffle carried, groups = keys.  mrhbm_checksum_result's out[3..5] keep their meaning;
   * in[0..2] == out[0..2] does not hold (a row holds a sum, not a value id).  The summing kernels are timed in
   * mrhbm_stats.ms_bigbins, inside ms_total.  Limits: fewer than 2^31 committed pairs per shuffle (else
   * MRHBM_E_INVAL).  Extra device memory: 11 bytes of value and 8 of offset per result row; and, in a shuffle with a
   * bin of more rows than one shared-memory sort takes, key slot + 8 bytes per result row of merge scratch and, for
   * the groups that span a chunk of such a bin, partial accumulators of 1096 bytes per slot, 2 ceil(rows / cap) + 2
   * slots (cap = 32 KB / record bytes). */
  MRHBM_RED_FSUM = 3,
  /* MRHBM_F_BYTE_VALUES only, with combiner MRHBM_COMBINE_NONE or MRHBM_COMBINE_DISTINCT (any other combination fails
   * mrhbm_init with MRHBM_E_INVAL; one GPU, as byte values are): the reducefn "the number of distinct values of the
   * key", COUNT(DISTINCT) -- unique visitors per page, the document frequency of a word, distinct sources per
   * destination -- computed on the device, no host reducefn runs.  After mrhbm_shuffle there is exactly one row per
   * key; its value is the number of distinct values among the key's committed pairs over all map jobs, encoded as the
   * 11-byte number of MRHBM_RED_FSUM (the bytes of tuple.encode_value(float(n))).  Values are equal when their bytes
   * are, exactly as in MRHBM_RED_DISTINCT: two emits of the same bytes under different value ids count once, the empty
   * value counts as a value, the numbers 1 and 1.0 have the same encoding and count once, while -0 and +0 have
   * different bytes and count twice.  Keys longer than the record class get the same count on the host, at their
   * place in the key order.  The result does not depend on emission order, map jobs, bins, runs, the distinct
   * combiner or any MRHBM_F_* layout flag: it is bit-identical across all of them.  Reading the result, as for
   * MRHBM_RED_FSUM: mrhbm_groups_next_values gives every group, long keys included, its one encoded count;
   * mrhbm_result_values gives one value per mrhbm_result_copy row, and the row's value field is the row index
   * (mrhbm_groups_next fails, mrhbm_result_copy needs sums = NULL).  mrhbm_result_info: pairs_in = committed pairs,
   * pairs_recv = distinct pairs the shuffle carried, groups = keys.  mrhbm_checksum_result's out[3..5] keep their
   * meaning; in[0..2] == out[0..2] does not hold (a row holds a count, not a value id).  The dedupe (the distinct set
   * of MRHBM_RED_DISTINCT, each surviving pair carrying the value 1) is timed in mrhbm_stats.ms_combine; the integer
   * sum of those 1s per key runs through the stages of MRHBM_RED_SUM and is timed where they are, all inside ms_total.
   * Hot keys cost what they cost MRHBM_RED_SUM: no value ordering runs.  Limits: fewer than 2^31 committed pairs per
   * shuffle (else MRHBM_E_INVAL), so every count is exact in a double.  Extra device memory: the distinct set of
   * MRHBM_RED_DISTINCT (16 bytes x a power of two >= 2 x pairs, plus 4 + record bytes per pair), and 11 bytes of value
   * and 8 of offset per result row. */
  MRHBM_RED_COUNT_DISTINCT = 4
};

/* built-in combinerfn, run on the map side (job.lua:92-96,198-202: reducing the combined values must give what
 * reducing the raw ones gives) */
enum {
  MRHBM_COMBINE_NONE = 0,
  MRHBM_COMBINE_REDUCER = 1, /* the built-in reducer (MRHBM_RED_SUM), at the shuffle: one pair per key */
  /* MRHBM_F_BYTE_VALUES only (any other combination fails mrhbm_init with MRHBM_E_INVAL): a combinerfn whose result
   * depends only on the SET of a key's values, such as an inverted index's "distinct files of a word".  At
   * mrhbm_map_commit the handle's pairs are reduced to their distinct (key, value) pairs: keys compare by their stored
   * slot bytes (long keys, see mrhbm_emit_str, by their bytes, on the host), values by their bytes (not by their value
   * id; the empty value is a value like any other).  The first copy in pool order (the handle's emission order)
   * survives; survivors keep their
   * relative order and their value ids.  Pairs of different map jobs are never merged (the host reducefn still sees
   * one copy per job), and replace-by-job-id and abort are unchanged; a commit that fails leaves the job uncommitted.
   * mrhbm_pool_read, mrhbm_checksum_input, mrhbm_result_info.pairs_in and everything after the commit see only the
   * surviving pairs.  The room of the dropped pairs and of their value bytes is not reused before mrhbm_reset.  Device
   * memory: a hash set of 16 bytes x (a power of two >= 2 x the job's pairs), kept across commits, plus 4 + record
   * bytes per pair of the job. */
  MRHBM_COMBINE_DISTINCT = 2,
  /* MRHBM_F_BYTE_VALUES and reducer MRHBM_RED_FSUM only (any other combination fails mrhbm_init with MRHBM_E_INVAL;
   * one GPU, as byte values are): the combinerfn "count = count + v" of a number-sum job, run on the device at
   * mrhbm_map_commit without rounding anything away.  Keys compare by their stored slot bytes (long keys, see
   * mrhbm_emit_str, by their bytes, on the host).  For each key of the handle's pairs, with m its values in this job
   * and S their exact sum:
   *   - a value that is not a number encoding (see MRHBM_RED_FSUM; a NaN encoding included), or +inf and -inf among
   *     the key's values, fails the commit with MRHBM_E_INVAL; the job stays uncommitted (the handle is consumed, an
   *     earlier commit under the same id stays), as a Lua combinerfn's count + v would break the map job;
   *   - infinities of one sign: one value, that infinity;
   *   - S = 0: one value, -0 if all m values are -0, else +0;
   *   - otherwise the greedy expansion: c1 = S rounded to the nearest double, ties to even (what MRHBM_RED_FSUM gives
   *     for these values alone), c(k+1) = S - c1 - ... - ck rounded the same way, until the remainder is 0 (one or
   *     two values in practice; two values never need more than two);
   *   - but if |S| >= 2^1024 - 2^970 (c1 would be +-inf) or the expansion has more than m terms, the key keeps its m
   *     values as emitted.
   * The surviving pairs are new pairs at the tail of the pool, ordered by the pool position of each key's first pair,
   * a key's values in the order c1, c2, ... (kept values in emission order).  Every survivor holds its own 11-byte
   * value and its value id is its own pool index, also in a job of mrhbm_map_words_value pieces.  mrhbm_pool_read,
   * mrhbm_checksum_input, mrhbm_result_info.pairs_in and everything after the commit see only the survivors.  The
   * job's original room is not reused before mrhbm_reset; survivors count against the 2^32 pairs between resets.
   * Replace-by-job-id, abort, reset and repeated shuffles are unchanged.  After mrhbm_shuffle every result is
   * bit-identical to the same commits without the combiner: mrhbm_groups_next_values, the rows of mrhbm_result_copy
   * with mrhbm_result_values (their order follows info.sorted, which the shuffle picks from the pairs
   * it carries), the groups count, and the shuffle's failures (+inf in one job and -inf in another still fail
   * it); pairs_in and pairs_recv count the survivors the shuffle carried.  The combine is not part of mrhbm_stats.  Limits: fewer than 2^31 pairs per map job (else
   * MRHBM_E_INVAL).  Device memory: the distinct combiner's hash set and per-pair scratch, plus 16 bytes x the set's
   * entries, 16 bytes per pair of the job, and 548 bytes per 4096 pairs; a commit where some key keeps its values
   * also copies the job's entries to the host and back. */
  MRHBM_COMBINE_FSUM = 3
};

typedef struct mrhbm_ctx mrhbm_ctx;
typedef struct mrhbm_map mrhbm_map;
typedef struct mrhbm_iter mrhbm_iter;

typedef struct mrhbm_config {
  uint32_t struct_size;    /* = sizeof(mrhbm_config) */
  int32_t device;          /* CUDA ordinal; -1 = current device */
  uint32_t key_kind;       /* MRHBM_KEY_* */
  uint32_t max_key_bytes;  /* STR: <=27 -> 32 B records, <=59 -> 64 B, <=123 -> 128 B */
  uint32_t num_partitions; /* P >= 1 (reduce jobs; server.lua:316-323) */
  uint32_t partitioner;    /* MRHBM_PART_* */
  uint32_t reducer;        /* MRHBM_RED_* */
  uint32_t combiner;       /* MRHBM_COMBINE_* (job.lua:92-96,198-202) */
  uint64_t reserve_pairs;  /* pre-size the HBM emit pool (0 = grow on demand) */
  uint32_t flags;          /* MRHBM_F_* */
  uint32_t reserved;
} mrhbm_config;
#define MRHBM_F_FORCE_RUNS 1u   /* always use hash sub-bins (skip the key-ordered attempt) */
#define MRHBM_F_SMALL_BINS 2u   /* test hook: tiny smem bins to exercise the overflow paths */
#define MRHBM_F_NO_OPTIMISTIC 4u /* always run the exact two-pass (histogram) partition layout */
/* Byte-string values (lua-mapreduce's emit(key, value) takes any Lua string or number, utils.lua:100-120): a value is
 * opaque bytes, 0 to 1 GiB long, carried through group-only mode.  Needs reducer = MRHBM_RED_NONE (or a byte-values
 * reducer: MRHBM_RED_DISTINCT, MRHBM_RED_FSUM, MRHBM_RED_COUNT_DISTINCT) and combiner
 * MRHBM_COMBINE_NONE or MRHBM_COMBINE_DISTINCT (else mrhbm_init fails with MRHBM_E_INVAL) and one GPU (mrhbm_comm_init with world > 1 fails).  On such a ctx:
 *   - pairs are emitted with mrhbm_emit_str_value / mrhbm_emit_u64_value / mrhbm_emit_batch_values /
 *     mrhbm_map_words_value / mrhbm_map_key_numbers; the integer-valued emits (emit_str, emit_u64, emit_batch, emit_device, map_gen_*,
 *     map_wordcount) fail with MRHBM_E_INVAL;
 *   - groups are read with mrhbm_groups_next_values (mrhbm_groups_next fails) and rows with mrhbm_result_values;
 *     mrhbm_result_copy needs sums = NULL;
 *   - the value field of a record (pool_read, result_copy) holds the pair's value id, its index in the emit pool,
 *     except that the pairs of one device piece of mrhbm_map_words_value share the id of the piece's first pair;
 *     fewer than 2^32 pairs may be emitted between mrhbm_reset calls, those of aborted and replaced jobs included.
 * The order of a key's values is unspecified with MRHBM_RED_NONE; MRHBM_RED_DISTINCT gives each key's distinct values
 * in ascending byte order; MRHBM_RED_FSUM gives each key one value, the exact sum of its numbers; MRHBM_RED_COUNT_DISTINCT
 * gives each key one value, the number of its distinct values.  The new calls fail with MRHBM_E_INVAL on a ctx
 * without the flag. */
#define MRHBM_F_BYTE_VALUES 8u

/* record layouts (little endian) moved by emit_batch / gen / result_copy:
 *   U64 : { uint64_t key; uint64_t value; }                             16 B
 *   STR : { uint8_t key[RB-4] zero padded, no NUL inside (see mrhbm_emit_str); uint32_t value; }  RB = 32/64/128 */
uint32_t mrhbm_record_bytes(const mrhbm_ctx *);

/* ---- lifecycle (replaces cnn(...) + fs.router(...), mapreduce/fs.lua:185-208) ---- */
int mrhbm_init(const mrhbm_config *, mrhbm_ctx **out);
void mrhbm_destroy(mrhbm_ctx *);
const char *mrhbm_last_error(const mrhbm_ctx *); /* owned by ctx; valid until next call */
int mrhbm_abi_version(void);

/* pinned host memory for zero-staging emit_batch / result_copy */
void *mrhbm_host_alloc(mrhbm_ctx *, size_t bytes);
void mrhbm_host_free(mrhbm_ctx *, void *);

/* ---- map side: job.lua:83-97 (emit) + job.lua:186-227 (sort/partition/spill) ---- */
int mrhbm_map_begin(mrhbm_ctx *, const char *map_job_id, mrhbm_map **out);
/* key bytes are copied before return (Lua strings may be collected).  Any byte string is a key: bytes 0x00 and
 * 0x01 are stored escaped (01 01 / 01 02, order preserving; each costs one more byte of the key slot), hashed by
 * the built-in partitioners as the original bytes and handed back unescaped by mrhbm_groups_next.  Key slots in
 * emit_batch records and in mrhbm_result_copy are in the stored (escaped) form.
 * A key LONGER than the ctx record class (max_key_bytes) is accepted too (the reference takes any key,
 * utils.lua:104-110): such pairs are assumed rare, stay on the host, are partitioned (same partitioner), exchanged
 * and grouped at the barrier, and mrhbm_groups_next hands them out at their place in the key order.  They follow
 * commit / abort / replace-by-job-id like every other pair; the combiner does not see them; the fixed-width bulk
 * calls (emit_batch, map_wordcount, result_copy, checksums) do not carry them. */
int mrhbm_emit_str(mrhbm_map *, const void *key, size_t klen, uint32_t value);
int mrhbm_emit_u64(mrhbm_map *, uint64_t key, uint64_t value); /* value < 2^53 keeps Lua-number sums exact */
/* n records in the ctx layout.  Pageable memory is consumed before return; memory from
 * mrhbm_host_alloc() is read asynchronously and must stay untouched until commit/abort. */
int mrhbm_emit_batch(mrhbm_map *, const void *records, size_t n);
/* records already in HBM (device pointer on the ctx device), copied device-to-device */
int mrhbm_emit_device(mrhbm_map *, const void *dev_records, size_t n);
/* device-side mapfn for the synthetic streams of SURVEY App. B (bench + parity tests):
 * u64: key=splitmix64(seed+i), val=splitmix64(seed+2^40+i)>>32, i in [start,start+n)
 * zipf: rank by lower-bound search of splitmix64(seed+2^41+i) in table[V] (host pointer),
 *       key = rank->string, val = 1 (needs 32 B records) */
int mrhbm_map_gen_u64(mrhbm_map *, uint64_t seed, uint64_t start, uint64_t n);
int mrhbm_map_gen_zipf(mrhbm_map *, uint64_t seed, uint64_t start, uint64_t n,
                       const uint64_t *table, uint64_t V);
/* device-side WordCount mapfn (examples/WordCount/mapfn.lua:3-9, misc/naive.lua:2-5): emits
 * (word, 1) for every maximal run of non-space bytes of `text`; the space class is C-locale
 * isspace (' ' \t \n \v \f \r), i.e. Lua's "[^%s]+".  A 64 MB piece of the text that holds a word longer than
 * the ctx record class (a URL in a corpus) is tokenised on the host instead, the long words going the way of
 * mrhbm_emit_str's long keys.  On failure nothing of the call is emitted.  *words (optional) receives the token count. */
int mrhbm_map_wordcount(mrhbm_map *, const void *text, size_t len, uint64_t *words);
/* host-side generator of the synthetic word-count text of SURVEY App. B (bench + tests; needs no ctx):
 * words first .. first+n-1 of the Zipf(table) word stream, one space between words, '\n' after every
 * words_per_line-th word.  *len receives the bytes the text needs; MRHBM_E_INVAL (nothing usable written) if
 * that exceeds cap.  Call with cap = 0 to size the buffer. */
int mrhbm_synth_zipf_text(uint64_t seed, uint64_t first, uint64_t n, uint32_t words_per_line,
                          const uint64_t *table, uint64_t V, void *out, size_t cap, size_t *len, int threads);
/* copies n committed pairs starting at pair index `first` (commit order) back to host
 * memory in the record layout (bench + tests: checks the device generators) */
int mrhbm_pool_read(mrhbm_ctx *, uint64_t first, uint64_t n, void *host_out);
/* atomic publish; a second commit under the same job id REPLACES the first
 * (job.lua:217-221 remove_file + build).  Consumes the handle. */
int mrhbm_map_commit(mrhbm_map *);
/* BROKEN job: nothing becomes visible (worker.lua:120-127).  Consumes the handle. */
void mrhbm_map_abort(mrhbm_map *);
/* MRHBM_F_BYTE_VALUES: one pair with the value bytes val[0 .. vlen) (copied before return; vlen <= 1 GiB, 0 allowed).
 * Keys follow mrhbm_emit_str / mrhbm_emit_u64, long string keys included. */
int mrhbm_emit_str_value(mrhbm_map *, const void *key, size_t klen, const void *val, size_t vlen);
int mrhbm_emit_u64_value(mrhbm_map *, uint64_t key, const void *val, size_t vlen);
/* MRHBM_F_BYTE_VALUES, bulk: n records in the ctx layout (their value field is ignored) and the value of record i at
 * vals[voff[i] .. voff[i+1]) (voff has n + 1 non-decreasing entries).  Pinned and pageable memory as for
 * mrhbm_emit_batch: all three buffers are pinned-or-pageable independently. */
int mrhbm_emit_batch_values(mrhbm_map *, const void *records, size_t n, const void *vals, const uint64_t *voff);
/* MRHBM_F_BYTE_VALUES: the device tokeniser of mrhbm_map_wordcount (same word rule, same pieces, same host fall-back
 * for words longer than the record class, same "nothing of a failed call is emitted"), emitting (word, val[0 .. vlen))
 * for every word instead of (word, 1): an inverted index's map job (examples/WordCount/mapfn.lua:3-9 with the file
 * name as the value).  val is copied before return (vlen <= 1 GiB, 0 allowed).  *words (optional) receives the token
 * count.  String-key ctx only. */
int mrhbm_map_words_value(mrhbm_map *, const void *text, size_t len, const void *val, size_t vlen, uint64_t *words);
/* MRHBM_F_BYTE_VALUES, string-key ctx only (else MRHBM_E_INVAL): the map side of a number sum over text lines
 * "key number" (bytes per URL, sales per product, edge weights per node), parsed on the device.
 *   - Lines: the text is cut into lines at '\n'; a last line without '\n' counts.  A line made only of C-locale white
 *     space (' ' \t \n \v \f \r) emits nothing.  A field is a maximal run of non-space bytes; every other line must
 *     have exactly two fields, the key, then the number.
 *   - Key: the first field's bytes, 0x00 and 0x01 escaped as in mrhbm_emit_str; a key longer than the record class
 *     takes the long-key path of mrhbm_emit_str_value (its 64 MB piece is parsed on the host).
 *   - Number: the second field must match [+-]?(D+(\.D*)?|\.D+)([eE][+-]?D+)? -- the decimal form Lua 5.2's tonumber
 *     takes through strtod.  Unlike Lua, hexadecimal numbers (0x10), inf, nan and anything else are refused.  Its
 *     value is the nearest double, ties to even (Python's float()): a magnitude beyond the largest double gives +-inf,
 *     underflow a correctly rounded subnormal or +-0, and -0 stays -0.  The value is stored as the 11-byte number
 *     encoding (see MRHBM_RED_FSUM), the bytes of tuple.encode_value(float(field)).
 *   - Pairs: one per line, in text order; each has its own 11-byte value and its value id is its own pool index.
 *   - Failure: a line that breaks these rules, or one longer than a 64 MB piece, fails the call with MRHBM_E_INVAL and
 *     a message giving the line's byte offset.  A failed call emits nothing.
 * *lines (optional) receives the number of pairs emitted. */
int mrhbm_map_key_numbers(mrhbm_map *, const void *text, size_t len, uint64_t *lines);

/* ---- barrier between MAP and REDUCE (server.lua:279-329) ---- */
/* hash-partition [+ NCCL all-to-all] + sort + segmented reduce of everything committed */
int mrhbm_shuffle(mrhbm_ctx *);
/* NON-EMPTY partitions owned by this rank, ascending -> red_jobs (server.lua:300-324) */
int mrhbm_partitions(mrhbm_ctx *, uint32_t *ids, size_t cap, size_t *n);
/* MRHBM_PART_RANGE: installs the num_partitions-1 splitters; splitter i is keys[off[i] .. off[i+1]) in original bytes
 * (u64 keys: 8 big-endian bytes).  Kept across mrhbm_reset.  Several GPUs: every rank must install the same splitters
 * (the next shuffle checks this and fails on all ranks with MRHBM_E_INVAL if they differ). */
int mrhbm_set_splitters(mrhbm_ctx *, const void *keys, const uint64_t *off, size_t n);
/* MRHBM_PART_RANGE: samples the committed pairs (collective on several GPUs, weighted by each rank's committed pairs),
 * installs num_partitions-1 quantile splitters and returns them in the form above (*need receives the key bytes).
 * They take at most (num_partitions-1) * key slot bytes (8 for u64 keys, mrhbm_record_bytes - 4 for strings): a
 * buffer of that size needs no sizing call (keys = NULL, cap = 0), which does the whole sample too.  off has
 * num_partitions entries.  Deterministic: the same committed pairs give the same splitters on every rank and call.
 * Keys longer than the record class (host side, see mrhbm_emit_str) are not sampled.  mrhbm_checksum_result refuses
 * (MRHBM_E_INVAL) once the splitters differ from those of the last shuffle. */
int mrhbm_sample_splitters(mrhbm_ctx *, void *keys, size_t cap, uint64_t *off, size_t *need);

/* ---- reduce side: utils.merge_iterator consumer (utils.lua:206-271, job.lua:264-284)
 *      and finalfn's pair iterator (server.lua:360-385) ---- */
int mrhbm_groups_open(mrhbm_ctx *, uint32_t partition, mrhbm_iter **out);
/* 1 = one group, 0 = end, <0 = error.  Ascending key order (C-locale bytewise; u64
 * numeric).  *key points at klen key bytes (u64 keys: 8 bytes big endian, SURVEY A.4);
 * values/nvalues is the reduced list (built-in sum: one value; MRHBM_RED_NONE: all values of the
 * key).  Pointers stay valid
 * until the next call on this iterator. */
int mrhbm_groups_next(mrhbm_iter *, const void **key, size_t *klen, const uint64_t **values,
                      size_t *nvalues);
/* MRHBM_F_BYTE_VALUES: the next group as mrhbm_groups_next gives it (same key order, long keys merged in, same pointer
 * lifetime), with its nvalues values packed in *vals: value i is (*vals)[(*voff)[i] .. (*voff)[i+1]). */
int mrhbm_groups_next_values(mrhbm_iter *, const void **key, size_t *klen, const void **vals, const uint64_t **voff,
                             size_t *nvalues);
void mrhbm_groups_close(mrhbm_iter *);

/* ---- bulk result access (finalfn feed without per-group calls) ---- */
typedef struct mrhbm_result_info {
  uint64_t pairs_in;   /* pairs committed on this rank */
  uint64_t pairs_recv; /* pairs this rank reduced (after the exchange) */
  uint64_t groups;     /* distinct keys owned by this rank */
  uint32_t key_bytes;  /* bytes per key slot in result_copy (8 or RB-4) */
  uint32_t sorted;     /* 1: each partition is one ascending run on the device (with MRHBM_PART_RANGE the
                          partition-major rows are then ascending as a whole);
                          0: a partition is several ascending runs, merged by the iterator */
  uint32_t runs_per_partition;
  uint32_t partitions_nonempty;
} mrhbm_result_info;
/* `groups` counts the rows mrhbm_result_copy returns; groups whose key is longer than a slot (mrhbm_emit_str) are not
 * among them -- mrhbm_partitions and mrhbm_groups_* see both kinds. */
int mrhbm_result_info_get(mrhbm_ctx *, mrhbm_result_info *);
/* copies all groups of this rank, partition-major, to host: keys (groups*key_bytes; u64
 * keys native little endian) and sums (groups*8); part_off[P+1] receives group offsets.
 * Inside a partition the order is ascending iff info.sorted, else run-major.
 * MRHBM_E_KEY when the result holds keys longer than a slot (see mrhbm_emit_str): iterate instead. */
int mrhbm_result_copy(mrhbm_ctx *, void *keys, uint64_t *sums, uint64_t *part_off);
/* MRHBM_F_BYTE_VALUES: the value bytes of this rank's rows in mrhbm_result_copy row order; row r's value is
 * vals[row_off[r] .. row_off[r+1]) (row_off: groups + 1 entries).  *need receives the bytes; vals = NULL only sizes
 * (row_off is then not written); MRHBM_E_INVAL when cap < *need.  MRHBM_E_KEY as for mrhbm_result_copy. */
int mrhbm_result_values(mrhbm_ctx *, void *vals, size_t cap, uint64_t *row_off, size_t *need);
/* size-independent parity properties computed on the device:
 *  in[0..3]  = { sum f1(key)*v, sum f2(key)*v, sum v, pairs }       over committed pairs
 *  out[0..3] = { sum f1(key)*s, sum f2(key)*s, sum s, groups }      over reduced groups
 *  out[4] = adjacent keys not strictly ascending inside a run, out[5] = groups whose
 *  partitioner(key) differs from the partition they sit in.  All mod 2^64.
 * Linearity of the sum makes in[0..2] == out[0..2] for a correct group-by. */
int mrhbm_checksum_input(mrhbm_ctx *, uint64_t in[4]);
int mrhbm_checksum_result(mrhbm_ctx *, uint64_t out[6]);

/* ---- measurement ---- */
typedef struct mrhbm_stats {
  float ms_total;     /* last shuffle, CUDA events on the ctx stream */
  float ms_combine, ms_hist, ms_plan, ms_scatter, ms_exchange, ms_sort_reduce, ms_bigbins;
  uint32_t launches;  /* kernels launched by the last shuffle */
  uint32_t bins, big_bins, sub_bins, attempts;
  uint64_t pairs, groups, bytes_exchanged;
  float ms_setup;     /* key sampling, job-wide agreement, buffer set-up, counter clears (between combine and hist/level 1) */
  float ms_finish;    /* offsets of the groups, totals, error flags back to the host (after the sort) */
} mrhbm_stats;
int mrhbm_stats_get(mrhbm_ctx *, mrhbm_stats *);
/* drops committed pairs and results, keeps buffers (next iteration of a "loop" task,
 * server.lua:386-404) */
int mrhbm_reset(mrhbm_ctx *);

/* ---- multi-GPU: one ctx per rank, partition p is owned by rank p % world ---- */
#define MRHBM_UNIQUE_ID_BYTES 128
int mrhbm_comm_unique_id(mrhbm_ctx *, void *id /* MRHBM_UNIQUE_ID_BYTES, rank 0 */);
int mrhbm_comm_init(mrhbm_ctx *, const void *id, int rank, int world);

#ifdef __cplusplus
}
#endif
#endif
