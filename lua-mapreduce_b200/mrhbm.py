"""ctypes binding of the C ABI in include/mrhbm.h -- the same entry points the Lua 5.2 C module
(lua/mrhbm_lua.c) binds.  Thin by design: every method is one C call plus error conversion to
the reference's ``nil, msg`` style (here: MrhbmError).  There is no CPU fallback: loading fails
loudly when lib/libmrhbm.so is missing, and Ctx() fails when no sm_90 GPU (H100) is present.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build

KEY_U64, KEY_STR = 0, 1
PART_FNV_LUA, PART_MULHASH, PART_WORDHASH, PART_RANGE = 0, 1, 2, 3
RED_SUM, RED_NONE, RED_DISTINCT, RED_FSUM, RED_COUNT_DISTINCT = 0, 1, 2, 3, 4
COMBINE_NONE, COMBINE_REDUCER, COMBINE_DISTINCT, COMBINE_FSUM = 0, 1, 2, 3
F_FORCE_RUNS, F_SMALL_BINS, F_NO_OPTIMISTIC, F_BYTE_VALUES = 1, 2, 4, 8
E_NODEVICE = -8
UNIQUE_ID_BYTES = 128


class MrhbmError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("mrhbm error %d: %s" % (code, msg))
        self.code = code


class Config(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("key_kind", C.c_uint32),
                ("max_key_bytes", C.c_uint32), ("num_partitions", C.c_uint32), ("partitioner", C.c_uint32),
                ("reducer", C.c_uint32), ("combiner", C.c_uint32), ("reserve_pairs", C.c_uint64),
                ("flags", C.c_uint32), ("reserved", C.c_uint32)]


class ResultInfo(C.Structure):
    _fields_ = [("pairs_in", C.c_uint64), ("pairs_recv", C.c_uint64), ("groups", C.c_uint64),
                ("key_bytes", C.c_uint32), ("sorted", C.c_uint32), ("runs_per_partition", C.c_uint32),
                ("partitions_nonempty", C.c_uint32)]


class Stats(C.Structure):
    _fields_ = [("ms_total", C.c_float), ("ms_combine", C.c_float), ("ms_hist", C.c_float),
                ("ms_plan", C.c_float), ("ms_scatter", C.c_float), ("ms_exchange", C.c_float),
                ("ms_sort_reduce", C.c_float), ("ms_bigbins", C.c_float), ("launches", C.c_uint32),
                ("bins", C.c_uint32), ("big_bins", C.c_uint32), ("sub_bins", C.c_uint32),
                ("attempts", C.c_uint32), ("pairs", C.c_uint64), ("groups", C.c_uint64),
                ("bytes_exchanged", C.c_uint64), ("ms_setup", C.c_float), ("ms_finish", C.c_float)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


EXPORTS = [
    "mrhbm_abi_version", "mrhbm_init", "mrhbm_destroy", "mrhbm_last_error", "mrhbm_record_bytes",
    "mrhbm_host_alloc", "mrhbm_host_free", "mrhbm_map_begin", "mrhbm_emit_str", "mrhbm_emit_u64",
    "mrhbm_emit_batch", "mrhbm_emit_device", "mrhbm_map_gen_u64", "mrhbm_map_gen_zipf", "mrhbm_map_wordcount", "mrhbm_synth_zipf_text", "mrhbm_pool_read", "mrhbm_map_commit",
    "mrhbm_map_abort", "mrhbm_shuffle", "mrhbm_partitions", "mrhbm_groups_open", "mrhbm_groups_next",
    "mrhbm_groups_close", "mrhbm_result_info_get", "mrhbm_result_copy", "mrhbm_checksum_input",
    "mrhbm_checksum_result", "mrhbm_stats_get", "mrhbm_reset", "mrhbm_comm_unique_id", "mrhbm_comm_init",
    "mrhbm_set_splitters", "mrhbm_sample_splitters", "mrhbm_emit_str_value", "mrhbm_emit_u64_value",
    "mrhbm_emit_batch_values", "mrhbm_groups_next_values", "mrhbm_result_values", "mrhbm_map_words_value",
    "mrhbm_map_key_numbers",
]

_lib = None


def lib_path():
    return _build.LIB


def load(build_if_missing=True):
    """dlopens lib/libmrhbm.so; raises if it cannot be built/loaded (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if build_if_missing and _build.needs_build():
        _build.build()
    if not os.path.exists(path):
        raise MrhbmError(-1, "libmrhbm.so is missing (%s) and there is no CPU fallback" % path)
    L = C.CDLL(path, mode=C.RTLD_GLOBAL)
    vp, sz, u64, u32, i = C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint32, C.c_int

    def sig(name, res, *args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = list(args)

    sig("mrhbm_abi_version", i)
    sig("mrhbm_init", i, C.POINTER(Config), C.POINTER(vp))
    sig("mrhbm_destroy", None, vp)
    sig("mrhbm_last_error", C.c_char_p, vp)
    sig("mrhbm_record_bytes", u32, vp)
    sig("mrhbm_host_alloc", vp, vp, sz)
    sig("mrhbm_host_free", None, vp, vp)
    sig("mrhbm_map_begin", i, vp, C.c_char_p, C.POINTER(vp))
    sig("mrhbm_emit_str", i, vp, C.c_char_p, sz, u32)
    sig("mrhbm_emit_u64", i, vp, u64, u64)
    sig("mrhbm_emit_batch", i, vp, vp, sz)
    sig("mrhbm_emit_device", i, vp, vp, sz)
    sig("mrhbm_map_gen_u64", i, vp, u64, u64, u64)
    sig("mrhbm_map_gen_zipf", i, vp, u64, u64, u64, vp, u64)
    sig("mrhbm_map_wordcount", i, vp, vp, sz, C.POINTER(u64))
    sig("mrhbm_synth_zipf_text", i, u64, u64, u64, u32, vp, u64, vp, sz, C.POINTER(sz), i)
    sig("mrhbm_pool_read", i, vp, u64, u64, vp)
    sig("mrhbm_map_commit", i, vp)
    sig("mrhbm_map_abort", None, vp)
    sig("mrhbm_shuffle", i, vp)
    sig("mrhbm_partitions", i, vp, vp, sz, C.POINTER(sz))
    sig("mrhbm_groups_open", i, vp, u32, C.POINTER(vp))
    sig("mrhbm_groups_next", i, vp, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.POINTER(sz))
    sig("mrhbm_groups_close", None, vp)
    sig("mrhbm_result_info_get", i, vp, C.POINTER(ResultInfo))
    sig("mrhbm_result_copy", i, vp, vp, vp, vp)
    sig("mrhbm_checksum_input", i, vp, vp)
    sig("mrhbm_checksum_result", i, vp, vp)
    sig("mrhbm_stats_get", i, vp, C.POINTER(Stats))
    sig("mrhbm_reset", i, vp)
    sig("mrhbm_comm_unique_id", i, vp, vp)
    sig("mrhbm_comm_init", i, vp, vp, i, i)
    sig("mrhbm_set_splitters", i, vp, vp, C.POINTER(u64), sz)
    sig("mrhbm_sample_splitters", i, vp, vp, sz, C.POINTER(u64), C.POINTER(sz))
    sig("mrhbm_emit_str_value", i, vp, C.c_char_p, sz, C.c_char_p, sz)
    sig("mrhbm_emit_u64_value", i, vp, u64, C.c_char_p, sz)
    sig("mrhbm_emit_batch_values", i, vp, vp, sz, vp, vp)
    sig("mrhbm_groups_next_values", i, vp, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.POINTER(vp), C.POINTER(sz))
    sig("mrhbm_result_values", i, vp, vp, sz, vp, C.POINTER(sz))
    sig("mrhbm_map_words_value", i, vp, vp, sz, C.c_char_p, sz, C.POINTER(u64))
    sig("mrhbm_map_key_numbers", i, vp, vp, sz, C.POINTER(u64))
    _lib = L
    return L


def synth_zipf_text(seed, first, n, table, words_per_line=25, out=None, threads=None):
    """SURVEY App. B word-count text of words [first, first+n) of the Zipf word stream (host side generator in
    libmrhbm).  Returns a uint8 array (a view of `out` when given)."""
    L = load()
    t = np.ascontiguousarray(table, dtype=np.uint64)
    threads = threads or min(os.cpu_count() or 1, 128)
    need = C.c_size_t()
    if out is None:
        L.mrhbm_synth_zipf_text(seed, first, n, words_per_line, t.ctypes.data, t.size, None, 0, C.byref(need), threads)
        out = np.empty(need.value, dtype=np.uint8)
    rc = L.mrhbm_synth_zipf_text(seed, first, n, words_per_line, t.ctypes.data, t.size, out.ctypes.data, out.nbytes,
                                 C.byref(need), threads)
    if rc != 0:
        raise MrhbmError(rc, "synth_zipf_text: the text needs %d bytes, the buffer holds %d" % (need.value, out.nbytes))
    return out[:need.value]


def splitter_bytes(key_kind, x):
    """A splitter in the C form: the original key bytes (u64 keys: 8 big-endian bytes)."""
    if key_kind == KEY_U64:
        if isinstance(x, (bytes, bytearray)):
            return bytes(x)
        return int(x).to_bytes(8, "big")
    return x.encode() if isinstance(x, str) else bytes(x)


def record_dtype(key_kind, max_key_bytes=27):
    """numpy dtype of one emit_batch record."""
    if key_kind == KEY_U64:
        return np.dtype([("key", "<u8"), ("val", "<u8")])
    rb = 32 if max_key_bytes <= 27 else 64 if max_key_bytes <= 59 else 128
    return np.dtype([("key", "S%d" % (rb - 4)), ("val", "<u4")])


class Map:
    """One map job's emit handle (mapreduce/job.lua:83-97)."""

    def __init__(self, ctx, job_id):
        self.ctx, self.h = ctx, C.c_void_p()
        ctx._chk(ctx.L.mrhbm_map_begin(ctx.h, str(job_id).encode(), C.byref(self.h)))

    def emit(self, key, value=1):
        if self.ctx.byte_values:  # any bytes (F_BYTE_VALUES)
            if not isinstance(value, (bytes, bytearray)):
                raise MrhbmError(-1, "a byte-values ctx takes bytes values, got %r" % type(value).__name__)
            v = bytes(value)
            if isinstance(key, int):
                rc = self.ctx.L.mrhbm_emit_u64_value(self.h, key, v, len(v))
            else:
                rc = self.ctx.L.mrhbm_emit_str_value(self.h, key, len(key), v, len(v))
            self.ctx._chk(rc)
            return
        # values are unsigned integers: < 2^32 in string records, < 2^53 (exact Lua numbers) with u64 keys;
        # ctypes would silently wrap or truncate anything else
        u64 = isinstance(key, int)
        if not (isinstance(value, (int, np.integer)) or float(value).is_integer()) or not 0 <= value < (1 << 53 if u64 else 1 << 32):
            raise MrhbmError(-1, "value must be an integer in [0, 2^%d), got %r" % (53 if u64 else 32, value))
        if u64:
            rc = self.ctx.L.mrhbm_emit_u64(self.h, key, int(value))
        else:
            rc = self.ctx.L.mrhbm_emit_str(self.h, key, len(key), int(value))
        self.ctx._chk(rc)

    def emit_batch(self, recs):
        a = np.ascontiguousarray(recs)
        assert a.dtype.itemsize == self.ctx.record_bytes, "record layout mismatch"
        self.ctx._chk(self.ctx.L.mrhbm_emit_batch(self.h, a.ctypes.data, a.shape[0]))

    def emit_batch_values(self, recs, blob, voff):
        """F_BYTE_VALUES: records in the ctx layout (value field ignored); value i is blob[voff[i]:voff[i+1]].
        numpy arrays (pinned ones from Ctx.pinned_array too) or bytes for the blob."""
        a = np.ascontiguousarray(recs)
        assert a.dtype.itemsize == self.ctx.record_bytes, "record layout mismatch"
        b = np.frombuffer(blob, dtype=np.uint8) if isinstance(blob, (bytes, bytearray)) else np.ascontiguousarray(blob)
        o = np.ascontiguousarray(voff, dtype=np.uint64)
        if o.shape[0] != a.shape[0] + 1:
            raise MrhbmError(-1, "emit_batch_values: %d records need %d offsets, got %d" % (a.shape[0], a.shape[0] + 1, o.shape[0]))
        if a.shape[0] and int(o[-1]) > b.nbytes:
            raise MrhbmError(-1, "emit_batch_values: offsets reach %d, the blob holds %d bytes" % (int(o[-1]), b.nbytes))
        self.ctx._chk(self.ctx.L.mrhbm_emit_batch_values(self.h, a.ctypes.data, a.shape[0], b.ctypes.data if b.nbytes else None,
                                                         o.ctypes.data))

    def emit_batch_ptr(self, ptr, n):
        self.ctx._chk(self.ctx.L.mrhbm_emit_batch(self.h, ptr, n))

    def emit_device(self, dev_ptr, n):
        self.ctx._chk(self.ctx.L.mrhbm_emit_device(self.h, dev_ptr, n))

    def gen_u64(self, seed, start, n):
        self.ctx._chk(self.ctx.L.mrhbm_map_gen_u64(self.h, seed, start, n))

    def gen_zipf(self, seed, start, n, table):
        t = np.ascontiguousarray(table, dtype=np.uint64)
        self.ctx._chk(self.ctx.L.mrhbm_map_gen_zipf(self.h, seed, start, n, t.ctypes.data, t.size))

    @staticmethod
    def _text(text, nbytes):
        """(address, bytes, object that keeps the memory alive) of a text buffer"""
        if isinstance(text, (bytes, bytearray)):
            keep = C.create_string_buffer(bytes(text), len(text)) if isinstance(text, bytearray) else text
            return C.cast(C.c_char_p(keep), C.c_void_p), len(text), keep
        if isinstance(text, np.ndarray):
            return C.c_void_p(text.ctypes.data), text.nbytes, text
        return C.c_void_p(int(text)), nbytes, None

    def wordcount(self, text, nbytes=None):
        """device-side WordCount mapfn over a text buffer (bytes, a uint8 numpy array, or an address with
        nbytes); returns the number of words emitted"""
        n = C.c_uint64()
        ptr, nbytes, keep = self._text(text, nbytes)
        self.ctx._chk(self.ctx.L.mrhbm_map_wordcount(self.h, ptr, nbytes, C.byref(n)))
        return n.value

    def words_value(self, text, value, nbytes=None):
        """F_BYTE_VALUES: the device tokeniser of wordcount emitting (word, value) for every word of the text (text
        as for wordcount, value bytes); returns the number of words emitted"""
        if not isinstance(value, (bytes, bytearray)):
            raise MrhbmError(-1, "words_value takes a bytes value, got %r" % type(value).__name__)
        v = bytes(value)
        n = C.c_uint64()
        ptr, nbytes, keep = self._text(text, nbytes)
        self.ctx._chk(self.ctx.L.mrhbm_map_words_value(self.h, ptr, nbytes, v, len(v), C.byref(n)))
        return n.value

    def key_numbers(self, text, nbytes=None):
        """F_BYTE_VALUES, string keys: every line "key number" of the text (text as for wordcount) becomes the pair
        (key, tuple.encode_value(float(number))), parsed on the device (see mrhbm_map_key_numbers); returns the number
        of pairs emitted"""
        n = C.c_uint64()
        ptr, nbytes, keep = self._text(text, nbytes)
        self.ctx._chk(self.ctx.L.mrhbm_map_key_numbers(self.h, ptr, nbytes, C.byref(n)))
        return n.value

    def commit(self):
        h, self.h = self.h, None
        self.ctx._chk(self.ctx.L.mrhbm_map_commit(h))

    def abort(self):
        if self.h:
            h, self.h = self.h, None
            self.ctx.L.mrhbm_map_abort(h)


class Ctx:
    """One GPU's shuffle context (storage = "hbm")."""

    def __init__(self, key_kind=KEY_STR, num_partitions=15, partitioner=None, max_key_bytes=27,
                 combiner=False, device=-1, reserve_pairs=0, flags=0, reducer=RED_SUM):
        self.L = load()
        if partitioner is None:
            partitioner = PART_MULHASH if key_kind == KEY_U64 else PART_FNV_LUA
        # combiner: a bool (False / True = COMBINE_REDUCER), COMBINE_DISTINCT or COMBINE_FSUM (byte values, see
        # include/mrhbm.h)
        combiner = combiner if combiner in (COMBINE_DISTINCT, COMBINE_FSUM) else int(bool(combiner))
        self.cfg = Config(C.sizeof(Config), device, key_kind, max_key_bytes, num_partitions, partitioner,
                          reducer, combiner, reserve_pairs, flags, 0)
        self.h = C.c_void_p()
        rc = self.L.mrhbm_init(C.byref(self.cfg), C.byref(self.h))
        if rc != 0:
            msg = self.L.mrhbm_last_error(self.h).decode() if self.h else "mrhbm_init failed"
            if self.h:
                self.L.mrhbm_destroy(self.h)
            self.h = None
            raise MrhbmError(rc, msg)
        self.key_kind = key_kind
        self.num_partitions = num_partitions
        self.byte_values = bool(flags & F_BYTE_VALUES)
        self.record_bytes = self.L.mrhbm_record_bytes(self.h)

    def _chk(self, rc):
        if rc < 0:
            raise MrhbmError(rc, self.L.mrhbm_last_error(self.h).decode())
        return rc

    def close(self):
        if getattr(self, "h", None):
            self.L.mrhbm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # -- map side
    def map_begin(self, job_id):
        return Map(self, job_id)

    def host_alloc(self, nbytes):
        p = self.L.mrhbm_host_alloc(self.h, nbytes)
        if not p:
            raise MrhbmError(-3, "pinned allocation failed")
        return p

    def host_free(self, p):
        self.L.mrhbm_host_free(self.h, p)

    def pinned_array(self, n, dtype):
        """numpy view over pinned host memory (free with host_free(arr.ctypes.data))."""
        dt = np.dtype(dtype)
        p = self.host_alloc(max(1, n * dt.itemsize))
        buf = (C.c_char * (n * dt.itemsize)).from_address(p)
        return np.frombuffer(buf, dtype=dt, count=n)

    def pool_read(self, first, n, out=None):
        if out is None:
            out = np.empty(n, dtype=record_dtype(self.key_kind, self.cfg.max_key_bytes))
        self._chk(self.L.mrhbm_pool_read(self.h, first, n, out.ctypes.data))
        return out

    # -- barrier
    def shuffle(self):
        self._chk(self.L.mrhbm_shuffle(self.h))

    def reset(self):
        self._chk(self.L.mrhbm_reset(self.h))

    def partitions(self):
        n = C.c_size_t()
        ids = (C.c_uint32 * self.num_partitions)()
        self._chk(self.L.mrhbm_partitions(self.h, ids, self.num_partitions, C.byref(n)))
        return list(ids[:n.value])

    # -- reduce side
    def groups(self, partition):
        """Yields (key bytes, [values]) in ascending key order (utils.merge_iterator order); with F_BYTE_VALUES the
        values are bytes."""
        it = C.c_void_p()
        self._chk(self.L.mrhbm_groups_open(self.h, partition, C.byref(it)))
        kp, kl, vp, vn, op = C.c_void_p(), C.c_size_t(), C.c_void_p(), C.c_size_t(), C.c_void_p()
        try:
            while True:
                if self.byte_values:
                    r = self._chk(self.L.mrhbm_groups_next_values(it, C.byref(kp), C.byref(kl), C.byref(vp), C.byref(op),
                                                                  C.byref(vn)))
                else:
                    r = self._chk(self.L.mrhbm_groups_next(it, C.byref(kp), C.byref(kl), C.byref(vp), C.byref(vn)))
                if r == 0:
                    return
                key = C.string_at(kp, kl.value) if kl.value else b""
                if self.byte_values:
                    off = (C.c_uint64 * (vn.value + 1)).from_address(op.value)
                    blob = C.string_at(vp, off[vn.value]) if off[vn.value] else b""
                    yield key, [blob[off[j]:off[j + 1]] for j in range(vn.value)]
                else:
                    yield key, list((C.c_uint64 * vn.value).from_address(vp.value))
        finally:
            self.L.mrhbm_groups_close(it)

    def result_info(self):
        info = ResultInfo()
        self._chk(self.L.mrhbm_result_info_get(self.h, C.byref(info)))
        return info

    def result_copy(self, keys=None, sums=None):
        """(keys, sums, part_off): all groups of this rank, partition-major (F_BYTE_VALUES: sums is None, see
        result_values)."""
        info = self.result_info()
        g = info.groups
        if keys is None:
            keys = np.empty(max(g, 1), dtype=np.uint64 if self.key_kind == KEY_U64 else "S%d" % info.key_bytes)
        if self.byte_values:  # rows carry value ids, their bytes come from result_values
            if keys.shape[0] < g:
                raise MrhbmError(-1, "result_copy: the key array holds %d groups, %d needed" % (keys.shape[0], g))
            po = np.empty(self.num_partitions + 1, dtype=np.uint64)
            self._chk(self.L.mrhbm_result_copy(self.h, keys.ctypes.data, None, po.ctypes.data))
            return keys[:g], None, po
        if sums is None:
            sums = np.empty(max(g, 1), dtype=np.uint64)
        if keys.shape[0] < g or sums.shape[0] < g:
            raise MrhbmError(-1, "result_copy: output arrays hold %d groups, %d needed" % (min(keys.shape[0], sums.shape[0]), g))
        po = np.empty(self.num_partitions + 1, dtype=np.uint64)
        self._chk(self.L.mrhbm_result_copy(self.h, keys.ctypes.data, sums.ctypes.data, po.ctypes.data))
        return keys[:g], sums[:g], po

    def result_values(self):
        """F_BYTE_VALUES: (uint8 blob, uint64 row_off) -- row r's value is blob[row_off[r]:row_off[r+1]], rows in
        result_copy order."""
        need = C.c_size_t()
        self._chk(self.L.mrhbm_result_values(self.h, None, 0, None, C.byref(need)))
        blob = np.empty(max(need.value, 1), dtype=np.uint8)
        row_off = np.empty(self.result_info().groups + 1, dtype=np.uint64)
        self._chk(self.L.mrhbm_result_values(self.h, blob.ctypes.data, blob.nbytes, row_off.ctypes.data, C.byref(need)))
        return blob[:need.value], row_off

    def checksum_input(self):
        a = (C.c_uint64 * 4)()
        self._chk(self.L.mrhbm_checksum_input(self.h, a))
        return list(a)

    def checksum_result(self):
        a = (C.c_uint64 * 6)()
        self._chk(self.L.mrhbm_checksum_result(self.h, a))
        return list(a)

    def stats(self):
        s = Stats()
        self._chk(self.L.mrhbm_stats_get(self.h, C.byref(s)))
        return s.asdict()

    # -- range partitioner
    def set_splitters(self, splitters):
        """PART_RANGE: installs the num_partitions - 1 non-decreasing splitters (bytes / str for string keys, ints for
        u64 keys); partition k then holds the keys k splitters are <= to (bisect_right)."""
        raw = [splitter_bytes(self.key_kind, x) for x in splitters]
        keys = b"".join(raw)
        off = (C.c_uint64 * (len(raw) + 1))()
        o = 0
        for i, r in enumerate(raw):
            off[i] = o
            o += len(r)
        off[len(raw)] = o
        buf = C.create_string_buffer(keys, max(1, len(keys)))
        self._chk(self.L.mrhbm_set_splitters(self.h, buf, off, len(raw)))

    def sample_splitters(self):
        """PART_RANGE: quantile splitters from a sample of the committed pairs (collective on several GPUs); installs
        and returns them (bytes for string keys, ints for u64 keys)."""
        n = self.num_partitions - 1
        off = (C.c_uint64 * (n + 1))()
        need = C.c_size_t()
        slot = 8 if self.key_kind == KEY_U64 else self.record_bytes - 4  # a splitter takes at most one key slot
        buf = C.create_string_buffer(max(1, n * slot))
        self._chk(self.L.mrhbm_sample_splitters(self.h, buf, max(1, n * slot), off, C.byref(need)))
        raw = buf.raw
        out = [raw[off[i]:off[i + 1]] for i in range(n)]
        return [int.from_bytes(x, "big") for x in out] if self.key_kind == KEY_U64 else out

    # -- multi-GPU
    def comm_unique_id(self):
        buf = (C.c_char * UNIQUE_ID_BYTES)()
        self._chk(self.L.mrhbm_comm_unique_id(self.h, buf))
        return bytes(buf)

    def comm_init(self, uid, rank, world):
        self._chk(self.L.mrhbm_comm_init(self.h, uid, rank, world))
