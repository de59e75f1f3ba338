"""Map and reduce job bodies (mapreduce/job.lua) over the HBM shuffle.

Map job (job.lua:83-97,166-227): `emit(k, v)` goes to mrhbm_emit_* instead of the Lua table;
keys_sorted / combiner / partitionfn / text spill are what mrhbm_shuffle does on the device.
Reduce job (job.lua:230-296): the (key, values) stream of utils.merge_iterator becomes
mrhbm_groups_next; the reducer algebra (job.lua:264-284) is kept."""
import importlib
import math
import time

from . import tuple as tuple_keys
from .utils import STATUS

_initialized = set()
_funcs = {}


def get_func(fname, func, args):
    """job.lua:64-76: require(fname), run its init once per process, return the module."""
    m = _funcs.get(fname)
    if m is None:
        m = importlib.import_module(fname)
        init = getattr(m, "init", None)
        if init is not None and init not in _initialized:
            init(args)
            _initialized.add(init)
        assert hasattr(m, func), "Module %s must provide %s" % (fname, func)
        _funcs[fname] = m
    return m


def _key_bytes(k):
    if isinstance(k, bytes):
        return k
    if isinstance(k, str):
        return k.encode()
    raise TypeError("hbm storage takes string keys (or ints with key_kind='u64'), got %r" % type(k))


class Job:
    def __init__(self, board, ns, doc, config):
        self.board, self.ns, self.doc, self.cfg = board, ns, doc, config
        self.written = False

    def get_id(self):
        return self.doc["_id"]

    def execute(self):
        t0 = time.process_time()
        self.t = time.time()
        (self._map if self.ns == "map_jobs" else self._reduce)()
        return time.process_time() - t0

    # ---- job.lua:166-227
    def _map(self):
        cfg, ctx = self.cfg, self.board.ctx
        mod = get_func(cfg["mapfn"], "mapfn", None)  # init(nil): the job.lua:369 quirk
        mapfn = mod.mapfn
        m = ctx.map_begin(self.get_id())
        try:
            hbm_mapfn = getattr(mod, "hbm_mapfn", None)
            if hbm_mapfn == "wordcount_file" and hasattr(m, "wordcount"):
                # declared built-in (same opt-in pattern as hbm_reducefn): the job value is a file
                # path, the device tokenises its bytes exactly like examples/WordCount/mapfn.lua:3-9
                with open(self.doc["value"], "rb") as fh:
                    m.wordcount(fh.read())
                mapfn = None
            elif hbm_mapfn == "words_file" and hasattr(m, "words_value"):
                # the same tokeniser pairing every word with the job value (the file path): an inverted index
                with open(self.doc["value"], "rb") as fh:
                    m.words_value(fh.read(), tuple_keys.encode_value(self.doc["value"]))
                mapfn = None
            elif hbm_mapfn == "key_numbers_file" and hasattr(m, "key_numbers"):
                # the job value is a file of lines "key number": the device parses them, emit(key, float(number))
                with open(self.doc["value"], "rb") as fh:
                    m.key_numbers(fh.read())
                mapfn = None
            kind = cfg["hbm"]["key_kind"]
            if kind == "u64":
                enc_key = int
            elif kind == "tuple":
                enc_key = tuple_keys.encode  # composite keys (tuple.lua): order-preserving byte strings across the C ABI
            else:
                enc_key = _key_bytes
            # value_kind = "bytes": Lua strings and numbers as tagged bytes (tuple.encode_value); else integers
            enc_val = tuple_keys.encode_value if cfg["hbm"].get("value_kind") == "bytes" else int

            def emit(key, value=1):
                m.emit(enc_key(key), enc_val(value))
            if mapfn is not None:
                mapfn(self.get_id(), self.doc["value"], emit)  # job.lua:182
            self.board.mark(self.doc, STATUS.FINISHED, finished_time=time.time())
            m.commit()  # atomic publish; replaces an earlier attempt (job.lua:217-221)
        except BaseException:
            m.abort()   # BROKEN job: nothing becomes visible (worker.lua:120-127)
            raise
        self.written = True
        self.board.mark(self.doc, STATUS.WRITTEN, written_time=time.time(), real_time=time.time() - self.t)

    def _bulk_groups(self, part):
        """[(key, [sum])] of one partition in ascending key order from ONE bulk copy of the shuffle's result
        (mrhbm_result_copy, cached on the board per shuffle) instead of one mrhbm_groups_next call per group.
        None when the ctx offers no bulk access (test stand-ins)."""
        import numpy as np
        b, ctx = self.board, self.board.ctx
        if not hasattr(ctx, "result_copy") or not hasattr(ctx, "result_info"):
            return None
        cache = getattr(b, "_bulk", None)
        if cache is None or cache[0] is not ctx or cache[1] != b.iteration:
            try:
                keys, sums, po = ctx.result_copy()
            except Exception as e:  # keys longer than a result slot live on the host side: the iterator merges them in
                if getattr(e, "code", None) != -4:  # MRHBM_E_KEY
                    raise
                b._bulk = (ctx, b.iteration, None, None, None, False)
                return None
            cache = b._bulk = (ctx, b.iteration, keys, sums, po, bool(ctx.result_info().sorted))
        _, _, keys, sums, po, is_sorted = cache
        if keys is None:
            return None
        a, e = int(po[part]), int(po[part + 1])
        k, v = keys[a:e], sums[a:e]
        if not is_sorted:  # several ascending runs (hash sub-bins): merge = stable sort by key
            order = np.argsort(k, kind="stable")
            k, v = k[order], v[order]
        if k.dtype.kind == "u":  # u64 keys are the reference's 8-byte big-endian strings (SURVEY A.4)
            ks = [int(x).to_bytes(8, "big") for x in k.tolist()]
        else:
            ks = k.tolist()  # numpy drops the zero padding
            if any(b"\x01" in x for x in ks):  # escaped 0x00 / 0x01 bytes (mrhbm_emit_str)
                ks = [x.replace(b"\x01\x01", b"\x00").replace(b"\x01\x02", b"\x01") if b"\x01" in x else x for x in ks]
        return [(kk, [vv]) for kk, vv in zip(ks, v.tolist())]

    def _bulk_numbers(self, part):
        """hbm_reducefn = "fsum" or "count_distinct": [(key, [number])] of one partition in ascending key order from
        one bulk copy of the shuffle's keys and values (mrhbm_result_copy + mrhbm_result_values, cached on the board
        per shuffle), the device's single number per key (a sum, or a count of distinct values) handed out as the
        reducefn's result.  None when the ctx offers no bulk access (keys longer than a result slot, test stand-ins):
        the iterator gives the same values."""
        import numpy as np
        b, ctx = self.board, self.board.ctx
        if not hasattr(ctx, "result_values"):
            return None
        cache = getattr(b, "_bulk_numbers", None)
        if cache is None or cache[0] is not ctx or cache[1] != b.iteration:
            try:
                keys, _, po = ctx.result_copy()
                blob, _ = ctx.result_values()
            except Exception as e:
                if getattr(e, "code", None) != -4:  # MRHBM_E_KEY
                    raise
                b._bulk_numbers = (ctx, b.iteration, None, None, None, False)
                return None
            cache = b._bulk_numbers = (ctx, b.iteration, keys, blob, po, bool(ctx.result_info().sorted))
        _, _, keys, blob, po, is_sorted = cache
        if keys is None:
            return None
        a, e = int(po[part]), int(po[part + 1])
        k = keys[a:e]
        # every row's value is the 11-byte number at 11 r: the sign-folded double in ten 7-bit groups
        g = blob[11 * a:11 * e].reshape(-1, 11)[:, 1:].astype(np.uint64) & np.uint64(0x7F)
        u = np.zeros(e - a, dtype=np.uint64)
        for j in range(10):
            u = (u << np.uint64(7)) | g[:, j]
        top = (u >> np.uint64(63)).astype(bool)
        bits = np.where(top, u & np.uint64(0x7FFFFFFFFFFFFFFF), ~u)
        v = bits.view(np.float64)
        if not is_sorted:  # several ascending runs (hash sub-bins): merge = stable sort by key
            order = np.argsort(k, kind="stable")
            k, v = k[order], v[order]
        if k.dtype.kind == "u":
            ks = [int(x).to_bytes(8, "big") for x in k.tolist()]
        else:
            ks = k.tolist()
            if any(b"\x01" in x for x in ks):  # escaped 0x00 / 0x01 bytes (mrhbm_emit_str)
                ks = [x.replace(b"\x01\x01", b"\x00").replace(b"\x01\x02", b"\x01") if b"\x01" in x else x for x in ks]
        # as tuple.decode_value gives them: integral numbers as ints, -0 as -0.0
        return [(kk, [int(f) if f.is_integer() and abs(f) <= (1 << 53) and not (f == 0 and math.copysign(1, f) < 0)
                      else f]) for kk, f in zip(ks, v.tolist())]

    # ---- job.lua:230-296
    def _reduce(self):
        cfg, ctx = self.cfg, self.board.ctx
        mod = get_func(cfg["reducefn"], "reducefn", None)
        aci = all(getattr(mod, f, False) for f in
                  ("associative_reducer", "commutative_reducer", "idempotent_reducer"))
        part = int(self.doc["_id"])
        out, result = [], []

        def emit(v):
            result.append(v)

        decode = tuple_keys.decode if cfg["hbm"]["key_kind"] == "tuple" else None
        byte_values = cfg["hbm"].get("value_kind") == "bytes"
        device_distinct = cfg["hbm"].get("reducer") == 2  # hbm_reducefn = "distinct": the values are its output
        # hbm_reducefn = "fsum" or "count_distinct": one number per key, in bulk
        one_number = cfg["hbm"].get("reducer") in (3, 4)
        if one_number and decode is None:
            numbers = self._bulk_numbers(part)
            if numbers is not None:
                self.doc["value"]["pairs"] = numbers
                self.written = True
                self.board.mark(self.doc, STATUS.WRITTEN, written_time=time.time(), real_time=time.time() - self.t)
                return
        device_distinct |= one_number  # (tuple keys, long keys: the iterator's one value per key)
        bulk = self._bulk_groups(part) if (aci and cfg["hbm"].get("reducer", 0) == 0 and decode is None) else None
        if bulk is not None:
            # built-in reducer + ACI flags: every value list is the singleton the device produced and the reference
            # passes singletons through untouched (job.lua:264-274) -- no per-group call into the library or reducefn
            self.doc["value"]["pairs"] = bulk
            self.written = True
            self.board.mark(self.doc, STATUS.WRITTEN, written_time=time.time(), real_time=time.time() - self.t)
            return
        for key, values in ctx.groups(part):
            if decode:
                key = decode(key)
            if byte_values:
                values = [tuple_keys.decode_value(v) for v in values]
            # The device applied the declared built-in (combiner semantics).  The reference
            # skips the reducer on singletons when the ACI flags are set (job.lua:264-274),
            # otherwise it always calls it (job.lua:275-284).
            if not device_distinct and not (aci and len(values) == 1):
                del result[:]
                mod.reducefn(key, values, emit)
                values = list(result)
            out.append((key, values))
        self.doc["value"]["pairs"] = out  # stands in for the GridFS file result.P<kk> (job.lua:287)
        self.written = True
        self.board.mark(self.doc, STATUS.WRITTEN, written_time=time.time(), real_time=time.time() - self.t)
