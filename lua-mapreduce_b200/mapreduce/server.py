"""mapreduce/server.lua mirrored: configure (server.lua:419-462), loop (466-611),
server_prepare_map (249-276), server_prepare_reduce (279-329), server_final (348-413).
The MongoDB task/job collections are an in-process board; GridFS spill files are the HBM
shuffle (storage "hbm").  Jobs run on attached workers or, when none is attached, inline."""
import bisect
import math
import importlib
import sys
import time

from . import task as _task
from .job import Job, get_func
from .utils import STATUS, TASK_STATUS, get_storage_from, count_digits

_BUILTIN_PART = {"fnv_lua": 0, "mulhash": 1, "wordhash": 2, "range": 3}


def range_splitters(part, nparts, key_kind):
    """The splitters a partitionfn module declares with hbm_partitionfn = "range": hbm_splitters = [...] (checked
    against the module's own partitionfn, since the declaration must mean what the function computes) or "sample"
    (the splitters are sampled from the map output at the MAP -> REDUCE barrier).  Returns the list as the ctx takes
    it (bytes, or ints for u64 keys) or "sample"."""
    spl = getattr(part, "hbm_splitters", None)
    if spl == "sample":
        return "sample"
    if not isinstance(spl, (list, tuple)):
        raise ValueError("hbm_partitionfn = 'range' needs hbm_splitters = [...] or hbm_splitters = 'sample'")
    if nparts != len(spl) + 1:
        raise ValueError("NUM_REDUCERS (%d) must equal the number of splitters + 1 (%d)" % (nparts, len(spl) + 1))
    u64 = key_kind == "u64"
    norm = [int(x) if u64 else (x.encode() if isinstance(x, str) else bytes(x)) for x in spl]
    if norm != sorted(norm):
        raise ValueError("hbm_splitters must be non-decreasing")
    for x in norm:
        for k in ([x, x - 1] if u64 and x > 0 else [x]):
            want, got = bisect.bisect_right(norm, k), part.partitionfn(k)
            if got != want:
                raise ValueError("partitionfn(%r) = %r, but the declared hbm_splitters put the key in partition %d: "
                                 "the declaration must describe the same key ranges as partitionfn" % (k, got, want))
    return norm


# Values the declaration hbm_combinerfn = "distinct" is checked on, one key per list: strings (repeated, distinct, the
# empty string) and numbers.  A list holds one type, as a Lua reducefn that sorts its values needs it.
_DISTINCT_PROBES = ([b"b", b"a", b"b", b"", b"a", b"", b"c"], [3, 1.5, 3, 0, 1.5])


def distinct_combiner(comb, value_kind):
    """Checks a combinerfn module that declares hbm_combinerfn = "distinct": the device then keeps one copy of each
    distinct (key, value) pair of a map job in its place, so the module's combinerfn must emit exactly the distinct
    values it is given (compared as the shuffle compares them, by their encoded bytes)."""
    from .tuple import encode_value
    if comb.hbm_combinerfn != "distinct":
        raise ValueError("unknown hbm_combinerfn %r (built-ins: 'distinct', 'fsum')" % (comb.hbm_combinerfn,))
    if value_kind != "bytes":
        raise ValueError("hbm_combinerfn = 'distinct' drops repeated string and number values: "
                         "configure hbm = {'value_kind': 'bytes'}")
    for values in _DISTINCT_PROBES:
        out = []
        try:
            comb.combinerfn(b"probe", list(values), out.append)
            got = sorted(encode_value(v) for v in out)
        except Exception as e:
            raise ValueError("hbm_combinerfn = 'distinct': combinerfn failed on the values %r: %r" % (values, e))
        if got != sorted({encode_value(v) for v in values}):
            raise ValueError("hbm_combinerfn = 'distinct', but combinerfn turns the values %r into %r instead of their "
                             "distinct values: the declaration must describe what the combinerfn computes" % (values, out))


# Number sums whose every summation order is exact (dyadic fractions, negatives, -0, cancellation across 2^60, in
# Python integers): any reducefn that adds its values one by one, in whatever order, gives the exact sum on them.  The
# sign of a zero sum is not checked: "count = 0; count = count + v" gives +0 where the device gives -0 for all -0.
_FSUM_PROBES = ([1, 2, 3], [0.5, 0.25, -1.75, 3], [2 ** 60, 1, -2 ** 60], [-0.0, -0.0], [0.0, -0.0],
                [-3.5], [1.5, -1.5, 0.125], [-2, -0.5, -0.75], [7])


def _check_sums(fn, name):
    """Raises unless fn (a reducefn or combinerfn, declared with hbm_<name> = "fsum") emits exactly one number, the sum,
    on every probe."""
    from fractions import Fraction
    for values in _FSUM_PROBES:
        out = []
        try:
            fn(b"probe", list(values), out.append)
        except Exception as e:
            raise ValueError("hbm_%s = 'fsum': %s failed on the values %r: %r" % (name, name, values, e))
        want = float(sum(Fraction(v) for v in values))
        ok = len(out) == 1 and isinstance(out[0], (int, float)) and not isinstance(out[0], bool) and out[0] == want
        if not ok:
            raise ValueError("hbm_%s = 'fsum', but %s turns the values %r into %r instead of their sum %r: "
                             "the declaration must describe what the %s computes" % (name, name, values, out, want, name))


def fsum_reducer(red, value_kind):
    """Checks a reducefn module that declares hbm_reducefn = "fsum": the device then hands every key the exact sum of
    its number values, rounded once, and the reducefn is not called, so it must emit exactly that one number."""
    if value_kind != "bytes":
        raise ValueError("hbm_reducefn = 'fsum' sums number values carried as bytes: configure hbm = {'value_kind': 'bytes'}")
    _check_sums(red.reducefn, "reducefn")


def fsum_combiner(comb, builtin_red, value_kind):
    """Checks a combinerfn module that declares hbm_combinerfn = "fsum": the device then replaces each map job's
    numbers per key by the exact expansion of their sum, which only the fsum reducer reads back exactly, so the
    combinerfn must emit exactly that one sum."""
    if builtin_red != "fsum" or value_kind != "bytes":
        raise ValueError("hbm_combinerfn = 'fsum' keeps each map job's sums exactly for the fsum reducer: it needs "
                         "hbm_reducefn = 'fsum' and hbm = {'value_kind': 'bytes'} (got hbm_reducefn = %r, value_kind "
                         "= %r)" % (builtin_red, value_kind))
    _check_sums(comb.combinerfn, "combinerfn")


def distinct_reducer(red, value_kind):
    """Checks a reducefn module that declares hbm_reducefn = "distinct": the device then hands every key its distinct
    values, ascending by their encoded bytes, and the reducefn is not called, so it must emit exactly that sequence."""
    from .tuple import encode_value
    if value_kind != "bytes":
        raise ValueError("hbm_reducefn = 'distinct' orders string and number values by their bytes: "
                         "configure hbm = {'value_kind': 'bytes'}")
    for values in _DISTINCT_PROBES:
        out = []
        try:
            red.reducefn(b"probe", list(values), out.append)
            got = [encode_value(v) for v in out]
        except Exception as e:
            raise ValueError("hbm_reducefn = 'distinct': reducefn failed on the values %r: %r" % (values, e))
        if got != sorted({encode_value(v) for v in values}):
            raise ValueError("hbm_reducefn = 'distinct', but reducefn turns the values %r into %r instead of their "
                             "distinct values in ascending order: the declaration must describe what the reducefn "
                             "computes" % (values, out))


def count_distinct_reducer(red, value_kind):
    """Checks a reducefn module that declares hbm_reducefn = "count_distinct": the device then hands every key the
    number of its distinct values (compared by their encoded bytes), and the reducefn is not called, so it must emit
    exactly that one number."""
    from .tuple import encode_value
    if value_kind != "bytes":
        raise ValueError("hbm_reducefn = 'count_distinct' compares string and number values by their bytes: "
                         "configure hbm = {'value_kind': 'bytes'}")
    for values in _DISTINCT_PROBES:
        out = []
        try:
            red.reducefn(b"probe", list(values), out.append)
        except Exception as e:
            raise ValueError("hbm_reducefn = 'count_distinct': reducefn failed on the values %r: %r" % (values, e))
        want = len({encode_value(v) for v in values})
        ok = len(out) == 1 and isinstance(out[0], (int, float)) and not isinstance(out[0], bool) and out[0] == want
        if not ok:
            raise ValueError("hbm_reducefn = 'count_distinct', but reducefn turns the values %r into %r instead of "
                             "the number of their distinct values, %d: the declaration must describe what the reducefn "
                             "computes" % (values, out, want))


class server:
    def __init__(self, connection_string, dbname, auth_table=None):
        self.cnn_string, self.dbname = connection_string, dbname
        self.board = _task.board(connection_string, dbname)
        self.configured = False
        self.finished = False
        self.ctx_factory = None  # tests inject a stand-in; default = the CUDA ctx

    @staticmethod
    def new(connection_string, dbname, auth_table=None):
        return server(connection_string, dbname, auth_table)

    # ---- server.lua:419-462
    def configure(self, params):
        params = dict(params)
        storage, path = get_storage_from(params.get("storage"), True)
        params["storage"] = "%s:%s" % (storage, path)
        self.result_ns = params.get("result_ns") or "result"
        assert all(params.get(k) for k in ("taskfn", "mapfn", "partitionfn", "reducefn")), \
            "Fields taskfn, mapfn, partitionfn and reducefn are mandatory"
        mods = {}
        for name in ("taskfn", "mapfn", "partitionfn", "reducefn", "finalfn", "combinerfn"):
            v = params.get(name)
            assert (isinstance(v, str)) or (not v and name in ("finalfn", "combinerfn")), \
                "Needs a %s module with %s function" % (name, name)
            if v:
                aux = importlib.import_module(v)
                assert hasattr(aux, name), "Module %s must return a table with the field %s" % (name, name)
                assert hasattr(aux, "init"), "Init function is needed: %s" % name
                mods[name] = aux
        self.init_args = params.get("init_args")
        self.taskfn = mods["taskfn"]
        self.finalfn = mods.get("finalfn")
        for init in {m.init for m in (self.taskfn, self.finalfn) if m is not None}:
            init(self.init_args)
        # ---- what the device evaluates: declared on the plugin modules (same pattern as the
        # associative/commutative/idempotent flags, examples/WordCount/reducefn.lua:10-14)
        red, part = mods["reducefn"], mods["partitionfn"]
        builtin_red = getattr(red, "hbm_reducefn", None)
        if builtin_red not in (None, "sum", "distinct", "fsum", "count_distinct"):
            raise NotImplementedError("unknown hbm_reducefn %r (built-ins: 'sum', 'distinct', 'fsum', 'count_distinct')"
                                      % (builtin_red,))
        # no declaration = general reducer: the device partitions, sorts and groups, reducefn runs
        # on the host per group (job.lua:264-284); values are unsigned integers < 2^32
        # A combinerfn only ever runs on the device, as the declared built-in (it must equal the reducefn there).
        # Any other combinerfn is SKIPPED: the reference's contract for it (job.lua:92-96,198-202) is that reducing
        # combined values equals reducing the raw ones, so the reducefn -- on the device if it is the built-in, per
        # group on the host otherwise -- sees the raw values and produces the same result, just without the saving.
        device_combiner = "combinerfn" in mods and builtin_red == "sum" and \
            getattr(mods["combinerfn"], "hbm_reducefn", None) == "sum"
        # hbm_combinerfn = "distinct" (value_kind = "bytes"): the combinerfn keeps one copy of each distinct value of a
        # key, so the device drops the repeated (key, value) pairs of each map job at its commit
        declared = getattr(mods["combinerfn"], "hbm_combinerfn", None) if "combinerfn" in mods else None
        # hbm_combinerfn = "fsum" (hbm_reducefn = "fsum", value_kind = "bytes"): each map job's numbers per key become
        # the exact expansion of their sum at its commit
        fsum_comb = declared == "fsum"
        distinct = declared is not None and not fsum_comb
        if "combinerfn" in mods and not device_combiner and not distinct and not fsum_comb:
            sys.stderr.write("# WARNING: combinerfn %s is not a device built-in (hbm_reducefn = 'sum'); it is skipped, "
                             "the reducefn sees the uncombined values\n" % params["combinerfn"])
        pname = getattr(part, "hbm_partitionfn", None)
        # a partitionfn runs on the device when it is one of the hash built-ins or a key range ("range" with
        # hbm_splitters)
        if pname not in _BUILTIN_PART:
            raise NotImplementedError("partitionfn module must declare hbm_partitionfn in %s" % sorted(_BUILTIN_PART))
        nparts = getattr(part, "NUM_REDUCERS", None) or getattr(part, "hbm_num_partitions", None)
        assert isinstance(nparts, int) and nparts >= 1, "partitionfn module must expose NUM_REDUCERS"
        hbm = dict(key_kind="str", max_key_bytes=123, device=-1, value_kind="int")
        hbm.update(params.get("hbm") or {})
        # value_kind = "bytes": values are Lua strings and numbers (tuple.encode_value), handed to a general reducefn
        if hbm["value_kind"] not in ("int", "bytes"):
            raise ValueError("hbm value_kind must be 'int' or 'bytes', got %r" % (hbm["value_kind"],))
        if fsum_comb:
            fsum_combiner(mods["combinerfn"], builtin_red, hbm["value_kind"])
        if hbm["value_kind"] == "bytes" and builtin_red not in (None, "distinct", "fsum", "count_distinct"):
            raise ValueError("hbm value_kind = 'bytes' hands string and number values to a general reducefn: "
                             "the reducefn module must not declare an hbm_reducefn other than 'distinct', 'fsum' or "
                             "'count_distinct' (it declares %r)" % (builtin_red,))
        if builtin_red == "distinct":  # every key's distinct values, ascending, on the device: reducefn is not called
            distinct_reducer(red, hbm["value_kind"])
        if builtin_red == "fsum":  # every key's numbers summed exactly on the device: reducefn is not called
            fsum_reducer(red, hbm["value_kind"])
            if distinct:  # a device combiner would drop repeated values before they are summed
                raise ValueError("hbm_reducefn = 'fsum' takes no device combiner: the combinerfn module declares "
                                 "hbm_combinerfn = %r" % (mods["combinerfn"].hbm_combinerfn,))
        if builtin_red == "count_distinct":  # every key's number of distinct values, on the device: reducefn is not called
            count_distinct_reducer(red, hbm["value_kind"])
        if getattr(mods["mapfn"], "hbm_mapfn", None) == "words_file" and hbm["value_kind"] != "bytes":
            raise ValueError("hbm_mapfn = 'words_file' pairs every word with the file name, a string value: "
                             "configure hbm = {'value_kind': 'bytes'}")
        if getattr(mods["mapfn"], "hbm_mapfn", None) == "key_numbers_file":
            if hbm["value_kind"] != "bytes":
                raise ValueError("hbm_mapfn = 'key_numbers_file' pairs every key with a number, a byte value: "
                                 "configure hbm = {'value_kind': 'bytes'}")
            if hbm["key_kind"] != "str":  # the host mapfn's u64 or tuple keys would be encoded differently
                raise ValueError("hbm_mapfn = 'key_numbers_file' emits the key field's bytes as a string key: it needs "
                                 "key_kind = 'str', not %r" % (hbm["key_kind"],))
        if distinct:
            distinct_combiner(mods["combinerfn"], hbm["value_kind"])
        hbm.update(partitioner=_BUILTIN_PART[pname], num_partitions=nparts,
                   combiner="distinct" if distinct else "fsum" if fsum_comb else device_combiner,
                   reducer={"sum": 0, "distinct": 2, "fsum": 3, "count_distinct": 4}.get(builtin_red, 1),
                   splitters=range_splitters(part, nparts, hbm["key_kind"]) if pname == "range" else None)
        self.config = dict(mapfn=params["mapfn"], reducefn=params["reducefn"], partitionfn=params["partitionfn"],
                           combinerfn=params.get("combinerfn"), init_args=self.init_args,
                           storage=params["storage"], hbm=hbm)
        self.configured = True

    def _make_ctx(self):
        h = self.config["hbm"]
        if self.ctx_factory is not None:
            return self.ctx_factory(h)
        from .. import mrhbm
        kind = mrhbm.KEY_U64 if h["key_kind"] == "u64" else mrhbm.KEY_STR
        combiner = {"distinct": mrhbm.COMBINE_DISTINCT, "fsum": mrhbm.COMBINE_FSUM}.get(h["combiner"], h["combiner"])
        ctx = mrhbm.Ctx(kind, h["num_partitions"], h["partitioner"], max_key_bytes=h["max_key_bytes"],
                        combiner=combiner, device=h["device"], reducer=h["reducer"],
                        flags=mrhbm.F_BYTE_VALUES if h.get("value_kind") == "bytes" else 0)
        if isinstance(h.get("splitters"), list):  # (kept across reset)
            ctx.set_splitters(h["splitters"])
        return ctx

    # ---- polling (server.lua:186-234) with inline execution when no worker is attached
    def _wait(self, ns):
        b = self.board
        while True:
            with b.cv:
                pend = b.pending(ns)
                if not pend:
                    break
                runnable = [j for j in pend if j["status"] in (STATUS.WAITING, STATUS.BROKEN)]
                if b.workers > 0 or not runnable:
                    b.cv.wait(timeout=0.05)
                    continue
            ns2, doc = b.take_next_job("server-inline")
            if doc is None:
                continue
            job = Job(b, ns2, doc, self.config)
            try:
                job.execute()
            except Exception as e:  # worker.lua:116-131
                b.mark_as_broken(doc, repr(e))
                sys.stderr.write("Error executing a job: %r\n" % (e,))
        return sum(1 for j in b.jobs[ns] if j["status"] == STATUS.FAILED)

    # ---- server.lua:466-611
    def loop(self):
        assert self.configured, "Call to server:configure(...) method is mandatory"
        b = self.board
        it = 0
        while True:
            it += 1
            t0 = time.time()
            with b.cv:
                if b.ctx is None or getattr(b.ctx, "h", True) is None:  # none yet, or closed by its owner
                    b.ctx = self._make_ctx()
                else:
                    b.ctx.reset()
                b.config, b.iteration = self.config, it
                b.jobs = {"map_jobs": [], "red_jobs": []}
                # server_prepare_map (server.lua:249-276)
                seen = set()

                def emit(key, value):
                    assert key not in seen, "Duplicate key: %s" % (key,)
                    seen.add(key)
                    b.jobs["map_jobs"].append(_task.make_job(key, value))
                self.taskfn.taskfn(emit)
                b.status = TASK_STATUS.MAP
                b.cv.notify_all()
            sys.stderr.write("# Iteration %d\n# \t Preparing MAP\n" % it)
            failed_maps = self._wait("map_jobs")
            # server_prepare_reduce (server.lua:279-329): one reduce job per NON-EMPTY partition
            if self.config["hbm"].get("splitters") == "sample":  # key ranges from this iteration's map output
                b.ctx.sample_splitters()
            b.ctx.shuffle()
            parts = b.ctx.partitions()
            digits = count_digits(max(parts) if parts else 0)
            with b.cv:
                for p in parts:
                    b.jobs["red_jobs"].append(_task.make_job(p, {
                        "file": "map_results.P%d" % p, "result": "%s.P%0*d" % (self.result_ns, digits, p)}))
                b.status = TASK_STATUS.REDUCE
                b.cv.notify_all()
            sys.stderr.write("# \t Preparing REDUCE\n")
            failed_reds = self._wait("red_jobs")
            self.stats = {"iteration": it, "map_count": len(b.jobs["map_jobs"]), "reduce_count": len(parts),
                          "failed_maps": failed_maps, "failed_reds": failed_reds,
                          "server_time": time.time() - t0, "shuffle": b.ctx.stats()}
            sys.stderr.write("# Server time %f\n" % self.stats["server_time"])
            reply = self._final()
            if reply != "loop":
                with b.cv:
                    b.status = TASK_STATUS.FINISHED
                    b.cv.notify_all()
                self.finished = True
                return

    # ---- server.lua:348-413
    def _final(self):
        b = self.board
        files = sorted(b.jobs["red_jobs"], key=lambda j: j["value"]["result"])  # server.lua:367

        def pair_iterator():
            for j in files:
                for key, values in j["value"].get("pairs", ()):
                    yield key, values

        self.results = files
        reply = self.finalfn.finalfn(pair_iterator()) if self.finalfn is not None else None
        if reply not in ("loop", True, False, None):
            sys.stderr.write("# WARNING!!! INCORRECT FINAL RETURN: %s\n" % (reply,))
        if reply == "loop":
            sys.stderr.write("# LOOP again\n")
        if reply is True or reply == "loop":  # remove results
            for j in files:
                j["value"].pop("pairs", None)
        return reply


    # ---- interchange with a stock lua-mapreduce deployment (SURVEY 8f rank 3)
    def export_results(self, directory):
        """Writes the kept results (finalfn returned false/nil) as the reference's result files: one file per
        non-empty partition named `<result_ns>.P<kk>` (server.lua:313-321), one line `return <key>,{<values>}`
        per key in ascending key order (job.lua:272-273).  Returns the file names."""
        import os
        from .utils import result_line
        names = []
        for j in getattr(self, "results", []):
            pairs = j["value"].get("pairs")
            if pairs is None:
                continue
            name = j["value"]["result"]
            with open(os.path.join(directory, name), "wb") as fh:
                for key, values in pairs:
                    fh.write(result_line(key, values))
            names.append(name)
        return names


new = server.new
