"""The emit pool's ledger (csrc/mrhbm_pool.h) on the CPU: room taken and given back, ranges per map job, commit as
replace-by-job-id, abort, rewind and reset, against a Python model that keeps a list of ranges and two counters.  The
driver tests/native/pool_ledger_check.cu is host-compiled from the same header."""
import copy
import os
import random
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPEN, COMMITTED, DEAD = range(3)


@pytest.fixture(scope="module")
def ledger(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path_factory.mktemp("ledger") / "pool_ledger_check")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "lua-mapreduce_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "pool_ledger_check.cu")])

    def run(cmds):
        text = "".join(" ".join(map(str, c)) + "\n" for c in cmds)
        out = subprocess.run([exe], input=text, capture_output=True, text=True, timeout=300, check=True)
        lines = out.stdout.splitlines()
        assert len(lines) == len(cmds)
        return lines
    return run


class Range:
    def __init__(self, job, owner, off, cnt, aoff):
        self.job, self.state, self.owner, self.off, self.cnt, self.aoff = job, OPEN, owner, off, cnt, aoff


class Session:
    """Applies every command to the model as it is issued and remembers the line the driver must print for it; check()
    then runs them all through the driver."""

    def __init__(self, byte_values=False):
        self.ranges, self.used, self.arena, self.owners, self.byte_values = [], 0, 0, 0, byte_values
        self.cmds, self.want, self.snaps = [], [], []
        if byte_values:
            self._log(("B",), "-")

    def _log(self, cmd, result):
        self.cmds.append(cmd)
        state = [self.used, self.arena] + [x for r in self.live() for x in r]
        self.want.append(f"{result} | " + " ".join(map(str, state)))

    def live(self):
        v = []
        for r in self.ranges:
            if r.state != COMMITTED or not r.cnt:
                continue
            if v and v[-1][0] + v[-1][1] == r.off:
                v[-1][1] += r.cnt
            else:
                v.append([r.off, r.cnt])
        return v

    def owner(self):
        self.owners += 1
        self._log(("O",), self.owners)
        return self.owners

    def take(self, n, nbytes):
        if self.byte_values and self.used + n >= 0xFFFFFFFF:
            self._log(("T", n, nbytes), "refused")
            return None
        off, aoff = self.used, self.arena
        self.used += n
        self.arena += nbytes
        self._log(("T", n, nbytes), f"{off} {aoff}")
        return off, aoff

    def add(self, owner, job, off, cnt, aoff):
        last = self.ranges[-1] if self.ranges else None
        if last and last.owner == owner and last.state == OPEN and last.off + last.cnt == off:
            last.cnt += cnt
        else:
            self.ranges.append(Range(job, owner, off, cnt, aoff))
        self._log(("A", owner, job, off, cnt, aoff), "-")

    def emit(self, owner, job, n, nbytes=0):
        off, aoff = self.take(n, nbytes)
        self.add(owner, job, off, n, aoff)
        return off, aoff

    def commit(self, owner, job):
        for r in self.ranges:
            if r.state == COMMITTED and r.job == job:
                r.state = DEAD
        for r in self.ranges:
            if r.owner == owner and r.state == OPEN:
                r.state = COMMITTED
        self._log(("C", owner, job), "-")

    def abort(self, owner):
        for r in self.ranges:
            if r.owner == owner and r.state == OPEN:
                r.state = DEAD
        while self.ranges and self.ranges[-1].state == DEAD and self.ranges[-1].off + self.ranges[-1].cnt == self.used:
            self.used, self.arena = self.ranges[-1].off, self.ranges[-1].aoff
            self.ranges.pop()
        self._log(("X", owner), "-")

    def mark(self):
        """the model keeps a copy of everything, the ledger four numbers"""
        self.snaps.append((copy.deepcopy(self.ranges), self.used, self.arena))
        self._log(("M",), len(self.snaps) - 1)
        return len(self.snaps) - 1

    def rewind(self, i):
        ranges, self.used, self.arena = self.snaps[i]
        self.ranges = copy.deepcopy(ranges)
        self._log(("W", i), "-")

    def reset(self):
        self.ranges, self.used, self.arena = [], 0, 0
        self._log(("R",), "-")

    def open_job(self):
        jobs = [r.job for r in self.ranges if r.state == OPEN]
        self._log(("J",), jobs[0] if jobs else "none")

    def state(self):
        return self.used, self.arena, self.live()

    def check(self, ledger):
        for i, (got, want) in enumerate(zip(ledger(self.cmds), self.want)):
            assert got == want, (i, self.cmds[max(0, i - 5):i + 1])


def test_abort_takes_back_the_tail_only(ledger):
    s = Session(byte_values=True)
    a, b, c = s.owner(), s.owner(), s.owner()
    s.emit(a, "ja", 10, 100)
    s.commit(a, "ja")
    s.emit(b, "jb", 5, 50)
    s.abort(b)  # at the tail: pool and arena come back
    assert s.state() == (10, 100, [[0, 10]])
    b = s.owner()
    s.emit(b, "jb", 5, 50)
    s.emit(c, "jc", 7, 70)
    s.open_job()
    s.abort(b)  # behind it lies c's open range: nothing comes back
    assert s.state() == (22, 220, [[0, 10]])
    s.abort(c)  # now both go, down to the committed range
    assert s.state() == (10, 100, [[0, 10]])
    s.open_job()
    s.abort(s.owner())  # a map that emitted nothing
    assert s.state() == (10, 100, [[0, 10]])
    s.check(ledger)


def test_recommit_replaces_the_job_and_dead_room_stays_until_reset(ledger):
    s = Session(byte_values=True)
    a, b, c = s.owner(), s.owner(), s.owner()
    s.emit(a, "j1", 10, 11)
    s.emit(b, "j2", 20, 22)
    s.emit(a, "j1", 3, 5)  # a's second range, behind b's
    s.commit(a, "j1")
    s.commit(b, "j2")
    assert s.state() == (33, 38, [[0, 33]])
    s.emit(c, "j1", 4, 4)
    assert s.live() == [[0, 33]]  # the first run of j1 counts until the second commits
    s.commit(c, "j1")
    assert s.state() == (37, 42, [[10, 20], [33, 4]])  # both earlier ranges of j1 are dead, j2 is untouched
    d = s.owner()
    s.emit(d, "j3", 1, 1)
    s.abort(d)  # takes back its own room; the dead ranges in the middle keep theirs
    assert s.state() == (37, 42, [[10, 20], [33, 4]])
    e = s.owner()
    s.emit(e, "j1", 2, 2)
    s.commit(e, "j1")  # third run: kills [33, 4), a dead range now lies right before the tail range
    f = s.owner()
    s.emit(f, "j4", 6, 6)
    s.abort(f)  # stops at e's committed range
    assert s.state() == (39, 44, [[10, 20], [37, 2]])
    s.reset()
    assert s.state() == (0, 0, [])
    g = s.owner()
    assert s.emit(g, "j1", 5, 5) == (0, 0)
    s.commit(g, "j1")
    assert s.state() == (5, 5, [[0, 5]])
    s.check(ledger)


def test_adds_merge_per_owner_and_keep_the_first_arena_offset(ledger):
    s = Session(byte_values=True)
    z = s.owner()
    s.emit(z, "jz", 4, 40)
    s.commit(z, "jz")
    a = s.owner()
    s.emit(a, "ja", 10, 100)
    s.emit(a, "ja", 5, 7)
    s.emit(a, "ja", 0, 0)
    s.emit(a, "ja", 1, 1)
    assert len(s.ranges) == 2 and s.ranges[-1].cnt == 16 and s.ranges[-1].aoff == 40
    s.abort(a)  # one range: everything back, to the arena offset of its first value
    assert s.state() == (4, 40, [[0, 4]])
    a, b = s.owner(), s.owner()
    for i in range(3):  # two owners that interleave: six ranges
        s.emit(a, "ja", 2, 20)
        s.emit(b, "jb", 3, 30)
    assert len(s.ranges) == 7
    s.abort(a)  # b's last range is the tail
    assert s.used == 19
    s.commit(b, "jb")
    assert s.state() == (19, 190, [[0, 4], [6, 3], [11, 3], [16, 3]])
    s.check(ledger)


def test_rewind_leaves_no_hole(ledger):
    s = Session(byte_values=True)
    a, b = s.owner(), s.owner()
    mk = s.mark()
    s.take(9, 90)  # room taken, never added: the emit failed
    s.rewind(mk)
    assert s.state() == (0, 0, [])
    s.emit(a, "ja", 10, 100)
    mk = s.mark()
    s.emit(a, "ja", 5, 50)  # merged into the range the mark saw
    s.take(7, 70)
    s.rewind(mk)
    assert (s.used, s.arena, s.ranges[-1].cnt) == (10, 100, 10)
    s.abort(a)  # no hole: the tail range still ends at used, so the abort takes it back
    assert s.state() == (0, 0, [])
    a = s.owner()
    s.emit(a, "ja", 10, 100)
    mk = s.mark()
    s.emit(b, "jb", 4, 40)  # ranges of its own behind the mark
    s.emit(a, "ja", 4, 40)
    s.take(1, 1)
    s.rewind(mk)
    assert len(s.ranges) == 1 and s.used == 10
    s.emit(b, "jb", 2, 20)
    s.commit(b, "jb")
    s.commit(a, "ja")
    assert s.state() == (12, 120, [[0, 12]])
    s.check(ledger)


def test_live_merges_adjacent_jobs(ledger):
    s = Session()
    a, b, c, d = s.owner(), s.owner(), s.owner(), s.owner()
    s.emit(a, "ja", 5)
    s.emit(b, "jb", 6)
    s.emit(c, "jc", 0)  # an empty range between them
    s.emit(d, "jd", 7)
    for o, j in ((a, "ja"), (b, "jb"), (c, "jc")):
        s.commit(o, j)
    assert s.state() == (18, 0, [[0, 11]])
    s.open_job()
    s.commit(d, "jd")
    assert s.live() == [[0, 18]]
    e = s.owner()
    s.emit(e, "jb", 1)
    s.commit(e, "jb")  # the middle job again: the merged run splits around its dead range
    assert s.live() == [[0, 5], [11, 8]]
    s.check(ledger)


def test_value_ids_stay_below_2_to_32(ledger):
    for byte_values in (True, False):
        s = Session(byte_values)
        a = s.owner()
        s.emit(a, "ja", 0xFFFFFFF0, 1)
        assert (s.take(15, 0) is None) == byte_values  # id 2^32 - 1 is never handed out
        s.emit(a, "ja", 14, 1)
        assert (s.take(1, 0) is None) == byte_values
        s.reset()
        assert s.take(1, 0) == (0, 0)
        s.check(ledger)


@pytest.mark.parametrize("seed", range(8))
def test_random_interleaved_maps(ledger, seed):
    rng = random.Random(seed)
    s = Session(byte_values=seed % 2 == 0)
    jobs = [f"j{i}" for i in range(5)]  # few ids: re-commits are common
    maps = {}  # owner -> job
    for _ in range(3000):
        x = rng.random()
        if x < 0.12 or not maps:
            maps[s.owner()] = rng.choice(jobs)
        elif x < 0.60:
            o = rng.choice(list(maps))
            s.emit(o, maps[o], rng.choice((0, 1, 2, 17, 65536)), rng.randrange(0, 300))
        elif x < 0.68:  # an emit that fails after taking its room
            mk = s.mark()
            s.take(rng.randrange(0, 100), rng.randrange(0, 300))
            s.rewind(mk)
        elif x < 0.74:  # a call of several emits that fails as a whole
            mk = s.mark()
            for _ in range(rng.randrange(1, 5)):
                o = rng.choice(list(maps))
                s.emit(o, maps[o], rng.randrange(0, 40), rng.randrange(0, 300))
            if rng.random() < 0.5:
                s.take(rng.randrange(0, 100), rng.randrange(0, 300))
            s.rewind(mk)
        elif x < 0.85:
            o = rng.choice(list(maps))
            s.commit(o, maps.pop(o))
        elif x < 0.95:
            o = rng.choice(list(maps))
            s.abort(o)
            del maps[o]
        elif x < 0.96:
            s.reset()
            maps = {}
        else:
            s.open_job()
    s.check(ledger)
