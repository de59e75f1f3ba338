"""The emit pool's ledger (csrc/mrhbm_pool.h) with the two operations of MRHBM_COMBINE_DISTINCT, on the CPU: open_ranges
lists a map's open ranges and shrink keeps the first records of one of them (its distinct pairs, moved forward at the
commit).  The Python model of tests/test_pool_ledger.py is extended by the same two operations and checked against
the driver tests/native/pool_ledger_shrink_check.cu, host-compiled from the header.  What the restatement pins: the
room behind a shrunk range's new end is never handed out again before reset, because a kept pair's value id may point
into it."""
import os
import random
import shutil
import subprocess

import pytest

from test_pool_ledger import OPEN, Session

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ledger(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path_factory.mktemp("ledger_shrink") / "pool_ledger_shrink_check")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "lua-mapreduce_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "pool_ledger_shrink_check.cu")])

    def run(cmds):
        text = "".join(" ".join(map(str, c)) + "\n" for c in cmds)
        out = subprocess.run([exe], input=text, capture_output=True, text=True, timeout=300, check=True)
        lines = out.stdout.splitlines()
        assert len(lines) == len(cmds)
        return lines
    return run


class ShrinkSession(Session):
    def open_ranges(self, owner):
        v = [(r.off, r.cnt) for r in self.ranges if r.owner == owner and r.state == OPEN and r.cnt]
        self._log(("P", owner), " ".join("%d %d" % x for x in v) if v else "none")
        return v

    def shrink(self, owner, off, cnt):
        r = next(r for r in self.ranges if r.owner == owner and r.state == OPEN and r.cnt and r.off == off)
        assert cnt <= r.cnt
        r.cnt = cnt
        self._log(("S", owner, off, cnt), "-")

    def commit_distinct(self, owner, job, keep):
        """the commit of a distinct-combining map: each open range keeps keep(count) records"""
        for off, cnt in self.open_ranges(owner):
            self.shrink(owner, off, keep(cnt))
        self.commit(owner, job)


def test_shrunk_room_is_not_handed_out_again(ledger):
    s = ShrinkSession(byte_values=True)
    a, b = s.owner(), s.owner()
    s.emit(a, "ja", 10, 100)
    s.emit(b, "jb", 4, 40)
    s.emit(a, "ja", 6, 60)  # a's second range, behind b's
    assert s.open_ranges(a) == [(0, 10), (14, 6)]
    s.commit_distinct(a, "ja", lambda n: n // 2)
    assert s.state() == (20, 200, [[0, 5], [14, 3]])
    s.abort(b)  # b's range lies between a's: nothing comes back
    assert s.state() == (20, 200, [[0, 5], [14, 3]])
    c = s.owner()
    s.emit(c, "jc", 2, 20)
    s.abort(c)  # the tail goes back, down to the end of a's room, not to the end of its kept records
    assert s.state() == (20, 200, [[0, 5], [14, 3]])
    c = s.owner()
    s.emit(c, "ja", 1, 1)
    s.commit(c, "ja")  # replace-by-job-id kills both shrunk ranges
    d = s.owner()
    s.emit(d, "jd", 3, 3)
    s.abort(d)
    assert s.state() == (21, 201, [[20, 1]])
    s.reset()
    assert s.state() == (0, 0, [])
    s.check(ledger)


def test_a_dead_shrunk_tail_keeps_its_room(ledger):
    s = ShrinkSession(byte_values=True)
    a = s.owner()
    s.emit(a, "ja", 8, 80)
    s.commit_distinct(a, "ja", lambda n: 3)
    b = s.owner()
    s.emit(b, "ja", 2, 2)
    s.commit_distinct(b, "ja", lambda n: n)  # nothing dropped; the first run of ja dies
    c = s.owner()
    s.emit(c, "jc", 5, 5)
    s.abort(c)  # back to b's committed range
    assert s.state() == (10, 82, [[8, 2]])
    e = s.owner()
    s.emit(e, "ja", 1, 1)
    s.commit(e, "ja")  # b's range dies too: a dead shrunk range and a dead full one
    f = s.owner()
    s.emit(f, "jf", 1, 1)
    s.abort(f)  # stops at e's committed range
    assert s.state() == (11, 83, [[10, 1]])
    s.check(ledger)


def test_shrink_to_nothing_and_merging(ledger):
    s = ShrinkSession()
    a, b = s.owner(), s.owner()
    s.emit(a, "ja", 4)
    s.emit(a, "ja", 4)  # merged into one range
    assert s.open_ranges(a) == [(0, 8)]
    s.commit_distinct(a, "ja", lambda n: 0)
    assert s.state() == (8, 0, [])
    s.emit(b, "jb", 3)
    s.commit_distinct(b, "jb", lambda n: n)
    assert s.live() == [[8, 3]]  # not merged with a's empty range
    assert s.open_ranges(b) == []
    c, d = s.owner(), s.owner()
    s.emit(c, "jc", 0)
    s.emit(d, "jd", 0)
    s.emit(c, "jc", 2)  # c now has an empty range and a range of records at the same offset
    assert s.open_ranges(c) == [(11, 2)]
    s.commit_distinct(c, "jc", lambda n: 1)
    s.commit(d, "jd")
    assert s.state() == (13, 0, [[8, 4]])
    s.check(ledger)


@pytest.mark.parametrize("seed", range(6))
def test_random_interleaved_maps_with_distinct_commits(ledger, seed):
    rng = random.Random(seed)
    s = ShrinkSession(byte_values=seed % 2 == 0)
    jobs = [f"j{i}" for i in range(5)]
    maps = {}
    for _ in range(3000):
        x = rng.random()
        if x < 0.12 or not maps:
            maps[s.owner()] = rng.choice(jobs)
        elif x < 0.60:
            o = rng.choice(list(maps))
            s.emit(o, maps[o], rng.choice((0, 1, 2, 17, 65536)), rng.randrange(0, 300))
        elif x < 0.68:
            mk = s.mark()
            s.take(rng.randrange(0, 100), rng.randrange(0, 300))
            s.rewind(mk)
        elif x < 0.78:
            o = rng.choice(list(maps))
            s.commit_distinct(o, maps.pop(o), lambda n: rng.randrange(0, n + 1))
        elif x < 0.83:
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
        # the room of every range, shrunk or not, lies below used()
        assert all(r.off + r.cnt <= s.used for r in s.ranges)
    s.check(ledger)
