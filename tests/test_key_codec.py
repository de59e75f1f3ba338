"""The host key codec (csrc/mrhbm_keys.h) on the CPU: escaping, slot order and decoding, the iterator's long-key
merge compare, the range partitioner's table image and the host partitioner, against Python models of the slot
format.  The driver tests/native/key_codec_check.cu is host-compiled from the same header."""
import bisect
import os
import random
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1
STR_KB = (28, 60, 124)  # the key bytes of the string record classes (32 / 64 / 128-byte records)


@pytest.fixture(scope="module")
def codec(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path_factory.mktemp("codec") / "key_codec_check")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "lua-mapreduce_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "key_codec_check.cu")])

    def run(cmds):
        """one output line (split into fields) per command: an op letter, then ints and byte strings"""
        field = lambda x: (x.hex() or "-") if isinstance(x, bytes) else str(x)
        text = "".join(" ".join(map(field, c)) + "\n" for c in cmds)
        out = subprocess.run([exe], input=text, capture_output=True, text=True, timeout=300, check=True)
        lines = out.stdout.splitlines()
        assert len(lines) == len(cmds)
        return [ln.split() for ln in lines]
    return run


def unhex(s):
    return b"" if s == "-" else bytes.fromhex(s)


def esc(key):
    return b"".join(b"\x01" + bytes([b + 1]) if b <= 1 else bytes([b]) for b in key)


def fits(key, kb):
    return len(esc(key)) < kb


def rich_bytes(rng, n, alphabet=(0, 1, 2, 0xFF, 0x61, 0x62)):
    return bytes(rng.choice(alphabet) for _ in range(n))


def test_escape_round_trip_and_order(codec):
    rng = random.Random(1)
    keys = [b"", b"\x00", b"\x01", b"\x02", b"\xff", b"a\x00", b"a\x01", b"ab"]
    keys += [rich_bytes(rng, rng.randrange(0, 14)) for _ in range(600)]
    for k, (e, n, u) in zip(keys, codec([("E", k) for k in keys])):
        assert unhex(e) == esc(k) and int(n) == len(esc(k)) and unhex(u) == k
    assert sorted(keys) == sorted(keys, key=esc)  # escaping preserves the byte order
    # a lone trailing 0x01 (no escape pair) is left as it is
    got = codec([("U", b"a\x01"), ("U", b"\x01"), ("U", b"\x01\x01"), ("U", b"\x01\x02\x01")])
    assert [unhex(g[0]) for g in got] == [b"a\x01", b"\x01", b"\x00", b"\x01\x01"]


def slot_order_keys(rng, kb):
    """keys that fit a kb-byte slot: shared prefixes, every length up to the slot, special bytes"""
    keys = [b"", b"\x00", b"\x01", b"\x00\x00", b"\xff", b"a", b"a\x00", b"a\x01", b"a\x02", b"ab"]
    for _ in range(400):
        k = rich_bytes(rng, rng.randrange(0, kb))
        while not fits(k, kb):
            k = k[:-1]
        keys.append(k)
        keys.append(k[:rng.randrange(0, len(k) + 1)])  # a prefix of another key
    base = b"b" * (kb - 1)  # the longest keys a slot holds, and their escaped neighbours
    keys += [base, base[:-1] + b"\xff", base[:-2] + b"\x00", base[:-2] + b"\x01", base[:-1]]
    return keys


@pytest.mark.parametrize("kb", STR_KB + (8,))
def test_slot_order_is_byte_order(codec, kb):
    rng = random.Random(kb)
    if kb == 8:  # u64 keys stand for their 8 big-endian bytes: numeric order is byte order
        ints = [0, 1, 255, 256, (1 << 32) - 1, 1 << 32, 1 << 63, M64, M64 - 1] + [rng.getrandbits(64) for _ in range(500)]
        ints += [rng.getrandbits(64) & ~0xFF for _ in range(100)] + ints[:50]
        keys = [v.to_bytes(8, "big") for v in ints]
        assert sorted(keys) == [v.to_bytes(8, "big") for v in sorted(ints)]
    else:
        keys = slot_order_keys(rng, kb)
        assert all(fits(k, kb) for k in keys)
    (out,) = codec([["O", kb] + keys])
    order, decoded = [int(x) for x in out[:len(keys)]], [unhex(x) for x in out[len(keys):]]
    assert order == sorted(range(len(keys)), key=lambda i: (keys[i], i))
    assert decoded == keys  # slot -> original bytes


@pytest.mark.parametrize("kb", STR_KB)
def test_long_key_against_slot_key(codec, kb):
    """the iterator's merge of a host-held key longer than a slot with the smallest slot key"""
    rng = random.Random(kb + 1)
    cmds = []
    for _ in range(300):
        lng = rich_bytes(rng, rng.randrange(kb - 1, kb + 20))
        while fits(lng, kb):
            lng += rich_bytes(rng, 1)
        cut = lng
        while not fits(cut, kb):
            cut = cut[:-1]
        shorts = [cut, cut[:len(cut) // 2], b""]  # proper prefixes of the long key
        shorts += [cut[:-1] + bytes([b]) for b in (0, 1, 2, 0xFE, 0xFF) if cut]
        shorts += [rich_bytes(rng, rng.randrange(0, kb // 2))]
        cmds += [("L", kb, lng, s) for s in shorts if fits(s, kb)]
    for (lk_, kb_, lng, s), (sign,) in zip(cmds, codec(cmds)):
        assert int(sign) == (lng > s) - (lng < s), (lng, s)


def splitter_sets(kb):
    """adversarial splitter lists (original bytes), non-decreasing"""
    u = b"a" * (kb - 1)
    sets = {
        "none": [],
        "plain": [b"b", b"d", b"f"],
        "empty_and_dup": [b"", b"", b"c", b"c", b"c"],
        "slot_long": [b"c" * kb, b"d" * kb],  # escaped size == kb: the whole slot, no padding left
        "longer": [b"b" * (kb + 5), b"c" * (kb + 1)],
        "carry": [b"a" + b"\xff" * (kb - 1) + b"z", b"b\x02" + b"\xff" * (kb - 2) + b"\x03"],
        "cut": [b"c", b"\xff" * (kb + 1), b"\xff" * (kb + 3)],  # above every slot key: fin < P - 1
        "special": [b"a\x00", b"a\x00\x01", b"a\x01", b"a\x01\xff", b"a\x02"],
        "pair_across": [u + b"\x00b", u + b"\x01", u + b"\x01c", u + b"b"],  # 01 xx with 01 the last slot byte
        "pair_across_ff": [b"\xff" * (kb - 1) + b"\x00q", b"\xff" * (kb - 1) + b"\x02"],
    }
    return sets


def probe_keys(rng, spl, kb):
    """keys that fit a slot, around every splitter: its prefixes and their neighbours"""
    keys = [b"", b"\x00", b"\x01", b"\xff" * (kb - 1)]
    for s in spl:
        for j in range(len(s) + 1):
            p = s[:j]
            keys.append(p)
            keys += [p + bytes([b]) for b in (0, 1, 2, 0x61, 0xFE, 0xFF)]
            if p:
                keys += [p[:-1] + bytes([(p[-1] + d) & 0xFF]) for d in (-1, 1)]
    keys += [rich_bytes(rng, rng.randrange(0, kb)) for _ in range(300)]
    return [k for k in keys if fits(k, kb)]


def parse_table(out, P, n, kb):
    fin, img = int(out[0]), unhex(out[1])
    words = lambda off, cnt: [int.from_bytes(img[off + 8 * i:off + 8 * i + 8], "little") for i in range(cnt)]
    inv = words(0, 2 * P)
    pre = words(16 * P, n)
    slots = [] if kb == 8 else [img[16 * P + 8 * n + i * kb:16 * P + 8 * n + (i + 1) * kb] for i in range(n)]
    assert len(img) == 16 * P + 8 * n + len(slots) * kb
    return fin, inv, pre, slots


def range_pid(slot, pre, slots, fin):
    """range_pid (mrhbm_dev.cuh) over the image: binary search on the 64-bit prefixes, then the walk over ties"""
    kp = int.from_bytes(slot[:8], "big")
    top = 1 if fin else 0
    while top and top * 2 <= fin:
        top *= 2
    pos, step = 0, top
    while step:
        q = pos + step
        if q <= fin and pre[q - 1] <= kp:
            pos = q
        step >>= 1
    while slots and pos > 0 and pre[pos - 1] == kp and slot[8:] < slots[pos - 1][8:]:
        pos -= 1
    return pos


@pytest.mark.parametrize("kb", STR_KB)
def test_range_table_strings(codec, kb):
    rng = random.Random(kb + 2)
    sets = splitter_sets(kb)
    for spl in sets.values():
        assert spl == sorted(spl)
    names = list(sets)
    outs = codec([["T", kb, len(sets[nm]) + 1] + sets[nm] for nm in names])
    for nm, out in zip(names, outs):
        spl = sets[nm]
        P, n = len(spl) + 1, len(spl)
        fin, inv, pre, slots = parse_table(out, P, n, kb)
        assert inv == [0] * (2 * P)
        assert (fin < n) == (nm == "cut"), nm
        assert all(p == 0 for p in pre[fin:]) and all(s == bytes(kb) for s in slots[fin:])
        for i in range(fin):
            assert pre[i] == int.from_bytes(slots[i][:8], "big")
        for k in probe_keys(rng, spl, kb):
            slot = esc(k).ljust(kb, b"\0")
            assert range_pid(slot, pre, slots, fin) == bisect.bisect_right(spl, k), (nm, k)


def test_range_table_u64(codec):
    rng = random.Random(3)
    sets = [[], [0], [M64], [5, 5, 5], [1, 2, 3], [0, 0, M64, M64], sorted(rng.getrandbits(64) for _ in range(200)),
            sorted(rng.getrandbits(20) for _ in range(50)) + [1 << 63]]
    outs = codec([["T", 8, len(s) + 1] + [v.to_bytes(8, "big") for v in s] for s in sets])
    for spl, out in zip(sets, outs):
        P, n = len(spl) + 1, len(spl)
        fin, inv, pre, _ = parse_table(out, P, n, 8)
        assert fin == n and pre == spl
        bounds = [0] + spl + [1 << 64]
        for p in range(P):
            w = bounds[p + 1] - bounds[p]
            f = ((1 << 128) - 1) // w if w else 0
            assert (inv[2 * p], inv[2 * p + 1]) == (f >> 64, f & M64), (p, w)
        keys = [0, M64] + [v + d for v in spl for d in (-1, 0, 1) if 0 <= v + d <= M64]
        keys += [rng.getrandbits(64) for _ in range(200)]
        for k in keys:
            assert range_pid(k.to_bytes(8, "big"), pre, [], fin) == bisect.bisect_right(spl, k)


def word_hash(stored):
    """the device word hash over the little-endian u32 words of the stored (escaped) bytes while non-zero"""
    stored += b"\0" * (-len(stored) % 4)
    h = 0x9E3779B97F4A7C15
    for i in range(0, len(stored), 4):
        w = int.from_bytes(stored[i:i + 4], "little")
        if w == 0:
            break
        h = ((h ^ w) * 0xBF58476D1CE4E5B9) & M64
        h ^= h >> 29
    h ^= h >> 32
    return (h * 0x94D049BB133111EB) & M64


def test_host_partition_range(codec):
    rng = random.Random(4)
    for kb in STR_KB:
        for spl in splitter_sets(kb).values():
            keys = probe_keys(rng, spl, kb) + [s + b"x" for s in spl] + [rich_bytes(rng, kb + 9) for _ in range(50)]
            (out,) = codec([["H", 3, len(spl) + 1, len(spl)] + spl + keys])
            assert [int(x) for x in out] == [bisect.bisect_right(spl, k) for k in keys]


def test_host_partition_fnv_lua_golden(codec, golden_vectors, golden_wordcount):
    known = golden_vectors["partitionfn_known_answers"]
    keys = [k.encode() for k in known] + [k for k, _, _ in golden_wordcount]
    want = [p for p, _ in known.values()] + [p for _, p, _ in golden_wordcount]
    (out,) = codec([["H", 0, 15, 0] + keys])
    assert [int(x) for x in out] == want


def test_host_partition_wordhash(codec):
    rng = random.Random(5)
    keys = [b"", b"a", b"abcd", b"abcde", b"\x00", b"\x01\x01", b"\xff" * 3]
    keys += [rich_bytes(rng, n) for n in (3, 4, 5, 27, 28, 29, 59, 60, 123, 124, 125, 300) for _ in range(20)]
    for P in (1, 7, 1024, 65537):
        (out,) = codec([["H", 2, P, 0] + keys])
        assert [int(x) for x in out] == [(word_hash(esc(k)) * P) >> 64 for k in keys]
