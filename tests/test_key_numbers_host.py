"""The decimal parser of mrhbm_map_key_numbers on the CPU: the shared grammar and conversion (csrc/mrhbm_decimal.cuh),
host-compiled from tests/native/decimal_parse_check.cu, against a reference regex and Python's float() on random and
adversarial tokens; its power-of-five table against Python's exact integers; and server.configure's refusals of the
declaration hbm_mapfn = "key_numbers_file"."""
import os
import random
import re
import shutil
import struct
import subprocess
from decimal import Decimal, localcontext
from fractions import Fraction

import pytest

import mrhbm_loader

mrhbm_loader.load()
from lua_mapreduce_b200.mapreduce import server  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRAMMAR = re.compile(r"[+-]?([0-9]+(\.[0-9]*)?|\.[0-9]+)([eE][+-]?[0-9]+)?\Z")


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def sig_digits(tok):
    """significant digits: first to last non-zero digit of the significand"""
    m = re.match(r"[+-]?([0-9.]*)", tok).group(1).replace(".", "").strip("0")
    return len(m)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    out = str(tmp_path_factory.mktemp("dec") / "decimal_parse_check")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "lua-mapreduce_b200", "csrc"),
                           "-o", out, os.path.join(ROOT, "tests", "native", "decimal_parse_check.cu")])
    return out


def run(exe, toks):
    out = subprocess.run([exe], input="\n".join(toks) + "\n", capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr
    res = out.stdout.splitlines()
    assert len(res) == len(toks)
    return res


def check(exe, toks):
    """every token: grammar as the regex; E tokens give float()'s bits on the device path; only >19-digit tokens
    (H19) and the ambiguous case (HEL, <= 19 digits, exponent outside -27..55) go to the host, which gives the bits
    too.  Returns the paths taken."""
    paths = {}
    for tok, line in zip(toks, run(exe, toks)):
        if not GRAMMAR.match(tok):
            assert line == "bad", (tok, line)
            continue
        want = "%016x" % bits(float(tok))
        path, dev, host = line.split()
        assert host == want, (tok, line, want)
        if path == "E":
            assert dev == want, (tok, line, want)
            assert sig_digits(tok) <= 19, tok
        elif path == "H19":
            assert sig_digits(tok) > 19, tok
        else:
            assert path == "HEL" and sig_digits(tok) <= 19, (tok, line)
        paths[path] = paths.get(path, 0) + 1
    return paths


def test_grammar_and_special_tokens(exe):
    toks = ["-0", "+.5", "5.", ".e1", "1e", "0x10", "inf", "nan", "1_0", "-0.0", "+0", "0", ".5", "-.5e-3", "5.e2",
            "1e+5", "1E-5", "1e999999999", "0e999999999", "-1e999999999", "1e-999999999", "-0e-999999999", "", "+",
            "-", ".", "e5", "1e5.5", "1.2.3", "--1", "+-1", "1e--5", " 1", "1 ", "0x1p3", "INF", "-nan", "Infinity",
            "1d5", "1,5", "١", "00000000000000000000000001", "0.000000000000000000000000000001000000000000000"]
    check(exe, toks)
    out = dict(zip(toks, run(exe, toks)))
    assert out["-0"].split()[1] == "8000000000000000"
    assert out["0e999999999"].split()[1] == "0000000000000000"
    assert out["1e999999999"].split()[1] == "7ff0000000000000"


def test_random_significands_and_exponents(exe):
    rng = random.Random(11)
    toks = []
    for _ in range(60000):
        nd = rng.randint(1, 19)
        d = str(rng.randrange(10 ** (nd - 1), 10 ** nd))
        form = rng.randrange(4)
        if form == 0:
            t = d + "e" + str(rng.randint(-360, 330))
        elif form == 1:
            k = rng.randint(0, nd)
            t = d[:k] + "." + d[k:] + ("e%d" % rng.randint(-40, 40) if rng.random() < 0.5 else "")
        elif form == 2:
            t = d + "e" + str(rng.randint(-30, 30))
        else:
            t = "0." + "0" * rng.randint(0, 330) + d
        if rng.random() < 0.3:
            t = rng.choice("+-") + t
        toks.append(t)
    for _ in range(20000):  # what text columns hold: %.2f, integers, repr()
        x = rng.uniform(-1e6, 1e6) * 10 ** rng.randint(-5, 5)
        toks += ["%.2f" % x, str(int(x)), repr(x)]
    for _ in range(5000):
        toks.append(repr(struct.unpack("<d", struct.pack("<Q", rng.getrandbits(63)))[0]))
    paths = check(exe, toks)
    assert paths.get("H19", 0) == 0 and paths.get("E", 0) > 0


def test_halfway_points(exe):
    """exact midpoints between neighbouring doubles, and their neighbours one unit in the last digit away"""
    rng = random.Random(12)
    pts = [0.0, 5e-324, 1e-323, 2.2250738585072014e-308, 2.225073858507201e-308, 1.0, 2.0 ** 53, 9007199254740993.0,
           1.7976931348623155e308]
    pts += [struct.unpack("<d", struct.pack("<Q", rng.getrandbits(62)))[0] for _ in range(300)]
    pts += [float(rng.randrange(1, 2 ** 53)) * 2.0 ** rng.randint(-1074, 40) for _ in range(300)]
    toks = []
    for a in pts:
        a = abs(a)
        b = struct.unpack("<d", struct.pack("<Q", bits(a) + 1))[0]
        if b == float("inf"):
            continue
        with localcontext() as dc:
            dc.prec = 1200  # exact: a midpoint has at most 767 significant digits
            h = (Decimal(a) + Decimal(b)) / 2
            assert Fraction(h) == (Fraction(a) + Fraction(b)) / 2
            s = format(h, "e")
        toks.append(s)
        toks.append("-" + s)
        m, e = s.split("e")
        # one unit in the last digit above and below the midpoint, and the midpoint cut to 17 and 19 digits
        ulp = Decimal(1).scaleb(int(e) - (len(m.replace(".", "")) - 1))
        with localcontext() as dc:
            dc.prec = 1200
            toks += [format(h + ulp, "e"), format(h - ulp, "e")]
        for nd in (17, 19):
            toks.append(format(h, ".%de" % (nd - 1)))
    toks += ["1.7976931348623158e308", "1.7976931348623159e308", "1.797693134862315807e308",
             "1.797693134862315808e308", "2.4703282292062327e-324", "2.4703282292062328e-324",
             "4.9406564584124654e-324", "2.2250738585072011e-308", "2.2250738585072012e-308",
             "9007199254740993", "9007199254740992.5", "9007199254740993.0000000000001"]
    paths = check(exe, toks)
    assert paths["H19"] > 0 and paths["E"] > 0


def test_long_tokens(exe):
    rng = random.Random(13)
    toks = []
    for _ in range(400):
        nd = rng.randint(20, 800)
        d = str(rng.randrange(1, 10)) + "".join(rng.choice("0123456789") for _ in range(nd - 1))
        k = rng.randint(0, nd)
        toks.append(d[:k] + "." + d[k:] + "e%d" % rng.randint(-400 - nd, 330))
    toks += ["1" + "0" * 30, "1" + "0" * 30 + ".000", "0." + "0" * 400 + "1", "1." + "0" * 790 + "1",
             "123456789012345678.9", "1234567890123456789.0", "12345678901234567890"]
    check(exe, toks)


def test_power_of_five_table(exe):
    out = subprocess.run([exe, "--table"], capture_output=True, text=True, timeout=300)
    lines = out.stdout.splitlines()
    assert len(lines) == 308 + 342 + 1
    for line in lines:
        q, hi, lo = line.split()
        q = int(q)
        if q >= 0:
            p = 5 ** q
            want = p << (128 - p.bit_length()) if p.bit_length() <= 128 else p >> (p.bit_length() - 128)
        else:
            p = 5 ** -q
            z = p.bit_length()
            c = (1 << (z + 127 if q >= -27 else 2 * z + 128)) // p + 1
            want = c >> max(0, c.bit_length() - 128)
        assert want.bit_length() == 128 and int(hi + lo, 16) == want, q


KNS = "lua_mapreduce_b200.mapreduce.examples.KeyNumberSum"


class StandIn:
    def __init__(self, h):
        self.h = dict(h)


def configure(**hbm):
    S = KNS + ".init"
    s = server.new("hbm://local", "key-numbers-configure")
    s.ctx_factory = StandIn
    s.configure(dict(taskfn=S, mapfn=KNS + ".mapfn_device", partitionfn=S, reducefn=KNS + ".reducefn_device",
                     finalfn=S, combinerfn=KNS + ".combinerfn", storage="hbm", hbm=hbm))
    return s


@pytest.mark.parametrize("hbm, msg", [
    (dict(value_kind="int"), "value_kind"),
    (dict(value_kind="bytes", key_kind="u64"), "key_kind"),
    (dict(value_kind="bytes", key_kind="tuple"), "key_kind"),
])
def test_configure_refuses_key_numbers_without_bytes_and_string_keys(hbm, msg):
    with pytest.raises(ValueError, match=msg):
        configure(**hbm)


def test_configure_accepts_key_numbers_on_bytes_and_string_keys():
    h = configure(value_kind="bytes").config["hbm"]
    assert h["key_kind"] == "str" and h["reducer"] == 3 and h["combiner"] == "fsum"
