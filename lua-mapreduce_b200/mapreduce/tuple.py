"""Composite (tuple) keys over the HBM shuffle (mapreduce/tuple.lua).

The reference interns immutable tuples so that they can be table keys (tuple.lua:252-301) and
defines `<` on them (tuple.lua:183-195).  The device only knows byte-string keys, so a tuple key
crosses the C ABI as an ORDER-PRESERVING, NUL-free byte string (<= 123 bytes, the long-key record
class) and is decoded again on the reduce side:

    key      := 0x7F component            -- a scalar key (tuple(x) returns x unchanged, tuple.lua:255-257)
              | (0x80 | n) component * n  -- a tuple of n <= 31 components; shorter tuples sort first
    component:= 0x10 num10                -- Lua number: IEEE double, sign-folded, 10 big-endian 7-bit groups | 0x80
              | 0x20 bytes 0x01           -- Lua string (bytes >= 0x02), a proper prefix sorts first
              | 0x30 key                  -- nested tuple

Values (server:configure{hbm = {value_kind = "bytes"}}) cross the C ABI as opaque bytes that keep the Lua type:

    value    := 0x10 num10                -- Lua number, the key encoding above, except that -0 stays -0
              | 0x20 bytes                -- Lua string: any bytes, any length

Bytewise order of the key encoding = length first, then component-wise lexicographic.  The reference's
`__lt` (shorter first; same length: "no component greater") is only a partial order; this is a
linear extension of it: whenever the reference says a < b, encode(a) < encode(b)
(tests/test_tuple_keys.py checks that against `lt`, the restatement of tuple.lua:183-195).
"""
import math
import struct

MAX_KEY_BYTES = 123  # include/mrhbm.h: the 128-byte record class

_SCALAR, _TUPLE = 0x7F, 0x80
_NUM, _STR, _TUP = 0x10, 0x20, 0x30
_END = 0x01


def tuple_(*args):
    """tuple.lua:252-301: one non-table argument is returned unchanged, tables (lists / tuples here)
    become immutable tuples, recursively.  Python tuples hash by value, which is what the
    reference's interning provides."""
    t = args[0] if len(args) == 1 else args
    if not isinstance(t, (list, tuple)):
        return t
    return tuple(tuple_(v) if isinstance(v, (list, tuple)) else v for v in t)


def lt(a, b):
    """The reference's tuple `<` (tuple.lua:183-195), restated: not a tuple on the right -> false;
    shorter first; identical -> false; otherwise true iff no component of a is greater."""
    if not isinstance(b, tuple):
        return False
    if len(a) != len(b):
        return len(a) < len(b)
    if a == b:
        return False
    for x, y in zip(a, b):
        if (lt(y, x) if isinstance(x, tuple) else x > y):
            return False
    return True


def _enc_num(x, out, key=True):
    if isinstance(x, bool) or not isinstance(x, (int, float)):
        raise TypeError("not a number: %r" % (x,))
    if isinstance(x, int) and abs(x) > (1 << 53):
        raise OverflowError("integer %d is not exact as a Lua number" % x)
    f = float(x)
    if math.isnan(f):
        # (as a value: the reference's "%.14g" spill line cannot load() it back either)
        raise ValueError("NaN cannot be a key (Lua rejects it as a table index)" if key else "NaN cannot be a value")
    if key and f == 0.0:
        f = 0.0  # -0 and 0 are the same Lua table key
    (u,) = struct.unpack(">Q", struct.pack(">d", f))
    u = u ^ 0xFFFFFFFFFFFFFFFF if u >> 63 else u | (1 << 63)  # total order of doubles as unsigned
    out.append(_NUM)
    out.extend(0x80 | ((u >> s) & 0x7F) for s in range(63, -1, -7))  # 1 + 9*7 bits, big endian


def _dec_num(b, i):
    u = 0
    for k in range(10):
        u = (u << 7) | (b[i + k] & 0x7F)
    u &= 0xFFFFFFFFFFFFFFFF
    u = u & ~(1 << 63) if u >> 63 else u ^ 0xFFFFFFFFFFFFFFFF
    (f,) = struct.unpack(">d", struct.pack(">Q", u))
    if f == 0.0 and math.copysign(1.0, f) < 0:
        return f, i + 10  # -0 (values only: keys fold it to 0)
    return (int(f) if f.is_integer() and abs(f) <= (1 << 53) else f), i + 10


def _enc_component(v, out):
    if isinstance(v, tuple):
        out.append(_TUP)
        _enc_key(v, out)
    elif isinstance(v, (bytes, str)):
        s = v.encode() if isinstance(v, str) else v
        if any(c < 2 for c in s):
            raise ValueError("string components must not contain the bytes 0x00 / 0x01")
        out.append(_STR)
        out.extend(s)
        out.append(_END)
    else:
        _enc_num(v, out)


def _enc_key(k, out):
    if isinstance(k, tuple):
        if len(k) > 31:
            raise ValueError("tuples of more than 31 components are not supported")
        out.append(_TUPLE | len(k))
        for v in k:
            _enc_component(v, out)
    else:
        out.append(_SCALAR)
        _enc_component(k, out)


def encode(key):
    """key (scalar, tuple, nested tuples) -> NUL-free bytes, at most MAX_KEY_BYTES."""
    out = bytearray()
    _enc_key(tuple_(key) if isinstance(key, (list, tuple)) else key, out)
    if len(out) > MAX_KEY_BYTES:
        raise ValueError("encoded key takes %d bytes, the limit is %d" % (len(out), MAX_KEY_BYTES))
    return bytes(out)


def _dec_component(b, i):
    tag = b[i]
    if tag == _NUM:
        return _dec_num(b, i + 1)
    if tag == _STR:
        j = b.index(_END, i + 1)
        return bytes(b[i + 1:j]), j + 1
    if tag == _TUP:
        return _dec_key(b, i + 1)
    raise ValueError("bad component tag 0x%02x" % tag)


def _dec_key(b, i):
    head = b[i]
    if head == _SCALAR:
        return _dec_component(b, i + 1)
    if not head & _TUPLE:
        raise ValueError("bad key header 0x%02x" % head)
    out = []
    i += 1
    for _ in range(head & 0x1F):
        v, i = _dec_component(b, i)
        out.append(v)
    return tuple(out), i


def decode(b):
    """inverse of encode (string components come back as bytes, integral numbers as ints)."""
    k, i = _dec_key(b, 0)
    if i != len(b):
        raise ValueError("trailing bytes after the key")
    return k


def encode_value(v):
    """Lua string (bytes / str) or number -> the opaque bytes of a byte-values shuffle (see the module text)."""
    if isinstance(v, (bytes, bytearray, str)):
        return bytes([_STR]) + (v.encode() if isinstance(v, str) else bytes(v))
    out = bytearray()
    _enc_num(v, out, key=False)
    return bytes(out)


def decode_value(b):
    """inverse of encode_value (strings come back as bytes, integral numbers as ints, -0 as -0.0)."""
    if not b:
        raise ValueError("empty value encoding")
    if b[0] == _STR:
        return bytes(b[1:])
    if b[0] == _NUM and len(b) == 11:
        return _dec_num(b, 1)[0]
    raise ValueError("bad value encoding (tag 0x%02x, %d bytes)" % (b[0], len(b)))
