"""Samsung V2 (SamsungV2Decompressor) for the tests: the constructor's checks and the 16-byte header
(SamsungV2Decompressor.cpp:85-143), the CPU restatement and stream writer of
tests/emu/samsung2_oracle.c, a bit writer for raw scripts, and synthetic content."""
import ctypes as C
import os
import re

import numpy as np

from helpers import compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "samsung2_oracle.c")
OUT = os.path.join(HERE, "emu", "_build", "libsamsung2_oracle.so")

# outcomes: 1..8 are the stream's (S2_* of samsung2_oracle.c, RSB200_S2_* of the C ABI), 9.. the
# constructor's
(OK, START_MOTION, MOTION_BEGIN, MOTION_END, UNDERFLOW, TOO_MANY, OVERREAD, SHORT, BYTESTREAM,
 CPP, BITS, DEPTH, FLAGS, DIMS, EXIF) = range(15)
MESSAGES = {
    START_MOTION: "At start of image and motion isn't 7. File corrupted?",
    MOTION_BEGIN: "Bad motion %d at the beginning of the row",
    MOTION_END: "Bad motion %d at the end of the row",
    UNDERFLOW: "Difference bits underflow. File corrupted?",
    TOO_MANY: "Too many difference bits (%u). File corrupted?",
    OVERREAD: "Buffer overflow read in BitStreamer",
    SHORT: "Bit stream size is smaller than MaxProcessBytes",
    BYTESTREAM: "Out of bounds access in ByteStream",
    CPP: "Unexpected component count / data type",
    BITS: "Unexpected bit per pixel (%u)",
    DEPTH: "Bit depth mismatch with container, %u vs %u",
    FLAGS: "Invalid opt flags %x",
    DIMS: "Unexpected image dimensions found: (%i; %i)",
    EXIF: "EXIF image dimensions do not match dimensions from raw header",
}
IOE_MSGS = {OVERREAD, SHORT, BYTESTREAM}
SKIP, MV, QP = 1, 2, 4
FILL_DEFAULT = 0xABCD  # what an image holds before the decode (pixels the decode never writes)
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(OUT) or os.path.getmtime(SRC) > os.path.getmtime(OUT):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            compile_shared(["gcc", "-std=c99", "-O2", "-Wall", "-fPIC", "-shared", "-o", OUT, SRC])
        L = C.CDLL(OUT)
        L.s2_decompress.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_void_p, C.c_int, C.POINTER(C.c_uint32), C.c_void_p]
        L.s2_encode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                C.c_uint64, C.c_void_p, C.c_void_p, C.c_int64]
        L.s2_encode.restype = C.c_int64
        _lib = L
    return _lib


def pitch_elems(w):
    """RawImageData::createData(): pitch = roundUp(w*2, 16) bytes."""
    return (w * 2 + 15) // 16 * 16 // 2


def strip_prefix(what):
    """The message of a reference exception's what(), without the "function, line N: " in front."""
    i = what.find(": ", what.find(", line ") + 1) if ", line " in what else -1
    return what[i + 2:] if i >= 0 else what


def message_id(text):
    """The outcome of a message (its printed values in place)."""
    for k, m in MESSAGES.items():
        pat = re.escape(m).replace("%d", "-?[0-9]+").replace("%u", "[0-9]+").replace("%i", "-?[0-9]+")
        if re.fullmatch(pat.replace("%x", "[0-9a-f]+"), text):
            return k
    raise ValueError("unexpected message: %r" % text)


# ---------------------------------------------------------------- header
def header(w, h, bits=12, flags=0, init=0, depth=None, nlc=0x0200, fmt=0, tile=0, raw=None):
    """The 16-byte header (MSB32): NLCVersion 16, ImgFormat 4, bitDepth - 1 4, NumBlkInRCUnit 4,
    CompressionRatio 4, width 16, height 16, TileWidth 16, reserved 4, optflags 4, OverlapWidth 8,
    reserved 8, Inc 8, reserved 2, initVal 14."""
    if raw is not None:
        return bytes(raw)
    b = BitWriter()
    b.put(nlc, 16)
    b.put(fmt, 4)
    b.put((bits if depth is None else depth) - 1, 4)
    b.put(0, 8)
    b.put(w, 16)
    b.put(h, 16)
    b.put(tile, 16)
    b.put(0, 4)
    b.put(flags, 4)
    b.put(0, 24)
    b.put(0, 2)
    b.put(init, 14)
    return b.bytes()


def parse_header(hdr):
    """-> dict of the header's fields (16 bytes)."""
    words = np.frombuffer(bytes(hdr[:16]), "<u4")
    v = 0
    for x in words:
        v = (v << 32) | int(x)

    def f(pos, n):
        return (v >> (128 - pos - n)) & ((1 << n) - 1)
    return {"depth": f(20, 4) + 1, "width": f(32, 16), "height": f(48, 16), "flags": f(84, 4),
            "init": f(114, 14)}


class BitWriter:
    """MSB32 bits: most significant bit first into 32-bit little-endian chunks."""

    def __init__(self):
        self.bits = []

    def put(self, v, n):
        for b in range(n - 1, -1, -1):
            self.bits.append((int(v) >> b) & 1)
        return self

    def pad_bytes(self, rng=None, to=1):
        """Fill to a multiple of `to` bytes (random bits if rng, else zeros)."""
        while len(self.bits) % (8 * to):
            self.bits.append(int(rng.integers(0, 2)) if rng is not None else 0)
        return self

    def bytes(self):
        bits = self.bits + [0] * (-len(self.bits) % 32)
        out = bytearray()
        for i in range(0, len(bits), 32):
            w = 0
            for b in bits[i:i + 32]:
                w = (w << 1) | b
            out += w.to_bytes(4, "little")
        return bytes(out)

    def nbytes(self):
        return (len(self.bits) + 7) // 8


# ---------------------------------------------------------------- restatement
def decompress(data, w, h, bits=12, cpp=1, fill=FILL_DEFAULT, ends=None):
    """SamsungV2Decompressor(RawImage(w, h, cpp), data, bits).decompress() ->
    (image (h, pitch) uint16 with untouched pixels at `fill`, outcome, where, message).
    where = value << 22 | row << 9 | block for the stream's failures (0 otherwise).  ends: an
    (h,) uint32 array that gets the data position behind each decoded row."""
    img = np.full((max(h, 1), pitch_elems(max(w, 1))), fill, dtype=np.uint16)
    if cpp != 1:
        return img, CPP, 0, MESSAGES[CPP]
    if bits not in (12, 14):
        return img, BITS, 0, MESSAGES[BITS] % bits
    data = bytes(data)
    if len(data) < 16:
        return img, BYTESTREAM, 0, MESSAGES[BYTESTREAM]
    hd = parse_header(data)
    if hd["depth"] != bits:
        return img, DEPTH, 0, MESSAGES[DEPTH] % (hd["depth"], bits)
    if hd["flags"] > 7:
        return img, FLAGS, 0, MESSAGES[FLAGS] % hd["flags"]
    hw, hh = hd["width"], hd["height"]
    if hw == 0 or hh == 0 or hw % 16 != 0 or hw > 6496 or hh > 4336:
        return img, DIMS, 0, MESSAGES[DIMS] % (hw, hh)
    if hw != w or hh != h:
        return img, EXIF, 0, MESSAGES[EXIF]
    where = C.c_uint32(0)
    rc = lib().s2_decompress(data[16:], len(data) - 16, bits, hd["flags"], hd["init"], w, h,
                             img.ctypes.data, img.shape[1], C.byref(where),
                             None if ends is None else ends.ctypes.data)
    return img, rc, where.value, message(rc, where.value)


def message(rc, where):
    """The text of a stream outcome (the value printed is where >> 22)."""
    if rc == OK:
        return ""
    m = MESSAGES[rc]
    return m % (where >> 22) if "%" in m else m


def consumed(rc, where):
    """RSB200 `consumed` of a stream outcome: code << 28 | where."""
    return 0 if rc == OK else (rc << 28 | where)


def encode(values, bits=12, flags=0, init=0, policy=0, seed=0):
    """The whole strip (header + data) that decodes to `values` (h, w) < 2^bits.  policy: 0 cheapest
    motion, 1 all 7 (left), 2 all up (3), 3 averaging (2 / 4), 4 random valid motions."""
    v = np.ascontiguousarray(np.asarray(values, np.uint16))
    h, w = v.shape
    tmp = np.zeros_like(v)
    cap = w * h * 4 + h * 32 + 64
    buf = np.zeros(cap, np.uint8)
    n = lib().s2_encode(v.ctypes.data, w, h, w, bits, flags, init, policy, seed, tmp.ctypes.data,
                        buf.ctypes.data, cap)
    assert n >= 0
    return header(w, h, bits, flags, init) + buf[:n].tobytes()


# ---------------------------------------------------------------- content
def natural_values(w, h, bits=12, seed=0):
    """Smooth gradients, texture and noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    s = (1 << bits) / 4096.0
    f = 1200 + 900 * np.sin(x / 157.0) * np.cos(y / 211.0) + 600 * (x / max(w, 1))
    f += 250 * np.sin((x + 2 * y) / 9.0)
    f = f * s + rng.normal(0, 24 * s, size=(h, w))
    return np.clip(f, 0, (1 << bits) - 1).astype(np.uint16)


def flat_values(w, h, bits=12, seed=0):
    return np.full((h, w), 1000 * (1 << bits) // 4096, np.uint16)


def random_values(w, h, bits=12, seed=0):
    return np.random.default_rng(seed).integers(0, 1 << bits, (h, w)).astype(np.uint16)


CONTENT = {"natural": natural_values, "flat": flat_values, "random": random_values}


def padded(values, fill=FILL_DEFAULT):
    """`values` (h, w) in an (h, pitch) buffer whose padding holds `fill`."""
    h, w = values.shape
    img = np.full((h, pitch_elems(w)), fill, np.uint16)
    img[:, :w] = values
    return img
