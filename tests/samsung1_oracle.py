"""Samsung V1 (SamsungV1Decompressor) for the tests: the CPU restatement and the stream writer of
tests/emu/samsung1_oracle.c, and synthetic frames."""
import ctypes as C
import os

import numpy as np

from helpers import compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "samsung1_oracle.c")
OUT = os.path.join(HERE, "emu", "_build", "libsamsung1_oracle.so")

# outcomes (S1_* of samsung1_oracle.c): the message the reference throws
OK, OOB, OVERREAD, SHORT, DIMS, BITS, CPP = range(7)
MESSAGES = {
    OOB: "decoded value out of bounds",
    OVERREAD: "Buffer overflow read in BitStreamer",
    SHORT: "Bit stream size is smaller than MaxProcessBytes",
    DIMS: "Unexpected image dimensions found",
    BITS: "Unexpected bit per pixel",
    CPP: "Unexpected component count / data type",
}
RDE_MSGS = {OOB, DIMS, BITS, CPP}
FILL_DEFAULT = 0xABCD  # what an image holds before the decode (pixels the decode never writes)
# SamsungV1Decompressor.cpp:88-101: (encLen, diffLen)
TAB = [(3, 4), (3, 7), (2, 6), (2, 5), (4, 3), (6, 0), (7, 9), (8, 10), (9, 11), (10, 12), (10, 13),
       (5, 1), (4, 8), (4, 2)]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(OUT) or os.path.getmtime(SRC) > os.path.getmtime(OUT):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            compile_shared(["gcc", "-std=c99", "-O2", "-Wall", "-fPIC", "-shared", "-o", OUT, SRC])
        L = C.CDLL(OUT)
        L.s1_decompress.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                    C.c_int, C.POINTER(C.c_uint32)]
        L.s1_encode.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        L.s1_encode.restype = C.c_int64
        _lib = L
    return _lib


def message_id(what):
    """The outcome of a reference exception message (what())."""
    for k, m in MESSAGES.items():
        if m in what:
            return k
    raise ValueError("unexpected message: %r" % what)


def pitch_elems(w):
    """RawImageData::createData(): pitch = roundUp(w*2, 16) bytes."""
    return (w * 2 + 15) // 16 * 16 // 2


def decompress(data, w, h, bit=12, cpp=1, fill=FILL_DEFAULT):
    """-> (image (h, pitch) uint16 with untouched pixels at `fill`, outcome, row << 14 | col).
    cpp: components per pixel of the image, which the constructor checks first."""
    img = np.full((max(h, 1), pitch_elems(max(w, 1))), fill, dtype=np.uint16)
    if cpp != 1:
        return img, CPP, 0
    where = C.c_uint32(0)
    rc = lib().s1_decompress(bytes(data), len(data), w, h, bit, img.ctypes.data, img.shape[1],
                             C.byref(where))
    return img, rc, where.value


def encode(diffs):
    """The stream (bytes) of the differences, in stream order (|d| < 8192)."""
    d = np.ascontiguousarray(np.asarray(diffs, np.int32).ravel())
    cap = (d.size * 23 + 7) // 8 + 16
    buf = np.zeros(cap, np.uint8)
    n = lib().s1_encode(d.ctypes.data, d.size, buf.ctypes.data, cap)
    assert n >= 0
    return buf[:n].tobytes()


def diffs_of(values):
    """Differences (h, w) int32 that make decompress() produce `values` (h, w)."""
    v = np.asarray(values, np.int32)
    d = v.copy()
    d[:, 2:] -= v[:, :-2]
    d[2:, :2] -= v[:-2, :2]
    return d


def make_stream(values, tail=8):
    """A stream that decodes to `values`, with `tail` zero bytes behind it (the decoder over-reads)."""
    return encode(diffs_of(values)) + bytes(tail)


def tstar(size):
    """First stream bit at which a symbol's refill fails."""
    return 0 if size < 4 else 32 * ((size + 8) // 4) + 10


# ---------------------------------------------------------------- content
def natural_values(w, h, seed=0):
    """Smooth gradients, texture and noise, 12-bit."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    f = 1200 + 900 * np.sin(x / 157.0) * np.cos(y / 211.0) + 600 * (x / max(w, 1))
    f += 250 * np.sin((x + 2 * y) / 9.0)
    f += rng.normal(0, 24, size=(h, w))
    return np.clip(f, 0, 4095).astype(np.uint16)


def flat_values(w, h, v=1000):
    return np.full((h, w), v, np.uint16)


def clipped_values(w, h, seed=0, rows=(0.3, 0.45)):
    """Natural content with a band of rows at 4095 (a clipped sky), longer than one range's halo."""
    v = natural_values(w, h, seed)
    v[int(rows[0] * h):int(rows[1] * h), :] = 4095
    return v


def longcode_values(w, h, seed=0):
    """Every difference of 12 or 13 bits: alternating extremes with noise."""
    rng = np.random.default_rng(seed)
    v = np.where((np.arange(w)[None, :] // 2 + np.arange(h)[:, None] // 2) % 2 == 0,
                 rng.integers(0, 64, (h, w)), rng.integers(4032, 4096, (h, w)))
    return v.astype(np.uint16)


CONTENT = {"natural": natural_values, "flat": lambda w, h, seed=0: flat_values(w, h),
           "clipped": clipped_values, "longcode": longcode_values}


def padded(values, fill=FILL_DEFAULT):
    """`values` (h, w) in an (h, pitch) buffer whose padding holds `fill`."""
    h, w = values.shape
    img = np.full((h, pitch_elems(w)), fill, np.uint16)
    img[:, :w] = values
    return img
