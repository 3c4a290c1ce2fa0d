"""Kodak DCR (KodakDecompressor) for the tests: the CPU restatement and stream writer of
tests/emu/kodak_oracle.c, the reference's tables (TableLookUp) in their three forms, and synthetic
content."""
import ctypes as C
import os
import re

import numpy as np

from helpers import compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "kodak_oracle.c")
OUT = os.path.join(HERE, "emu", "_build", "libkodak_oracle.so")

# outcomes: VALUE and OVERFLOW are the stream's (RSB200_KODAK_* of the C ABI), the rest the constructor's
OK, VALUE, OVERFLOW, CPP, DIMS, BPS, BYTESTREAM = range(7)
MESSAGES = {
    VALUE: "Value out of bounds %d (bps = %i)",
    OVERFLOW: "Buffer overflow: image file may be truncated",
    CPP: "Unexpected component count / data type",
    DIMS: "Unexpected image dimensions found: (%d; %d)",
    BPS: "Unexpected bits per sample: %i",
    BYTESTREAM: "Out of bounds access in ByteStream",
}
IOE_MSGS = {OVERFLOW, BYTESTREAM}
NONE, PLAIN, DITHER = 0, 1, 2  # table modes
FILL_DEFAULT = 0xABCD  # what an image holds before the decode (pixels the decode never writes)
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(OUT) or os.path.getmtime(SRC) > os.path.getmtime(OUT):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            compile_shared(["gcc", "-std=c99", "-O2", "-Wall", "-fPIC", "-shared", "-o", OUT, SRC])
        L = C.CDLL(OUT)
        P, i = C.c_void_p, C.c_int
        L.kd_decompress.argtypes = [C.c_char_p, C.c_uint32, i, i, i, i, i, P, P, i,
                                    C.POINTER(i), C.POINTER(i), C.POINTER(i)]
        L.kd_write.argtypes = [P, P, i, i, P, C.c_int64]
        L.kd_write.restype = C.c_int64
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
    for k, m in MESSAGES.items():
        pat = re.escape(m).replace("%d", "-?[0-9]+").replace("%i", "-?[0-9]+")
        if re.fullmatch(pat, text):
            return k
    raise ValueError("unexpected message: %r" % text)


def message(rc, w, h, bps, value):
    """The reference's text for outcome rc."""
    if rc == OK:
        return ""
    if rc == VALUE:
        return MESSAGES[VALUE] % (value, bps)
    if rc == DIMS:
        return MESSAGES[DIMS] % (w, h)
    if rc == BPS:
        return MESSAGES[BPS] % bps
    return MESSAGES[rc]


# ---------------------------------------------------------------- tables
def lookup_table(curve, dither):
    """TableLookUp::setTable (common/TableLookUp.cpp:50-85) of table 0: 65536 entries, or 2 x 65536
    {base, delta} when dithered."""
    curve = [int(c) for c in curve]
    n = len(curve)
    if not dither:
        t = np.empty(65536, np.uint16)
        t[:n] = curve
        t[n:] = curve[-1]
        return t
    t = np.zeros(2 * 65536, np.uint16)
    for i, c in enumerate(curve):
        lo = min(curve[i - 1] if i > 0 else c, c)
        hi = max(curve[i + 1] if i < n - 1 else c, c)
        t[2 * i] = min(max(c - (hi - lo + 2) // 4, 0), 65535)
        t[2 * i + 1] = hi - lo
    t[2 * n::2] = curve[-1]
    return t


def device_table(table, mode):
    """The plan's 65536-entry table for a RawImage table: entries 2*v of a dithered one."""
    return np.ascontiguousarray(table[0::2] if mode == DITHER else table, np.uint16)


# ---------------------------------------------------------------- restatement
def decompress(data, w, h, bps, mode=NONE, table=None, cpp=1, fill=FILL_DEFAULT):
    """-> (image (h, pitch) uint16, outcome, row, col, value)."""
    img = np.full((max(h, 1), pitch_elems(max(w, 1))), fill, np.uint16)
    r, c, v = C.c_int(), C.c_int(), C.c_int()
    tab = None if table is None else np.ascontiguousarray(table, np.uint16)
    data = bytes(data)
    rc = lib().kd_decompress(data, len(data), w, h, bps, cpp, mode,
                             None if tab is None else tab.ctypes.data, img.ctypes.data, img.shape[1],
                             C.byref(r), C.byref(c), C.byref(v))
    return img, rc, r.value, c.value, v.value


def consumed(rc, row, col):
    """rsb200_scan_result.consumed of a job failing with rc at (row, col)."""
    return 0 if rc == OK else rc << 28 | row << 13 | col


# ---------------------------------------------------------------- writer
def diffs(values):
    """Per-segment, per-parity differences of an (h, w) array of values (the predictors start at 0 in
    every segment of 256 pixels)."""
    v = np.asarray(values, np.int64)
    d = v.copy()
    d[:, 2:] -= v[:, :-2]
    for c in range(0, v.shape[1], 256):
        d[:, c:c + 2] = v[:, c:c + 2]
    return d


def codes_of(d):
    """-> (lens, codes) of differences |d| < 2^15: the only length that represents d (extend())."""
    d = np.asarray(d, np.int64)
    a = np.abs(d)
    lens = np.zeros(d.shape, np.uint8)
    for L in range(1, 16):
        lens[a >= (1 << (L - 1))] = L
    codes = np.where(d > 0, d, d + (1 << lens.astype(np.int64)) - 1)
    codes = np.where(lens == 0, 0, codes) & 0xFFFF
    return lens, codes.astype(np.uint16)


def write(lens, codes, w, h):
    """Stream bytes of raw per-pixel lengths and codes ((h, w) each)."""
    lens = np.ascontiguousarray(lens, np.uint8).reshape(-1)
    codes = np.ascontiguousarray(codes, np.uint16).reshape(-1)
    assert lens.size == w * h and codes.size == w * h
    cap = h * ((w + 255) // 256) * 700
    out = np.zeros(cap, np.uint8)
    n = lib().kd_write(lens.ctypes.data, codes.ctypes.data, w, h, out.ctypes.data, cap)
    assert n >= 0
    return out[:n].tobytes()


def encode(values):
    """Stream bytes that decode to the (h, w) values (any ints whose differences fit 15 bits)."""
    v = np.asarray(values)
    lens, codes = codes_of(diffs(v))
    return write(lens, codes, v.shape[1], v.shape[0])


def natural(w, h, bps, seed=0):
    """Smooth content with noise, within [0, 2^bps)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    top = (1 << bps) - 1
    base = (top * 0.5 * (1 + np.sin(x / 97.0 + seed) * np.cos(y / 61.0))).astype(np.int64)
    noise = rng.integers(-40, 41, size=(h, w))
    return np.clip(base + noise, 0, top)


def random_values(w, h, bps, seed=0):
    return np.random.default_rng(seed).integers(0, 1 << bps, size=(h, w))


def max_read(w, h):
    """The most bytes a frame of w x h can read: 608 per full segment and the tail's maximum per row."""
    t = w % 256
    row = 608 * (w // 256)
    if t:
        e = 2 if t % 8 == 4 else 0
        row += t // 2 + e + 4 * ((max(0, 15 * t - 8 * e) + 31) // 32)
    return row * h
