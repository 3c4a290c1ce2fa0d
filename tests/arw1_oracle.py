"""Sony ARW1 (SonyArw1Decompressor) for the tests: the CPU restatement and the stream writer of
tests/emu/arw1_oracle.c, and synthetic frames."""
import ctypes as C
import os

import numpy as np

from helpers import compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "arw1_oracle.c")
OUT = os.path.join(HERE, "emu", "_build", "libarw1_oracle.so")

OK, RDE, IOE, CTOR = 0, 1, 2, 3
FILL_DEFAULT = 0xABCD  # what an image holds before the decode (pixels the decode never writes)
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(OUT) or os.path.getmtime(SRC) > os.path.getmtime(OUT):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            compile_shared(["gcc", "-std=c99", "-O2", "-Wall", "-fPIC", "-shared", "-o", OUT, SRC])
        L = C.CDLL(OUT)
        L.arw1_decompress.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                      C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
        L.arw1_decompress.restype = C.c_int
        L.arw1_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int]
        L.arw1_encode.restype = C.c_int64
        _lib = L
    return _lib


def pitch_elems(w):
    """RawImageData::createData(): pitch = roundUp(w*2, 16) bytes."""
    return (w * 2 + 15) // 16 * 16 // 2


def decompress(data, w, h, fill=FILL_DEFAULT):
    """-> (image (h, pitch) uint16 with untouched pixels at `fill`, status, where)."""
    data = np.ascontiguousarray(np.frombuffer(bytes(data), dtype=np.uint8))
    img = np.full((max(h, 1), pitch_elems(max(w, 1))), fill, dtype=np.uint16)
    where, cons = C.c_uint32(0), C.c_uint64(0)
    buf = data if data.size else np.zeros(1, np.uint8)
    rc = lib().arw1_decompress(buf.ctypes.data, data.size, w, h, img.ctypes.data, img.shape[1],
                               C.byref(where), C.byref(cons))
    return img, rc, where.value


def encode(diffs, lens=None, pad_bit=0):
    """One symbol per difference (stream order); lens[i] >= 0 forces a symbol's length."""
    d = np.ascontiguousarray(diffs, dtype=np.int32)
    ln = None if lens is None else np.ascontiguousarray(lens, dtype=np.int8)
    cap = 4 * d.size + 16
    out = np.zeros(cap, np.uint8)
    n = lib().arw1_encode(d.ctypes.data, None if ln is None else ln.ctypes.data, d.size,
                          out.ctypes.data, cap, pad_bit)
    assert n >= 0, "difference out of range"
    return out[:n].tobytes()


def stream_rows_cols(w, h):
    """(row, col) of every stream index: columns from the right, even rows then odd rows."""
    i = np.arange(w * h, dtype=np.int64)
    col = w - 1 - i // h
    k = i % h
    row = np.where(k < h // 2, 2 * k, 2 * (k - h // 2) + 1)
    return row, col


def frame_diffs(frame):
    """Differences in stream order that decode to `frame` (h, w) of 0..4095 values."""
    h, w = frame.shape
    row, col = stream_rows_cols(w, h)
    v = frame[row, col].astype(np.int64)
    return np.diff(v, prepend=0).astype(np.int32)


def encode_frame(frame, pad_bit=0):
    return encode(frame_diffs(frame), pad_bit=pad_bit)


def natural_frame(w, h, seed=0):
    """Smooth gradients, texture and noise, 12-bit."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    f = 1200 + 900 * np.sin(x / 157.0) * np.cos(y / 211.0) + 600 * (x / max(w, 1))
    f += 250 * np.sin((x + 2 * y) / 9.0)
    f += rng.normal(0, 24, size=(h, w))
    return np.clip(f, 0, 4095).astype(np.uint16)


def uniform_frame(w, h, value=512):
    return np.full((h, w), value, dtype=np.uint16)


def clipped_frame(w, h, c0, ncols, seed=0):
    """A natural frame with columns c0..c0+ncols-1 clipped to 4095 (a flat run in the stream)."""
    f = natural_frame(w, h, seed)
    f[:, c0:c0 + ncols] = 4095
    return f
