"""Samsung V0 (SamsungV0Decompressor) for the tests: the CPU restatement and the row-stream writer of
tests/emu/samsung0_oracle.c, and synthetic frames."""
import ctypes as C
import os

import numpy as np

from helpers import compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "samsung0_oracle.c")
OUT = os.path.join(HERE, "emu", "_build", "libsamsung0_oracle.so")

# outcomes (S0_* of samsung0_oracle.c): the message the reference throws
OK, LEN_NEG, LEN_BIG, UP_FIRST, UP_LAST, OVERREAD, SHORT, DIMS, OFFSETS, BS_SKIP, BS_STREAM = range(11)
MESSAGES = {
    LEN_NEG: "Bit length less than 0.",
    LEN_BIG: "Bit Length more than 16.",
    UP_FIRST: "Upward prediction for the first two rows. Raw corrupt",
    UP_LAST: "Upward prediction for the last block of pixels. Raw corrupt",
    OVERREAD: "Buffer overflow read in BitStreamer",
    SHORT: "Bit stream size is smaller than MaxProcessBytes",
    DIMS: "Unexpected image dimensions found",
    OFFSETS: "Line offsets are out of sequence or slice is empty.",
    BS_SKIP: "Out of bounds access in ByteStream",
    BS_STREAM: "Buffer overflow: image file may be truncated",
}
RDE_MSGS = {LEN_NEG, LEN_BIG, UP_FIRST, UP_LAST, DIMS, OFFSETS}
CTOR_MSGS = {DIMS, OFFSETS, BS_SKIP, BS_STREAM}
FILL_DEFAULT = 0xABCD  # what an image holds before the decode (pixels the decode never writes)
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(OUT) or os.path.getmtime(SRC) > os.path.getmtime(OUT):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            compile_shared(["gcc", "-std=c99", "-O2", "-Wall", "-fPIC", "-shared", "-o", OUT, SRC])
        L = C.CDLL(OUT)
        L.s0_decompress.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_int, C.c_int,
                                    C.c_void_p, C.c_int, C.POINTER(C.c_uint32)]
        L.s0_write_row.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_int64]
        L.s0_write_row.restype = C.c_int64
        L.s0_fit.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def message_id(what):
    """The S0_* outcome of a reference exception message (what())."""
    for k, m in MESSAGES.items():
        if m in what:
            return k
    raise ValueError("unexpected message: %r" % what)


def pitch_elems(w):
    """RawImageData::createData(): pitch = roundUp(w*2, 16) bytes."""
    return (w * 2 + 15) // 16 * 16 // 2


def decompress(bso, bsr, w, h, fill=FILL_DEFAULT):
    """-> (image (h, pitch) uint16 with untouched pixels at `fill`, outcome, row << 9 | block)."""
    img = np.full((max(h, 1), pitch_elems(max(w, 1))), fill, dtype=np.uint16)
    where = C.c_uint32(0)
    rc = lib().s0_decompress(bytes(bso), len(bso), bytes(bsr), len(bsr), w, h, img.ctypes.data,
                             img.shape[1], C.byref(where))
    return img, rc, where.value


def nblocks(w):
    return (w + 15) // 16


def fit(values, dirs):
    """Stream choices for `values` (h, w) before the red/blue swap: -> (op, setlen, adj)."""
    h, w = values.shape
    nb = nblocks(w)
    v = np.ascontiguousarray(values, dtype=np.uint16)
    d = np.ascontiguousarray(dirs, dtype=np.uint8).reshape(h, nb)
    op = np.zeros((h, nb, 4), np.uint8)
    setlen = np.zeros((h, nb, 4), np.uint8)
    adj = np.zeros((h, nb, 16), np.int32)
    rc = lib().s0_fit(w, h, v.ctypes.data, d.ctypes.data, op.ctypes.data, setlen.ctypes.data, adj.ctypes.data)
    assert rc == 0, "a group needs 16 bits from a length below 15"
    return op, setlen, adj


def write_rows(dirs, op, setlen, adj):
    """Row streams (list of bytes) for per-block directions, ops, set lengths and adjs (stream order)."""
    h, nb = dirs.shape
    rows = []
    for r in range(h):
        d = np.ascontiguousarray(dirs[r], np.uint8)
        o = np.ascontiguousarray(op[r], np.uint8)
        s = np.ascontiguousarray(setlen[r], np.uint8)
        a = np.ascontiguousarray(adj[r], np.int32)
        cap = nb * 48 + 64
        buf = np.zeros(cap, np.uint8)
        n = lib().s0_write_row(r, nb, d.ctypes.data, o.ctypes.data, s.ctypes.data, a.ctypes.data,
                               buf.ctypes.data, cap)
        assert n >= 0
        rows.append(buf[:n].tobytes())
    return rows


def pack(rows, first=0):
    """(bso, bsr) for row streams laid back to back in bsr from byte `first`."""
    offs = np.cumsum([0] + [len(r) for r in rows[:-1]], dtype=np.int64) + first
    return offs.astype("<u4").tobytes(), bytes(first) + b"".join(rows)


def make_frame(values, dirs, first=0):
    """(bso, bsr, rows) of a frame that decodes to `values` (before the swap) with directions `dirs`."""
    op, setlen, adj = fit(values, dirs)
    rows = write_rows(np.asarray(dirs, np.uint8).reshape(values.shape[0], -1), op, setlen, adj)
    bso, bsr = pack(rows, first)
    return bso, bsr, rows


# ---------------------------------------------------------------- content and directions
def natural_values(w, h, seed=0):
    """Smooth gradients, texture and noise, 12-bit."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    f = 1200 + 900 * np.sin(x / 157.0) * np.cos(y / 211.0) + 600 * (x / max(w, 1))
    f += 250 * np.sin((x + 2 * y) / 9.0)
    f += rng.normal(0, 24, size=(h, w))
    return np.clip(f, 0, 4095).astype(np.uint16)


def _up_allowed(w, h):
    """Blocks that may predict upwards: rows from 2, and col + 16 < width."""
    nb = nblocks(w)
    ok = np.zeros((h, nb), bool)
    ok[2:, :] = (16 * np.arange(nb) + 16 < w)[None, :]
    return ok


def dirs_left(w, h):
    return np.zeros((h, nblocks(w)), np.uint8)


def dirs_up(w, h):
    """Every block that may predict upwards does."""
    return _up_allowed(w, h).astype(np.uint8)


def dirs_alternating(w, h):
    nb = nblocks(w)
    r, k = np.mgrid[0:h, 0:nb]
    return (_up_allowed(w, h) & ((r + k) % 2 == 1)).astype(np.uint8)


def dirs_staircase(w, h):
    """Block k predicts upwards below row s_k = k (h - 1) / (nb - 1) and from the left on it: the
    chain from the bottom right walks up and left through every row and block (depth ~ h + nb)."""
    nb = nblocks(w)
    r, k = np.mgrid[0:h, 0:nb]
    s = (k * (h - 1)) // max(nb - 1, 1)
    return (_up_allowed(w, h) & (r > s)).astype(np.uint8)


def dirs_random(w, h, seed=0):
    rng = np.random.default_rng(seed)
    return (_up_allowed(w, h) & (rng.random((h, nblocks(w))) < 0.5)).astype(np.uint8)


DIRS = {"left": dirs_left, "up": dirs_up, "alternating": dirs_alternating, "staircase": dirs_staircase}


def swap_rb(values, pitch):
    """The image decompress() leaves for `values` (h, w): the red/blue swap, in an (h, pitch) buffer
    whose padding holds FILL_DEFAULT."""
    h, w = values.shape
    v = values.copy()
    n = w // 2   # pairs (col, col + 1), col even, col < w - 1
    t = v[0:h - 1:2, 1:2 * n:2].copy()
    v[0:h - 1:2, 1:2 * n:2] = v[1:h:2, 0:2 * n:2]
    v[1:h:2, 0:2 * n:2] = t
    img = np.full((h, pitch), FILL_DEFAULT, np.uint16)
    img[:, :w] = v
    return img
