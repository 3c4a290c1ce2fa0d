"""Kodak DCR kernels (rawspeed_b200/csrc/kodak.cuh) without a GPU: the kernel bodies compiled by g++
against tests/emu/cuda_emu.h and run in the plan's order and layout, with every CTA's threads as fibers
in forward and in reverse order, compared with the restatement of KodakDecompressor
(tests/emu/kodak_oracle.c, pinned against the reference in tests/test_oracle_kodak.py): the whole output
buffer with sentinels around every frame, status, `consumed` and the printed value.  The candidate
entries are checked directly: every one is a failure or a candidate within 0..ncand - 1, and on the
true chain each row start leads to the next.  Parity of the real kernels is tests/test_gpu_kodak.py's
job."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import compile_shared

import kodak_oracle as K
import test_oracle_kodak as T

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "kodak_emu.cpp")
OUT = os.path.join(HERE, "emu", "_build", "libkodak_emu.so")
DEPS = [SRC, os.path.join(HERE, "emu", "cuda_emu.h"),
        os.path.join(HERE, "..", "rawspeed_b200", "csrc", "kodak.cuh")]
FILL = K.FILL_DEFAULT
GAP = 32  # sentinel pixels before every frame and behind the last
FAIL = 1 << 31
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in DEPS):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            compile_shared(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas",
                            "-Wno-unused-function", "-fPIC", "-shared", "-o", OUT, SRC])
        L = C.CDLL(OUT)
        P = C.c_void_p
        L.kd_emu_run.argtypes = [P, C.c_uint64, C.c_int] + [P] * 12 + [C.c_int, P, C.c_uint64, P, C.c_uint64, P, P]
        L.kd_emu_run.restype = C.c_uint64
        _lib = L
    return _lib


def stride(w):
    t = w % 256
    return 4 if (t // 2 + (2 if t % 8 == 4 else 0)) % 4 == 0 else 2


def run_emu(frames, reverse, skew=0):
    """frames: [(data, w, h, bps, mode, table)] -> (images, results, values, tables)."""
    n = len(frames)
    blob, ioff, tabs, tix = bytearray(), [], [], []
    for data, w, h, bps, mode, table in frames:
        blob += bytes((-len(blob)) % 16 + skew)
        ioff.append(len(blob))
        blob += data
        if mode == K.NONE:
            tix.append(0xFFFFFFFF)
        else:
            tix.append(65536 * len(tabs))
            tabs.append(K.device_table(table, mode))
    u32 = lambda xs: np.array(xs, np.uint32)  # noqa: E731
    isz, w, h, bps = (u32([f[i] if i else len(f[0]) for f in frames]) for i in (0, 1, 2, 3))
    oo, op, layout, pos = [], [], [], 0
    for data, fw, fh, *_ in frames:
        pitch = K.pitch_elems(fw)
        pos += GAP
        oo.append(2 * pos)
        op.append(2 * pitch)
        layout.append((pos, fh, pitch))
        pos += fh * pitch
    pos += GAP
    out = np.full(pos, FILL, np.uint16)
    res = np.zeros(2 * n, np.uint32)
    vals = np.zeros(n, np.int32)
    fail = np.zeros(2 * n, np.uint32)
    counts = np.zeros(2, np.uint64)
    ncand = sum(len(f[0]) // stride(f[1]) + 1 for f in frames)
    tab = np.zeros(ncand, np.uint32)
    rows = np.zeros(int(h.sum()), np.uint32)
    tables = np.concatenate(tabs) if tabs else np.zeros(1, np.uint16)
    ioff, tix = np.array(ioff, np.uint64), u32(tix)
    oo, op = np.array(oo, np.uint64), u32(op)
    b = bytes(blob)
    outside = lib().kd_emu_run(b, len(b), n, ioff.ctypes.data, isz.ctypes.data, w.ctypes.data, h.ctypes.data,
                               bps.ctypes.data, tix.ctypes.data, tables.ctypes.data, oo.ctypes.data, op.ctypes.data,
                               out.ctypes.data, res.ctypes.data, vals.ctypes.data, int(reverse), tab.ctypes.data,
                               ncand, rows.ctypes.data, rows.size, fail.ctypes.data, counts.ctypes.data)
    assert outside == 0, "loads outside the input"
    assert list(counts) == [ncand, rows.size]
    imgs, seen = [], np.zeros(pos, bool)
    for p, fh, pitch in layout:
        imgs.append(out[p:p + fh * pitch].reshape(fh, pitch))
        seen[p:p + fh * pitch] = True
    assert np.all(out[~seen] == FILL), "a store outside the frames' images"
    return imgs, [(int(res[2 * i]), int(res[2 * i + 1])) for i in range(n)], list(vals), (tab, rows, fail)


def check_tables(frames, tables):
    """Candidate entries bounded; on the true chain every row start leads to the next."""
    tab, rows, fail = tables
    c0 = r0 = 0
    for k, (data, w, h, *_) in enumerate(frames):
        st = stride(w)
        nc = len(data) // st + 1
        ft = tab[c0:c0 + nc]
        assert np.all((ft & FAIL) | (ft < nc)), k
        starts = []
        segs, end = T.segment_starts(data, w, h, starts)
        starts += [end] if end is not None else []
        nseg = (w + 255) // 256
        frow = len(segs) // nseg if end is None else h
        assert int(fail[2 * k]) == frow, k
        for r in range(min(frow + 1, h)):
            assert starts[r] % st == 0 and rows[r0 + r] * st == starts[r], (k, r)
            e = int(ft[rows[r0 + r]])
            if r < frow:
                assert e * st == starts[r + 1], (k, r, hex(e))
            else:
                assert e == FAIL | (len(segs) % nseg), (k, r, hex(e))
                assert int(fail[2 * k + 1]) == len(segs) % nseg
        c0 += nc
        r0 += h


def check(frames, reverse, skew=0):
    imgs, res, vals, tables = run_emu(frames, reverse, skew)
    for k, ((data, w, h, bps, mode, table), img, got, val) in enumerate(zip(frames, imgs, res, vals)):
        want, rc, r, c, v = K.decompress(data, w, h, bps, mode, table, fill=FILL)
        st = 0 if rc == K.OK else (2 if rc in K.IOE_MSGS else 1)
        assert got == (st, K.consumed(rc, r, c)), (k, got, rc, r, c)
        assert val == (v if rc == K.VALUE else 0), (k, val, v)
        assert np.array_equal(img, want), k
    check_tables(frames, tables)


def small_pinned():
    out = []
    for name, case in T.golden_cases():
        data, w, h, bps, cpp, curve, dither, uncorrected = case
        if T.run_case(*case)[1] < K.CPP and w * h <= 4 * 800:
            mode, table = T.case_table(curve, dither, uncorrected)
            out.append((data, w, h, bps, mode, table))
    return out


@pytest.mark.parametrize("reverse", [False, True])
def test_pinned_cases_one_plan(reverse):
    """The pinned cases that fit the replay, all in one plan (mixed outcomes)."""
    check(small_pinned(), reverse)


@pytest.mark.parametrize("reverse", [False, True])
def test_tall_frames_failing_past_checkpoints(reverse):
    """Frames of 100 rows (four checkpoints) failing at chosen rows, both kinds, skewed input."""
    frames = []
    for w in (8, 260, 264):
        v = K.natural(w, 100, 12, seed=w)
        data = K.encode(v)
        frames.append((data, w, 100, 12, K.NONE, None))
        segs, _ = T.segment_starts(data, w, 100)
        nseg = (w + 255) // 256
        for row in (31, 32, 33, 64, 99):
            frames.append((data[:max(segs[row * nseg][2] + 1, w * 50)], w, 100, 12, K.NONE, None))
            vv = v.copy()
            vv[row, w - 1] = 4096
            frames.append((K.encode(vv), w, 100, 12, K.NONE, None))
    check(frames, reverse, skew=5)


@pytest.mark.parametrize("reverse", [False, True])
def test_random_payloads(reverse):
    rng = np.random.default_rng(23)
    frames = []
    for k in range(24):
        w, h, bps = 4 * int(rng.integers(1, 100)), int(rng.integers(1, 12)), (10, 12)[k % 2]
        if k % 2:
            data = K.encode(K.random_values(w, h, bps, seed=k))
            data = data[:max(len(data) - int(rng.integers(0, 40)), w * h // 2)]
        else:
            data = rng.integers(0, 256, int(rng.integers(w * h // 2, 2 * w * h + 1)), dtype=np.uint8).tobytes()
        frames.append((data, w, h, bps, K.NONE, None))
    check(frames, reverse)
