"""The plan's order of the thread path (thread_shape_order, rawspeed_b200/csrc/ljpeg_host.h) without a GPU:
the order itself, and what it does to k2_stream_kernel's output stage in the CPU replay
(tests/emu/ljpeg_stream_order_emu.cpp), whose lanes go through rows and units in step as the GPU's do:
a run is stored by the whole warp only where all 32 lanes flush at the same row and unit."""
import ctypes as C
import os

import numpy as np
import pytest

from rawspeed_b200 import _abi
from oracle import port, synth
from helpers import dng_ljpeg_scans, compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "ljpeg_stream_order_emu.cpp")
OUT = os.path.join(HERE, "emu", "_build", "libljpeg_stream_order_emu.so")
CSRC = os.path.join(HERE, "..", "rawspeed_b200", "csrc")
DEPS = [SRC, os.path.join(HERE, "emu", "cuda_emu.h")] + [
    os.path.join(CSRC, f) for f in ("ljpeg_stream.cuh", "ljpeg_lane.cuh", "ljpeg_host.h", "ljpeg_types.h")]


@pytest.fixture(scope="module")
def olib():
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in DEPS):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        compile_shared(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                        "-fPIC", "-shared", "-o", OUT, SRC])
    L = C.CDLL(OUT)
    L.order_emu_run.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int]
    L.order_emu_shape_order.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.order_emu_runs.restype = C.c_ulonglong
    return L


def _order(olib, scans, ntab):
    sarr = (_abi.LJpegScan * len(scans))(*scans)
    perm = np.zeros(len(scans), np.uint32)
    assert olib.order_emu_shape_order(sarr, len(scans), ntab, perm.ctypes.data) == 0
    return perm


def _shape(s):
    return (s.mcu_w * s.mcu_h, s.frame_w * s.mcu_w * s.mcu_h, s.rows, s.store_w)


def _model_whole_runs(scans, order):
    """Runs stored by whole warps when the lanes of a warp (32 consecutive threads) go in step: a warp whose
    32 lanes run one kernel body (one G) flushes together at each row and staged group all of them have."""
    whole = 0
    for w in range(0, len(order) - 31, 32):
        lanes = [scans[i] for i in order[w:w + 32]]
        if len({s.mcu_w * s.mcu_h for s in lanes}) == 1:
            whole += 32 * min(s.rows for s in lanes) * min(s.store_w // 32 for s in lanes)
    return whole


def test_order_is_a_stable_grouping_by_shape(olib):
    """A permutation; each shape class contiguous; classes by descending samples, then stored width;
    inside a class, scan order."""
    rng = np.random.default_rng(5)
    t = synth.make_dng_ljpeg(synth.image_model(256, 16, 3), 128, 16)
    _, (tpl, _) = dng_ljpeg_scans(t, port.image_pitch(256))
    scans = []
    for _ in range(700):
        s = _abi.LJpegScan.from_buffer_copy(tpl)
        s.mcu_w = int(rng.choice([1, 2, 4]))
        s.frame_w = int(rng.choice([16, 32, 64])) // s.mcu_w * 4
        s.rows = int(rng.choice([4, 8, 16]))
        s.store_w = int(rng.choice([s.frame_w * s.mcu_w, 40, 64]))
        s.out_pitch = 4096
        s.table[:] = [0, 0, 0, 0]
        scans.append(s)
    perm = [int(p) for p in _order(olib, scans, 1)]
    assert sorted(perm) == list(range(len(scans)))
    keys = [_shape(scans[i]) for i in perm]
    seen, runs = set(), []
    for k, key in enumerate(keys):
        if k == 0 or key != keys[k - 1]:
            assert key not in seen, key
            seen.add(key)
            runs.append(key)
    assert len(runs) > 20
    work = [(-(r[1] * r[2]), -r[3]) for r in runs]
    assert work == sorted(work)
    for key in runs:
        members = [i for i in perm if _shape(scans[i]) == key]
        assert members == sorted(members)


def test_headline_lane_structure(olib):
    """The headline's tiles in miniature: 256 x 8 tiles over 8256 x 172, so 33 x 22 tiles, the last column 64
    wide (two staged groups of eight) and the last row 4 high, as in the 8256 x 5504 frames of 256 x 256
    tiles.  In scan order nearly every warp holds a right-edge tile, whose lane leaves the other lanes from
    the third group of a row on: about a quarter of the runs are stored by whole warps.  In the plan's
    order every warp but the one at a class boundary and the last, partial one is.  The whole output buffer
    (and its guard bytes) equals the oracle's either way, from both output bases, both ways of flushing."""
    w, h = 8256, 172
    img = synth.image_model(w, h, 17)
    t = synth.make_dng_ljpeg(img, 256, 8)
    pitch = port.image_pitch(w)
    tabs, scans = dng_ljpeg_scans(t, pitch)
    assert len(scans) == 33 * 22 and len(tabs.tabs) == 1 and olib.order_emu_staged(1)
    assert {s.store_w for s in scans} == {256, 64} and {s.rows for s in scans} == {8, 4}
    want = port.new_image(w, h)
    want[...] = 0x5A5A
    port.dng_decompress(t.blob, t.offsets, t.lengths, want, w, 1, 256, 8, 7)
    runs = sum(s.rows * (s.store_w // 32) for s in scans)
    perm = [int(p) for p in _order(olib, scans, 1)]
    tarr = (_abi.HuffTable * len(tabs.tabs))(*tabs.tabs)
    sarr = (_abi.LJpegScan * len(scans))(*scans)
    blob = np.ascontiguousarray(t.blob)
    shared_of = {}
    for shape_order in (0, 1):
        for out_base in (0, 16):
            for gather in (0, 1):
                got = port.new_image(w, h)
                got[...] = 0x5A5A
                rc = olib.order_emu_run(blob.ctypes.data, blob.size, tarr, 1, sarr, len(scans), got.ctypes.data,
                                        got.nbytes, out_base, gather, gather, shape_order)
                assert rc == 0, rc
                bad = np.argwhere(got != want)
                assert bad.size == 0, (shape_order, out_base, gather, bad[:5])
                shared, own = olib.order_emu_runs(1), olib.order_emu_runs(0)
                assert shared + own == runs
                if gather:
                    shared_of.setdefault(shape_order, set()).add(shared)
                else:
                    assert shared == 0
    scan = shared_of[0].pop()
    shaped = shared_of[1].pop()
    assert not shared_of[0] and not shared_of[1]      # the same from both output bases
    assert scan == _model_whole_runs(scans, list(range(len(scans))))
    assert shaped == _model_whole_runs(scans, perm)
    assert 0.2 < scan / runs < 0.35, scan / runs
    # plan's order: 21 warps of interior tiles, one of the 21 right-edge tiles and 11 bottom tiles (whole
    # at the rows and groups all of them have), then the last 22 tiles
    interior = 32 * 21 * 8 * 8
    assert shaped == interior + 32 * 4 * 2, (shaped, runs)
    assert shaped / runs > 0.97
