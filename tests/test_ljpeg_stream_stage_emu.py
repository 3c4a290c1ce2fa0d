"""The output stage of k2_stream_kernel's full-launch form (rawspeed_b200/csrc/ljpeg_stream.cuh) without a
GPU: the kernel body compiled by g++ against tests/emu/cuda_emu.h (tests/emu/ljpeg_stream_stage_emu.cpp).
The warp-wide flush is replayed with every lane alone and with the running lanes of a warp meeting;
pixels of the whole output buffer (and guard bytes around it) must match either way, and every staged
64-byte run must leave exactly once."""
import ctypes as C
import os

import numpy as np
import pytest

from rawspeed_b200 import _abi
from oracle import port, synth
from helpers import dng_ljpeg_scans, compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "ljpeg_stream_stage_emu.cpp")
OUT = os.path.join(HERE, "emu", "_build", "libljpeg_stream_stage_emu.so")
CSRC = os.path.join(HERE, "..", "rawspeed_b200", "csrc")
DEPS = [SRC, os.path.join(HERE, "emu", "cuda_emu.h")] + [
    os.path.join(CSRC, f) for f in ("ljpeg_stream.cuh", "ljpeg_lane.cuh", "ljpeg_host.h", "ljpeg_types.h")]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in DEPS):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        compile_shared(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
                        "-fPIC", "-shared", "-o", OUT, SRC])
    L = C.CDLL(OUT)
    L.stage_emu_run.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int]
    L.stage_emu_runs.restype = C.c_ulonglong
    L.stage_emu_smem_bytes.restype = C.c_ulonglong
    return L


def _decode(lib, t, tabs, scans, out, out_base, gather):
    tarr = (_abi.HuffTable * len(tabs.tabs))(*tabs.tabs)
    sarr = (_abi.LJpegScan * len(scans))(*scans)
    blob = np.ascontiguousarray(t.blob)
    rc = lib.stage_emu_run(blob.ctypes.data, blob.size, tarr, len(tabs.tabs), sarr, len(scans), out.ctypes.data,
                           out.nbytes, out_base, gather, gather)
    assert rc == 0, "emu rc %d (-4 read outside the input, -6 store outside the output, -7 status)" % rc
    return lib.stage_emu_runs(1), lib.stage_emu_runs(0)


def _check(lib, img, tile_w, tile_h, shift=0, **kw):
    """Every tile at its place moved right by `shift` samples, from both output bases, both ways of
    meeting at the flush.  Returns the runs stored by whole warps when the lanes meet."""
    h, w = img.shape
    ntab = kw.pop("ntab", None)
    t = synth.make_dng_ljpeg(img, tile_w, tile_h, **kw)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(w + 24))
    assert ntab is None or len(tabs.tabs) == ntab
    for s in scans:
        s.out_x += shift
    staged = lib.stage_emu_staged(len(tabs.tabs))
    runs = sum(s.rows * (s.store_w // 32) for s in scans) if staged else 0
    shared_when_gathered = None
    for out_base in (0, 16):
        for gather in (0, 1):
            got = port.new_image(w + 24, h)
            got[...] = 0x5A5A
            want = got.copy()
            want[:, shift:shift + w] = img
            shared, own = _decode(lib, t, tabs, scans, got, out_base, gather)
            bad = np.argwhere(got != want)
            assert bad.size == 0, (out_base, gather, bad[:5])
            assert shared + own == runs, (out_base, gather, shared, own, runs)
            if gather == 0:
                assert shared == 0
            else:
                shared_when_gathered = shared
    return shared_when_gathered, len(scans)


@pytest.mark.parametrize("shift", [0, 8, 16, 24])
def test_whole_warps_and_mixed_lanes(lib, shift):
    """147 tiles of 48 x 16 in two CTAs (the second a partial warp); the last tile of a row 40 samples
    wide and the tiles of the last row 4 rows high, so one warp holds lanes with different row counts
    and store_w tails (units behind the last whole run are stored directly); row starts at 0, 16, 32
    and 48 bytes modulo 64."""
    shared, n = _check(lib, synth.image_model(1000, 100, 41), 48, 16, shift)
    assert n == 147 and shared > 0


def test_two_tables_are_staged(lib):
    tabs = synth.default_tables(2)
    shared, _ = _check(lib, synth.image_model(512, 64, 43), 64, 16, 8, tabs=tabs, tab_of_comp=[0, 1])
    assert lib.stage_emu_staged(2) and shared > 0


def test_four_tables_store_directly(lib):
    """No room for the stage: pairs of units leave as whole sectors, or single units."""
    d, a = synth.default_tables(2)
    tabs = [d, a, port.Huff(d.ncpl, bytes(reversed(d.values))), port.Huff(a.ncpl, bytes(reversed(a.values)))]
    shared, _ = _check(lib, synth.image_model(512, 64, 47), 128, 16, 0, ncomp=4, tabs=tabs,
                       tab_of_comp=[0, 1, 2, 3], ntab=4)
    assert shared == 0


def test_stream_smem_fits_six_ctas(lib):
    """For every table count the plan gives the stream kernel (1 to 4), 6 CTAs fit an SM (228 KB, 1 KB of
    it reserved per CTA); the output stage (64 bytes per thread) is there with one or two tables."""
    for ntab in range(1, 5):
        assert 6 * (lib.stage_emu_smem_bytes(ntab) + 1024) <= 228 * 1024, ntab
        assert lib.stage_emu_staged(ntab) == (ntab <= 2), ntab
