"""k2_stream_kernel (rawspeed_b200/csrc/ljpeg_stream.cuh) without a GPU: the kernel body is compiled
by g++ against tests/emu/cuda_emu.h and run on the descriptors the plan builder produces, then
compared with the oracle -- pixels of the whole padded buffer, `consumed`, status.  The warp vote
that schedules the fill steps is replaced by its two extremes ("only when I am low myself" and
"always"): results must not depend on it.  A segment whose last symbols read behind the end of its
data is only flagged here (`redo`): the plan hands it to the tile kernel (exact, tested in
test_ljpeg_tile_emu.py); every case that is NOT flagged must match the oracle in status, `consumed`
and pixels.
Parity of the real kernel is the GPU tests' job (tests/test_gpu_ljpeg.py)."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import _abi
from oracle import port, synth
from helpers import dng_ljpeg_scans, compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "ljpeg_stream_emu.cpp")
OUT = os.path.join(HERE, "emu", "_build", "libljpeg_stream_emu.so")
CSRC = os.path.join(HERE, "..", "rawspeed_b200", "csrc")
DEPS = [SRC, os.path.join(HERE, "emu", "cuda_emu.h")] + [
    os.path.join(CSRC, f) for f in ("ljpeg_stream.cuh", "ljpeg_lane.cuh", "ljpeg_host.h", "ljpeg_types.h")]


@pytest.fixture(scope="module", params=["default", "st256", "lut32", "pipe0", "pipe2"])
def emu(request):
    """The instantiations of the kernel: 128-bit output stores, whole 32-byte sectors (two units stored back to back), and
    the 32-bit LUT entries of the straight-line decode, and the FMA-pipe forms of its field arithmetic."""
    out = OUT if request.param == "default" else OUT.replace(".so", "_%s.so" % request.param)
    flags = {"default": [], "st256": ["-DRSB200_EMU_WIDE=true"],
             "lut32": ["-DRSB200_EMU_WIDE=true", "-DRSB200_S_LUT32=1"],
             "pipe0": ["-DRSB200_EMU_WIDE=true", "-DRSB200_S_PIPE=0"],
             "pipe2": ["-DRSB200_EMU_WIDE=true", "-DRSB200_S_PIPE=2", "-DRSB200_S_FILL2=1"]}[request.param]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in DEPS):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        compile_shared(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas",
                               "-Wno-unused-function", "-fPIC", "-shared"] + flags + ["-o", out, SRC])
    lib = C.CDLL(out)
    lib.stream_emu_run.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                   C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.stream_emu_sector_stores.restype = C.c_ulonglong
    lib.wide = request.param != "default"
    return lib


def run_emu(lib, blob, tabs, scans, out, reverse=False, any_mode=0, in_base=0, out_base=0, may_redo=True):
    """One launch of the replay.  in_base / out_base: the input and output buffers start at this
    offset (0 or 16) from a 32-byte boundary; the replay copies them there itself.  may_redo=False: no
    segment may be handed to the tile kernel (the plan's segments that it cannot take)."""
    tarr = (_abi.HuffTable * len(tabs))(*tabs)
    sarr = (_abi.LJpegScan * len(scans))(*scans)
    res = (_abi.ScanResult * len(scans))()
    redo = np.zeros(len(scans), dtype=np.uint32)
    blob = np.ascontiguousarray(blob)
    assert out.flags.c_contiguous
    rc = lib.stream_emu_run(blob.ctypes.data, blob.size, in_base, tarr, len(tabs), sarr, len(scans),
                            out.ctypes.data, out.nbytes, out_base, res, redo.ctypes.data, int(reverse), any_mode,
                            int(may_redo))
    assert rc == 0, ("emu rc %d (-1 = a scan is not eligible for the thread kernels, "
                     "-4 = a read outside the readable input)" % rc)
    return [(r.status, r.consumed, int(f)) for r, f in zip(res, redo)]


def _sector_rows(scans, out_base):
    """Whether the WIDE form stores whole 32-byte sectors for some segment: its first output row
    and its pitch are 32-byte aligned, and a row holds at least two units."""
    for s in scans:
        row0 = out_base + s.out_offset + s.out_y * s.out_pitch + 2 * s.out_x
        if ((row0 | s.out_pitch) & 31) == 0 and s.store_w >= 16 and s.rows > 0:
            return True
    return False


def check_tiles(lib, img, tile_w, tile_h, **kw):
    h, w = img.shape
    cpp = kw.pop("cpp", 1)
    w //= cpp
    t = synth.make_dng_ljpeg(img, tile_w, tile_h, cpp=cpp, **kw)
    want = port.new_image(w, h, cpp)
    port.dng_decompress(t.blob, t.offsets, t.lengths, want, w, cpp, tile_w, tile_h, 7,
                        fix_ljpeg=kw.get("fix16", False), nthreads=4)
    tabs, scans = dng_ljpeg_scans(t, want.shape[1] * 2, fix16=kw.get("fix16", False))
    for out_base in (0, 16):
        for any_mode in (0, 1):
            got = port.new_image(w, h, cpp)
            res = run_emu(lib, t.blob, tabs.tabs, scans, got, reverse=bool(any_mode), any_mode=any_mode,
                          out_base=out_base)
            assert all(s == 0 and f == 0 for s, _, f in res), (out_base, any_mode, res[:4])
            bad = np.argwhere(got != want)
            assert bad.size == 0, (out_base, any_mode, bad[:5], got[tuple(bad[0])], want[tuple(bad[0])])
            # the WIDE form takes its sector branch exactly where rows and pitch are 32-byte aligned
            # (output base 0 with a pitch that is a multiple of 32 bytes; never at base 16 for these tiles), the
            # narrow form never
            sectors = lib.stream_emu_sector_stores()
            assert (sectors > 0) == (lib.wide and _sector_rows(scans, out_base)), (out_base, sectors)
            if lib.wide and want.strides[0] % 32 == 0:
                assert (sectors > 0) == (out_base == 0), (out_base, sectors)
    return t, tabs, scans


def test_single_tile(emu):
    img = synth.image_model(256, 64, 1)
    check_tiles(emu, img, 256, 64)


def test_tiles_ragged_edges(emu):
    img = synth.image_model(600, 200, 7)
    check_tiles(emu, img, 256, 64)


def test_wild_noise_long_codes(emu):
    img = synth.image_model(512, 96, 9, wild=True)
    check_tiles(emu, img, 256, 32)


def test_sixteen_bit_ssss16(emu):
    """More than two bytes per sample for a while: lanes run dry and fill on their own."""
    img = synth.image_model(256, 64, 11, wild=True, bits=16)
    img[0, 0:8] = [0, 0x8000, 0, 0x8000, 0xFFFF, 0x7FFF, 0, 0x8000]
    check_tiles(emu, img, 256, 64, prec=16)
    check_tiles(emu, img, 256, 64, prec=16, fix16=True)


def test_components_1_and_4(emu):
    img = synth.image_model(512, 48, 13)
    check_tiles(emu, img, 256, 24, ncomp=1)
    check_tiles(emu, img, 512, 48, ncomp=4)


def test_two_tables_long_code_of_one_is_a_short_code_of_the_other(emu):
    """The straight-line unit counts on "a miss repeats" (same window, same table).  With two tables a
    window that starts with a 12-bit code of the first can be a 3-bit code of the second: such segments
    must go symbol by symbol (found in round 2: the shipped kernel decoded garbage here)."""
    rng = np.random.default_rng(5)
    img = np.zeros((32, 256), np.uint16)
    img[:, 0::2] = rng.integers(0, 1 << 14, (32, 128))
    img[:, 1::2] = 8192 + rng.integers(0, 60, (32, 128))
    tabs = [synth.default_tables(1)[0], port.Huff(bytes([0, 0, 8] + [0] * 13), bytes(range(8)))]
    check_tiles(emu, img, 256, 32, tabs=tabs, tab_of_comp=[0, 1])
    check_tiles(emu, img, 256, 32, ncomp=4, tabs=tabs, tab_of_comp=[0, 1, 0, 1])


def test_restart_intervals(emu):
    img = synth.image_model(320, 96, 17)
    check_tiles(emu, img, 160, 48, restart_rows=1)
    check_tiles(emu, img, 160, 48, restart_rows=5)


def test_big_tile(emu):
    img = synth.image_model(512, 256, 23)
    check_tiles(emu, img, 512, 256)


def test_flat_image_two_bits_per_sample(emu):
    """Lanes with room but no need: the ring stays full, steps are skipped."""
    img = np.full((128, 1024), 2000, dtype=np.uint16)
    check_tiles(emu, img, 512, 128)
    img[::7, ::5] += 3
    check_tiles(emu, img, 512, 128)


def test_stuffing_everywhere(emu):
    """Streams full of FF bytes: every pattern of the selector table, FF at word and block ends."""
    rng = np.random.default_rng(5)
    img = np.zeros((64, 512), dtype=np.uint16)
    img[:, 0::2] = 0x3FFF
    img[:, 1::2] = 0
    img[::3, 2::4] = 0x3FFF
    check_tiles(emu, img, 256, 32)
    img = rng.integers(0, 1 << 14, size=(64, 512)).astype(np.uint16)
    check_tiles(emu, img, 256, 32)


def test_many_offsets_of_the_segment_start(emu):
    """The same tiles at every offset modulo 32 of the first byte (bytes before it in the sector),
    from an input base on a 32-byte boundary and from one 16 bytes behind it."""
    img = synth.image_model(256, 32, 31)
    t = synth.make_dng_ljpeg(img, 128, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    want = port.new_image(256, 32)
    port.dng_decompress(t.blob, t.offsets, t.lengths, want, 256, 1, 128, 32, 7, nthreads=1)
    for in_base, shift in itertools.product((0, 16), range(32)):
        blob = np.concatenate([np.full(shift, 0xFF, dtype=np.uint8), t.blob])
        sc = [rs.LJpegScan.from_buffer_copy(s) for s in scans]
        for s in sc:
            s.in_offset += shift
        got = port.new_image(256, 32)
        res = run_emu(emu, blob, tabs.tabs, sc, got, in_base=in_base)
        assert all(s == 0 and f == 0 for s, _, f in res), (in_base, shift, res)
        assert np.array_equal(got, want), (in_base, shift)


def test_consumed_matches_the_oracle(emu):
    img = synth.image_model(512, 64, 21)
    t, tabs, scans = check_tiles(emu, img, 256, 32)
    hts = synth.default_tables(1)
    got = port.new_image(512, 64)
    res = run_emu(emu, t.blob, tabs.tabs, scans, got)
    for (status, consumed, redo), s, off, ln in zip(res, scans, t.offsets, t.lengths):
        data = t.blob[s.in_offset:off + ln]
        o = port.new_image(512, 64)
        want = port.ljpeg_decompress(o, 512, 1, (s.out_x, s.out_y, s.store_w, s.rows),
                                     (2, 1), (s.frame_w, s.rows), [hts[0], hts[0]],
                                     [1 << 13] * 2, s.rows, data)
        assert (status, consumed, redo) == (0, want, 0)


def _one_scan_outcome(s, data, hts, w, h):
    """The oracle on one segment: (status, consumed, image)."""
    o = port.new_image(w, h)
    try:
        c = port.ljpeg_decompress(o, w, 1, (s.out_x, s.out_y, s.store_w, s.rows), (2, 1),
                                  (s.frame_w, s.rows), [hts[0], hts[0]], [1 << 13] * 2, s.rows, data)
        return 0, c, o
    except port.IOException:
        return 2, None, o
    except port.RawDecoderException:
        return 1, None, o


def _check_against(emu, blob, tabs, s, want, w, h, in_base=0):
    want_status, want_cons, want_img = want
    for any_mode in (0, 1):
        got = port.new_image(w, h)
        (status, consumed, redo), = run_emu(emu, blob, tabs.tabs, [s], got, any_mode=any_mode, in_base=in_base)
        if redo:
            assert status == 0   # handed to the tile kernel, which decides
            continue
        assert status == want_status
        if want_status == 0:
            assert consumed == want_cons
            assert np.array_equal(got, want_img)
    return redo


@pytest.mark.parametrize("cut", list(range(1, 34)) + [40, 64, 100])
def test_streams_that_end_early(emu, cut):
    """A segment truncated by `cut` bytes (the buffer ends; no marker).  Either the last symbol
    still lies inside the data (then everything matches the oracle) or the segment is flagged."""
    img = synth.image_model(256, 32, 53)
    t = synth.make_dng_ljpeg(img, 256, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    hts = synth.default_tables(1)
    s = rs.LJpegScan.from_buffer_copy(scans[0])
    s.in_size = scans[0].in_size - cut
    blob = t.blob[:s.in_offset + s.in_size].copy()
    want = _one_scan_outcome(s, blob[s.in_offset:], hts, 256, 32)
    _check_against(emu, blob, tabs, s, want, 256, 32)


@pytest.mark.parametrize("cut", [2, 3, 5, 8, 11, 16, 19, 24, 27, 32, 40])
def test_streams_with_an_early_marker(emu, cut):
    img = synth.image_model(256, 32, 57)
    t = synth.make_dng_ljpeg(img, 256, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    hts = synth.default_tables(1)
    s = rs.LJpegScan.from_buffer_copy(scans[0])
    blob = t.blob.copy()
    end = s.in_offset + s.in_size          # behind EOI
    pos = end - 2 - cut
    if blob[pos - 1] == 0xFF:              # do not turn a stuffing pair into something else
        pos -= 2
    blob[pos] = 0xFF
    blob[pos + 1] = 0xD9
    want = _one_scan_outcome(s, blob[s.in_offset:end], hts, 256, 32)
    _check_against(emu, blob[:end], tabs, s, want, 256, 32)


def test_marker_split_over_a_block_boundary(emu):
    """FF as the last byte of a 16-byte block, D9 as the first of the next one -- at every offset
    modulo 32, from both input bases."""
    img = synth.image_model(256, 32, 61)
    t = synth.make_dng_ljpeg(img, 256, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    hts = synth.default_tables(1)
    s0 = scans[0]
    end = s0.in_offset + s0.in_size
    for in_base, shift in itertools.product((0, 16), range(32)):
        blob = np.concatenate([np.zeros(shift, dtype=np.uint8), t.blob[:end]])
        s = rs.LJpegScan.from_buffer_copy(s0)
        s.in_offset += shift
        want = _one_scan_outcome(s, blob[s.in_offset:], hts, 256, 32)
        assert want[0] == 0
        redo = _check_against(emu, blob, tabs, s, want, 256, 32, in_base=in_base)
        assert redo == 0


def test_garbage_behind_the_last_symbol(emu):
    """Rows below the crop are not decoded: the stream goes on behind the last needed symbol."""
    img = synth.image_model(256, 64, 59)
    t = synth.make_dng_ljpeg(img, 256, 64)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    hts = synth.default_tables(1)
    s = rs.LJpegScan.from_buffer_copy(scans[0])
    s.rows = 40
    want = _one_scan_outcome(s, t.blob[s.in_offset:], hts, 256, 64)
    assert want[0] == 0
    assert _check_against(emu, t.blob, tabs, s, want, 256, 64) == 0


def test_bad_huffman_code(emu):
    img = synth.image_model(256, 32, 23, wild=True)
    t = synth.make_dng_ljpeg(img, 256, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    blob = t.blob.copy()
    s = scans[0]
    blob[s.in_offset + 40:s.in_offset + 49] = [0xFF, 0, 0xFF, 0, 0xFF, 0, 0xFF, 0, 0xFE]
    (status, _, redo), = run_emu(emu, blob, tabs.tabs, scans[:1], port.new_image(256, 32))
    assert (status, redo) == (1, 0)


def inject_bad_code(data, rng, pos):
    """An unassigned code of the default table at byte `pos` of entropy-coded data (in place): FF 00 FF 00 FE,
    23 one-bits where no code of that table starts with more than 15, then 2 .. 11 random bytes that are not
    FF, so that the decode behind the code goes on out of step.  The last two bytes (EOI) stay."""
    junk = rng.integers(0, 255, int(rng.integers(2, 12)))
    new = np.concatenate([[0xFF, 0, 0xFF, 0, 0xFE], junk]).astype(np.uint8)
    if data[pos - 1] == 0xFF:    # (not between an FF and its stuffing byte)
        pos += 1
    n = max(0, min(new.size, data.size - 2 - pos))
    data[pos:pos + n] = new[:n]


@pytest.mark.parametrize("seed", range(4))
def test_unassigned_code_then_a_run_past_the_end(emu, seed):
    """A segment the tile kernel cannot take (may_redo cleared) with an unassigned code inside its data:
    the kernel decodes on behind the code, out of step, and often runs past the end of the data.  The
    reference throws at the code (RawDecoderException), so the kernel must report status 1, not the
    IOException of a segment that merely ran out of data."""
    img = synth.image_model(256, 32, 53)
    t = synth.make_dng_ljpeg(img, 256, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    hts = synth.default_tables(1)
    rng = np.random.default_rng(900 + seed)
    n_rde = 0
    for trial in range(25):
        s = rs.LJpegScan.from_buffer_copy(scans[0])
        data = t.blob[s.in_offset:s.in_offset + s.in_size].copy()
        inject_bad_code(data, rng, int(rng.integers(8, data.size - 8)))
        s.in_offset = 0
        want_status, want_cons, want_img = _one_scan_outcome(s, data, hts, 256, 32)
        for any_mode in (0, 1):
            got = port.new_image(256, 32)
            (status, consumed, redo), = run_emu(emu, data, tabs.tabs, [s], got, any_mode=any_mode, may_redo=False)
            assert redo == 0
            if want_status == 2:
                assert status == 2, (trial, status)
            elif want_status == 1:
                assert status == 1, (trial, status)
            else:   # (no second opinion: an end of stream the kernel cannot settle stays an IOException)
                assert status in (0, 2), (trial, status)
                if status == 0:
                    assert consumed == want_cons and np.array_equal(got, want_img)
        n_rde += want_status == 1
    assert n_rde >= 20


def _random_table(rng, nvalues, maxlen=16):
    """A random COMPLETE canonical code over SSSS values 0 .. nvalues-1 (every leaf of a random binary
    tree with depths <= maxlen), values in random order: short complete tables, long tails, anything."""
    depths = [1, 1]
    while len(depths) < nvalues:
        cand = [i for i, d in enumerate(depths) if d < maxlen]
        i = int(rng.choice(cand))
        d = depths.pop(i)
        depths += [d + 1, d + 1]
    ncpl = [0] * 16
    for d in depths:
        ncpl[d - 1] += 1
    return port.Huff(bytes(ncpl), bytes(int(v) for v in rng.permutation(nvalues)))


@pytest.mark.parametrize("seed", range(24))
def test_random_tables_and_components(emu, seed):
    """Differential fuzz: 1 / 2 / 4 components, one to four random complete tables (codes up to 16 bits:
    most symbols of some tables miss the 11-bit LUT, others are resolved by every window), noise from a
    few bits to the full range; the compiled reference, the oracle and the replay agree bit for bit."""
    from oracle import ref
    rng = np.random.default_rng(7000 + seed)
    ncomp = int(rng.choice([1, 2, 4]))
    ntab = int(rng.integers(1, min(ncomp, 4) + 1))
    bits = int(rng.choice([3, 6, 10, 14]))
    h, tw = int(rng.choice([8, 16, 24])), int(rng.choice([64, 128, 256]))
    w = tw * int(rng.integers(1, 3))
    img = (8192 + rng.integers(0, 1 << bits, (h, w)) - (1 << bits) // 2).astype(np.uint16) & 0x3FFF
    tabs = [_random_table(rng, 16) for _ in range(ntab)]     # SSSS 0 .. 15: every 14-bit difference
    tab_of_comp = [int(rng.integers(0, ntab)) for _ in range(ncomp)]
    for t in range(ntab):                                     # (every table is used by some component)
        if t not in tab_of_comp:
            tab_of_comp[t % ncomp] = t
    t, tabset, scans = check_tiles(emu, img, tw, h, ncomp=ncomp, tabs=tabs, tab_of_comp=tab_of_comp)
    if ref.available():
        r = port.new_image(w, h)
        ref.dng_decompress(t.blob, t.offsets, t.lengths, r, w, 1, tw, h, 7)
        assert np.array_equal(r[:, :w], img)
