"""Seeded differential fuzz of the kernels developed against CPU replays (K9 scaling, K10 DNG
opcodes, K11 bad pixels, Panasonic V4): random geometries and parameters, three ways --
compiled reference (where built), oracle, CPU replay of the kernel's thread program -- all
bit-exact.  Sized to run in a few seconds."""
import ctypes as C

import numpy as np
import pytest

from oracle import port, ref, synth as S
from rawspeed_b200._abi import BadPixJob, ScaleJob
from test_scale_emu import emu as scale_emu, job as scale_job, run as scale_run   # noqa: F401
from test_dngop_emu import emu as dngop_emu, replay as dngop_replay               # noqa: F401
from test_badpix_emu import emu as badpix_emu, job as badpix_job                  # noqa: F401
from test_pana4_emu import emu as pana4_emu, v4_payload                           # noqa: F401
from test_lookup_emu import emu as lookup_emu, job as lookup_job                  # noqa: F401
from rawspeed_b200._abi import LookupJob

HAVE_REF = ref.checkable()   # the compiled reference, or its recorded results


def rnd_image(rng, w, h, cpp=1, hi=65536):
    a = port.new_image(w, h, cpp)
    a[:, :] = rng.integers(0, hi, size=a.shape, dtype=np.uint16)
    return a


@pytest.mark.parametrize("seed", range(40))
def test_scale_fuzz(scale_emu, seed):
    rng = np.random.default_rng(1000 + seed)
    w, h = int(rng.integers(9, 400)), int(rng.integers(1, 24))
    cw, ch = int(rng.integers(1, w + 1)), int(rng.integers(1, h + 1))
    crop = (int(rng.integers(0, w - cw + 1)), int(rng.integers(0, h - ch + 1)), cw, ch)
    bits = int(rng.choice([10, 12, 14, 16]))
    white = int(rng.integers((1 << bits) // 2, 1 << bits))
    black = [int(v) for v in rng.integers(0, white // 4 + 1, 4)]
    dither = bool(rng.integers(0, 2))
    a = rnd_image(rng, w, h, 1, 1 << bits)
    want = a.copy()
    port.scale_values(want, w, crop, black, white, dither=dither)
    if HAVE_REF:
        r = a.copy()
        ref.scale_values(r, w, crop, black, white, dither=dither)
        assert np.array_equal(r, want)
    assert scale_run(scale_emu, a, [scale_job(0, a, w, h, 1, crop, black, white, dither)]) == 1
    assert np.array_equal(a, want)


def _random_opcode_list(rng, w, h, cpp, is_f32):
    """A valid random list over the crop (w, h) (ROIs relative to it)."""
    ops = []
    cw, ch = w, h
    for _ in range(int(rng.integers(1, 7))):
        top, left = int(rng.integers(0, ch)), int(rng.integers(0, cw))
        bottom, right = int(rng.integers(top + 1, ch + 1)), int(rng.integers(left + 1, cw + 1))
        first = int(rng.integers(0, cpp))
        planes = int(rng.integers(1, cpp - first + 1))
        rp, cp = int(rng.integers(1, bottom - top + 1)), int(rng.integers(1, right - left + 1))
        rp, cp = min(rp, 5), min(cp, 9)
        area = S.dng_pixel_area((top, left, bottom, right), first, planes, rp, cp)
        nrow, ncol = -(-(bottom - top) // rp), -(-(right - left) // cp)
        kind = int(rng.choice([7, 8, 10, 11, 12, 13] if not is_f32 else [10, 11, 12, 13]))
        if kind == 7:
            n = int(rng.integers(1, 65537))
            ops.append(S.dng_map_table(area, rng.integers(0, 65536, n).astype(np.uint16)))
        elif kind == 8:
            ops.append(S.dng_map_polynomial(area, (rng.random(int(rng.integers(1, 6))) - 0.3).tolist()))
        elif kind in (10, 11):
            n = nrow if kind == 10 else ncol
            vals = (rng.random(n, dtype=np.float32) * 2 - 1) * (0.02 if not is_f32 else 5.0)
            ops.append(S.dng_delta(kind, area, vals))
        else:
            n = nrow if kind == 12 else ncol
            ops.append(S.dng_delta(kind, area, rng.random(n, dtype=np.float32) * 3))
        if not is_f32 and cpp == 1 and rng.integers(0, 4) == 0:
            ops.append(S.dng_fix_bad_constant(int(rng.integers(0, 4))))
        if rng.integers(0, 5) == 0:
            ops.append(S.dng_fix_bad_list(points=[(int(rng.integers(0, h)), int(rng.integers(0, w)))]))
        if rng.integers(0, 5) == 0 and cw > 4 and ch > 4:
            t, l = int(rng.integers(0, 2)), int(rng.integers(0, 2))
            b, r = ch - int(rng.integers(0, 2)), cw - int(rng.integers(0, 2))
            ops.append(S.dng_trim_bounds(t, l, b, r))
            cw, ch = r - l, b - t
    return S.dng_opcode_list(ops)


@pytest.mark.parametrize("seed", range(40))
def test_dng_opcodes_fuzz(dngop_emu, seed):
    rng = np.random.default_rng(2000 + seed)
    is_f32 = seed % 4 == 3
    cpp = int(rng.integers(1, 4))
    w, h = int(rng.integers(6, 90)), int(rng.integers(3, 20))
    if is_f32:
        a = port.new_image_f32(w, h, cpp)
        a[:, :] = (rng.random(a.shape, dtype=np.float32) * 100).view(np.uint32)
    else:
        a = rnd_image(rng, w, h, cpp, 4 if seed % 3 == 0 else 65536)
    # the list is built for the uncropped image; FixBadPixelsList points use uncropped coordinates too
    blob = _random_opcode_list(rng, w, h, cpp, is_f32)
    crop = [0, 0, w, h]
    want = a.copy()
    wcrop, wbad = port.dng_opcodes(want, w, cpp, crop, blob)
    if HAVE_REF:
        r = a.copy()
        rcrop, rbad = ref.dng_opcodes(r, w, cpp, crop, blob)
        assert np.array_equal(r, want) and rcrop == wcrop and rbad == wbad
    gcrop, gbad, gerr = dngop_replay(dngop_emu, a, w, cpp, crop, blob)
    assert gerr is None
    assert np.array_equal(a, want)
    assert gcrop == wcrop and gbad == wbad


@pytest.mark.parametrize("seed", range(40))
def test_bad_pixels_fuzz(badpix_emu, seed):
    rng = np.random.default_rng(3000 + seed)
    w, h = int(rng.integers(17, 200)), int(rng.integers(1, 30))
    cfa = bool(rng.integers(0, 2))
    n = int(rng.integers(1, max(2, w * h // int(rng.choice([2, 8, 40])))))
    p = ((rng.integers(0, h, n).astype(np.uint32) << 16) | rng.integers(0, w, n).astype(np.uint32))
    a = rnd_image(rng, w, h)
    want = a.copy()
    port.fix_bad_pixels(want, w, 1, p, cfa)
    if HAVE_REF:
        r = a.copy()
        ref.fix_bad_pixels(r, w, 1, p, cfa, nthreads=2)
        assert np.array_equal(r, want)
    err = C.create_string_buffer(256)
    assert badpix_emu.badpix_emu_run(a.ctypes.data, (BadPixJob * 1)(badpix_job(0, a, w, cfa, 0, n)), 1,
                                     p.ctypes.data, n, seed & 1, err, 256) >= 0, err.value
    assert np.array_equal(a, want)


@pytest.mark.parametrize("seed", range(20))
def test_panasonic_v4_fuzz(pana4_emu, seed):
    rng = np.random.default_rng(4000 + seed)
    w, h = 14 * int(rng.integers(1, 120)), int(rng.integers(1, 40))
    split = int(rng.choice([0, 0x2008, 0x1FF8, 0x4000, int(rng.integers(1, 0x4000))]))
    zero_ok = bool(rng.integers(0, 2))
    data = v4_payload(w, h, split, 4000 + seed, zero_every=int(rng.choice([0, 3, 7, 50])))
    want = port.new_image(w, h)
    zwant = port.panasonic_v4(want, w, data, zero_ok, split, cap=1 << 20)
    if HAVE_REF:
        r = port.new_image(w, h)
        zr = ref.panasonic_v4(r, w, data, zero_ok, split, nthreads=2)
        assert np.array_equal(r, want) and zr == zwant
    got = port.new_image(w, h)
    zl = np.zeros(1 << 20, dtype=np.uint32)
    nz = C.c_uint32(0)
    buf = np.concatenate([data, np.zeros(16, np.uint8)])
    pana4_emu.pana4_emu_run(buf.ctypes.data, 0, got.ctypes.data, 0, got.shape[1] * 2, w, h, split,
                            int(zero_ok), zl.ctypes.data, zl.size, C.byref(nz))
    assert np.array_equal(got, want)
    assert sorted(zl[:nz.value].tolist()) == zwant


@pytest.mark.parametrize("seed", range(30))
def test_lookup_fuzz(lookup_emu, seed):
    rng = np.random.default_rng(5000 + seed)
    cpp = int(rng.integers(1, 4))
    w, h = int(rng.integers(1, 700)), int(rng.integers(1, 14))
    dither = bool(seed & 1)
    cv = np.sort(rng.integers(0, 65536, int(rng.integers(1, 5000)))).astype(np.uint16)
    a = rnd_image(rng, w, h, cpp)
    want = a.copy()
    t = port.build_table(cv, dither)
    port.sixteen_bit_lookup(want, w, cpp, t, dither)
    if HAVE_REF:
        r = a.copy()
        ref.sixteen_bit_lookup(r, w, cpp, [0, 0, w, h], cv, dither, nthreads=2)
        assert np.array_equal(r, want)
    err = C.create_string_buffer(256)
    assert lookup_emu.lookup_emu_run(a.ctypes.data, (LookupJob * 1)(lookup_job(0, a, w, cpp)), 1,
                                     t.ctypes.data, 1, int(dither), err, 256) == 0, err.value
    assert np.array_equal(a, want)


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref/libref.so not built")
@pytest.mark.parametrize("seed", range(250))
def test_mutated_opcode_lists_fail_alike(seed):
    """Byte-level mutations of valid opcode lists (what fuzz/librawspeed/common/DngOpcodes.cpp
    feeds the reference): the compiled reference, the oracle and the host mirror's parser agree
    on success / exception class / stage, and reference and oracle on the image and the lists."""
    from rawspeed_b200 import host
    rng = np.random.default_rng(6000 + seed)
    cpp = int(rng.integers(1, 3))
    w, h = int(rng.integers(8, 40)), int(rng.integers(4, 12))
    a = rnd_image(rng, w, h, cpp, 64)
    blob = _random_opcode_list(rng, w, h, cpp, False).copy()
    for _ in range(int(rng.integers(1, 4))):
        kind = int(rng.integers(0, 4))
        i = int(rng.integers(0, blob.size))
        if kind == 0:
            blob[i] = rng.integers(0, 256)
        elif kind == 1:
            blob[i] ^= 1 << int(rng.integers(0, 8))
        elif kind == 2 and blob.size > 8:
            blob = blob[:int(rng.integers(4, blob.size))].copy()
        else:
            blob = np.concatenate([blob, rng.integers(0, 256, int(rng.integers(1, 6))).astype(np.uint8)])
    crop = [0, 0, w, h]
    res = {}
    for name, mod in (("ref", ref), ("port", port)):
        im = a.copy()
        try:
            out = mod.dng_opcodes(im, w, cpp, crop, blob)
            res[name] = ("ok", out, im)
        except Exception as ex:   # noqa: BLE001
            res[name] = (type(ex).__name__, tuple(mod.dng_opcodes.partial[:2]), im)
    assert res["ref"][0] == res["port"][0], (res["ref"][0], res["port"][0])
    assert tuple(res["ref"][1]) == tuple(res["port"][1])
    assert np.array_equal(res["ref"][2], res["port"][2])
    # the mirror: constructor errors raise from dngop_lower; setup()/apply() errors come back in "error"
    stage = ref.dng_opcodes.stage
    try:
        low = host.dngop_lower(a, w, cpp, crop, blob)
        got = "ok" if low["error"] is None else type(low["error"]).__name__
        assert stage != 1, "the reference's constructor threw, the mirror's did not"
    except Exception as ex:   # noqa: BLE001
        got = type(ex).__name__
        assert stage == 1, "the mirror's constructor threw (%s), the reference's did not" % ex
    assert got == res["ref"][0]
