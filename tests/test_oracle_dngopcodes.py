"""DngOpcodes (SURVEY 8(f)3): the oracle's restatement (parse + validate + apply) against the
compiled reference -- uint16 and float images, crops, every implemented opcode, list order of
mBadPixelPositions, and the error class / stage of malformed lists."""
import numpy as np
import pytest

from oracle import port, ref, synth as S

needs_ref = pytest.mark.skipif(not ref.checkable(), reason="oracle/_ref/libref.so not built")


def u16_image(w, h, cpp, seed, lo=0, hi=65536):
    rng = np.random.default_rng(seed)
    a = port.new_image(w, h, cpp)
    a[:, :] = rng.integers(lo, hi, size=a.shape, dtype=np.uint16)
    return a


def f32_image(w, h, cpp, seed):
    rng = np.random.default_rng(seed)
    a = port.new_image_f32(w, h, cpp)
    a[:, :] = rng.random(a.shape, dtype=np.float32).view(np.uint32)
    return a


def both(img, w, cpp, crop, blob):
    a, b = img.copy(), img.copy()
    ra = ref.dng_opcodes(a, w, cpp, crop, blob)
    rb = port.dng_opcodes(b, w, cpp, crop, blob)
    assert np.array_equal(a, b)
    assert ra == rb
    return ra, a


FULL = lambda w, h: (0, 0, h, w)   # noqa: E731  (top, left, bottom, right)


def scenarios():
    """(name, image, w, cpp, crop, opcode list) -- shared with the CPU replay of the kernel
    (tests/test_dngop_emu.py) and the GPU tests (tests/test_gpu_dngopcodes.py)."""
    out = []
    rng = np.random.default_rng(77)
    small = lambda n: (rng.random(n, dtype=np.float32) * 2 - 1) * 0.01     # noqa: E731
    w, h = 64, 20
    table = (np.arange(1000, dtype=np.uint32) * 37 % 65536).astype(np.uint16)
    out.append(("lookup", u16_image(w, h, 1, 1), w, 1, [0, 0, w, h], S.dng_opcode_list([
        S.dng_map_table(S.dng_pixel_area((2, 4, 18, 60), 0, 1, 2, 2), table),
        S.dng_map_polynomial(S.dng_pixel_area(FULL(w, h)), [0.01, 0.9, 0.2, -0.1]),
        S.dng_map_polynomial(S.dng_pixel_area((1, 1, 19, 63), 0, 1, 3, 5), [0.0] * 8 + [1.0])])))
    for cpp in (1, 3):
        w, h = 60, 24
        out.append(("delta_u16_cpp%d" % cpp, u16_image(w, h, cpp, 2), w, cpp, [3, 2, 50, 20], S.dng_opcode_list([
            S.dng_delta(10, S.dng_pixel_area((0, 0, 20, 50), 0, cpp, 1, 1), small(20)),
            S.dng_delta(11, S.dng_pixel_area((1, 2, 19, 47), cpp - 1, 1, 2, 3), small(15)),
            S.dng_delta(12, S.dng_pixel_area((2, 0, 20, 50), 0, 1, 4, 1), np.abs(small(5)) * 150),
            S.dng_delta(13, S.dng_pixel_area((0, 5, 20, 45), 0, cpp, 1, 7), np.abs(small(6)) * 90 + 0.5)])))
    for cpp in (1, 2):
        w, h = 36, 10
        out.append(("delta_f32_cpp%d" % cpp, f32_image(w, h, cpp, 3), w, cpp, [0, 0, w, h], S.dng_opcode_list([
            S.dng_delta(10, S.dng_pixel_area((1, 0, 9, 36), 0, cpp, 2, 1), rng.random(4, dtype=np.float32)),
            S.dng_delta(13, S.dng_pixel_area((0, 3, 10, 33), 0, 1, 1, 4), rng.random(8, dtype=np.float32) * 3),
            S.dng_delta(11, S.dng_pixel_area(FULL(36, 10), cpp - 1, 1, 1, 1), -rng.random(36, dtype=np.float32)),
            S.dng_delta(12, S.dng_pixel_area(FULL(36, 10), 0, cpp, 3, 2), rng.random(4, dtype=np.float32) + 1e30)])))
    w, h = 48, 16
    out.append(("bad_lists_trim", u16_image(w, h, 1, 4, 0, 8), w, 1, [0, 0, w, h], S.dng_opcode_list([
        S.dng_fix_bad_constant(3),
        S.dng_fix_bad_list(points=[(2, 5), (15, 47)], rects=[(1, 1, 3, 4), (0, 0, 0, 9)]),
        S.dng_trim_bounds(2, 4, 14, 40),
        S.dng_fix_bad_constant(5),
        S.dng_delta(10, S.dng_pixel_area((0, 0, 12, 36)), np.full(12, 0.001, np.float32)),
        S.dng_fix_bad_list(points=[(0, 0)]),
        S.dng_trim_bounds(1, 1, 11, 35)])))
    w, h = 300, 9
    out.append(("wide_mixed", u16_image(w, h, 1, 12), w, 1, [4, 1, 290, 7], S.dng_opcode_list([
        S.dng_delta(11, S.dng_pixel_area((0, 0, 7, 290), 0, 1, 1, 1), small(290)),
        S.dng_map_table(S.dng_pixel_area((1, 3, 6, 287), 0, 1, 1, 2), (65535 - np.arange(65536)).astype(np.uint16)),
        S.dng_fix_bad_constant(65535),
        S.dng_delta(12, S.dng_pixel_area((0, 1, 7, 289), 0, 1, 3, 16), np.array([0.5, 1.5, 31.9], np.float32))])))
    # setup() errors after opcodes that did run
    w, h = 32, 8
    area = S.dng_pixel_area(FULL(w, h))
    out.append(("error_after_prefix", u16_image(w, h, 1, 9), w, 1, [0, 0, w, h], S.dng_opcode_list([
        S.dng_delta(11, area, np.full(w, 0.25, np.float32)), S.dng_fix_bad_list(points=[(1, 1)]),
        S.dng_delta(12, area, np.full(8, -0.5, np.float32)), S.dng_delta(10, area, np.zeros(8, np.float32))])))
    out.append(("empty_trim_after_prefix", u16_image(w, h, 1, 9), w, 1, [0, 0, w, h], S.dng_opcode_list([
        S.dng_delta(11, area, np.full(w, 0.25, np.float32)), S.dng_trim_bounds(3, 3, 3, 9)])))
    return out


@needs_ref
def test_map_table_and_polynomial_u16():
    w, h = 64, 20
    img = u16_image(w, h, 1, 1)
    table = (np.arange(1000, dtype=np.uint32) * 37 % 65536).astype(np.uint16)
    blob = S.dng_opcode_list([
        S.dng_map_table(S.dng_pixel_area((2, 4, 18, 60), 0, 1, 2, 2), table),
        S.dng_map_polynomial(S.dng_pixel_area(FULL(w, h)), [0.01, 0.9, 0.2, -0.1]),
        S.dng_map_polynomial(S.dng_pixel_area((1, 1, 19, 63), 0, 1, 3, 5), [0.0] * 8 + [1.0]),
    ])
    both(img, w, 1, [0, 0, w, h], blob)


@needs_ref
@pytest.mark.parametrize("cpp", [1, 3])
def test_delta_and_scale_u16_planes_pitches_crop(cpp):
    w, h = 60, 24
    img = u16_image(w, h, cpp, 2)
    crop = [3, 2, 50, 20]      # ROI coordinates are relative to this crop
    rng = np.random.default_rng(5)
    rows = lambda n: (rng.random(n, dtype=np.float32) * 2 - 1) * 0.01     # noqa: E731
    blob = S.dng_opcode_list([
        S.dng_delta(10, S.dng_pixel_area((0, 0, 20, 50), 0, cpp, 1, 1), rows(20)),
        S.dng_delta(11, S.dng_pixel_area((1, 2, 19, 47), cpp - 1, 1, 2, 3), rows(15)),
        S.dng_delta(12, S.dng_pixel_area((2, 0, 20, 50), 0, 1, 4, 1), np.abs(rows(5)) * 150),
        S.dng_delta(13, S.dng_pixel_area((0, 5, 20, 45), 0, cpp, 1, 7), np.abs(rows(6)) * 90 + 0.5),
    ])
    both(img, w, cpp, crop, blob)


@needs_ref
@pytest.mark.parametrize("cpp", [1, 2])
def test_delta_and_scale_f32(cpp):
    w, h = 36, 10
    img = f32_image(w, h, cpp, 3)
    rng = np.random.default_rng(6)
    blob = S.dng_opcode_list([
        S.dng_delta(10, S.dng_pixel_area((1, 0, 9, 36), 0, cpp, 2, 1), rng.random(4, dtype=np.float32)),
        S.dng_delta(13, S.dng_pixel_area((0, 3, 10, 33), 0, 1, 1, 4), rng.random(8, dtype=np.float32) * 3),
        S.dng_delta(11, S.dng_pixel_area(FULL(36, 10), cpp - 1, 1, 1, 1), -rng.random(36, dtype=np.float32)),
        S.dng_delta(12, S.dng_pixel_area(FULL(36, 10), 0, cpp, 3, 2), rng.random(4, dtype=np.float32) + 1e30),
    ])
    both(img, w, cpp, [0, 0, w, h], blob)


@needs_ref
def test_bad_pixel_lists_trim_bounds_and_list_order():
    w, h = 48, 16
    img = u16_image(w, h, 1, 4, 0, 8)      # few distinct values: the constant 3 occurs often
    blob = S.dng_opcode_list([
        S.dng_fix_bad_constant(3),
        S.dng_fix_bad_list(points=[(2, 5), (15, 47)], rects=[(1, 1, 3, 4), (0, 0, 0, 9)]),
        S.dng_trim_bounds(2, 4, 14, 40),
        S.dng_fix_bad_constant(5),                         # scans the trimmed crop only
        S.dng_delta(10, S.dng_pixel_area((0, 0, 12, 36)), np.full(12, 0.001, np.float32)),
        S.dng_fix_bad_list(points=[(0, 0)]),               # inserted at the beginning again
        S.dng_trim_bounds(1, 1, 11, 35),
    ])
    (crop, bad), _ = both(img, w, 1, [0, 0, w, h], blob)
    assert crop == [5, 3, 34, 10]
    assert bad[0] == 0 and len(bad) > 20


@needs_ref
def test_optional_unsupported_opcodes_are_skipped():
    w, h = 16, 4
    img = u16_image(w, h, 1, 8)
    # (only with an empty payload: the reference insists that every opcode's bytes are consumed,
    # DngOpcodes.cpp:717-718, and never reads an unsupported opcode's)
    blob = S.dng_opcode_list([(9, b"", 1), (1, b"", 1),
                              S.dng_delta(11, S.dng_pixel_area(FULL(w, h)), np.zeros(16, np.float32) + 0.5)])
    both(img, w, 1, [0, 0, w, h], blob)
    _err_both(img, w, 1, [0, 0, w, h], S.dng_opcode_list([(9, b"\x00" * 40, 1)]))


def _err_both(img, w, cpp, crop, blob):
    """Same exception class, same stage (constructor vs apply), same image afterwards."""
    a, b = img.copy(), img.copy()
    errs = []
    for mod, im in ((ref, a), (port, b)):
        with pytest.raises(Exception) as ei:
            mod.dng_opcodes(im, w, cpp, crop, blob)
        errs.append(ei.value)
    assert type(errs[0]).__name__ == type(errs[1]).__name__, errs
    assert np.array_equal(a, b)
    assert (ref.dng_opcodes.stage == 1) == (port.dng_opcodes.partial[2] == 0 and np.array_equal(b, img)) or ref.dng_opcodes.stage == 2
    return type(errs[0]).__name__, ref.dng_opcodes.stage


@needs_ref
def test_malformed_lists_same_error_class_and_stage():
    w, h = 32, 8
    img = u16_image(w, h, 1, 9)
    area = S.dng_pixel_area(FULL(w, h))
    ok_delta = S.dng_delta(10, area, np.zeros(8, np.float32))
    cases = {
        "truncated": S.dng_opcode_list([ok_delta])[:-3],
        "count_too_big": np.concatenate([S.dng_opcode_list([ok_delta]), np.zeros(0, np.uint8)]).copy(),
        "unknown_code": S.dng_opcode_list([(99, b"")]),
        "unsupported_mandatory": S.dng_opcode_list([(9, b"\x00" * 8, 0)]),
        "roi_outside": S.dng_opcode_list([S.dng_delta(10, S.dng_pixel_area((0, 0, h + 1, w)), np.zeros(9, np.float32))]),
        "roi_inverted": S.dng_opcode_list([S.dng_trim_bounds(5, 5, 4, 10)]),
        "bad_planes": S.dng_opcode_list([S.dng_delta(10, S.dng_pixel_area(FULL(w, h), 1, 1), np.zeros(8, np.float32))]),
        "zero_pitch": S.dng_opcode_list([S.dng_delta(10, S.dng_pixel_area(FULL(w, h), 0, 1, 0, 1), np.zeros(8, np.float32))]),
        "pitch_too_big": S.dng_opcode_list([S.dng_delta(10, S.dng_pixel_area(FULL(w, h), 0, 1, 1, w + 1), np.zeros(8, np.float32))]),
        "wrong_count": S.dng_opcode_list([S.dng_delta(11, area, np.zeros(8, np.float32))]),
        "nan_delta": S.dng_opcode_list([S.dng_delta(10, area, np.array([np.nan] * 8, np.float32))]),
        "table_empty": S.dng_opcode_list([S.dng_map_table(area, np.zeros(0, np.uint16))]),
        "poly_degree_9": S.dng_opcode_list([S.dng_map_polynomial(area, [0.0] * 10)]),
        "trailing_bytes": S.dng_opcode_list([(6, S.dng_roi(0, 0, h, w) + b"\x00")]),
        "bad_point": S.dng_opcode_list([S.dng_fix_bad_list(points=[(h, 0)])]),
        "bad_rect": S.dng_opcode_list([S.dng_fix_bad_list(rects=[(0, 0, h + 1, 2)])]),
        "list_count_overflow": S.dng_opcode_list([(5, b"\x00\x00\x00\x00\xff\xff\xff\xff\x00\x00\x00\x00")]),
        # setup()/apply() errors: earlier opcodes stay applied
        "offset_too_large": S.dng_opcode_list([ok_delta, S.dng_delta(10, area, np.full(8, 1.5, np.float32))]),
        "scale_negative": S.dng_opcode_list([S.dng_delta(11, area, np.full(w, 0.25, np.float32)),
                                             S.dng_delta(12, area, np.full(8, -0.5, np.float32))]),
        "scale_too_large": S.dng_opcode_list([S.dng_delta(13, area, np.full(w, 40000.0, np.float32))]),
        "empty_trim": S.dng_opcode_list([S.dng_delta(11, area, np.full(w, 0.25, np.float32)),
                                         S.dng_trim_bounds(3, 3, 3, 9)]),
    }
    cases["count_too_big"][3] = 2     # says two opcodes, holds one
    seen = {}
    for name, blob in cases.items():
        seen[name] = _err_both(img, w, 1, [0, 0, w, h], blob)
    assert seen["truncated"][0] == "IOException" and seen["unknown_code"] == ("RawDecoderException", 1)
    assert seen["offset_too_large"][1] == 2 and seen["empty_trim"][1] == 2


@needs_ref
def test_setup_errors_on_wrong_image_type():
    w, h = 16, 4
    f = f32_image(w, h, 1, 1)
    area = S.dng_pixel_area(FULL(w, h))
    for blob in (S.dng_opcode_list([S.dng_map_table(area, np.arange(16, dtype=np.uint16))]),
                 S.dng_opcode_list([S.dng_fix_bad_constant(0)])):
        assert _err_both(f, w, 1, [0, 0, w, h], blob) == ("RawDecoderException", 2)
    u3 = u16_image(w, h, 3, 2)
    assert _err_both(u3, w, 3, [0, 0, w, h], S.dng_opcode_list([S.dng_fix_bad_constant(0)])) == \
        ("RawDecoderException", 2)


@needs_ref
@pytest.mark.parametrize("k", range(9))
def test_shared_scenarios_match_reference(k):
    name, img, w, cpp, crop, blob = scenarios()[k]
    if "error" in name or "empty_trim" in name:
        assert _err_both(img, w, cpp, crop, blob)[1] == 2
        assert ref.dng_opcodes.partial == port.dng_opcodes.partial[:2]
    else:
        both(img, w, cpp, crop, blob)
