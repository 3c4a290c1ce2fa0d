"""RawImageDataU16::scaleValues (SURVEY 8(f)3 groundwork): the oracle's restatement of
both the SSE2 and the plain path against the compiled reference's scaleBlackWhite()."""
import numpy as np
import pytest

from oracle import port, ref

needs_ref = pytest.mark.skipif(not ref.checkable(), reason="oracle/_ref/libref.so not built")


def _image(w, h, seed, lo=0, hi=65536):
    rng = np.random.default_rng(seed)
    img = port.new_image(w, h)
    img[:, :] = rng.integers(lo, hi, size=img.shape, dtype=np.uint16)
    return img


CASES = [
    # w, h, crop, black_sep, white
    (64, 16, (0, 0, 64, 16), (256, 256, 256, 256), 16383),          # 14 bit, app_scale ~ 4
    (70, 11, (3, 1, 61, 9), (60, 64, 68, 72), 4095),                # odd crop offsets, 12 bit
    (37, 9, (2, 3, 30, 5), (1000, 1010, 990, 1024), 15000),         # width not a multiple of 8
    (48, 8, (1, 0, 40, 8), (0, 0, 0, 0), 65535),                    # identity scale
    (40, 6, (0, 1, 40, 4), (2048, 2000, 2100, 2047), 3000),         # app_scale ~ 68 -> plain path
    (33, 7, (5, 2, 20, 4), (100, 200, 300, 400), 1023),             # 10 bit -> plain path
    (24, 4, (0, 0, 24, 4), (5000, 100, 100, 100), 6200),            # app_scale ~ 54, big multipliers elsewhere
]


@needs_ref
@pytest.mark.parametrize("dither", [True, False])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_scale_values_matches_reference(case, dither):
    w, h, crop, black, white = CASES[case]
    a = _image(w, h, 100 + case)
    b = a.copy()
    ref.scale_values(a, w, crop, black, white, dither=dither)
    port.scale_values(b, w, crop, black, white, dither=dither)
    assert np.array_equal(a, b)


@needs_ref
def test_scale_values_rows_are_independent_of_threading():
    w, h, crop, black, white = 96, 40, (2, 2, 90, 36), (64, 65, 66, 67), 16000
    a = _image(w, h, 7)
    b = a.copy()
    c = a.copy()
    ref.scale_values(a, w, crop, black, white, nthreads=1)
    ref.scale_values(b, w, crop, black, white, nthreads=4)
    port.scale_values(c, w, crop, black, white)
    assert np.array_equal(a, b) and np.array_equal(a, c)


def test_path_choice():
    assert port.scale_uses_sse2((256,) * 4, 16383)
    assert not port.scale_uses_sse2((0,) * 4, 1023)


def test_sse2_path_touches_whole_rows_plain_path_only_the_crop():
    # scaleValues_SSE2 walks x over roundDown(uncropped width, 8); scaleValues_plain over dim.x
    w, h, crop = 32, 6, (8, 1, 16, 4)
    black = (100, 100, 100, 100)
    for white, sse2 in ((16383, True), (1000, False)):
        a = _image(w, h, 3, 100, 1000)
        b = a.copy()
        port.scale_values(b, w, crop, black, white, dither=False)
        changed = a != b
        assert not changed[0].any() and not changed[5].any()
        assert changed[1:5, 8:24].any()
        assert changed[1:5, :8].any() == sse2


def test_plain_path_without_dither_is_the_rounded_affine_map():
    w, h = 16, 4
    a = _image(w, h, 9, 0, 1024)
    b = a.copy()
    port.scale_values(b, w, (0, 0, w, h), (64, 64, 64, 64), 1023, dither=False, sse2=False)
    mul = int(np.float32(16384.0) * np.float32(65535.0) / np.float32(1023 - 64))
    want = np.clip(((a[:, :w].astype(np.int64) - 64) * mul + 8192) >> 14, 0, 65535)
    assert np.array_equal(b[:, :w], want.astype(np.uint16))


# ---- scaleBlackWhite + calculateBlackAreas ------------------------------------------------

def _sensor(w, h, seed, black=512, white=15000, masked_cols=16, masked_rows=8):
    """A sensor-like frame: masked left columns / top rows near `black`, the rest a ramp."""
    rng = np.random.default_rng(seed)
    img = port.new_image(w, h)
    img[:, :] = rng.integers(black, white, size=img.shape, dtype=np.uint16)
    # the optically black strips: black + a little per-position noise
    img[:, :masked_cols] = (black + rng.integers(-6, 7, size=(h, masked_cols))).astype(np.uint16)
    img[:masked_rows, :] = (black + 3 + rng.integers(-6, 7, size=(masked_rows, img.shape[1]))).astype(np.uint16)
    return img


SBW = [
    # name, w, h, crop, kwargs
    ("vertical_area", 96, 40, (16, 8, 80, 32), dict(white=15000, areas=[(1, 0, 16)])),
    ("horizontal_area", 96, 40, (16, 8, 80, 32), dict(white=15000, areas=[(0, 0, 8)])),
    ("both_odd_sizes", 97, 41, (17, 9, 80, 32), dict(white=15000, areas=[(1, 1, 15), (0, 1, 7)])),
    ("not_cfa_average", 96, 40, (16, 8, 80, 32), dict(white=15000, areas=[(1, 0, 16)], is_cfa=False)),
    ("black_level_only", 64, 24, (0, 0, 64, 24), dict(black_level=500, white=15000)),
    ("separate_given", 64, 24, (2, 2, 60, 20), dict(black_sep=[500, 510, 505, 515], white=15000)),
    ("nothing_to_do", 64, 24, (0, 0, 64, 24), dict(black_level=0, white=65535)),
    ("empty_areas_zero_pixels", 64, 24, (0, 0, 64, 24), dict(black_level=300, white=12000, areas=[(1, 0, 1)])),
    ("estimate_both", 640, 560, (4, 4, 620, 540), dict()),
    ("estimate_white", 640, 560, (4, 4, 620, 540), dict(black_level=600)),
    ("estimate_black", 640, 560, (4, 4, 620, 540), dict(white=14000)),
]


@needs_ref
@pytest.mark.parametrize("case", SBW, ids=[c[0] for c in SBW])
def test_scale_black_white_matches_reference(case):
    name, w, h, crop, kw = case
    a = _sensor(w, h, sum(map(ord, name)))
    b = a.copy()
    ra = ref.scale_black_white(a, w, crop, **kw)
    rb = port.scale_black_white(b, w, crop, **kw)
    assert np.array_equal(a, b)
    assert ra == rb
    if name == "nothing_to_do":
        assert ra[0] is None


@needs_ref
def test_black_area_beyond_image_same_error():
    a = _sensor(64, 24, 5)
    for areas, msg in (([(0, 20, 8)], "height"), ([(1, 60, 8)], "width")):
        errs = []
        for mod in (ref, port):
            with pytest.raises(Exception) as ei:
                mod.scale_black_white(a.copy(), 64, (0, 0, 64, 24), white=15000, areas=areas)
            errs.append(ei.value)
        assert all(msg in str(x) for x in errs)


def test_histogram_counters_are_16_bit():
    # calculateBlackAreas counts in uint16_t: 65536 equal samples of one bin wrap to zero
    # and the median walks past it (RawImageDataU16.cpp:63-64)
    w, h = 1024 + 8, 520
    img = port.new_image(w, h)
    img[:, :] = 2000
    img[:, 0] = 100     # the one sampled column of the vertical area
    sep, white = port.scale_black_white(img, w, (8, 0, 1024, 512), white=4000,
                                        areas=[(1, 0, 512)], dither=False)
    # 512 rows * 512 columns / 4 positions = 65536 hits per histogram -> all counters wrapped to 0
    assert sep == [65535] * 4


@needs_ref
@pytest.mark.parametrize("white", [15000, 900])     # SSE2 path / plain path
def test_three_components_per_pixel(white):
    # cpp = 3 (not CFA): the SSE2 loop still bounds x by the PIXEL width (only the first
    # roundDown(w, 8) of the 3*w samples of a row are scaled); the plain loop covers dim.x*cpp
    w, h, cpp = 40, 10, 3
    rng = np.random.default_rng(white)
    a = port.new_image(w, h, cpp)
    a[:, :] = rng.integers(100, white, size=a.shape, dtype=np.uint16)
    b = a.copy()
    kw = dict(black_sep=[100, 100, 100, 100], white=white, is_cfa=False, cpp=cpp)
    ra = ref.scale_black_white(a, w, (2, 1, 30, 8), **kw)
    rb = port.scale_black_white(b, w, (2, 1, 30, 8), **kw)
    assert ra == rb and np.array_equal(a, b)
