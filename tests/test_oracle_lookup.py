"""RawImageData::sixteenBitLookup / RawImageDataU16::doLookup (SURVEY 8(f)3): the oracle's
restatement against the compiled reference -- plain and dithered tables, cpp 1 to 3, with and
without a crop (the APPLY_LOOKUP worker always covers the whole uncropped buffer)."""
import numpy as np
import pytest

from oracle import port, ref, synth

needs_ref = pytest.mark.skipif(not ref.checkable(), reason="oracle/_ref/libref.so not built")


def image(w, h, cpp, seed, hi=65536):
    rng = np.random.default_rng(seed)
    a = port.new_image(w, h, cpp)
    a[:, :] = rng.integers(0, hi, size=a.shape, dtype=np.uint16)
    return a


def curve(n, seed):
    rng = np.random.default_rng(seed)
    c = np.sort(rng.integers(0, 65536, n)).astype(np.uint16)
    return c


CASES = [(64, 12, 1, [0, 0, 64, 12], 4096), (70, 9, 1, [3, 2, 60, 5], 65536), (40, 8, 3, [0, 0, 40, 8], 1000),
         (333, 5, 1, [1, 1, 300, 3], 16384), (16, 3, 2, [0, 1, 16, 2], 2)]


@needs_ref
@pytest.mark.parametrize("dither", [False, True])
@pytest.mark.parametrize("k", range(len(CASES)))
def test_lookup_matches_reference(k, dither):
    w, h, cpp, crop, ncurve = CASES[k]
    a = image(w, h, cpp, k)
    b = a.copy()
    cv = curve(ncurve, 10 + k)
    ref.sixteen_bit_lookup(a, w, cpp, crop, cv, dither, nthreads=3)
    port.sixteen_bit_lookup(b, w, cpp, port.build_table(cv, dither), dither)
    assert np.array_equal(a, b)


@needs_ref
def test_no_table_is_a_no_op():
    a = image(32, 4, 1, 1)
    b = a.copy()
    ref.sixteen_bit_lookup(a, 32, 1, [0, 0, 32, 4], None, False)
    port.sixteen_bit_lookup(b, 32, 1, None, False)
    assert np.array_equal(a, b) and np.array_equal(a, image(32, 4, 1, 1))


@needs_ref
def test_sony_curve_with_dither_on_a_large_row_count():
    # rows whose seed (w + 13 y) ^ 0x45694584 has a low half of 0xFFFF step twice above the modulus
    w, h = 40, 3700
    a = image(w, h, 1, 3, 4096 * 2)
    b = a.copy()
    cv = synth.sony_curve()
    ref.sixteen_bit_lookup(a, w, 1, [0, 0, w, h], cv, True, nthreads=4)
    port.sixteen_bit_lookup(b, w, 1, port.build_table(cv, True), True)
    assert np.array_equal(a, b)
