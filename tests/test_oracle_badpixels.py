"""RawImageData::fixBadPixels (SURVEY 8(f)3): the oracle's restatement against the compiled
reference -- CFA (step 2) and non-CFA (step 1) images, clusters of bad pixels, bad pixels at the
borders, whole bad rows / columns, cpp 3, and the (w + 15) / 32 block rule."""
import numpy as np
import pytest

from oracle import port, ref

needs_ref = pytest.mark.skipif(not ref.checkable(), reason="oracle/_ref/libref.so not built")


def image(w, h, cpp, seed):
    rng = np.random.default_rng(seed)
    a = port.new_image(w, h, cpp)
    a[:, :] = rng.integers(0, 65536, size=a.shape, dtype=np.uint16)
    return a


def pos(points):
    return np.array([(y << 16) | x for y, x in points], dtype=np.uint32)


def scenarios():
    rng = np.random.default_rng(5)
    out = []
    w, h = 64, 24
    scattered = [(int(y), int(x)) for y, x in zip(rng.integers(0, h, 60), rng.integers(0, w, 60))]
    out.append(("scattered_cfa", w, h, 1, True, scattered))
    out.append(("scattered_plain", w, h, 1, False, scattered))
    out.append(("corners_edges", w, h, 1, True, [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (0, 1), (1, 0),
                                                  (h - 2, w - 2), (5, 0), (5, w - 1), (0, 7), (h - 1, 9)]))
    out.append(("cluster", w, h, 1, True, [(y, x) for y in range(8, 14) for x in range(20, 29)]))
    out.append(("whole_row_and_column", w, h, 1, True, [(6, x) for x in range(w)] + [(y, 11) for y in range(h)]))
    out.append(("same_parity_all_bad_in_row", w, h, 1, True, [(3, x) for x in range(0, w, 2)]))
    out.append(("duplicates", w, h, 1, False, [(2, 2), (2, 2), (2, 3), (2, 2)]))
    out.append(("cpp3", 40, 12, 3, False, [(1, 1), (5, 20), (11, 30), (0, 0), (6, 31), (6, 30)]))
    out.append(("width_48_only_first_32", 48, 6, 1, True, [(2, 5), (2, 31), (2, 32), (3, 47)]))
    out.append(("width_49_all", 49, 6, 1, True, [(2, 5), (2, 31), (2, 32), (3, 48)]))
    out.append(("everything_bad", 34, 5, 1, True, [(y, x) for y in range(5) for x in range(34)]))
    return out


@needs_ref
@pytest.mark.parametrize("k", range(11))
def test_fix_bad_pixels_matches_reference(k):
    name, w, h, cpp, cfa, points = scenarios()[k]
    a = image(w, h, cpp, k)
    b = a.copy()
    keep = a.copy()
    ref.fix_bad_pixels(a, w, cpp, pos(points), cfa, nthreads=3)
    port.fix_bad_pixels(b, w, cpp, pos(points), cfa)
    assert np.array_equal(a, b)
    if name == "width_48_only_first_32":
        assert a[2, 32] == keep[2, 32] and a[3, 47] == keep[3, 47] and a[2, 5] != keep[2, 5]


def test_no_positions_is_a_no_op():
    a = image(32, 4, 1, 1)
    b = a.copy()
    port.fix_bad_pixels(b, 32, 1, np.zeros(0, np.uint32))
    assert np.array_equal(a, b)


def test_isolated_bad_pixel_is_the_mean_of_its_four_neighbours():
    a = port.new_image(32, 9)       # (a 16 pixel wide image has (16 + 15) / 32 = 0 blocks: untouched)
    a[:, :] = 0
    a[4, 6], a[4, 10], a[2, 8], a[6, 8] = 100, 200, 300, 400      # step 2 neighbours of (4, 8)
    a[4, 8] = 9999
    port.fix_bad_pixels(a, 32, 1, pos([(4, 8)]))
    assert a[4, 8] == (100 * 128 + 200 * 128 + 300 * 128 + 400 * 128) >> 9
