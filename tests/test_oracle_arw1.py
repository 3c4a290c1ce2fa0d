"""Sony ARW1 on the CPU: the restatement of SonyArw1Decompressor in tests/emu/arw1_oracle.c against
the outcomes of the reference's own decompressor (tests/golden/arw1_ref.json, recorded by
tools/arw1_ref_golden.py), against a second, bit-by-bit Python reading of
SonyArw1Decompressor.cpp:58-92, and its stream writer."""
import hashlib
import json
import os

import numpy as np
import pytest

import arw1_oracle as A


def py_decompress(data, w, h):
    """Straight Python reading of the reference loop (small frames only)."""
    if w <= 0 or h <= 0 or h % 2 or w > 4600 or h > 3072:
        return None, A.CTOR, 0
    size = len(data)
    if size < 4:   # BitStreamerMSB's constructor
        return np.full((h, A.pitch_elems(w)), 0xABCD, np.uint16), A.IOE, 0
    bits = np.unpackbits(np.frombuffer(bytes(data) + bytes(64), np.uint8))
    img = np.full((h, A.pitch_elems(w)), 0xABCD, np.uint16)
    pos, pred = 0, 0

    def get(n):
        nonlocal pos
        v = 0
        for _ in range(n):
            v = (v << 1) | int(bits[pos])
            pos += 1
        return v
    for col in range(w - 1, -1, -1):
        rows = list(range(0, h, 2)) + list(range(1, h, 2))
        for row in rows:
            refills = (pos >> 5) + 1 + (1 if pos & 31 else 0)   # BitStreamerMSB fill(32)
            if refills >= (size + 8) // 4 + 2:
                return img, A.IOE, 0
            ln = 4 - get(2)
            if ln == 3 and get(1):
                ln = 0
            if ln == 4:
                while ln < 17 and not get(1):
                    ln += 1
            d = 0
            if ln:
                v = get(ln)
                d = v if v >> (ln - 1) else v - ((1 << ln) - 1)
            pred += d
            if not 0 <= pred <= 4095:
                return img, A.RDE, (row << 14) | col
            img[row, col] = pred
    return img, A.OK, 0


def check(data, w, h):
    got, rc, where = A.decompress(data, w, h)
    want, rc2, where2 = py_decompress(data, w, h)
    assert (rc, where) == (rc2, where2)
    if rc != A.CTOR:
        assert np.array_equal(got, want)
    return rc, where


@pytest.mark.parametrize("w,h", [(1, 2), (3, 2), (17, 6), (40, 12)])
def test_round_trip(w, h):
    f = A.natural_frame(w, h, seed=w * h)
    data = A.encode_frame(f)
    rc, _ = check(data, w, h)
    assert rc == A.OK
    img, _, _ = A.decompress(data, w, h)
    assert np.array_equal(img[:, :w], f)


def test_round_trip_dslr_frame():
    w, h = 3872, 2592
    f = A.natural_frame(w, h, seed=5)
    img, rc, _ = A.decompress(A.encode_frame(f), w, h)
    assert rc == A.OK and np.array_equal(img[:, :w], f)


def test_every_length():
    """Lengths 0..17: the writer's codes are the reference's, value by value."""
    w, h = 5, 8
    d = []
    for ln in range(18):
        if ln == 0:
            d.append(0)
            continue
        v = (1 << (ln - 1)) + 1 if ln > 1 else 1
        d += [v, -v]                       # up and back: pred stays 0..4095 while |d| < 4096
    d += [0] * (w * h - len(d))
    data = A.encode(np.array(d[:w * h]))
    rc, where = check(data, w, h)
    # the first length >= 13 (|d| >= 4096) is the first violation
    first = next(i for i, x in enumerate(d) if abs(x) >= 4096)
    row, col = A.stream_rows_cols(w, h)
    assert rc == A.RDE and where == (int(row[first]) << 14) | int(col[first])


@pytest.mark.parametrize("seed", range(6))
def test_random_streams_and_cuts(seed):
    rng = np.random.default_rng(seed)
    w, h = int(rng.integers(1, 9)), 2 * int(rng.integers(1, 5))
    data = rng.integers(0, 256, int(rng.integers(0, 48)), dtype=np.uint8).tobytes()
    check(data, w, h)
    f = A.natural_frame(w, h, seed)
    full = A.encode_frame(f)
    for cut in range(0, min(41, len(full) + 1)):
        check(full[:len(full) - cut], w, h)


@pytest.mark.parametrize("fill", [0x00, 0xFF])
def test_constant_streams(fill):
    for n in (0, 1, 7, 64):
        check(bytes([fill]) * n, 6, 4)


@pytest.mark.parametrize("w,h", [(0, 2), (4, 0), (4, 3), (4601, 2), (4, 3074), (-1, 2)])
def test_constructor_rejects(w, h):
    _, rc, _ = A.decompress(b"\x00" * 16, w, h)
    assert rc == A.CTOR


# ---------------------------------------------------------------- pinned against the reference
def digest(rc, img):
    """Outcome class and the whole padded image after the call (None: the constructor threw)."""
    h = hashlib.sha256(bytes([rc]))
    if img is not None:
        h.update(np.ascontiguousarray(img).tobytes())
    return h.hexdigest()


def golden_cases():
    """(name, (data, w, h)) for every case pinned against the reference."""
    for w, h in [(1, 2), (3, 2), (17, 6), (640, 480), (3872, 2592)]:
        yield "size_%dx%d" % (w, h), (A.encode_frame(A.natural_frame(w, h, seed=w + h)), w, h)
    w, h = 5, 8
    for first_long in range(13, 18):
        d = [0]
        for ln in range(1, 13):
            v = (1 << (ln - 1)) + 1 if ln > 1 else 1
            d += [v, -v]
        v = (1 << (first_long - 1)) + 1
        d += [v, -v, 7] + [0] * (w * h)
        yield "lengths_to_%d" % first_long, (A.encode(np.array(d[:w * h])), w, h)
    for d0 in (65541, -65540, 32773):
        d = np.zeros(16, np.int32)
        d[0], d[5] = 100, d0
        yield "long_%d" % d0, (A.encode(d), 4, 4)
    w, h = 70, 130
    f = A.natural_frame(w, h, 3)
    row, cc = A.stream_rows_cols(w, h)
    for half in (0, 1):
        for c in (w - 1, 33, 0):
            for sign in (-1, 1):
                d = A.frame_diffs(f).astype(np.int64)
                i = int(np.nonzero((row == 34 + half) & (cc == c))[0][0])
                d[i] += sign * 5000
                d[min(i + 40, d.size - 1)] -= sign * 9000
                yield "violation_%d_%d_%d" % (half, c, sign), (A.encode(d), w, h)
    w, h = 24, 10
    f = A.natural_frame(w, h, 7)
    d2 = A.frame_diffs(f)
    d2[-3] += 6000
    for tag, s in (("clean", A.encode_frame(f)), ("viol", A.encode(d2))):
        for cut in range(41):
            yield "cut_%s_%d" % (tag, cut), (s[:max(len(s) - cut, 0)], w, h)
    for fill in (0x00, 0xFF):
        for n in (0, 1, 7, 64, 4096):
            yield "const_%02x_%d" % (fill, n), (bytes([fill]) * n, 6, 4)
    for w, h in [(0, 2), (4, 0), (4, 3), (4601, 2), (4, 3074)]:
        yield "ctor_%dx%d" % (w, h), (b"\x00" * 16, w, h)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "arw1_ref.json")


def test_oracle_matches_reference_outcomes():
    with open(GOLDEN) as f:
        want = json.load(f)
    cases = dict(golden_cases())
    assert set(cases) == set(want)
    for name, (data, w, h) in cases.items():
        img, rc, _ = A.decompress(data, w, h, fill=A.FILL_DEFAULT)
        assert digest(rc, img if rc != A.CTOR else None) == want[name], name
