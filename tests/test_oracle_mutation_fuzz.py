"""Byte-level mutation fuzz of whole lossless-JPEG tiles (markers + entropy-coded data) and of
packed strips: the oracle against the compiled reference on CORRUPT input -- same success /
exception class, and the same pixels whenever the decode still succeeds (the reference-side
driver hands the image back only then).  (The happy path is
covered by tests/test_oracle_vs_ref.py; this is the unhappy one: bad Huffman codes, early
markers, truncated streams, broken SOF / DHT / SOS fields.)"""
import numpy as np
import pytest

from oracle import port, ref, synth

pytestmark = pytest.mark.skipif(not ref.checkable(), reason="oracle/_ref/libref.so not built")


def _mutate(rng, blob, lo=0):
    blob = blob.copy()
    for _ in range(int(rng.integers(1, 4))):
        kind = int(rng.integers(0, 5))
        i = int(rng.integers(lo, blob.size))
        if kind == 0:
            blob[i] = rng.integers(0, 256)
        elif kind == 1:
            blob[i] ^= 1 << int(rng.integers(0, 8))
        elif kind == 2:
            blob[i] = 0xFF
        elif kind == 3 and blob.size > lo + 8:
            blob = blob[:int(rng.integers(lo + 4, blob.size))].copy()
        else:
            j = int(rng.integers(lo, blob.size))
            blob[i], blob[j] = blob[j], blob[i]
    return blob


def _both(fn_ref, fn_port, shape_img):
    out = []
    for fn in (fn_ref, fn_port):
        im = shape_img.copy()
        try:
            fn(im)
            out.append(("ok", im))
        except Exception as ex:   # noqa: BLE001
            out.append((type(ex).__name__, im))
    return out


@pytest.mark.parametrize("seed", range(150))
def test_mutated_ljpeg_tile(seed):
    rng = np.random.default_rng(7000 + seed)
    ncomp = int(rng.choice([1, 2, 3, 4]))
    tw, th = 8 * ncomp * int(rng.integers(1, 5)), int(rng.integers(2, 12))
    img = synth.image_model(tw, th, seed, bits=14)
    two_tabs = ncomp >= 2 and bool(rng.integers(0, 2))
    t = synth.make_dng_ljpeg(img, tw, th, ncomp=ncomp, tabs=synth.default_tables(2 if two_tabs else 1),
                             tab_of_comp=[c % 2 if two_tabs else 0 for c in range(ncomp)],
                             restart_rows=int(rng.choice([0, 0, 1, 2])))
    blob = _mutate(rng, t.blob)
    base = port.new_image(tw, th)
    (ra, ia), (rb, ib) = _both(lambda im: ref.ljpeg_decode(blob, im, tw, 1, (0, 0), (tw, th), (tw, th)),
                               lambda im: port.ljpeg_decode(blob, im, tw, 1, (0, 0), (tw, th), (tw, th)), base)
    assert ra == rb, (ra, rb)
    if ra == "ok":
        assert np.array_equal(ia, ib)


@pytest.mark.parametrize("seed", range(60))
def test_truncated_or_short_packed_strips(seed):
    rng = np.random.default_rng(8000 + seed)
    bps = int(rng.choice([8, 10, 12, 14, 16]))
    order = int(rng.integers(0, 4))
    w = 8 * int(rng.integers(1, 30))
    h = int(rng.integers(1, 9))
    in_pitch = w * bps // 8 + int(rng.choice([0, 0, 3]))
    n = in_pitch * h
    data = synth.lcg_bytes(n, seed)
    cut = int(rng.integers(max(0, n - 2 * in_pitch), n + 1))
    data = data[:cut].copy()
    base = port.new_image(w, h)
    (ra, ia), (rb, ib) = _both(lambda im: ref.unpack(data, im, w, 1, (0, 0, w, h), in_pitch, bps, order),
                               lambda im: port.unpack(data, im, w, 1, (0, 0, w, h), in_pitch, bps, order), base)
    assert ra == rb, (ra, rb)
    if ra == "ok":
        assert np.array_equal(ia, ib)


def _classes(fa, fb, w, h):
    a, b = port.new_image(w, h), port.new_image(w, h)
    out = []
    for fn, im in ((fa, a), (fb, b)):
        try:
            fn(im)
            out.append("ok")
        except Exception as ex:   # noqa: BLE001
            out.append(type(ex).__name__)
    assert out[0] == out[1], out
    if out[0] == "ok":
        assert np.array_equal(a, b)
    return out[0]


@pytest.mark.parametrize("seed", range(80))
def test_mutated_pentax(seed):
    rng = np.random.default_rng(9000 + seed)
    modern = bool(rng.integers(0, 2))
    be = bool(rng.integers(0, 2)) if modern else True
    meta = synth.pentax_modern_meta(be) if modern else None
    w, h = 2 * int(rng.integers(1, 40)), int(rng.integers(1, 12))
    img = (synth.image_model(w, h, seed=seed, bits=12) & 0x0FFF).astype(np.uint16)
    data = np.frombuffer(bytes(synth.make_pentax(img, port.pentax_table(meta, be))), dtype=np.uint8).copy()
    if modern and rng.integers(0, 2):
        meta = _mutate(rng, np.frombuffer(bytes(meta), dtype=np.uint8).copy())
    else:
        data = _mutate(rng, data)
    _classes(lambda im: ref.pentax_decompress(im, w, data, meta, be),
             lambda im: port.pentax_decompress(im, w, data, meta, be), w, h)


@pytest.mark.parametrize("seed", range(80))
def test_mutated_nikon(seed):
    rng = np.random.default_rng(9500 + seed)
    kind = str(rng.choice(["lossless", "table", "segments", "z7", "skip"]))
    bits = int(rng.choice([12, 14]))
    be = bool(rng.integers(0, 2))
    w, h = 2 * int(rng.integers(1, 40)), int(rng.integers(1, 12))
    half = 1 << (bits - 1)
    pup = [half, half + 2, half - 8, half - 2]
    meta = np.frombuffer(bytes(synth.nikon_meta(kind, bits, (pup[0], pup[2], pup[1], pup[3]), be)), dtype=np.uint8).copy()
    su = port.nikon_setup(meta, be, bits, w, h)
    img = (synth.image_model(w, h, seed=seed, bits=bits) & ((1 << bits) - 1)).astype(np.uint16)
    data = np.frombuffer(bytes(synth.make_nikon(img, su["huff_select"], pup)), dtype=np.uint8).copy()
    if rng.integers(0, 2):
        meta = _mutate(rng, meta)
    else:
        data = _mutate(rng, data)
    unc = bool(rng.integers(0, 2))
    _classes(lambda im: ref.nikon_decompress(im, w, meta, be, bits, data, unc),
             lambda im: port.nikon_decompress(im, w, meta, be, bits, data, unc), w, h)


@pytest.mark.parametrize("seed", range(80))
def test_mutated_cr2(seed):
    rng = np.random.default_rng(9800 + seed)
    ncomp = int(rng.choice([2, 4]))
    nslices = int(rng.integers(0, 3))
    sw = ncomp * int(rng.integers(2, 10))                   # slice width in samples
    w = sw * (nslices + 1)
    h = int(rng.integers(2, 10))
    slicing = (nslices, sw, sw)
    img = port.new_image(w, h)
    img[:, :w] = synth.image_model(w, h, seed, bits=14)
    two = bool(rng.integers(0, 2))
    blob = port.cr2_encode(img, w, (ncomp, 1, 1), (w // ncomp, h), slicing, 14,
                           synth.default_tables(2 if two else 1), [c % 2 if two else 0 for c in range(ncomp)])
    blob = _mutate(rng, np.ascontiguousarray(blob))
    _classes(lambda im: ref.cr2_ljpeg_decode(blob, im, w, slicing),
             lambda im: port.cr2_ljpeg_decode(blob, im, w, slicing), w, h)
