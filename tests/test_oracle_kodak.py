"""Kodak DCR on the CPU: the restatement of KodakDecompressor in tests/emu/kodak_oracle.c against the
outcomes of the reference's own decompressor (tests/golden/kodak_ref.json, recorded by
tools/kodak_ref_golden.py): the message thrown, printed values included, and the whole padded image
after the call.  Also the stream writer against the restatement, and the closed form of a segment's
length that the device's row walk relies on."""
import hashlib
import json
import os

import numpy as np

import kodak_oracle as K

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kodak_ref.json")


def digest(message, img):
    return hashlib.sha256(message.encode() + b"\0" + np.ascontiguousarray(img).tobytes()).hexdigest()


GAMMA = [int(65535 * (i / 4095.0) ** 0.45) for i in range(4096)]
ZIGZAG = [(i * 37) % 1000 + (i & 1) * 30000 for i in range(4096)]  # non-monotonic
SHORT = [100 + 3 * i for i in range(300)]  # values past its end take the last entry


def segment_starts(data, w, h, row_start=None):
    """Offsets of every segment by the closed form len = h + e + 4 ceil(max(0, S - 8e) / 32), until one
    reads past the end: [(row, col, offset)], and the offset behind the last (or None).  row_start, a
    list, gets the start of every row reached."""
    row_start = [] if row_start is None else row_start
    out, p = [], 0
    for r in range(h):
        for c in range(0, w, 256):
            b = min(256, w - c)
            hb, e = b // 2, (2 if b % 8 == 4 else 0)
            if c == 0:
                row_start.append(p)
            if p + hb > len(data):
                return out, None
            s = sum((x & 15) + (x >> 4) for x in data[p:p + hb])
            n = hb + e + 4 * ((max(0, s - 8 * e) + 31) // 32)
            if p + n > len(data):
                return out, None
            out.append((r, c, p))
            p += n
    return out, p


def case_table(curve, dither, uncorrected):
    """(mode, table) of the restatement for a RawImage with `curve` (or none)."""
    if uncorrected or curve is None:
        return K.NONE, None
    return (K.DITHER if dither else K.PLAIN), K.lookup_table(curve, dither)


def golden_cases():
    """[(name, (data, w, h, bps, cpp, curve, dither, uncorrected))]"""
    out = []

    def add(name, data, w, h, bps=12, cpp=1, curve=None, dither=False, uncorrected=True):
        out.append((name, (bytes(data), w, h, bps, cpp, curve, dither, uncorrected)))

    # widths: t == 0, t % 8 == 0, t % 8 == 4, under 256; both depths
    for w in (4, 8, 100, 252, 256, 260, 264, 280, 300, 512, 516, 520, 772):
        for bps in (10, 12):
            h = 3 if w < 600 else 2
            add("dims_%d_%d" % (w, bps), K.encode(K.natural(w, h, bps, seed=w + bps)), w, h, bps)
    # table modes: uncorrected with a table set, plain, dithered, non-monotonic and short curves
    v = K.natural(300, 3, 12, seed=5)
    data = K.encode(v)
    for cname, curve in (("gamma", GAMMA), ("zigzag", ZIGZAG), ("short", SHORT)):
        for dither in (False, True):
            add("table_%s_%d" % (cname, dither), data, 300, 3, 12, curve=curve, dither=dither, uncorrected=False)
        add("table_%s_uncorrected" % cname, data, 300, 3, 12, curve=curve, uncorrected=True)
    add("table_none_corrected", data, 300, 3, 12, uncorrected=False)
    # values at the edges: 0, 2^bps - 1 decode; 2^bps and -1 fail
    for bps in (10, 12):
        for name, x in (("zero", 0), ("top", (1 << bps) - 1), ("over", 1 << bps), ("neg", -1)):
            for col in (0, 1, 255, 256, 299):
                vv = K.natural(300, 2, bps, seed=col)
                vv[1, col] = x
                add("edge_%s_%d_%d" % (name, bps, col), K.encode(vv), 300, 2, bps, curve=GAMMA, dither=True,
                    uncorrected=False)
    # lengths 0 (flat) and 15 (out of range either way)
    add("flat", K.encode(np.zeros((3, 516), np.int64)), 516, 3, 12)
    for sign in (1, -1):
        lens = np.zeros((2, 260), np.uint8)
        codes = np.zeros((2, 260), np.uint16)
        lens[1, 7] = 15
        codes[1, 7] = (1 << 14) + 5 if sign > 0 else 3
        add("len15_%+d" % sign, K.write(lens, codes, 260, 2), 260, 2, 12)
    # raw scripts: random lengths and codes (out-of-range values)
    rng = np.random.default_rng(7)
    for k in range(6):
        w, h = (260, 100, 516, 8, 264, 300)[k], 2
        lens = rng.integers(0, 16, (h, w)).astype(np.uint8)
        codes = rng.integers(0, 1 << 16, (h, w)).astype(np.uint16)
        add("script_%d" % k, K.write(lens, codes, w, h), w, h, (10, 12)[k % 2])
    # truncation: inside a header, inside the two-byte prefix, inside a refill, exactly enough, one short
    for w in (260, 300, 516, 100):
        v = K.natural(w, 3, 12, seed=w)
        v[:, ::3] = (v[:, ::3] * 7) % 4096  # long differences: several refills per segment
        data = K.encode(v)
        segs, end = segment_starts(data, w, 3)
        assert end == len(data)
        r, c, p = segs[len(segs) // 2 + 1]
        b = min(256, w - c)
        add("cut_header_%d" % w, data[:p + b // 4], w, 3)
        if b % 8 == 4:
            add("cut_prefix_%d" % w, data[:p + b // 2 + 1], w, 3)
        add("cut_refill_%d" % w, data[:p + b // 2 + (2 if b % 8 == 4 else 0) + 6], w, 3)
        add("cut_exact_%d" % w, data, w, 3)
        add("cut_one_short_%d" % w, data[:-1], w, 3)
        add("cut_extra_%d" % w, data + bytes(40), w, 3)
    # the constructor: cpp, every dimension check, bps, the size check
    d = K.encode(K.natural(8, 2, 12))
    add("ctor_cpp", d, 8, 2, 12, cpp=2)
    for name, (w, h) in (("w0", (0, 2)), ("h0", (8, 0)), ("w6", (6, 2)), ("w4520", (4520, 2)),
                         ("h3013", (8, 3013)), ("wneg", (-4, 2))):
        add("ctor_dims_%s" % name, d, w, h, 12)
    for bps in (8, 11, 14, 16):
        add("ctor_bps_%d" % bps, d, 8, 2, bps)
    add("ctor_size", bytes(63), 16, 8, 12)
    add("ctor_size_ok", bytes(64), 16, 8, 12)
    # random bytes
    for k in range(10):
        w, h = 4 * int(rng.integers(1, 200)), int(rng.integers(1, 5))
        n = int(rng.integers(w * h // 2, w * h * 2 + 1))
        add("random_%d" % k, rng.integers(0, 256, n, dtype=np.uint8).tobytes(), w, h, (10, 12)[k % 2])
    # real sensor sizes
    add("full_4500x3000_12", K.encode(K.natural(4500, 3000, 12, seed=1)), 4500, 3000, 12)
    add("full_4516x3012_10", K.encode(K.natural(4516, 3012, 10, seed=2)), 4516, 3012, 10, curve=GAMMA,
        dither=True, uncorrected=False)
    return out


def run_case(data, w, h, bps, cpp, curve, dither, uncorrected):
    mode, table = case_table(curve, dither, uncorrected)
    img, rc, r, c, v = K.decompress(data, w, h, bps, mode, table, cpp)
    return img, rc, r, c, v, K.message(rc, w, h, bps, v)


def test_golden_outcomes():
    with open(GOLDEN) as f:
        want = json.load(f)
    cases = dict(golden_cases())
    assert set(cases) == set(want)
    for name, case in cases.items():
        img, _, _, _, _, msg = run_case(*case)
        assert digest(msg, img) == want[name], name


def test_cases_reach_every_outcome():
    seen = {run_case(*case)[1] for _, case in golden_cases()}
    assert seen == set(range(7))


def test_messages_parse_back():
    for name, case in golden_cases():
        _, rc, _, _, _, msg = run_case(*case)
        if rc != K.OK:
            assert K.message_id(msg) == rc, name


def test_round_trip():
    for w in (4, 100, 256, 260, 300, 772):
        for bps in (10, 12):
            v = K.random_values(w, 5, bps, seed=w)
            img, rc, _, _, _ = K.decompress(K.encode(v), w, 5, bps)
            assert rc == K.OK
            assert np.array_equal(img[:, :w], v)


def test_closed_form_segment_length():
    """Where the closed form says the stream ends (or over-reads) is where the restatement does."""
    rng = np.random.default_rng(3)
    for k in range(200):
        w, h = 4 * int(rng.integers(1, 150)), int(rng.integers(1, 4))
        data = rng.integers(0, 256, int(rng.integers(w * h // 2, 3 * w * h)), dtype=np.uint8).tobytes()
        segs, end = segment_starts(data, w, h)
        _, rc, r, c, _ = K.decompress(data, w, h, 12)
        if end is None:
            nxt = len(segs)
            fr, fc = divmod(nxt, (w + 255) // 256)
            if rc == K.OVERFLOW:
                assert (r, c) == (fr, 256 * fc), k
            else:  # a value out of range in an earlier segment
                assert rc == K.VALUE and (r, c) < (fr, 256 * fc), k
        else:
            assert rc in (K.OK, K.VALUE), k
