"""GoPro VC-5 on the CPU: the restatement of VC5Decompressor in tests/emu/vc5_oracle.c against the
outcomes of the reference's own decompressor (tests/golden/vc5_ref.json, recorded by
tools/vc5_ref_golden.py): the message thrown, printed values included, and the whole padded image after
the call.  Also the band writer against the restatement's band decoder."""
import hashlib
import json
import os

import numpy as np

import vc5_oracle as V

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vc5_ref.json")
PS2 = [[2, 2, 2]] * 4  # unit gain per level


def digest(message, img):
    return hashlib.sha256(message.encode() + b"\0" + np.ascontiguousarray(img).tobytes()).hexdigest()


def parts(w, h, content, prec=16, quants=None):
    """(payloads, params) of band content, as V.encode writes them."""
    dims = V.band_dims(w, h)
    payloads, params = [], []
    for ch in range(4):
        pl, pa = [], []
        for s in range(10):
            bw, bh = dims[V.level_of(s)]
            v = np.asarray(content[ch][s]).reshape(bh, bw)
            q = 1 if quants is None else quants[ch][s]
            pl.append(V.lowpass_bytes(v, prec) if s == 0 else V.pack(V.band_symbols(v, q)))
            pa.append(prec if s == 0 else q)
        payloads.append(pl)
        params.append(pa)
    return payloads, params


def band_script(w, h, kind, subband):
    """Symbols of a high-pass band of w x h (image dims) that fails with `kind` (or decodes, kind OK)."""
    bw, bh = V.band_dims(w, h)[V.level_of(subband)]
    area = bw * bh
    one, z12, end = V.entry(1, 0), V.entry(12, 0), V.entry(0, 1)
    fill = [[one, 0]] * (area - 1)
    if kind == V.OK:
        return fill + [[one, 0], [end, 0]]
    if kind == V.EARLY_END:
        return fill[:area // 2] + [[end, 0]]
    if kind == V.OVERRUN:
        return fill[:area - 5] + [[z12, 0], [end, 0]]
    if kind == V.NO_END:
        return fill + [[one, 0], [one, 0]]
    if kind == V.QUANT:
        return fill[:area // 3] + [[V.entry(1, 255), 1]] + fill[area // 3:] + [[one, 0], [end, 0]]
    raise ValueError(kind)


def failing_block(w, h, fails, content=None, quant_big=None):
    """A datablock of natural content in which fails[(ch, s)] = kind makes that band fail."""
    content = V.natural(w, h, seed=w * h) if content is None else content
    payloads, params = parts(w, h, content)
    for (ch, s), kind in fails.items():
        if kind == V.SHORT:
            payloads[ch][s] = b""
        elif kind == V.OVERREAD:
            # 4 zero bytes: one-bit zero symbols, the pump's zero fill behind the payload included, up to
            # bit 8 * 4 + 64; the band needs more (area > 97)
            payloads[ch][s] = bytes(4)
        else:
            payloads[ch][s] = V.pack(band_script(w, h, kind, s))
            if kind == V.QUANT:
                params[ch][s] = 200
    return V.datablock(w, h, payloads, params, PS2)


def golden_cases():
    """[(name, (data, w, h, white, cfa))]"""
    out = []

    def add(name, data, w, h, white=4095, cfa=V.RGGB):
        out.append((name, (bytes(data), w, h, white, cfa)))

    # dims: every even remainder mod 16, non-square, odd band sizes at each level
    for k in range(8):
        w, h = 34 + 2 * k, 48 - 2 * k + 16 * (k & 1)
        add("dims_%d_%d" % (w, h), V.encode(w, h, V.natural(w, h, seed=k), prescale=PS2), w, h)
    add("dims_98_66", V.encode(98, 66, V.natural(98, 66, seed=9), prescale=PS2), 98, 66)
    # output bits 1..16 (white levels 1, 3, 7, ... and one not of the form 2^k - 1)
    v = V.natural(256, 224, seed=3)
    rng = np.random.default_rng(3)
    for ch in range(4):  # random low pass, gain 1/4 at wavelet 1: pre-table values cover 0..4095 and beyond
        v[ch][0] = rng.integers(0, 18400, size=v[ch][0].shape) if ch == 0 else rng.integers(6000, 10400, v[ch][0].shape)
    data = V.encode(256, 224, v, prescale=[[0, 2, 2]] * 4)
    for bits in range(1, 17):
        add("bits_%d" % bits, data, 256, 224, white=(1 << bits) - 1)
    add("bits_white_1000", data, 256, 224, white=1000)
    # both phases
    for cfa in (V.RGGB, V.GBRG):
        add("phase_%d" % cfa, V.encode(50, 40, V.natural(50, 40, seed=cfa), prescale=PS2), 50, 40, cfa=cfa)
    # prescale 0, 1, 2, 3 per wavelet, per channel (every wavelet's prescale is set: the reference leaves
    # one that no PrescaleShift sets indeterminate)
    for p in range(4):
        pre = [[p, (p + 1) % 4, (p + 2) % 4], [2, p, 2], [p, 2, 2], [2, 2, p]]
        add("prescale_%d" % p, V.encode(40, 36, V.natural(40, 36, seed=p, span=300), prescale=pre), 40, 36)
    # quantization: 1, large, negative, 0
    for q in (1, 37, 120, -3, 0):
        c = V.natural(48, 40, seed=abs(q), quant=q) if q else V.flat(48, 40)
        quants = [[q] * 10 for _ in range(4)]
        add("quant_%d" % q, V.encode(48, 40, c, quants=quants, prescale=PS2), 48, 40)
    # dense content (long codes), flat content (runs crossing rows and band ends), low-pass precisions
    add("noise", V.encode(52, 44, V.noise(52, 44, seed=1), prescale=PS2), 52, 44)
    add("flat", V.encode(70, 34, V.flat(70, 34, 777), prescale=PS2), 70, 34)
    for prec in (8, 12, 15):
        add("prec_%d" % prec, V.encode(36, 36, V.natural(36, 36, seed=prec, span=250), prec=prec, prescale=PS2),
            36, 36)
    # each band message in a level-3, level-2 and level-1 band; two bands at once; end marker sign 1
    for kind in (V.QUANT, V.EARLY_END, V.OVERRUN, V.NO_END, V.SHORT, V.OVERREAD):
        w, h = (176, 160) if kind == V.OVERREAD else (46, 38)
        for ch, s in ((1, 2), (2, 5), (3, 9)):
            add("fail_%d_ch%d_sb%d" % (kind, ch, s), failing_block(w, h, {(ch, s): kind}), w, h)
    add("fail_two_a", failing_block(46, 38, {(0, 7): V.SHORT, (3, 1): V.EARLY_END}), 46, 38)
    add("fail_two_b", failing_block(46, 38, {(2, 4): V.NO_END, (1, 4): V.OVERRUN}), 46, 38)
    w, h = 40, 40
    c = V.flat(w, h)
    payloads, params = parts(w, h, c)
    syms = V.band_symbols(c[0][8], 1)
    syms[-1][1] = 1
    payloads[0][8] = V.pack(syms)
    add("end_marker_sign", V.datablock(w, h, payloads, params, PS2), w, h)
    # constructor checks
    good = V.encode(36, 34, V.natural(36, 34, seed=1), prescale=PS2)
    add("ctor_dims", good, 0, 34)
    add("ctor_width", good, 35, 34)
    add("ctor_height", good, 36, 33)
    add("ctor_cfa", good, 36, 34, cfa=4)
    for cfa in (1, 3):
        add("ctor_phase_%d" % cfa, good, 36, 34, cfa=cfa)
    for white in (0, 65536, -5):
        add("ctor_white_%d" % white, good, 36, 34, white=white)
    # the tag walk
    cp, pp = parts(36, 34, V.natural(36, 34, seed=2))
    base = [(0x0014, 36), (0x0015, 34)] + V.HEADER_TAGS
    add("tag_magic", b"VC-6" + good[4:], 36, 34)
    for name, t, v in (("channels", 0x000c, 3), ("width", 0x0014, 38), ("height", 0x0015, 30),
                       ("format", 0x0054, 3), ("subbands", 0x000e, 9), ("bpc", 0x0066, 14),
                       ("pat_w", 0x006a, 4), ("pat_h", 0x006b, 1), ("cps", 0x006c, 3),
                       ("prec_low", 0x0023, 7), ("prec_high", 0x0023, 17), ("channel_no", 0x003e, 4),
                       ("subband_no", 0x0030, 10), ("unknown", 0x0123, 5), ("unknown_small", 0x4123, 1),
                       ("optional_skip", -0x4123 & 0xFFFF, 1), ("optional_large", -0x2101 & 0xFFFF, 7),
                       ("optional_min", 0x8000, 3)):
        add("tag_" + name, V.datablock(36, 34, cp, pp, PS2, header=base + [(t, v)]), 36, 34)
    hdr = b"VC-5" + b"".join(V.tag(t, v) for t, v in base)
    lp = cp[0][0]
    add("tag_no_subband", hdr + V.tag(0x0023, 16) + V.chunk(lp), 36, 34)
    add("tag_no_precision", hdr + V.tag(0x0030, 0) + V.chunk(lp), 36, 34)
    add("tag_no_quant", hdr + V.tag(0x0030, 1) + V.chunk(cp[0][1]), 36, 34)
    add("tag_seen", hdr + V.tag(0x0023, 16) + V.tag(0x0030, 0) + V.chunk(lp) + V.tag(0x0023, 16) +
        V.tag(0x0030, 0) + V.chunk(lp), 36, 34)
    add("tag_seen_high", hdr + V.tag(0x003e, 2) + V.tag(0x0035, 1) + V.tag(0x0030, 5) + V.chunk(cp[2][5]) +
        V.tag(0x0035, 1) + V.tag(0x0030, 5) + V.chunk(cp[2][5]), 36, 34)
    add("tag_short_lowpass", hdr + V.tag(0x0023, 16) + V.tag(0x0030, 0) + V.chunk(lp[:-8]), 36, 34)
    add("tag_lowpass_precision_18", hdr + V.tag(0x0023, 8) + V.tag(0x0030, 0) + V.chunk(lp), 36, 34)
    for cut in (2, 5, 8, 100, len(good) - 3):
        add("truncated_%d" % cut, good[:cut], 36, 34)
    add("truncated_chunk", hdr + V.tag(0x0023, 16) + V.tag(0x0030, 0) + V.chunk(lp)[:-4], 36, 34)
    add("truncated_skip", hdr + V.tag(-0x4123 & 0xFFFF, 4) + b"\0" * 12, 36, 34)
    # channel order and the PrescaleShift quirk: a PrescaleShift before ChannelNumber applies to the
    # channel before (channel 0 gets 0 here; channel 1 still gets its own)
    blk = V.datablock(40, 36, *parts(40, 36, V.natural(40, 36, seed=11, span=200)), prescale=PS2)
    ps1 = V.tag(0x006d, 2 << 14 | 2 << 12 | 2 << 10)
    add("prescale_before_channel", blk.replace(V.tag(0x003e, 1) + ps1, V.tag(0x006d, 0) + V.tag(0x003e, 1) + ps1),
        40, 36)
    return out


def run_case(data, w, h, white, cfa):
    """-> (image, outcome, message)"""
    img, rc, args = V.decompress(data, w, h, white, cfa)
    return img, rc, V.message(rc, args)


def test_golden_outcomes():
    with open(GOLDEN) as f:
        gold = json.load(f)
    cases = golden_cases()
    assert sorted(n for n, _ in cases) == sorted(gold)
    bad = []
    for name, case in cases:
        img, rc, msg = run_case(*case)
        if digest(msg, img) != gold[name]:
            bad.append((name, rc, msg))
    assert not bad, bad


def test_cases_reach_every_outcome():
    seen = {run_case(*c)[1] for _, c in golden_cases()}
    assert {V.TOO_MANY + k for k in V.BAND_MESSAGES} <= seen
    assert set(V.CTOR_MESSAGES) <= seen | {35}  # (35 is reached: unknown tags)
    assert 35 in seen and V.OK in seen


def test_log_table_fully_reached():
    """The content of the bits_* cases reaches every log-table entry: each value of the 16-bit table
    is in the image."""
    lut = {int(65535 * ((113.0 ** (i / 4095.0) - 1) / 112.0)) for i in range(4096)}
    for name, case in golden_cases():
        if name == "bits_16":
            img, rc, _ = run_case(*case)
            assert rc == V.OK
            assert lut <= set(np.unique(img[:224, :256]).tolist())


def test_writer_round_trip():
    """Band content -> symbols -> bytes -> the restatement's band decoder."""
    rng = np.random.default_rng(5)
    cb = V.codebook()
    for q in (1, 7, -2, 0):
        for w, h in ((5, 3), (17, 9), (60, 1)):
            mags = V.magnitudes(q)
            v = np.where(rng.random((h, w)) < 0.3, rng.choice([-1, 1], (h, w)) * mags[rng.integers(0, 256, (h, w))],
                         0) * (1 if q >= 0 else -1)
            data = V.pack(V.band_symbols(v, q))
            out = np.zeros(w * h, np.int16)
            rc = V.lib().vc_decode_band(data, len(data), w, h, q, cb.ctypes.data, cb.shape[0], out.ctypes.data)
            assert rc == V.OK and np.array_equal(out, v.reshape(-1)), (q, w, h, rc)


def test_codebook_fixture_is_a_complete_prefix_code():
    cb = V.codebook()
    assert cb.shape == (264, 4)
    assert sum(2.0 ** -int(s) for s in cb[:, 0]) == 1.0
    codes = sorted((int(b) << (26 - int(s)), int(s)) for s, b, _, _ in cb)
    for (a, la), (b, _) in zip(codes, codes[1:]):
        assert a + (1 << (26 - la)) <= b


def golden_cases_by_name():
    return dict(golden_cases())
