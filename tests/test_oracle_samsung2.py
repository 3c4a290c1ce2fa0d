"""Samsung V2 on the CPU: the restatement of SamsungV2Decompressor in tests/emu/samsung2_oracle.c
(with the constructor's checks in tests/samsung2_oracle.py) against the outcomes of the reference's
own decompressor (tests/golden/samsung_v2_ref.json, recorded by tools/samsung2_ref_golden.py): the
message thrown, printed values included, and the whole padded image after the call.  Also the
stream writer against the restatement."""
import hashlib
import json
import os

import numpy as np

import samsung2_oracle as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "samsung_v2_ref.json")


def digest(message, img):
    return hashlib.sha256(message.encode() + b"\0" + np.ascontiguousarray(img).tobytes()).hexdigest()


# ---------------------------------------------------------------- raw scripts
def script(w, h, bits=12, flags=0, init=0, seed=0, motion=None, scale=None, skip=None, lens=None,
           cut=0, hdr=None):
    """A strip written block by block.  Callbacks of (row, block), each None for the default:
    motion -> 0..7 to set (1 + 3 bits; under MV 3 or 7) or None to keep; scale -> 0..2 or
    (3, twelve bits); skip -> bool; lens -> four length flags, a flag 3 as (3, length).  Defaults: keep
    the motion, scale code 0, no skip, flag 3 with a random length up to bits + 1.  Differences are
    random.  Rows end in random bits and bytes up to the next multiple of 16; `cut` bytes come off
    the end."""
    rng = np.random.default_rng(seed)
    out = bytearray(S.header(w, h, bits, flags, init) if hdr is None else hdr)
    for r in range(h):
        b = S.BitWriter()
        state = [7 if r < 2 else 4] * 4
        for k in range(w // 16):
            if not (flags & S.QP) and k % 4 == 0:
                sc = 0 if scale is None else scale(r, k)
                if isinstance(sc, tuple):
                    b.put(3, 2).put(sc[1], 12)
                else:
                    b.put(sc, 2)
            m = None if motion is None else motion(r, k)
            if flags & S.MV:
                b.put(1 if m == 3 else 0, 1)
            elif m is None:
                b.put(1, 1)
            else:
                b.put(0, 1).put(m, 3)
            if not (flags & S.SKIP):
                sk = bool(skip(r, k)) if skip is not None else False
                b.put(int(sk), 1)
                if sk:
                    continue
            fl = lens(r, k) if lens is not None else [(3, int(rng.integers(0, bits + 2))) for _ in range(4)]
            ln = []
            for g, f in enumerate(fl):
                code = f[0] if isinstance(f, tuple) else f
                b.put(code, 2)
                ln.append(f[1] if code == 3 else max(0, state[g] + (0, 1, -1)[code]))
            for g, f in enumerate(fl):
                if isinstance(f, tuple):
                    b.put(f[1], 4)
            state = ln
            for i in range(16):
                n = min(ln[i >> 2], 15)
                if n:
                    b.put(int(rng.integers(0, 1 << n)), n)
        b.pad_bytes(rng, 16)
        out += bytes(b.bytes()[:b.nbytes()])
    return bytes(out[:len(out) - cut]) if cut else bytes(out)


def natural(w, h, bits=12, flags=0, init=0, policy=0, seed=0):
    return S.encode(S.natural_values(w, h, bits, seed), bits, flags, init, policy, seed)


def row_ends(data, w, h, bits=12):
    ends = np.zeros(h, np.uint32)
    S.decompress(data, w, h, bits, ends=ends)
    return ends


# ---------------------------------------------------------------- cases
def golden_cases():
    """-> [(name, (data, w, h, bits, cpp))]"""
    cases = []

    def add(name, data, w, h, bits=12, cpp=1):
        cases.append((name, (bytes(data), w, h, bits, cpp)))

    # every opt-flag value at both bit depths: natural content, random valid motions
    for bits in (12, 14):
        for f in range(8):
            add("flags_%d_%d" % (bits, f), natural(64, 6, bits, f, init=321 * f, policy=4, seed=f), 64, 6, bits)
            add("flags_%d_%d_script" % (bits, f),
                script(96, 5, bits, f, init=77, seed=10 + f,
                       motion=lambda r, k: (k * 3 + r) % 7 if r >= 2 and 1 <= k <= 3 else 7,
                       lens=lambda r, k: [(3, 3), 1, 0, 2]), 96, 5, bits)
    # every motion on interior blocks, and the policies of the writer
    for m in range(8):
        add("motion_%d" % m, script(128, 6, 12, 0, init=2000, seed=20 + m,
                                    motion=lambda r, k, m=m: m if r >= 2 and 1 <= k <= 6 else 7,
                                    lens=lambda r, k: [(3, 4), (3, 2), (3, 5), (3, 1)]), 128, 6)
    for pol in range(5):
        for bits in (12, 14):
            add("policy_%d_%d" % (pol, bits), natural(80, 7, bits, 0, init=5, policy=pol, seed=pol), 80, 7, bits)
    # bad motion at the first and the last block (each motion), in rows 0 and 1, and averages at the edge
    for m in range(7):
        add("bad_first_%d" % m, script(64, 4, 12, 0, seed=30 + m, motion=lambda r, k, m=m: m if (r, k) == (2, 0) else 7),
            64, 4)
        add("bad_last_%d" % m, script(64, 4, 12, 0, seed=40 + m, motion=lambda r, k, m=m: m if (r, k) == (3, 3) else 7),
            64, 4)
        add("row0_motion_%d" % m, script(48, 3, 12, 0, seed=50 + m, motion=lambda r, k, m=m: m if (r, k) == (0, 1) else None),
            48, 3)
        add("row1_motion_%d" % m, script(48, 3, 12, 0, seed=60 + m, motion=lambda r, k, m=m: m if (r, k) == (1, 0) else None),
            48, 3)
    add("row0_mv", script(48, 3, 12, S.MV, seed=70, motion=lambda r, k: 3 if (r, k) == (0, 2) else 7), 48, 3)
    add("row1_mv_last", script(48, 3, 12, S.MV, seed=71, motion=lambda r, k: 3 if (r, k) == (1, 2) else 7), 48, 3)
    add("mv_last_block", script(48, 4, 12, S.MV, seed=72, motion=lambda r, k: 3 if (r, k) == (3, 2) else 7), 48, 4)
    for w in (16, 32):
        for m in (2, 4, 5, 6):
            add("narrow_%d_%d" % (w, m), script(w, 3, 12, 0, seed=73 + m, motion=lambda r, k, m=m: m if r == 2 else 7), w, 3)
    # skip blocks, with and without SKIP, and a skip keeping the lengths of the block before
    for f in (0, S.SKIP, S.SKIP | S.QP, S.QP):
        add("skip_%d" % f, script(128, 5, 12, f, init=900, seed=80 + f, skip=lambda r, k: (r + k) % 3 == 0,
                                  lens=lambda r, k: [0, 1, 2, 0] if k % 2 else [(3, 5), (3, 6), (3, 3), (3, 2)]),
            128, 5)
    # scale codes, negative scale, clamping at 0 and 2^bits - 1
    for bits in (12, 14):
        add("scale_codes_%d" % bits, script(320, 4, bits, 0, init=1000, seed=90 + bits,
                                            scale=lambda r, k: (k // 4) % 3 if k % 8 else (3, 37 * r + k)), 320, 4, bits)
        add("scale_negative_%d" % bits, script(512, 3, bits, 0, init=10, seed=92 + bits, scale=lambda r, k: 1), 512, 3, bits)
        add("scale_big_%d" % bits, script(256, 3, bits, 0, init=(1 << bits) - 5, seed=94 + bits,
                                          scale=lambda r, k: (3, 4095)), 256, 3, bits)
        add("clamp_low_%d" % bits, script(64, 4, bits, S.QP, init=0, seed=96 + bits,
                                          lens=lambda r, k: [(3, bits + 1)] * 4), 64, 4, bits)
        add("clamp_high_%d" % bits, script(64, 4, bits, 0, init=(1 << 14) - 1, seed=98 + bits,
                                           scale=lambda r, k: (3, 4095)), 64, 4, bits)
    # length flags: underflow, explicit lengths at and above bitDepth + 1, +1 past the limit
    for bits in (12, 14):
        for L in (bits, bits + 1, bits + 2, 15):
            add("explicit_%d_%d" % (bits, L), script(48, 3, bits, 0, seed=100 + L,
                                                     lens=lambda r, k, L=L: [(3, 2), (3, L if (r, k) == (2, 1) else 3), 0, 0]),
                48, 3, bits)
        add("plus_one_%d" % bits, script(48, 3, bits, 0, seed=110 + bits,
                                         lens=lambda r, k: [(3, bits + 1) if k == 0 else 1, 0, 0, 0]), 48, 3, bits)
    for g in range(4):
        add("underflow_%d" % g, script(64, 4, 12, 0, seed=120 + g,
                                       lens=lambda r, k, g=g: [(3, 0) if (i == g and k == 1) else (2 if (i == g and k == 2 and r == 3) else (3, 3)) for i in range(4)]),
            64, 4)
        add("underflow_row_start_%d" % g, script(64, 4, 12, 0, seed=124 + g,
                                                 lens=lambda r, k, g=g: [2 if i == g else 0 for i in range(4)]), 64, 4)
    # rows ending at every residue mod 16 (natural content of many widths) and random payloads
    for w in (16, 48, 64, 80, 112, 160, 208):
        for h in (1, 2, 3, 4):
            add("dims_%d_%d" % (w, h), natural(w, h, 12, 0, init=w, policy=0, seed=w * h), w, h)
    add("wide_6496", natural(6496, 2, 12, 0, init=3, policy=0, seed=1), 6496, 2)
    add("wide_6496_14", natural(6496, 3, 14, S.SKIP, init=3, policy=4, seed=2), 6496, 3, 14)
    add("tall_4336", natural(16, 4336, 12, 0, init=3, policy=0, seed=3), 16, 4336)
    rng = np.random.default_rng(1234)
    for i in range(24):
        w, h = 16 * int(rng.integers(1, 9)), int(rng.integers(1, 7))
        bits = (12, 14)[i % 2]
        body = rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8).tobytes()
        add("random_%02d" % i, S.header(w, h, bits, int(rng.integers(0, 8)), int(rng.integers(0, 1 << 14))) + body,
            w, h, bits)
    # cuts: the last 40 bytes, and around an interior row end
    base = natural(64, 4, 12, 0, init=100, policy=4, seed=5)
    for c in range(41):
        add("cut_tail_%02d" % c, base[:len(base) - c], 64, 4)
    full = natural(96, 3, 12, 0, init=100, policy=0, seed=6)
    e0 = int(row_ends(full, 96, 3)[0])
    for d in range(-10, 22):
        add("cut_row_%+03d" % d, full[:16 + e0 + d], 96, 3)
    # constructor rejections
    good = natural(64, 2, 12, 0, seed=7)
    add("ctor_cpp", good, 64, 2, 12, 2)
    for b in (0, 8, 13, 16):
        add("ctor_bits_%d" % b, good, 64, 2, b)
    for n in (0, 1, 15):
        add("ctor_short_%d" % n, good[:n], 64, 2)
    add("ctor_depth", S.header(64, 2, 12, depth=14) + good[16:], 64, 2)
    add("ctor_depth_16", S.header(64, 2, 12, depth=16) + good[16:], 64, 2, 14)
    for f in (8, 15):
        add("ctor_flags_%d" % f, S.header(64, 2, 12, flags=f) + good[16:], 64, 2)
    for (w, h) in ((0, 2), (64, 0), (24, 2), (6512, 2), (64, 4337), (65520, 65535)):
        add("ctor_dims_%d_%d" % (w, h), S.header(w, h, 12) + good[16:], 64, 2)
    add("ctor_exif_w", good, 48, 2)
    add("ctor_exif_h", good, 64, 3)
    add("ctor_header_only", good[:16], 64, 2)
    add("ctor_header_plus3", good[:19], 64, 2)
    return cases


def tall_cases():
    """Frames taller than a few row-start checkpoints (64 rows each) that fail at chosen rows: cuts at
    and around row ends (the end-of-row skip, the alignment skip past the end, fewer than 4 bytes at a
    row start, an over-read), a bad motion and a length underflow in the first row of a chunk and
    deeper.  -> [(name, (data, w, h, bits, cpp))]"""
    cases = []
    w, h = 48, 200
    full = natural(w, h, 12, 0, init=50, policy=4, seed=11)
    ends = row_ends(full, w, h)
    for r in (1, 2, 65, 66, 129, 130, 198):
        for d in (-1, 0, 1, 2):
            cases.append(("tall_cut_%d_%+d" % (r, d), (full[:16 + int(ends[r]) + d], w, h, 12, 1)))
        a = (int(ends[r]) + 15) // 16 * 16  # (the next row's start)
        for d in (0, 3, 4):
            cases.append(("tall_cut_%d_next_%d" % (r, d), (full[:16 + a + d], w, h, 12, 1)))
    for r in (66, 130, 199):
        cases.append(("tall_motion_%d" % r, (script(w, h, 12, 0, seed=r, motion=lambda y, k, r=r: 0 if (y, k) == (r, 0) else 7,
                                                    lens=lambda y, k: [(3, 3)] * 4), w, h, 12, 1)))
        cases.append(("tall_underflow_%d" % r, (script(w, h, 14, 0, seed=r + 1,
                                                       lens=lambda y, k, r=r: [(3, 0), 2 if (y, k) == (r, 1) else (3, 0), 1, 1]),
                                                w, h, 14, 1)))
    cases.append(("tall_ok", (full, w, h, 12, 1)))
    return cases


def test_tall_cases_fail_where_chosen():
    rows = {}
    for name, (data, w, h, bits, cpp) in tall_cases():
        _, rc, where, _ = S.decompress(data, w, h, bits, cpp)
        rows.setdefault(rc, set()).add((where >> 9) & 0x1FFF)
    assert {S.OK, S.OVERREAD, S.SHORT, S.BYTESTREAM, S.MOTION_BEGIN, S.UNDERFLOW} <= set(rows)
    for rc in (S.OVERREAD, S.SHORT, S.BYTESTREAM):
        assert max(rows[rc]) >= 66, rc
    assert {66, 130, 199} <= rows[S.MOTION_BEGIN] and {66, 130, 199} <= rows[S.UNDERFLOW]


def test_round_trip():
    for bits in (12, 14):
        for f in range(8):
            for pol in range(5):
                for w, h in [(16, 1), (48, 3), (80, 5), (208, 4)]:
                    for name, fn in S.CONTENT.items():
                        v = fn(w, h, bits, seed=w + h + pol)
                        data = S.encode(v, bits, f, init=1234, policy=pol, seed=f)
                        img, rc, _, msg = S.decompress(data, w, h, bits)
                        assert rc == S.OK, (bits, f, pol, w, h, name, msg)
                        assert np.array_equal(img, S.padded(v)), (bits, f, pol, w, h, name)


def test_golden_outcomes():
    with open(GOLDEN) as f:
        want = json.load(f)
    cases = dict(golden_cases())
    assert set(cases) == set(want)
    for name, (data, w, h, bits, cpp) in cases.items():
        img, rc, _, msg = S.decompress(data, w, h, bits, cpp)
        assert digest(msg, img) == want[name], name


def test_cases_reach_every_outcome():
    seen = set()
    for name, (data, w, h, bits, cpp) in golden_cases():
        seen.add(S.decompress(data, w, h, bits, cpp)[1])
    assert seen == set(range(15))


def test_rows_end_at_every_residue():
    seen = set()
    for name, (data, w, h, bits, cpp) in golden_cases():
        if name.startswith(("dims_", "flags_", "policy_")):
            ends = np.zeros(h, np.uint32)
            if S.decompress(data, w, h, bits, ends=ends)[1] == S.OK:
                seen |= {int(e) % 16 for e in ends}
    assert seen == set(range(16))


def test_messages_parse_back():
    for name, (data, w, h, bits, cpp) in golden_cases():
        _, rc, _, msg = S.decompress(data, w, h, bits, cpp)
        if rc != S.OK:
            assert S.message_id(msg) == rc, name
