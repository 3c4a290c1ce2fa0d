"""Samsung V1 on the CPU: the restatement of SamsungV1Decompressor in tests/emu/samsung1_oracle.c
against the outcomes of the reference's own decompressor (tests/golden/samsung_v1_ref.json,
recorded by tools/samsung1_ref_golden.py): the message thrown (which fixes the class) and the
whole padded image after the call.  Also the stream writer against the restatement, and the end
rule (fill(23): the first symbol that starts at or after T* fails) against a bit-level count."""
import hashlib
import json
import os

import numpy as np
import pytest

import samsung1_oracle as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "samsung_v1_ref.json")


def test_round_trip():
    for w, h in [(32, 2), (64, 4), (96, 6), (160, 10), (1024, 8), (5664, 2)]:
        for name, fn in S.CONTENT.items():
            v = fn(w, h, seed=w + h)
            img, rc, _ = S.decompress(S.make_stream(v), w, h)
            assert rc == S.OK, (w, h, name)
            assert np.array_equal(img, S.padded(v)), (w, h, name)


# ---------------------------------------------------------------- cases
def script(w, h, d):
    """A case from a raw difference script (h, w) in stream order."""
    return S.encode(np.asarray(d, np.int32).reshape(h, w)) + bytes(8)


def sym_case(L, sign, ext):
    """Every other column of row 0 .. 1 carries +-x, then -+x back: |x| = 2^(L-1) (min) or 2^L - 1
    (max).  From 0 for positive x, from 4095 for negative x; SSSS 13 leaves 0..4095 at once."""
    x = 0 if L == 0 else (1 << (L - 1) if ext == "min" else (1 << L) - 1)
    x *= sign
    w, h = 32, 2
    d = np.zeros((h, w), np.int32)
    base = 0 if sign > 0 else 4095
    d[:, 0:2] = base
    d[:, 2::4] = x
    d[:, 4::4] = -x
    return script(w, h, d), w, h, 12, 1


def oob_case(w, h, row, col, sign):
    """Natural content with a difference that takes pixel (row, col) just out of 0..4095."""
    v = S.natural_values(w, h, seed=row * 7 + col)
    d = S.diffs_of(v)
    d[row, col] += (4096 - int(v[row, col])) if sign > 0 else -(int(v[row, col]) + 1)
    return script(w, h, d), w, h, 12, 1


def chain_case(w, h, col, sign):
    """Columns 0 / 1 walk down the row - 2 chain (+-600 every second row) until they leave."""
    d = np.zeros((h, w), np.int32)
    d[0:2, 0:2] = 2048
    d[2:, col] = 600 * sign
    return script(w, h, d), w, h, 12, 1


def scratch_diff(data, i):
    """The difference the range decoder decodes for symbol i of `data` (zero bits behind the data)."""
    import ctypes as C
    d = np.zeros(i + 1, np.int16)
    st = np.zeros(i + 1, np.uint64)
    S.lib().s1_parse.argtypes = [C.c_char_p, C.c_uint32, C.c_int64, C.c_void_p, C.c_void_p]
    S.lib().s1_parse(bytes(data), len(data), i + 1, d.ctypes.data, st.ctypes.data)
    return int(d[i]), int(st[i])


def tie_cases(limit=3):
    """Cuts whose failing refill falls on a pixel that its decoded difference (zero bits: 000 0000 is
    -15) also takes out of 0..4095: columns 0 / 1 hold 5, the rest 4000, so the zero symbols behind
    the data end a row harmlessly and the failing one starts the next row from 5.  The refill wins."""
    w, h = 32, 8
    v = np.full((h, w), 4000, np.uint16)
    v[:, :2] = 5
    full = S.encode(S.diffs_of(v))
    out = []
    for n in range(4, len(full)):
        data = full[:n]
        img, rc, at = S.decompress(data, w, h)
        if rc != S.OVERREAD or (at & 0x3FFF) != 0 or (at >> 14) < 2 or n % 4 == 0:
            continue
        i = (at >> 14) * w
        d, start = scratch_diff(data, i)
        assert S.tstar(n) <= start < 8 * n + 74   # (the range decoder decodes it from zero bits)
        if not 0 <= int(img[(at >> 14) - 2, 0]) + d <= 4095:
            out.append((data, w, h, 12, 1))
        if len(out) == limit:
            break
    return out


def golden_cases():
    cases = []
    for k, c in enumerate(tie_cases()):
        cases.append(("tie_%d" % k, c))
    cases.append(("sym_L0", sym_case(0, 1, "min")))
    for L in range(1, 14):
        for sign, sn in ((1, "pos"), (-1, "neg")):
            for ext in ("min", "max") if L > 1 else ("min",):
                cases.append(("sym_L%d_%s_%s" % (L, sn, ext), sym_case(L, sign, ext)))
    for w, h in [(32, 2), (64, 2), (96, 4), (128, 2), (480, 4), (1024, 2), (2048, 2), (5664, 2)]:
        v = S.natural_values(w, h, seed=w)
        cases.append(("width_%d_%d" % (w, h), (S.make_stream(v), w, h, 12, 1)))
    w, h = 64, 6
    for sign, sn in ((1, "high"), (-1, "neg")):
        for where, (r, c) in {"first": (0, 0), "middle": (3, 29), "last": (h - 1, w - 1),
                              "col0_row2": (2, 0), "col1_row3": (3, 1), "col1_row0": (0, 1)}.items():
            cases.append(("oob_%s_%s" % (where, sn), oob_case(w, h, r, c, sign)))
        for col in (0, 1):
            cases.append(("chain_col%d_%s" % (col, sn), chain_case(32, 16, col, sign)))
    # cuts of the last bytes: T* = 32 floor((size + 8) / 4) + 10 moves by 32 bits every 4 bytes;
    # three contents put the symbol boundaries at other residues around it
    for seed, (w, h) in enumerate([(64, 4), (96, 2), (32, 8)]):
        full = S.encode(S.diffs_of(S.natural_values(w, h, seed=100 + seed)))
        for cut in range(0, 41):
            cases.append(("cut_%d_%02d" % (seed, cut), (full[:max(len(full) - cut, 0)], w, h, 12, 1)))
    flat = S.encode(S.diffs_of(S.flat_values(64, 4)))
    for cut in range(0, 24):
        cases.append(("cutflat_%02d" % cut, (flat[:len(flat) - cut], 64, 4, 12, 1)))
    for n in range(4):
        cases.append(("size_%d" % n, (bytes(range(0xA0, 0xA0 + n)), 32, 2, 12, 1)))
    rng = np.random.default_rng(5)
    for k in range(6):
        cases.append(("random_%d" % k, (rng.integers(0, 256, 64 + 37 * k, dtype=np.uint8).tobytes(),
                                        32 * (k + 1), 2, 12, 1)))
    ok = S.make_stream(S.natural_values(32, 2))
    for name, (w, h, bit, cpp) in {"dims_w0": (0, 2, 12, 1), "dims_h0": (32, 0, 12, 1),
                                   "dims_w33": (33, 2, 12, 1), "dims_w5696": (5696, 2, 12, 1),
                                   "dims_h3": (32, 3, 12, 1), "dims_h3716": (32, 3716, 12, 1),
                                   "bits_14": (32, 2, 14, 1), "bits_0": (32, 2, 0, 1),
                                   "bits_14_dims_w33": (33, 2, 14, 1), "cpp_2": (32, 2, 12, 2),
                                   "cpp_2_bits_14": (32, 2, 14, 2)}.items():
        cases.append((name, (ok, w, h, bit, cpp)))
    return cases


def digest(msg, img):
    """Outcome (message id) and the whole padded image after the call."""
    hh = hashlib.sha256(bytes([msg]))
    hh.update(np.ascontiguousarray(img).tobytes())
    return hh.hexdigest()


def test_oracle_matches_reference_outcomes():
    with open(GOLDEN) as f:
        want = json.load(f)
    cases = dict(golden_cases())
    assert set(cases) == set(want)
    for name, (data, w, h, bit, cpp) in cases.items():
        img, rc, _ = S.decompress(data, w, h, bit, cpp)
        assert digest(rc, img) == want[name], name


def test_cases_reach_every_outcome():
    seen = set()
    for name, (data, w, h, bit, cpp) in golden_cases():
        seen.add(S.decompress(data, w, h, bit, cpp)[1])
    assert seen == set(range(7))


def test_symbol_cases_decode_or_leave_range_as_built():
    for name, (data, w, h, bit, cpp) in golden_cases():
        if name.startswith("sym_"):
            L = int(name.split("_")[1][1:])
            assert S.decompress(data, w, h)[1] == (S.OOB if L == 13 else S.OK), name


@pytest.mark.parametrize("where", [(0, 0), (3, 29), (5, 63), (2, 0), (3, 1), (0, 1)])
@pytest.mark.parametrize("sign", [1, -1])
def test_violation_lands_where_placed(where, sign):
    data, w, h, _, _ = oob_case(64, 6, where[0], where[1], sign)
    _, rc, at = S.decompress(data, w, h)
    assert rc == S.OOB and at == (where[0] << 14 | where[1])


def parse_lengths(data, n):
    """Bit lengths of the first n symbols of `data` read as the reference reads it (zero bits behind)."""
    enc = []
    for el, dl in S.TAB:
        enc += [(el, dl)] * (1024 >> el)
    bits = np.unpackbits(np.frombuffer(bytes(data) + bytes(4 * n), np.uint8))
    out, p = [], 0
    for _ in range(n):
        c = int("".join(map(str, bits[p:p + 10])), 2)
        el, dl = enc[c]
        out.append(el + dl)
        p += el + dl
    return np.array(out, np.int64)


def _fail_index(lens, size, fill_bits):
    """Symbol index whose refill throws under fill(fill_bits) (None if all decode): refills before the
    symbol at bit T are ceil((T + fill_bits) / 32); refill (size + 8) // 4 + 2 throws."""
    starts = np.concatenate([[0], np.cumsum(lens)])[:-1]
    refills = (starts + fill_bits + 31) // 32
    bad = np.nonzero(refills >= (size + 8) // 4 + 2)[0]
    return int(bad[0]) if bad.size else None


def test_end_rule_is_tstar():
    """The cut cases fail exactly at the first symbol that starts at or after T*, and some of them at
    a symbol where a fill(32) pump would not have failed yet."""
    differs = 0
    for seed, (w, h) in enumerate([(64, 4), (96, 2), (32, 8)]):
        v = S.natural_values(w, h, seed=100 + seed)
        d = S.diffs_of(v).ravel()
        full = S.encode(d)
        for cut in range(0, 41):
            data = full[:len(full) - cut]
            img, rc, at = S.decompress(data, w, h)
            lens = parse_lengths(data, len(d))
            i23 = _fail_index(lens, len(data), 23)
            starts = np.concatenate([[0], np.cumsum(lens)])[:-1]
            first = np.nonzero(starts >= S.tstar(len(data)))[0]
            assert (int(first[0]) if first.size else None) == i23
            ends = starts + lens
            n = len(d) if i23 is None else i23
            got = img[:, :w].ravel()
            # symbols that end inside the data decode to their pixels; later ones read zero bits
            whole = ends[:n] <= 8 * len(data)
            assert np.array_equal(got[:n][whole], v.ravel()[:n][whole]), (seed, cut)
            assert np.all(got[n:] == S.FILL_DEFAULT), (seed, cut)
            if i23 is None:
                assert rc == S.OK
            else:
                assert rc == S.OVERREAD and at == ((i23 // w) << 14 | (i23 % w)), (seed, cut)
            differs += i23 != _fail_index(lens, len(data), 32)
    assert differs > 0


def test_tie_cases_exist():
    assert len(tie_cases()) == 3
