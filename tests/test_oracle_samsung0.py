"""Samsung V0 on the CPU: the restatement of SamsungV0Decompressor in tests/emu/samsung0_oracle.c
against the outcomes of the reference's own decompressor (tests/golden/samsung_v0_ref.json,
recorded by tools/samsung0_ref_golden.py): the message thrown (which fixes the class) and the
whole padded image after the call.  Also the stream writer against the restatement."""
import hashlib
import json
import os

import numpy as np
import pytest

import samsung0_oracle as S


def test_round_trip_every_mode():
    for w, h in [(16, 1), (17, 2), (31, 3), (40, 7), (100, 20), (333, 41)]:
        for name, fn in S.DIRS.items():
            v = S.natural_values(w, h, seed=w + h)
            bso, bsr, _ = S.make_frame(v, fn(w, h))
            img, rc, _ = S.decompress(bso, bsr, w, h)
            assert rc == S.OK, (w, h, name)
            assert np.array_equal(img, S.swap_rb(v, S.pitch_elems(w))), (w, h, name)


def test_round_trip_staircase_full_size():
    w, h = 5546, 3714
    v = S.natural_values(w, h, seed=3)
    bso, bsr, _ = S.make_frame(v, S.dirs_staircase(w, h))
    img, rc, _ = S.decompress(bso, bsr, w, h)
    assert rc == S.OK and np.array_equal(img, S.swap_rb(v, S.pitch_elems(w)))


# ---------------------------------------------------------------- cases
def script(w, h, seed, dirs=None):
    """A valid frame's stream choices: (dirs, op, setlen, adj), each per row and block."""
    v = S.natural_values(w, h, seed)
    d = S.dirs_random(w, h, seed) if dirs is None else dirs
    op, setlen, adj = S.fit(v, d)
    return d.copy(), op, setlen, adj


def frame(d, op, setlen, adj, first=0):
    rows = S.write_rows(d, op, setlen, adj)
    bso, bsr = S.pack(rows, first)
    return bso, bsr


def length_walk(w, h, seed):
    """Every op on every group, lengths walking 0 <-> 16 (set, step down to 0, step up to 16), with
    random values of each length."""
    rng = np.random.default_rng(seed)
    nb = S.nblocks(w)
    d = np.zeros((h, nb), np.uint8)
    op = np.zeros((h, nb, 4), np.uint8)
    setlen = np.zeros((h, nb, 4), np.uint8)
    for r in range(h):
        for i in range(4):
            L = 7 if r < 2 else 4
            phase = (r + i) % 3
            for k in range(nb):
                if phase == 0:      # down to 0, then set 15 and up to 16
                    q = 2 if L > 0 else 3
                elif phase == 1:    # up to 16, then set 0 and keep
                    q = 1 if L < 16 else 3
                else:
                    q = int(rng.integers(0, 4))
                    if (q == 2 and L == 0) or (q == 1 and L == 16):
                        q = 0
                s = int(rng.integers(0, 16)) if q == 3 else 0
                if q == 3 and phase == 0:
                    s = 15
                if q == 3 and phase == 1:
                    s = 0
                op[r, k, i] = q
                setlen[r, k, i] = s
                L = s if q == 3 else L + (1 if q == 1 else (-1 if q == 2 else 0))
    up = S._up_allowed(w, h) & (rng.random((h, nb)) < 0.4)
    d[up] = 1
    adj = rng.integers(-40000, 40000, (h, nb, 16)).astype(np.int32)
    return frame(d, op, setlen, adj)


def violation(w, h, kind, row, k, seed=0):
    """A valid frame with the first RawDecoderException of `kind` at (row, block k)."""
    d, op, setlen, adj = script(w, h, seed)
    if kind == S.LEN_NEG:          # block k - 1 sets length 0, block k steps down
        op[row, k - 1, 0], setlen[row, k - 1, 0] = 3, 0
        op[row, k, 0] = 2
    elif kind == S.LEN_BIG:        # set 15, step to 16, step to 17
        op[row, k - 2, 3], setlen[row, k - 2, 3] = 3, 15
        op[row, k - 1, 3] = 1
        op[row, k, 3] = 1
    else:                          # UP_FIRST (row < 2) / UP_LAST (last block)
        d[row, k] = 1
    return frame(d, op, setlen, adj)


def golden_cases():
    """(name, (bso, bsr, w, h)) for every case pinned against the reference."""
    widths = [16, 17, 31, 32] + [48 + m for m in range(16)]
    for w in widths:
        for h in (1, 2, 3, 6, 7):
            d, op, setlen, adj = script(w, h, seed=w * 7 + h)
            yield "size_%dx%d" % (w, h), frame(d, op, setlen, adj) + (w, h)
    for name, fn in S.DIRS.items():
        for w, h in [(100, 21), (64, 10), (333, 40)]:
            v = S.natural_values(w, h, seed=w + h)
            yield "mode_%s_%dx%d" % (name, w, h), S.make_frame(v, fn(w, h))[:2] + (w, h)
    for seed in range(4):
        yield "lengths_%d" % seed, length_walk(77, 9, seed) + (77, 9)
    w, h = 70, 9
    nb = S.nblocks(w)
    for kind, rows, blocks in [(S.LEN_NEG, (0, 4, h - 1), (1, 2, nb - 1)),
                               (S.LEN_BIG, (0, 4, h - 1), (2, 3, nb - 1)),
                               (S.UP_FIRST, (0, 1), (0, 2, nb - 1)),
                               (S.UP_LAST, (2, 4, h - 1), (nb - 1,))]:
        for r in rows:
            for k in blocks:
                yield "viol_%d_r%d_b%d" % (kind, r, k), violation(w, h, kind, r, k, seed=r + k) + (w, h)
    # cuts of one row's stream: from "the row fits" down past the 8-byte rule, and 1..3 bytes
    w, h = 40, 6
    d, op, setlen, adj = script(w, h, seed=11)
    rows = S.write_rows(d, op, setlen, adj)
    for r in (0, 3, h - 1):
        for n in range(len(rows[r]) + 1, 0, -1):
            rr = list(rows)
            rr[r] = (rows[r] + b"\x5a" * 4)[:n]
            yield "cut_r%d_%d" % (r, n), S.pack(rr) + (w, h)
    # offsets: equal, decreasing, past bsr, the first one past bsr, short bso
    base = S.pack(rows)
    offs = np.frombuffer(base[0], "<u4").astype(np.int64)
    for tag, r, val in [("equal", 2, None), ("decr", 3, -5), ("past", 4, 10 ** 6), ("first_past", 0, 10 ** 6),
                        ("first_end", 0, len(base[1])), ("last_end", h - 1, len(base[1]))]:
        o = offs.copy()
        o[r] = o[r - 1] if val is None else (o[r] + val if val < 0 else val)
        yield "offsets_%s" % tag, (o.astype("<u4").tobytes(), base[1], w, h)
    yield "offsets_first_skip", S.pack(rows, first=13) + (w, h)
    for n in (0, 3, 4 * h - 1):
        yield "short_bso_%d" % n, (base[0][:n], base[1], w, h)
    for w2, h2 in [(15, 4), (0, 4), (16, 0), (5547, 2), (16, 3715)]:
        yield "ctor_%dx%d" % (w2, h2), (base[0], base[1], w2, h2)


def digest(msg, img):
    """Outcome (message id) and the whole padded image after the call."""
    hh = hashlib.sha256(bytes([msg]))
    hh.update(np.ascontiguousarray(img).tobytes())
    return hh.hexdigest()


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "samsung_v0_ref.json")


def test_oracle_matches_reference_outcomes():
    with open(GOLDEN) as f:
        want = json.load(f)
    cases = dict(golden_cases())
    assert set(cases) == set(want)
    for name, (bso, bsr, w, h) in cases.items():
        img, rc, _ = S.decompress(bso, bsr, w, h)
        assert digest(rc, img) == want[name], name


def test_cases_reach_every_outcome():
    seen = set()
    for name, (bso, bsr, w, h) in golden_cases():
        seen.add(S.decompress(bso, bsr, w, h)[1])
    assert seen == set(range(11))


@pytest.mark.parametrize("kind", [S.LEN_NEG, S.LEN_BIG, S.UP_FIRST, S.UP_LAST])
def test_violation_lands_where_placed(kind):
    w, h = 70, 9
    nb = S.nblocks(w)
    r, k = (0 if kind == S.UP_FIRST else 3), (nb - 1 if kind == S.UP_LAST else 2)
    bso, bsr = violation(w, h, kind, r, k)
    _, rc, where = S.decompress(bso, bsr, w, h)
    assert rc == kind and where == (r << 9 | k)
