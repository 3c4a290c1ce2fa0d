"""Samsung V0 on the GPU (rsb200_samsung0_plan_create, samsung0.cuh) against the CPU restatement of
SamsungV0Decompressor (tests/emu/samsung0_oracle.c, pinned against the reference's outcomes): the
whole output buffer byte for byte with sentinel bytes around every job, status and the failing row and
block, through the C ABI and through the host mirror SamsungV0Decompressor."""
import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
import samsung0_oracle as S
import test_oracle_samsung0 as T
from test_samsung0_emu import expect, golden_decodable, strips_of

pytestmark = pytest.mark.gpu

GAP = 48  # sentinel bytes before, between and after the jobs' images


def run_plan(ctx, frames, skews=None, shuffle_seed=None):
    """frames: [(bso, bsr, w, h)] with valid offset tables.  Each frame's rows go to the input at
    in_offset & 15 == skews[i] (default 0), in row order or (shuffle_seed) in a random order with random
    gaps.  -> (whole output buffer, expected buffer, results, plan)."""
    import torch
    rng = np.random.default_rng(shuffle_seed)
    blob = bytearray()
    jobs, strips = [], []
    out_off = GAP
    want = []
    for i, (bso, bsr, w, h) in enumerate(frames):
        rows = strips_of(bso, bsr, h)
        blob += bytes((-len(blob)) % 16 + (0 if skews is None else skews[i]))
        first = len(strips)
        if shuffle_seed is None:
            base = len(blob)
            blob += bsr
            strips += [(base + o, n) for o, n in rows]
        else:
            at = [0] * h
            for r in rng.permutation(h):
                blob += bytes(int(rng.integers(0, 7)))
                at[r] = len(blob)
                o, n = rows[r]
                blob += bsr[o:o + n]
            strips += [(at[r], rows[r][1]) for r in range(h)]
        j = rs.SamsungV0Job()
        pitch = S.pitch_elems(w) * 2
        j.out_offset, j.out_pitch, j.width, j.height, j.first_strip = out_off, pitch, w, h, first
        jobs.append(j)
        img, rc, where = S.decompress(bso, bsr, w, h)
        want.append((out_off, img, expect(rc, where)))
        out_off += pitch * h + GAP
    sa = []
    for o, n in strips:
        s = rs.SamsungV0Strip()
        s.in_offset, s.in_size = o, n
        sa.append(s)
    plan = rs.samsung0_plan(ctx, jobs, sa)
    exp = np.full(out_off // 2, S.FILL_DEFAULT, np.uint16)
    for off, img, _ in want:
        exp[off // 2: off // 2 + img.size] = img.ravel()
    d_in = torch.from_numpy(np.frombuffer(bytes(blob) + b"\x5a" * 64, np.uint8).copy()).cuda()
    out = torch.from_numpy(np.full(out_off // 2, S.FILL_DEFAULT, np.uint16).view(np.int16)).cuda()
    plan.run((d_in.data_ptr(), len(blob)), out)
    torch.cuda.synchronize()
    res = plan.results(check=False)
    got = out.cpu().numpy().view(np.uint16)
    return got, exp, res, [r for _, _, r in want]


def assert_same(got, exp):
    if not np.array_equal(got, exp):
        i = int(np.nonzero(got != exp)[0][0])
        raise AssertionError("first differing byte at %d: %#06x != %#06x" % (2 * i, got[i], exp[i]))


def check(ctx, frames, skews=None, shuffle_seed=None, mirror=True):
    got, exp, res, want = run_plan(ctx, frames, skews, shuffle_seed)
    assert res == want
    assert_same(got, exp)
    if mirror:
        for bso, bsr, w, h in frames:
            host_check(bso, bsr, w, h)
    return res


def host_check(bso, bsr, w, h):
    """SamsungV0Decompressor(img, bso, bsr).decompress() through the host mirror."""
    want, rc, _ = S.decompress(bso, bsr, w, h)
    img = np.full((h, S.pitch_elems(w)), S.FILL_DEFAULT, np.uint16)
    try:
        host.samsung_v0(img, w, bso, bsr)
        assert rc == S.OK
    except rs.RawDecoderException as e:
        assert rc in S.RDE_MSGS and S.MESSAGES[rc] in e.msg, (rc, e.msg)
    except rs.IOException as e:
        assert rc not in S.RDE_MSGS and rc != S.OK and S.MESSAGES[rc] in e.msg, (rc, e.msg)
    assert np.array_equal(img, want)


@pytest.mark.parametrize("chunk", range(4))
def test_golden_cases(ctx, chunk):
    """Every decodable case pinned against the reference: sizes, modes, lengths 0..16 with every op,
    each RawDecoderException at the first, a middle and the last block and row, strip cuts across the
    8-byte rule and strips of 1..3 bytes; 12 frames per plan at every in_offset & 15."""
    cases = [c for i, (_, c) in enumerate(golden_decodable()) if i % 4 == chunk]
    for i in range(0, len(cases), 12):
        part = cases[i:i + 12]
        check(ctx, part, skews=[(i + k) % 16 for k in range(len(part))])


def test_constructor_errors_host_mirror():
    for name, (bso, bsr, w, h) in T.golden_cases():
        if S.decompress(bso, bsr, w, h)[1] in S.CTOR_MSGS and w > 0 and h > 0:
            host_check(bso, bsr, w, h)


@pytest.mark.parametrize("w,h", [(15, 4), (5547, 2), (16, 3715), (16, 0), (0, 4)])
def test_constructor_dimensions_refused(ctx, w, h):
    j = rs.SamsungV0Job()
    j.out_pitch, j.width, j.height = 2 * 5600, w, h
    s = rs.SamsungV0Strip()
    s.in_size = 64
    with pytest.raises(rs.RawDecoderException, match="Unexpected image dimensions found"):
        rs.samsung0_plan(ctx, [j], [s] * max(h, 1))


@pytest.mark.parametrize("field,value", [("out_offset", 3), ("out_pitch", 99), ("out_pitch", 62),
                                         ("first_strip", 1)])
def test_refused_layout(ctx, field, value):
    """An odd out_offset or out_pitch, a pitch below the row, strips outside the array: never launched."""
    j = rs.SamsungV0Job()
    j.out_offset, j.out_pitch, j.width, j.height = 0, 64, 32, 2
    setattr(j, field, value)
    s = rs.SamsungV0Strip()
    s.in_size = 64
    with pytest.raises(rs.Rsb200Error) as e:
        rs.samsung0_plan(ctx, [j], [s, s])
    assert e.value.code == 4   # RSB200_ERR_ARG


def test_shuffled_strips_every_skew(ctx):
    frames = []
    for k in range(16):
        w, h = 40 + 37 * k, 3 + 5 * k
        v = S.natural_values(w, h, seed=k)
        mode = sorted(S.DIRS)[k % 4]
        bso, bsr, _ = S.make_frame(v, S.DIRS[mode](w, h))
        frames.append((bso, bsr, w, h))
    check(ctx, frames, skews=list(range(16)), shuffle_seed=5, mirror=False)


@pytest.mark.parametrize("seed", range(3))
def test_random_payloads(ctx, seed):
    rng = np.random.default_rng(100 + seed)
    cases = []
    for _ in range(6):
        w, h = int(rng.integers(16, 600)), int(rng.integers(1, 90))
        cases.append(T.length_walk(w, h, int(rng.integers(1 << 30))) + (w, h))
        d, op, setlen, adj = T.script(w, h, int(rng.integers(1 << 30)))
        rows = S.write_rows(d, op, setlen, adj)
        r = int(rng.integers(0, h))
        rows[r] = rng.integers(0, 256, len(rows[r]), dtype=np.uint8).tobytes()
        cases.append(S.pack(rows) + (w, h))
    check(ctx, cases, skews=[int(x) for x in rng.integers(0, 16, len(cases))])


def test_full_size_frames(ctx):
    """5546 x 3714 (the constructor's limit): staircase (the deepest chains), all up, all left."""
    w, h = 5546, 3714
    frames = []
    for k, mode in enumerate(["staircase", "up", "left"]):
        v = S.natural_values(w, h, seed=20 + k)
        bso, bsr, _ = S.make_frame(v, S.DIRS[mode](w, h))
        frames.append((bso, bsr, w, h))
    res = check(ctx, frames, skews=[0, 5, 11], mirror=False)
    assert res == [(0, 0)] * 3
    host_check(*frames[0])


def test_plan_reports_bytes_and_kernels(ctx):
    w, h = 100, 21
    v = S.natural_values(w, h, seed=1)
    bso, bsr, _ = S.make_frame(v, S.dirs_staircase(w, h))
    j = rs.SamsungV0Job()
    j.out_pitch, j.width, j.height = S.pitch_elems(w) * 2, w, h
    sa = []
    for o, n in strips_of(bso, bsr, h):
        s = rs.SamsungV0Strip()
        s.in_offset, s.in_size = o, n
        sa.append(s)
    plan = rs.samsung0_plan(ctx, [j], sa)
    assert plan.bytes() == (len(bsr), 2 * w * h, w * h)
    assert "s0_jump_kernel" in plan.kernels
