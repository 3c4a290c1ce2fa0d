"""Samsung V1 on the GPU (rsb200_samsung1_plan_create: the multi-CTA range decoder with the LUT-only
table, samsung1.cuh's reconstruction and end-of-stream scan) against the CPU restatement of
SamsungV1Decompressor (tests/emu/samsung1_oracle.c, pinned against the reference's outcomes): the
whole output buffer with sentinels around every job, status and the reported pixel, through the C
ABI and through the host mirror SamsungV1Decompressor."""
import ctypes as C

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
import samsung1_oracle as S
import test_oracle_samsung1 as T

pytestmark = pytest.mark.gpu

FILL = S.FILL_DEFAULT
GAP = 32  # sentinel pixels before every job and behind the last


def run_frames(ctx, frames, in_skews=None):
    """frames: [(data bytes, w, h)] -> ([image], [(status, consumed)], [redo flag]); asserts that the
    sentinels around every job's output are untouched."""
    import torch
    blob, jobs, outs, off = bytearray(), [], [], 0
    for k, (data, w, h) in enumerate(frames):
        skew = 0 if in_skews is None else in_skews[k]
        blob += bytes((-len(blob)) % 16 + skew)
        j = rs.SamsungV1Job()
        j.in_offset, j.in_size = len(blob), len(data)
        blob += data
        j.bits, j.width, j.height = 12, w, h
        pitch = S.pitch_elems(w)
        off += GAP
        j.out_offset, j.out_pitch = off * 2, pitch * 2
        outs.append((off, h, pitch))
        off += pitch * h
        jobs.append(j)
    off += GAP
    plan = rs.samsung1_plan(ctx, jobs)
    d_in = torch.from_numpy(np.frombuffer(bytes(blob) + b"\x5a" * 64, np.uint8).copy()).cuda()
    out = torch.full((off,), FILL, dtype=torch.int32).to(torch.int16).cuda()
    plan.run((d_in.data_ptr(), len(blob)), out)
    torch.cuda.synchronize()
    res = plan.results(check=False)
    f = plan.ctx._lib.rsb200_debug_range_redo
    f.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_int]
    arr = (C.c_uint32 * plan.nunits)()
    plan.ctx.check(f(plan.h, arr, plan.nunits))
    o = out.cpu().numpy().view(np.uint16)
    imgs, seen = [], np.zeros(off, bool)
    for p, h, pitch in outs:
        imgs.append(o[p:p + h * pitch].reshape(h, pitch))
        seen[p:p + h * pitch] = True
    assert np.all(o[~seen] == FILL), "a store outside the jobs' images"
    return imgs, res, list(arr)


def host_run(data, w, h, bit=12, cpp=1):
    """SamsungV1Decompressor(img, data, bit).decompress() through the host mirror -> (image, outcome)."""
    img = np.full((max(h, 1), S.pitch_elems(max(w, 1) * cpp)), FILL, np.uint16)
    try:
        host.samsung_v1(img, w, np.frombuffer(bytes(data), np.uint8).copy(), bit, cpp)
        return img, S.OK
    except (rs.RawDecoderException, rs.IOException) as e:
        mid = S.message_id(str(e))
        assert isinstance(e, rs.RawDecoderException) == (mid in S.RDE_MSGS)
        return img, mid


def expect(data, w, h):
    """-> (image, status, consumed) the plan must report."""
    want, rc, where = S.decompress(data, w, h, fill=FILL)
    st = {S.OK: 0, S.OOB: 1, S.OVERREAD: 2, S.SHORT: 2}[rc]
    cons = (0x80000000 | where) if rc == S.OOB else (where if rc == S.OVERREAD else 0)
    return want, st, cons, rc


def check(ctx, frames, in_skews=None, mirror=True):
    imgs, res, redo = run_frames(ctx, frames, in_skews)
    for k, ((data, w, h), img, got) in enumerate(zip(frames, imgs, res)):
        want, st, cons, rc = expect(data, w, h)
        assert got == (st, cons), (k, got, st, cons)
        assert np.array_equal(img, want), k
        if mirror:
            himg, hrc = host_run(data, w, h)
            assert hrc == rc and np.array_equal(himg, want), k
    return res, redo


def decodable_cases():
    return [(n, (d, w, h)) for n, (d, w, h, bit, cpp) in T.golden_cases()
            if bit == 12 and cpp == 1 and w > 0 and h > 0 and w % 32 == 0 and h % 2 == 0
            and w <= 5664 and h <= 3714]


def test_golden_cases_through_mirror(ctx):
    """Every pinned case, one plan each, through the host mirror and the C ABI."""
    for name, fr in decodable_cases():
        check(ctx, [fr])


@pytest.mark.parametrize("skew", range(16))
def test_golden_cases_every_alignment(ctx, skew):
    """All pinned cases in one plan, every input at in_offset & 15 == skew."""
    frames = [fr for _, fr in decodable_cases()]
    check(ctx, frames, [skew] * len(frames), mirror=False)


def test_outcomes_reached():
    seen = {expect(d, w, h)[3] for _, (d, w, h) in decodable_cases()}
    assert seen == {S.OK, S.OOB, S.OVERREAD, S.SHORT}


def test_random_payloads_several_per_plan(ctx):
    rng = np.random.default_rng(11)
    frames = []
    for k in range(24):
        w, h = 32 * int(rng.integers(1, 12)), 2 * int(rng.integers(1, 8))
        n = int(rng.integers(0, w * h * 2))
        frames.append((rng.integers(0, 256, n, dtype=np.uint8).tobytes(), w, h))
    check(ctx, frames, [int(x) for x in rng.integers(0, 16, len(frames))], mirror=False)


def test_natural_frames_and_cuts_several_per_plan(ctx):
    frames = []
    for k, (w, h) in enumerate([(5664, 16), (2048, 64), (640, 480), (96, 2)]):
        v = S.natural_values(w, h, seed=k)
        data = S.make_stream(v)
        frames += [(data, w, h), (data[:len(data) * 3 // 4], w, h)]
    res, redo = check(ctx, frames, [3 * k % 16 for k in range(len(frames))])
    assert [r[0] for r in res[0::2]] == [0] * 4


@pytest.mark.parametrize("content", sorted(S.CONTENT))
def test_full_size_not_redone(ctx, content):
    """5664 x 3714 frames (two per plan) decode exactly and no range seam fails."""
    w, h = 5664, 3714
    frames = [(S.make_stream(S.CONTENT[content](w, h, seed=s)), w, h) for s in (1, 2)]
    res, redo = check(ctx, frames, [0, 5], mirror=(content == "natural"))
    assert [r[0] for r in res] == [0, 0]
    assert redo == [0, 0], (content, redo)


def test_clipped_band_longer_than_halo(ctx):
    """Rows of 4095 over far more than a range's 8 KiB halo: zero differences, code 110100."""
    w, h = 5664, 512
    v = S.natural_values(w, h, seed=4)
    v[100:400, :] = 4095
    data = S.make_stream(v)
    assert len(S.encode(np.zeros(w * 300, np.int32))) > 8 * 8192
    res, redo = check(ctx, [(data, w, h)])
    assert res[0][0] == 0 and redo == [0]


def test_forced_redo_periodic_run_is_exact(ctx):
    """Every difference +1 (code 11011 + one bit: 110111 repeated): speculative starts on a wrong
    residue never resynchronise, a seam fails and the exact single-CTA decoder redoes the frame."""
    w, h = 5664, 512
    d = np.ones((h, w), np.int32)
    data = S.encode(d) + bytes(8)
    res, redo = check(ctx, [(data, w, h), (data[:len(data) // 2], w, h)])
    assert res[0][0] == 0 and res[1][0] == 2
    assert redo[0] == 1


@pytest.mark.parametrize("w,h,bit,msg", [(0, 2, 12, S.DIMS), (32, 0, 12, S.DIMS), (33, 2, 12, S.DIMS),
                                         (5696, 2, 12, S.DIMS), (32, 3, 12, S.DIMS),
                                         (32, 3716, 12, S.DIMS), (32, 2, 14, S.BITS),
                                         (33, 2, 14, S.BITS)])
def test_constructor_rejections(ctx, w, h, bit, msg):
    j = rs.SamsungV1Job()
    j.in_offset, j.in_size, j.bits, j.width, j.height = 0, 64, bit, w, h
    j.out_offset, j.out_pitch = 0, max(2 * w, 4) + 16
    with pytest.raises(rs.RawDecoderException) as e:
        rs.samsung1_plan(ctx, [j])
    assert S.message_id(e.value.msg) == msg
    if w > 0 and h > 0:
        _, hrc = host_run(bytes(64), w, h, bit)
        assert hrc == msg


def test_mirror_component_check(ctx):
    img, hrc = host_run(S.make_stream(S.natural_values(32, 2)), 32, 2, cpp=2)
    assert hrc == S.CPP and np.all(img == FILL)


@pytest.mark.parametrize("field,value", [("out_offset", 2), ("out_pitch", 130), ("out_pitch", 60),
                                         ("in_size", 1 << 28), ("reserved", 1)])
def test_refused_layout(ctx, field, value):
    j = rs.SamsungV1Job()
    j.in_offset, j.in_size, j.bits, j.width, j.height = 0, 64, 12, 32, 2
    j.out_offset, j.out_pitch = 0, 128
    setattr(j, field, value)
    with pytest.raises(rs.Rsb200Error) as e:
        rs.samsung1_plan(ctx, [j])
    assert e.value.code == 4   # RSB200_ERR_ARG


def test_mid_size_clipped_not_redone(ctx):
    """The 3008x2000 clipped band, the slowest class of tools/samsung_v1_time.py: exact, no redo."""
    w, h = 3008, 2000
    frames = [(S.make_stream(S.clipped_values(w, h, seed=1)), w, h)]
    res, redo = check(ctx, frames, mirror=False)
    assert res[0][0] == 0 and redo == [0]


def test_more_frames_than_a_grid_dimension(ctx):
    """65537 frames in one plan (the row kernels put every frame's CTAs along one grid dimension)."""
    import torch
    w, h, n = 32, 2, 65537
    data = S.make_stream(S.natural_values(w, h, seed=5))
    want, rc, _ = S.decompress(data, w, h, fill=FILL)
    assert rc == S.OK
    pitch = S.pitch_elems(w)
    jobs = (rs.SamsungV1Job * n)()
    for k in range(n):
        j = jobs[k]
        j.in_offset, j.in_size, j.bits, j.width, j.height = 0, len(data), 12, w, h
        j.out_offset, j.out_pitch = k * pitch * h * 2, pitch * 2
    plan = rs.samsung1_plan(ctx, list(jobs))
    d_in = torch.from_numpy(np.frombuffer(data + bytes(64), np.uint8).copy()).cuda()
    out = torch.full((n * pitch * h,), FILL, dtype=torch.int32).to(torch.int16).cuda()
    plan.run((d_in.data_ptr(), len(data)), out)
    torch.cuda.synchronize()
    assert set(plan.results()) == {(0, 0)}
    o = out.cpu().numpy().view(np.uint16).reshape(n, h, pitch)
    assert np.array_equal(o, np.broadcast_to(want, o.shape))
