"""Samsung V2 on the GPU (rsb200_samsung2_plan_create, samsung2.cuh) against the CPU restatement of
SamsungV2Decompressor (tests/emu/samsung2_oracle.c, pinned against the reference's outcomes): the
whole output buffer with sentinels around every job, status and `consumed`, through the C ABI and
through the host mirror SamsungV2Decompressor, whose message text must be the reference's."""
import re

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
import samsung2_oracle as S
import test_oracle_samsung2 as T

pytestmark = pytest.mark.gpu

FILL = S.FILL_DEFAULT
GAP = 32  # sentinel pixels before every job and behind the last


def make_job(data, w, h, bits, in_offset, out_offset, pitch):
    j = rs.SamsungV2Job()
    j.in_offset, j.in_size, j.bits, j.width, j.height = in_offset, len(data), bits, w, h
    for i, b in enumerate(bytes(data[:16]).ljust(16, b"\0")):
        j.header[i] = b
    j.out_offset, j.out_pitch = out_offset, pitch
    return j


def run_frames(ctx, frames, in_skews=None):
    """frames: [(data, w, h, bits)] -> ([image], [(status, consumed)]); asserts that the sentinels
    around every job's output are untouched."""
    import torch
    blob, jobs, outs, off = bytearray(), [], [], 0
    for k, (data, w, h, bits) in enumerate(frames):
        skew = 0 if in_skews is None else in_skews[k]
        blob += bytes((-len(blob)) % 16 + skew)
        pitch = S.pitch_elems(w)
        off += GAP
        jobs.append(make_job(data, w, h, bits, len(blob), off * 2, pitch * 2))
        blob += data
        outs.append((off, h, pitch))
        off += pitch * h
    off += GAP
    plan = rs.samsung2_plan(ctx, jobs)
    d_in = torch.from_numpy(np.frombuffer(bytes(blob) + b"\x5a" * 64, np.uint8).copy()).cuda()
    out = torch.full((off,), FILL, dtype=torch.int32).to(torch.int16).cuda()
    plan.run((d_in.data_ptr(), len(blob)), out)
    torch.cuda.synchronize()
    res = plan.results(check=False)
    o = out.cpu().numpy().view(np.uint16)
    imgs, seen = [], np.zeros(off, bool)
    for p, h, pitch in outs:
        imgs.append(o[p:p + h * pitch].reshape(h, pitch))
        seen[p:p + h * pitch] = True
    assert np.all(o[~seen] == FILL), "a store outside the jobs' images"
    return imgs, res


def host_run(data, w, h, bits=12, cpp=1):
    """SamsungV2Decompressor(img, data, bits).decompress() through the host mirror -> (image, message)."""
    img = np.full((max(h, 1), S.pitch_elems(max(w, 1) * cpp)), FILL, np.uint16)
    try:
        host.samsung_v2(img, w, np.frombuffer(bytes(data), np.uint8).copy(), bits, cpp)
        return img, ""
    except (rs.RawDecoderException, rs.IOException) as e:
        text = re.sub(r"^rsb200 error -?[0-9]+: ", "", str(e))
        assert isinstance(e, rs.IOException) == (S.message_id(text) in S.IOE_MSGS), text
        return img, text


def rejected(data, rc):
    """Whether the constructor rejects the case (a strip under 16 bytes fails its bs.check(16))."""
    return rc >= S.CPP or len(data) < 16


def decodes(data, w, h, bits):
    """Whether the constructor accepts the case (the plan runs it)."""
    return not rejected(data, S.decompress(data, w, h, bits)[1])


def check(ctx, frames, in_skews=None, mirror=True):
    imgs, res = run_frames(ctx, frames, in_skews)
    for k, ((data, w, h, bits), img, got) in enumerate(zip(frames, imgs, res)):
        want, rc, where, msg = S.decompress(data, w, h, bits, fill=FILL)
        st = 0 if rc == S.OK else (2 if rc in S.IOE_MSGS else 1)
        assert got == (st, S.consumed(rc, where)), (k, got, rc, where)
        assert np.array_equal(img, want), k
        if mirror:
            himg, text = host_run(data, w, h, bits)
            assert text == msg and np.array_equal(himg, want), (k, text, msg)


def pinned():
    return [(d, w, h, bits) for _, (d, w, h, bits, cpp) in T.golden_cases() if cpp == 1 and decodes(d, w, h, bits)]


def test_golden_cases_through_mirror(ctx):
    """Every pinned case the constructor accepts, one plan each, through the C ABI and the host mirror."""
    for fr in pinned():
        check(ctx, [fr])


@pytest.mark.parametrize("skew", range(16))
def test_golden_cases_every_alignment(ctx, skew):
    """All pinned cases in one plan (mixed outcomes), every strip at in_offset & 15 == skew."""
    frames = pinned()
    check(ctx, frames, [skew] * len(frames), mirror=False)


def test_random_payloads_several_per_plan(ctx):
    rng = np.random.default_rng(17)
    frames = []
    for k in range(40):
        w, h, bits = 16 * int(rng.integers(1, 20)), int(rng.integers(1, 9)), (12, 14)[k % 2]
        if k % 3 == 0:
            v = S.random_values(w, h, bits, seed=k)
            data = S.encode(v, bits, int(rng.integers(0, 8)), int(rng.integers(0, 1 << bits)), int(k % 5), k)
            data = data[:len(data) - int(rng.integers(0, 24))]
        else:
            data = S.header(w, h, bits, int(rng.integers(0, 8)), int(rng.integers(0, 1 << 14))) + \
                rng.integers(0, 256, int(rng.integers(0, 64 * w)), dtype=np.uint8).tobytes()
        frames.append((data, w, h, bits))
    check(ctx, frames)


@pytest.mark.parametrize("dims", [(6496, 4336), (5472, 3648)])
@pytest.mark.parametrize("bits", [12, 14])
@pytest.mark.parametrize("content", ["natural", "up", "average", "flat"])
def test_full_frames(ctx, dims, bits, content):
    w, h = dims
    pol = {"natural": 0, "up": 2, "average": 3, "flat": 1}[content]
    fn = S.flat_values if content == "flat" else S.natural_values
    v = fn(w, h, bits, seed=w + bits)
    data = S.encode(v, bits, S.SKIP if content == "flat" else 0, 77, pol, seed=bits)
    imgs, res = run_frames(ctx, [(data, w, h, bits)])
    assert res[0] == (0, 0)
    assert np.array_equal(imgs[0], S.padded(v))


def test_failure_in_a_full_frame(ctx):
    """A frame cut in its middle: rows before the failing one, and the failing row's blocks, as the
    restatement leaves them."""
    w, h = 2048, 600
    v = S.natural_values(w, h, 12, seed=3)
    data = S.encode(v, 12, 0, 5, 0, seed=3)
    check(ctx, [(data[:len(data) // 2 + 5], w, h, 12)], mirror=True)


def test_tall_frames_failing_past_checkpoints(ctx):
    """Frames of 200 rows failing at chosen rows past the first row-start checkpoints: cuts at and
    around row ends (end-of-row skip, alignment skip past the end, a short pump, over-reads), a bad
    motion and a length underflow in row 66 (the first row of the second chunk) and deeper; one plan,
    then each through the host mirror."""
    frames = [(d, w, h, bits) for _, (d, w, h, bits, _) in T.tall_cases()]
    check(ctx, frames, [3] * len(frames), mirror=False)
    for fr in frames:
        check(ctx, [fr])


def test_mirror_with_long_data_behind_the_frame(ctx):
    """More data behind a frame than it can read (the host mirror hands the plan no more than that)
    decodes as the restatement does."""
    for w, h in ((16, 2), (64, 5)):
        data = T.natural(w, h, 12, 0, init=3, policy=4, seed=w) + bytes(range(256)) * 400
        want, rc, _, msg = S.decompress(data, w, h, 12, fill=FILL)
        img, text = host_run(data, w, h, 12)
        assert rc == S.OK and text == msg and np.array_equal(img, want)


def test_more_than_65535_frames(ctx):
    base = [S.encode(S.random_values(16, 2, 12, seed=i), 12, i % 8, i, i % 5, i) for i in range(7)]
    frames = [(base[i % 7], 16, 2, 12) for i in range(65537)]
    frames[40000] = (base[0][:20], 16, 2, 12)
    imgs, res = run_frames(ctx, frames)
    for k in list(range(0, 65537, 997)) + [40000, 65536]:
        data, w, h, bits = frames[k]
        want, rc, where, _ = S.decompress(data, w, h, bits, fill=FILL)
        assert res[k] == (0 if rc == S.OK else (2 if rc in S.IOE_MSGS else 1), S.consumed(rc, where)), k
        assert np.array_equal(imgs[k], want), k


def test_refused_layouts(ctx):
    data = S.encode(S.natural_values(64, 2), 12, 0, 0, 0)
    for kw in ({"out_offset": 2}, {"out_pitch": 130}, {"out_pitch": 64}, {"reserved": 1},
               {"in_size": 1 << 28}):
        j = make_job(data, 64, 2, 12, 0, 0, 128)
        for k, val in kw.items():
            setattr(j, k, val)
        with pytest.raises(rs.Rsb200Error):
            rs.samsung2_plan(ctx, [j])


def test_constructor_rejections(ctx):
    """The constructor's rejections: plan creation fails with the reference's class and message, and
    the host mirror throws it."""
    for name, (data, w, h, bits, cpp) in T.golden_cases():
        _, rc, _, msg = S.decompress(data, w, h, bits, cpp)
        if not rejected(data, rc):
            continue
        img, text = host_run(data, w, h, bits, cpp)
        assert text == msg, (name, text, msg)
        if cpp == 1 and w > 0 and h > 0:
            exc = rs.IOException if rc in S.IOE_MSGS else rs.RawDecoderException
            with pytest.raises(exc) as e:
                rs.samsung2_plan(ctx, [make_job(data, w, h, bits, 0, 0, S.pitch_elems(w) * 2)])
            assert msg in str(e.value), (name, str(e.value))
