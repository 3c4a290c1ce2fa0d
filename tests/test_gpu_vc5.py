"""GoPro VC-5 on the GPU (rsb200_vc5_plan_create, vc5.cuh) against the CPU restatement of
VC5Decompressor (tests/emu/vc5_oracle.c, pinned against the reference's outcomes): the whole output
buffer with sentinels around every job, status and `consumed`, on every golden case the tag walk
accepts, mixed batches, every ABI-legal output alignment, GoPro-sized frames, and the refusals."""
import numpy as np
import pytest

import rawspeed_b200 as rs
import test_oracle_vc5 as T
import vc5_oracle as V

pytestmark = pytest.mark.gpu


def gpu_run(ctx, frames, skew=0, pitch_extra=0, gap=32, codes=None):
    """-> ([image], [(status, consumed)], plan launches) of one plan over `frames`; asserts that
    everything outside the jobs' images is untouched."""
    import torch
    blob, jobs, bands, outs, total = V.plan_inputs(frames, skew, pitch_extra, gap)
    plan = rs.vc5_plan(ctx, V.codebook() if codes is None else codes, jobs, bands)
    d_in = torch.from_numpy(np.frombuffer(blob + b"\x5a" * 64, np.uint8).copy()).cuda()
    out = torch.from_numpy(np.full(total, V.FILL_DEFAULT, np.uint16).view(np.int16)).cuda()
    plan.run((d_in.data_ptr(), len(blob)), out)
    torch.cuda.synchronize()
    res = plan.results(check=False)
    launches = plan.launches
    plan.close()
    o = out.cpu().numpy().view(np.uint16)
    imgs, seen = [], np.zeros(total, bool)
    for off, h, pitch in outs:
        imgs.append(o[off:off + h * pitch].reshape(h, pitch))
        seen[off:off + h * pitch] = True
    assert np.all(o[~seen] == V.FILL_DEFAULT), "a store outside the jobs' images"
    return imgs, res, launches


def check(ctx, frames, **kw):
    imgs, res, _ = gpu_run(ctx, frames, **kw)
    want = V.expected(frames, pitch_extra=kw.get("pitch_extra", 0))
    for k, ((wimg, wres), img, got) in enumerate(zip(want, imgs, res)):
        assert tuple(got) == wres, (k, got, wres)
        assert np.array_equal(img, wimg), k


def accepted():
    return [(n, c) for n, c in T.golden_cases() if V.parse(*c)[0] == V.OK]


def test_golden_cases(ctx):
    for name, case in accepted():
        check(ctx, [case])


@pytest.mark.parametrize("skew,pitch_extra,gap", [(0, 0, 32), (1, 2, 34), (2, 4, 36), (3, 6, 38), (5, 2, 40)])
def test_golden_cases_one_plan(ctx, skew, pitch_extra, gap):
    """All accepted cases in one plan (different dims, phases, depths; failing jobs next to good ones), every
    payload at in_offset & 15 == skew, images at every 4-byte-aligned offset and pitch."""
    frames = [c for n, c in accepted() if not n.startswith("bits_")] + [accepted()[0][1]]
    check(ctx, frames, skew=skew, pitch_extra=pitch_extra, gap=gap)


def frame(w, h, kind, seed):
    content = {"natural": lambda: V.natural(w, h, seed=seed),
               "noise": lambda: V.noise(w, h, seed=seed, top=40),
               "flat": lambda: V.flat(w, h, 900 + seed)}[kind]()
    return (V.encode(w, h, content, prescale=T.PS2), w, h, 4095, V.RGGB if seed % 2 == 0 else V.GBRG)


def test_gopro_frame(ctx):
    """One 4000x3000 frame: many segments per band, bit-exact."""
    check(ctx, [frame(4000, 3000, "natural", 0)])


def test_batch_of_16(ctx):
    """16 frames of mixed sizes and content in one plan; two of them fail."""
    frames = []
    for i in range(16):
        w, h = ((4000, 3000), (1280, 962), (2048, 1536), (998, 674))[i % 4]
        frames.append(frame(w, h, ("natural", "flat", "noise")[i % 3], i))
    frames[5] = T.failing_block(176, 160, {(1, 4): V.OVERREAD}), 176, 160, 4095, V.RGGB
    frames[11] = T.failing_block(46, 38, {(3, 9): V.QUANT, (0, 2): V.NO_END}), 46, 38, 4095, V.RGGB
    check(ctx, frames)


def test_launches_do_not_grow_with_frames(ctx):
    one = frame(640, 480, "natural", 1)
    _, _, l1 = gpu_run(ctx, [one])
    _, _, l8 = gpu_run(ctx, [one] * 8)
    assert l1 == l8


def refused(ctx, frames=None, codes=None, mutate=None):
    blob, jobs, bands, outs, total = V.plan_inputs(frames or [frame(64, 48, "natural", 3)])
    if mutate:
        mutate(jobs, bands)
    with pytest.raises(rs.Rsb200Error) as e:
        rs.vc5_plan(ctx, V.codebook() if codes is None else codes, jobs, bands)
    return e


def test_refusals(ctx):
    cb = V.codebook()
    for bad in (cb[:-1],                                          # incomplete
                np.concatenate([cb[:-1], cb[-2:-1]]),             # a code twice
                np.where(np.arange(len(cb))[:, None] == 0, [27, 0, 1, 0], cb),  # length 27
                cb * np.array([1, 1, 0, 1]) + np.array([0, 0, 512, 0]),          # count 512
                np.where(np.arange(len(cb))[:, None] == 3, cb + [0, 0, 0, 300], cb)):  # value > 255
        refused(ctx, codes=np.ascontiguousarray(bad, np.int64))

    def job(field, value):
        return lambda jobs, bands: setattr(jobs[0], field, value)

    for m in (job("width", 32), job("height", 30), job("width", 63), job("output_bits", 0), job("output_bits", 17),
              job("phase", 1), job("out_offset", 66), job("out_pitch", 126), job("out_pitch", 98),
              job("reserved", 1), job("first_band", 1)):
        refused(ctx, mutate=m)

    def prescale(jobs, bands):
        jobs[0].prescale[2][1] = 4

    def band(i, field, value):
        return lambda jobs, bands: setattr(bands[i], field, value)

    for m in (prescale, band(3, "in_size", 6), band(3, "in_size", (1 << 28) + 4), band(3, "param", 40000),
              band(0, "param", 7), band(0, "param", 17), band(10, "in_size", 8)):
        refused(ctx, mutate=m)
    # the smallest accepted image: 34 x 34
    check(ctx, [frame(34, 34, "natural", 4)])


def test_host_mirror_route(ctx):
    """rsb200h_vc5: every golden case (constructor rejections included) through the host mirror, whose
    text, exception class and image are the reference's; the smallest images the plan refuses excepted."""
    from test_host_vc5 import host_run
    for name, (data, w, h, white, cfa) in T.golden_cases():
        if w <= 0 or h <= 0:
            continue
        want, rc, args = V.decompress(data, w, h, white, cfa)
        img, text, ioe = host_run(data, w, h, white, cfa)
        assert text == V.message(rc, args), (name, text)
        assert ioe == V.is_ioe(rc), name
        assert np.array_equal(img, want[:h]), name
    # a 4000x3000 frame
    data, w, h, white, cfa = frame(4000, 3000, "natural", 2)
    want, rc, _ = V.decompress(data, w, h, white, cfa)
    img, text, _ = host_run(data, w, h, white, cfa)
    assert rc == V.OK and text == "" and np.array_equal(img, want[:h])
