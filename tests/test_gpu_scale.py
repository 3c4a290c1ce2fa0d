"""K9 parity: CUDA black/white scaling vs the oracle (pinned against the compiled reference in
tests/test_oracle_scale.py), through the C ABI (device-resident, in place) and through the
C++ host mirror's RawImageData::scaleBlackWhite(); bit-exact, dither included."""
import os

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
from rawspeed_b200._abi import SCALE_AUTO, SCALE_PLAIN, SCALE_SSE2
from oracle import port

pytestmark = pytest.mark.gpu


def _job(offset, img, w, h, cpp, crop, black, white, dither=True, path=SCALE_AUTO):
    j = rs.ScaleJob()
    j.offset, j.pitch, j.width, j.height, j.cpp = offset, img.shape[1] * 2, w, h, cpp
    j.crop_x, j.crop_y, j.crop_w, j.crop_h = crop
    for i in range(4):
        j.black_separate[i] = black[i]
    j.white_point, j.dither, j.path = white, int(dither), path
    return j


def _image(w, h, cpp, seed, lo=0, hi=65536):
    rng = np.random.default_rng(seed)
    a = port.new_image(w, h, cpp)
    a[:, :] = rng.integers(lo, hi, size=a.shape, dtype=np.uint16)
    return a


def _run_in_place(plan, img):
    import torch
    d = torch.from_numpy(img.view(np.int16).copy()).cuda()
    plan.run(None, d)
    torch.cuda.synchronize()
    assert plan.results()[0][0] == 0
    return d.cpu().numpy().view(np.uint16)


CASES = [
    (64, 16, 1, (0, 0, 64, 16), (256, 256, 256, 256), 16383),
    (70, 11, 1, (3, 1, 61, 9), (60, 64, 68, 72), 4095),
    (37, 9, 1, (2, 3, 30, 5), (1000, 1010, 990, 1024), 15000),
    (1000, 6, 1, (8, 0, 980, 6), (512, 512, 512, 512), 16383),
    (33, 7, 1, (5, 2, 20, 4), (100, 200, 300, 400), 1023),
    (530, 9, 1, (11, 2, 515, 6), (10, 20, 30, 40), 900),
    (40, 10, 3, (2, 1, 30, 8), (100, 100, 100, 100), 15000),
    (40, 10, 3, (3, 1, 30, 8), (100, 100, 100, 100), 900),
    (8256, 37, 1, (8, 1, 8240, 35), (1008, 1010, 1009, 1011), 16383),
]


@pytest.mark.parametrize("path", [SCALE_AUTO, SCALE_SSE2, SCALE_PLAIN])
@pytest.mark.parametrize("dither", [True, False])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_scale_matches_oracle(ctx, case, dither, path):
    w, h, cpp, crop, black, white = CASES[case]
    a = _image(w, h, cpp, 40 + case)
    want = a.copy()
    sse2 = None if path == SCALE_AUTO else path == SCALE_SSE2
    port.scale_black_white(want, w, crop, black_sep=list(black), white=white, dither=dither,
                           sse2=sse2, cpp=cpp, is_cfa=cpp == 1)
    plan = rs.scale_plan(ctx, [_job(0, a, w, h, cpp, crop, black, white, dither, path)])
    assert plan.launches == 1
    got = _run_in_place(plan, a)
    assert np.array_equal(got, want)


def test_batch_of_images_both_loops(ctx):
    specs = [(64, 13, (1, 1, 60, 11), (256,) * 4, 16383), (48, 9, (3, 0, 40, 9), (64,) * 4, 1023),
             (96, 6, (0, 2, 96, 3), (10, 20, 30, 40), 4095)]
    imgs = [_image(w, h, 1, 7 + i) for i, (w, h, *_) in enumerate(specs)]
    sizes = [(im.nbytes + 255) // 256 * 256 for im in imgs]
    buf = np.zeros(sum(sizes) // 2, dtype=np.uint16)
    jobs, offs = [], []
    o = 0
    for im, sz, (w, h, crop, black, white) in zip(imgs, sizes, specs):
        buf[o // 2:o // 2 + im.size] = im.reshape(-1)
        jobs.append(_job(o, im, w, h, 1, crop, black, white))
        offs.append(o)
        o += sz
    plan = rs.scale_plan(ctx, jobs)
    assert plan.launches == 2
    got = _run_in_place(plan, buf)
    for im, o, (w, h, crop, black, white) in zip(imgs, offs, specs):
        want = im.copy()
        port.scale_values(want, w, crop, black, white)
        assert np.array_equal(got[o // 2:o // 2 + im.size].reshape(im.shape), want)


def test_decode_then_scale_stays_on_the_device(ctx):
    """The use the kernel exists for: a packed frame is unpacked and scaled without leaving HBM."""
    import torch
    w, h, bps = 4000, 64, 12
    rng = np.random.default_rng(3)
    packed = rng.integers(0, 256, size=h * w * bps // 8, dtype=np.uint8)
    want = port.new_image(w, h)
    port.unpack(packed, want, w, 1, (0, 0, w, h), w * bps // 8, bps, rs.MSB)
    port.scale_values(want, w, (0, 0, w, h), (256, 256, 256, 256), 4095)
    uj = rs.UnpackJob()
    uj.in_offset, uj.in_size, uj.out_offset, uj.out_pitch = 0, packed.size, 0, port.image_pitch(w)
    uj.row0, uj.rows, uj.samples, uj.out_col0 = 0, h, w, 0
    uj.in_pitch, uj.bps, uj.order = w * bps // 8, bps, rs.MSB
    up = rs.unpack_plan(ctx, [uj])
    a = port.new_image(w, h)
    sp = rs.scale_plan(ctx, [_job(0, a, w, h, 1, (0, 0, w, h), (256,) * 4, 4095)])
    d_in = torch.from_numpy(packed).cuda()
    d_img = torch.from_numpy(a.view(np.int16).copy()).cuda()
    up.run(d_in, d_img)
    sp.run(None, d_img)
    torch.cuda.synchronize()
    assert np.array_equal(d_img.cpu().numpy().view(np.uint16), want)


@pytest.mark.parametrize("kw", [
    dict(white=15000, areas=[(1, 0, 16)]),
    dict(black_level=500, white=15000),
    dict(black_sep=[500, 510, 505, 515], white=15000, dither=False),
    dict(black_level=0, white=65535),                      # nothing to do
    dict(black_sep=[64, 64, 64, 64], white=1000),          # plain loop
])
def test_host_mirror_scale_black_white(kw):
    rng = np.random.default_rng(11)
    w, h, crop = 96, 40, (16, 8, 80, 32)
    a = port.new_image(w, h)
    a[:, :] = rng.integers(400, 15000, size=a.shape, dtype=np.uint16)
    a[:, :16] = 512
    want = a.copy()
    r_want = port.scale_black_white(want, w, crop, **kw)
    r_got = host.scale_black_white(a, w, crop, **kw)
    assert r_got == r_want
    assert np.array_equal(a[:, :w], want[:, :w])
