"""K11 parity: bad-pixel interpolation on the GPU vs the oracle (pinned against the compiled
reference in tests/test_oracle_badpixels.py), through the C ABI on a device-resident image and
through the C++ host mirror's RawImageData::fixBadPixels()."""
import os

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
from oracle import port
from test_oracle_badpixels import scenarios, image, pos

pytestmark = pytest.mark.gpu

CPP1 = [k for k, s in enumerate(scenarios()) if s[3] == 1]


def _job(offset, img, w, cfa, first, n):
    j = rs.BadPixJob()
    j.offset, j.pitch, j.width, j.height = offset, img.shape[1] * 2, w, img.shape[0]
    j.is_cfa, j.first_position, j.num_positions, j.prior_map = int(cfa), first, n, None
    return j


@pytest.mark.parametrize("k", CPP1)
def test_abi_device_resident(ctx, k):
    import torch
    name, w, h, cpp, cfa, points = scenarios()[k]
    a = image(w, h, 1, k)
    want = a.copy()
    port.fix_bad_pixels(want, w, 1, pos(points), cfa)
    plan = rs.badpix_plan(ctx, [_job(0, a, w, cfa, 0, len(points))], pos(points))
    d = torch.from_numpy(a.view(np.int16).copy()).cuda()
    plan.run(None, d)
    torch.cuda.synchronize()
    assert np.array_equal(d.cpu().numpy().view(np.uint16), want)


@pytest.mark.parametrize("k", CPP1)
def test_host_mirror(k):
    name, w, h, cpp, cfa, points = scenarios()[k]
    a = image(w, h, 1, k)
    want = a.copy()
    port.fix_bad_pixels(want, w, 1, pos(points), cfa)
    host.fix_bad_pixels(a, w, 1, pos(points), cfa)
    assert np.array_equal(a[:, :w], want[:, :w])


def test_large_frame_sparse_defects(ctx):
    import torch
    w, h = 8256, 5504
    rng = np.random.default_rng(3)
    a = port.new_image(w, h)
    a[:, :] = rng.integers(0, 16384, size=a.shape, dtype=np.uint16)
    n = 20000
    p = ((rng.integers(0, h, n).astype(np.uint32) << 16) | rng.integers(0, w, n).astype(np.uint32))
    want = a.copy()
    port.fix_bad_pixels(want, w, 1, p, True)
    plan = rs.badpix_plan(ctx, [_job(0, a, w, True, 0, n)], p)
    d = torch.from_numpy(a.view(np.int16).copy()).cuda()
    plan.run(None, d)
    torch.cuda.synchronize()
    assert np.array_equal(d.cpu().numpy().view(np.uint16), want)
