"""K12 parity: whole-image table lookup on the GPU vs the oracle (pinned against the compiled
reference in tests/test_oracle_lookup.py), through the C ABI on a device-resident image and
through the C++ host mirror's RawImageData::sixteenBitLookup()."""
import os

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
from oracle import port, synth
from test_oracle_lookup import CASES, image, curve

pytestmark = pytest.mark.gpu


def _job(offset, img, w, cpp, table=0):
    j = rs.LookupJob()
    j.offset, j.pitch, j.width, j.height, j.cpp, j.table = offset, img.shape[1] * 2, w, img.shape[0], cpp, table
    return j


@pytest.mark.parametrize("dither", [False, True])
@pytest.mark.parametrize("k", range(len(CASES)))
def test_abi_device_resident(ctx, k, dither):
    import torch
    w, h, cpp, crop, ncurve = CASES[k]
    a = image(w, h, cpp, k)
    want = a.copy()
    t = port.build_table(curve(ncurve, 10 + k), dither)
    port.sixteen_bit_lookup(want, w, cpp, t, dither)
    plan = rs.lookup_plan(ctx, [_job(0, a, w, cpp)], t, dither)
    d = torch.from_numpy(a.view(np.int16).copy()).cuda()
    plan.run(None, d)
    torch.cuda.synchronize()
    assert np.array_equal(d.cpu().numpy().view(np.uint16), want)
    assert plan.launches == 1


@pytest.mark.parametrize("dither", [False, True])
@pytest.mark.parametrize("k", range(len(CASES)))
def test_host_mirror(k, dither):
    w, h, cpp, crop, ncurve = CASES[k]
    a = image(w, h, cpp, k)
    want = a.copy()
    cv = curve(ncurve, 10 + k)
    port.sixteen_bit_lookup(want, w, cpp, port.build_table(cv, dither), dither)
    host.sixteen_bit_lookup(a, w, cpp, cv, dither)
    assert np.array_equal(a[:, :w * cpp], want[:, :w * cpp])


def test_full_frame_sony_curve_dithered(ctx):
    import torch
    w, h = 8256, 5504
    a = image(w, h, 1, 5, 4096 * 2)
    want = a.copy()
    t = port.build_table(synth.sony_curve(), True)
    port.sixteen_bit_lookup(want, w, 1, t, True)
    plan = rs.lookup_plan(ctx, [_job(0, a, w, 1)], t, True)
    d = torch.from_numpy(a.view(np.int16).copy()).cuda()
    plan.run(None, d)
    torch.cuda.synchronize()
    assert np.array_equal(d.cpu().numpy().view(np.uint16), want)
