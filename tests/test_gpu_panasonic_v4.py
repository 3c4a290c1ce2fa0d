"""K7 / V4 parity: CUDA PanasonicV4 decode vs the oracle (pinned against the compiled reference
in tests/test_oracle_panasonic.py), through the C ABI and the C++ host mirror; bit-exact
pixels and the same set of bad (zero) pixel positions."""
import os

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
from oracle import port
from helpers import gpu_run
from test_pana4_emu import v4_payload

pytestmark = pytest.mark.gpu


def _job(w, h, size, split, zero_ok, in_offset=0, out_offset=0):
    j = rs.PanaJob()
    j.in_offset, j.in_size, j.out_offset = in_offset, size, out_offset
    j.out_pitch, j.width, j.height, j.version, j.bps = port.image_pitch(w), w, h, 4, 12
    j.zero_is_not_bad, j.section_split_offset = int(zero_ok), split
    return j


CASES = [(14, 1, 0, True), (28, 3, 0, False), (1400, 25, 0x1FF8, True), (2800, 13, 0x1FF8, False),
         (1414, 9, 0, False), (4200, 6, 0x2008, False), (1428, 11, 0x4000, False),
         (1428, 30, 0x1235, False), (5600, 12, 0x3FFF, False), (4592 // 14 * 14, 3448, 0x2008, False)]


@pytest.mark.parametrize("w,h,split,zero_ok", CASES)
def test_v4_abi_matches_oracle(ctx, w, h, split, zero_ok):
    data = v4_payload(w, h, split, w + h, zero_every=7 if h < 100 else 0)
    want = port.new_image(w, h)
    zwant = port.panasonic_v4(want, w, data, zero_ok, split, cap=1 << 22)
    plan = rs.pana_plan(ctx, [_job(w, h, data.size, split, zero_ok)])
    got, _ = gpu_run(plan, data, port.new_image(w, h))
    assert np.array_equal(got, want)
    n, pos = plan.bad_pixels(0, cap=1 << 22)
    assert n == len(zwant) and sorted(pos) == zwant


def test_v4_batch_with_other_versions_and_rerun(ctx):
    """Two V4 images (one collecting bad pixels) and a V5 image in one plan, odd input offsets;
    a second run gives the same list (the counters are reset per run)."""
    from test_oracle_panasonic import payload
    specs = [(4, 1400, 9, 0x2008, False), (5, 40, 30, 0, True), (4, 2800, 5, 0, True)]
    jobs, blobs, wants, zw = [], [], [], []
    pos, opos = 3, 0
    for k, (v, w, h, split, zero_ok) in enumerate(specs):
        if v == 4:
            d = v4_payload(w, h, split, 90 + k)
            j = _job(w, h, d.size, split, zero_ok, pos, opos)
            want = port.new_image(w, h)
            zw.append(port.panasonic_v4(want, w, d, zero_ok, split))
        else:
            d = payload(5, w, h, 12, 50)
            j = rs.PanaJob()
            j.in_offset, j.in_size, j.out_offset = pos, d.size, opos
            j.out_pitch, j.width, j.height, j.version, j.bps = port.image_pitch(w), w, h, 5, 12
            want = port.new_image(w, h)
            port.panasonic(5, want, w, d, 12)
            zw.append([])
        jobs.append(j)
        blobs.append((pos, d))
        wants.append((opos, want))
        pos += d.size + 5
        opos += (want.size * 2 + 255) // 256 * 256
    buf = np.zeros(pos + 16, dtype=np.uint8)
    for p, d in blobs:
        buf[p:p + d.size] = d
    out = np.full(opos // 2, 0xA5A5, dtype=np.uint16)
    plan = rs.pana_plan(ctx, jobs)
    for _ in range(2):
        got, _ = gpu_run(plan, buf, out)
        for (o, want), (v, w, *_), z in zip(wants, specs, zw):
            g = got[o // 2:o // 2 + want.size].reshape(want.shape)
            assert np.array_equal(g[:, :w], want[:, :w])
        for i, z in enumerate(zw):
            n, p = plan.bad_pixels(i)
            assert n == len(z) and sorted(p) == z


@pytest.mark.parametrize("w,h,split,zero_ok", CASES[:8])
def test_v4_host_mirror(w, h, split, zero_ok):
    data = v4_payload(w, h, split, w + h)
    want = port.new_image(w, h)
    zwant = port.panasonic_v4(want, w, data, zero_ok, split)
    got = port.new_image(w, h)
    zgot = host.panasonic_v4(got, w, data, zero_ok, split)
    assert np.array_equal(got[:, :w], want[:, :w])
    assert zgot == zwant
