"""K10 parity: the fused DNG opcode pass on the GPU vs the oracle (pinned against the compiled
reference in tests/test_oracle_dngopcodes.py): through the C++ host mirror's
DngOpcodes(ri, bs).applyOpCodes(ri) (pixels, crop, mBadPixelPositions in order, error class and
stage) and through the C ABI with a device-resident image."""
import os

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
from oracle import port
from test_oracle_dngopcodes import scenarios

pytestmark = pytest.mark.gpu


def _oracle(img, w, cpp, crop, blob):
    want = img.copy()
    try:
        crop2, bad = port.dng_opcodes(want, w, cpp, crop, blob)
        return want, crop2, bad, None
    except Exception as ex:   # noqa: BLE001
        return want, port.dng_opcodes.partial[0], port.dng_opcodes.partial[1], ex


@pytest.mark.parametrize("k", range(9))
def test_host_mirror_apply_opcodes(k):
    name, img, w, cpp, crop, blob = scenarios()[k]
    want, wcrop, wbad, werr = _oracle(img, w, cpp, crop, blob)
    got = img.copy()
    try:
        gcrop, gbad = host.dng_opcodes(got, w, cpp, crop, blob)
        gerr = None
    except Exception as ex:   # noqa: BLE001
        gerr = ex
        gcrop, gbad = host.dng_opcodes.partial
        assert host.dng_opcodes.stage == 2
    assert np.array_equal(got, want)
    assert gcrop == wcrop and gbad == wbad
    assert (gerr is None) == (werr is None)
    if werr is not None:
        assert type(gerr).__name__ == type(werr).__name__


@pytest.mark.parametrize("k", [0, 1, 2, 3, 6])
def test_abi_device_resident(ctx, k):
    """The list lowered by the mirror, run through rsb200_dngop_plan_create on an image that
    stays in HBM; two images in one plan (the second a copy at another offset)."""
    import torch
    name, img, w, cpp, crop, blob = scenarios()[k]
    want, _, _, _ = _oracle(img, w, cpp, crop, blob)
    low = host.dngop_lower(img, w, cpp, crop, blob)
    nbytes = (img.nbytes + 255) // 256 * 256
    jobs, ops = [], []
    for f in range(2):
        j = rs.DngOpJob()
        j.offset, j.pitch, j.width, j.height = f * nbytes, img.shape[1] * img.itemsize, w, img.shape[0]
        j.cpp, j.is_f32, j.first_op, j.num_ops = cpp, int(img.dtype == np.uint32), len(ops), len(low["ops"])
        jobs.append(j)
        ops += [rs.DngOp.from_buffer_copy(o) for o in low["ops"]]
    plan = rs.dngop_plan(ctx, jobs, ops, low["tables"], low["deltas"])
    buf = np.zeros(2 * nbytes, dtype=np.uint8)
    for f in range(2):
        buf[f * nbytes:f * nbytes + img.nbytes] = img.reshape(-1).view(np.uint8)
    d = torch.from_numpy(buf).cuda()
    plan.run(None, d)
    torch.cuda.synchronize()
    got = d.cpu().numpy()
    for f in range(2):
        g = got[f * nbytes:f * nbytes + img.nbytes].view(img.dtype).reshape(img.shape)
        assert np.array_equal(g, want)
    assert plan.launches == 1


def test_large_image_many_opcodes(ctx):
    """A 4000 x 3000 frame with eight opcodes: one pass, bit-exact."""
    import torch
    from oracle import synth as S
    w, h = 4000, 3000
    rng = np.random.default_rng(1)
    img = port.new_image(w, h)
    img[:, :] = rng.integers(0, 65536, size=img.shape, dtype=np.uint16)
    area = S.dng_pixel_area((0, 0, h, w))
    blob = S.dng_opcode_list([
        S.dng_delta(12, area, (rng.random(h, dtype=np.float32) + 0.5)),
        S.dng_delta(13, S.dng_pixel_area((0, 0, h, w), 0, 1, 1, 2), (rng.random(w // 2, dtype=np.float32) + 0.5)),
        S.dng_delta(10, S.dng_pixel_area((1, 1, h, w), 0, 1, 2, 2), (rng.random(h // 2, dtype=np.float32) - 0.5) * 0.01),
        S.dng_delta(11, area, (rng.random(w, dtype=np.float32) - 0.5) * 0.01),
        S.dng_map_polynomial(area, [0.0, 0.8, 0.3, -0.1]),
        S.dng_map_table(S.dng_pixel_area((0, 1, h, w), 0, 1, 2, 2), (np.arange(65536) ^ 1).astype(np.uint16)),
        S.dng_fix_bad_constant(65535),
        S.dng_delta(13, S.dng_pixel_area((8, 8, h - 8, w - 8), 0, 1, 1, 16), rng.random((w - 16 + 15) // 16, dtype=np.float32) + 0.25),
    ])
    want = img.copy()
    wcrop, wbad = port.dng_opcodes(want, w, 1, [0, 0, w, h], blob, cap=1 << 22)
    got = img.copy()
    gcrop, gbad = host.dng_opcodes(got, w, 1, [0, 0, w, h], blob, cap=1 << 22)
    assert np.array_equal(got, want) and gcrop == wcrop and gbad == wbad
