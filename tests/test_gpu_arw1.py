"""Sony ARW1 on the GPU (rsb200_arw1_plan_create: complemented copy, the multi-CTA range decoder,
arw1.cuh's frame-wide scan) against the CPU restatement of SonyArw1Decompressor
(tests/emu/arw1_oracle.c, pinned against the reference's outcomes): pixels of the whole padded
buffer, status and the reported pixel, through the C ABI and through the host mirror
SonyArw1Decompressor."""
import ctypes as C

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
import arw1_oracle as A

pytestmark = pytest.mark.gpu

FILL = 0xABCD


def run_frames(ctx, frames, in_skews=None):
    """frames: [(data bytes, w, h)] -> ([image], [(status, consumed)], [redo flag])."""
    import torch
    blob, jobs, outs, off_out = bytearray(), [], [], 0
    for k, (data, w, h) in enumerate(frames):
        skew = 0 if in_skews is None else in_skews[k]
        blob += bytes((-len(blob)) % 16 + skew)
        j = rs.Arw1Job()
        j.in_offset, j.in_size = len(blob), len(data)
        blob += data
        j.width, j.height = w, h
        pitch = A.pitch_elems(w)
        j.out_offset, j.out_pitch = off_out, pitch * 2
        off_out += pitch * 2 * h
        jobs.append(j)
        outs.append((h, pitch))
    plan = rs.arw1_plan(ctx, jobs)
    d_in = torch.from_numpy(np.frombuffer(bytes(blob) + b"\x5a" * 64, np.uint8).copy()).cuda()
    out = torch.full((off_out // 2 + 64,), FILL, dtype=torch.int32).to(torch.int16).cuda()
    plan.run((d_in.data_ptr(), len(blob)), out)
    torch.cuda.synchronize()
    res = plan.results(check=False)
    f = plan.ctx._lib.rsb200_debug_range_redo
    f.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_int]
    arr = (C.c_uint32 * plan.nunits)()
    plan.ctx.check(f(plan.h, arr, plan.nunits))
    o = out.cpu().numpy().view(np.uint16)
    imgs, p = [], 0
    for h, pitch in outs:
        imgs.append(o[p:p + h * pitch].reshape(h, pitch))
        p += h * pitch
    return imgs, res, list(arr)


def host_run(data, w, h):
    """SonyArw1Decompressor(img).decompress(data) through the host mirror -> (image, status)."""
    img = np.full((h, A.pitch_elems(w)), FILL, np.uint16)
    try:
        host.arw1_decompress(img, w, np.frombuffer(bytes(data), np.uint8).copy())
        return img, A.OK
    except rs.RawDecoderException:
        return img, A.RDE
    except rs.IOException:
        return img, A.IOE


def check(ctx, frames, in_skews=None, mirror=True):
    imgs, res, redo = run_frames(ctx, frames, in_skews)
    for (data, w, h), img, (st, cons) in zip(frames, imgs, res):
        want, rc, where = A.decompress(data, w, h, fill=FILL)
        assert st == rc, (st, rc)
        if rc == A.RDE:
            assert cons == 0x80000000 | where
        assert np.array_equal(img, want)
        if mirror:
            got, hrc = host_run(data, w, h)
            assert hrc == rc and np.array_equal(got, want)
    return res, redo


@pytest.mark.parametrize("w,h", [(1, 2), (3, 2), (17, 6), (640, 480)])
def test_sizes(ctx, w, h):
    res, redo = check(ctx, [(A.encode_frame(A.natural_frame(w, h, w + h)), w, h)])
    assert res[0][0] == 0 and redo == [0]


def test_every_length(ctx):
    w, h = 5, 8
    for first_long in range(13, 18):
        d = [0]
        for ln in range(1, 13):
            v = (1 << (ln - 1)) + 1 if ln > 1 else 1
            d += [v, -v]
        v = (1 << (first_long - 1)) + 1
        d += [v, -v, 7]
        d += [0] * (w * h - len(d))
        res, _ = check(ctx, [(A.encode(np.array(d[:w * h])), w, h)])
        assert res[0][0] == A.RDE


def test_len17_small_mod_2_16(ctx):
    """65541 = 5 mod 2^16: a length-17 difference is a violation, never a small step."""
    w, h = 4, 4
    for d0 in (65541, 65536, -65540, 70000, 32768 + 5):
        d = np.zeros(w * h, np.int32)
        d[0] = 100
        d[5] = d0
        res, _ = check(ctx, [(A.encode(d), w, h)])
        assert res[0][0] == A.RDE


@pytest.mark.parametrize("half,col,sign", [(0, "first", -1), (0, "last", 1), (1, "first", 1),
                                           (1, "last", -1), (0, "mid", 1), (1, "mid", -1)])
def test_first_violation(ctx, half, col, sign):
    """The first violation in stream order is reported; a later one must not win."""
    w, h = 70, 130
    f = A.natural_frame(w, h, 3).astype(np.int64)
    c = {"first": w - 1, "last": 0, "mid": 33}[col]   # stream order starts at the right
    r = 2 * 17 + half
    d = A.frame_diffs(f).astype(np.int64)
    row, cc = A.stream_rows_cols(w, h)
    i = int(np.nonzero((row == r) & (cc == c))[0][0])
    d[i] += sign * 5000
    d[min(i + 40, d.size - 1)] += -sign * 9000       # a later violation (never reached)
    res, _ = check(ctx, [(A.encode(d), w, h)])
    assert res[0] == (A.RDE, 0x80000000 | (r << 14) | c)


@pytest.mark.parametrize("trailing", [False, True])
def test_cuts(ctx, trailing):
    """Streams cut by 0..40 bytes, with and without bytes behind in_size; violation before and
    after the over-read."""
    w, h = 24, 10
    f = A.natural_frame(w, h, 7)
    full = A.encode_frame(f)
    d = A.frame_diffs(f)
    d2 = d.copy()
    d2[-3] += 6000                                      # a violation near the end
    viol = A.encode(d2)
    frames = []
    for cut in range(41):
        for s in (full, viol):
            frames.append((s[:max(len(s) - cut, 0)], w, h))
    skews = [(k * 5) % 16 for k in range(len(frames))]
    if trailing:   # the next frame's bytes follow each cut stream in the buffer
        check(ctx, frames, skews, mirror=False)
    else:          # one frame per plan: only padding behind the stream (and the host mirror)
        for k, fr in enumerate(frames):
            check(ctx, [fr], [skews[k]])


@pytest.mark.parametrize("fill", [0x00, 0xFF])
def test_constant_streams(ctx, fill):
    check(ctx, [(bytes([fill]) * n, 6, 4) for n in (0, 1, 7, 64, 4096)])


@pytest.mark.parametrize("w,h", [(0, 2), (4, 0), (4, 3), (4601, 2), (4, 3074)])
def test_constructor_rejects(ctx, w, h):
    j = rs.Arw1Job()
    j.in_size, j.width, j.height, j.out_pitch = 16, w, h, 2 * max(w, 1)
    with pytest.raises(rs.RawDecoderException, match="Unexpected image dimensions"):
        rs.arw1_plan(ctx, [j])


def test_two_frames_every_offset(ctx):
    a = A.encode_frame(A.natural_frame(300, 64, 1))
    b = A.encode_frame(A.natural_frame(129, 38, 2))
    for s in range(16):
        check(ctx, [(a, 300, 64), (b, 129, 38)], [s, (s * 7) % 16])


DSLR = (3872, 2592)


@pytest.mark.parametrize("kind", ["natural", "uniform", "uniform4095", "clipped8", "clipped12",
                                  "clipped13", "clipped14"])
def test_dslr_frames(ctx, kind):
    """Flat areas (runs of zero differences, which never resynchronise a parse started on the wrong
    residue) must verify without the single-CTA redo: bands of 8 to 14 full columns at several
    offsets, and whole uniform frames."""
    w, h = DSLR
    if kind == "natural":
        f = A.natural_frame(w, h, 9)
    elif kind.startswith("uniform"):
        f = A.uniform_frame(w, h, 4095 if kind == "uniform4095" else 512)
    else:
        ncols = int(kind[len("clipped"):])
        c0 = {8: 2000, 12: 100, 13: 1931, 14: 3700}[ncols]
        f = A.clipped_frame(w, h, c0, ncols, seed=4)
    data = A.encode_frame(f)
    res, redo = check(ctx, [(data, w, h)], mirror=kind == "natural")
    assert res[0][0] == 0
    assert redo == [0]
