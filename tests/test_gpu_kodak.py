"""Kodak DCR on the GPU (rsb200_kodak_plan_create, kodak.cuh) against the CPU restatement of
KodakDecompressor (tests/emu/kodak_oracle.c, pinned against the reference's outcomes): the whole output
buffer with sentinels around every job, status, `consumed` and the printed value, through the C ABI
and through the host mirror KodakDecompressor, whose message text must be the reference's."""
import re

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import host
import kodak_oracle as K
import test_oracle_kodak as T

pytestmark = pytest.mark.gpu

FILL = K.FILL_DEFAULT
GAP = 32  # sentinel pixels before every job and behind the last


def run_frames(ctx, frames, in_skews=None):
    """frames: [(data, w, h, bps, mode, table)] (table: the RawImage's TableLookUp content) ->
    ([image], [(status, consumed)], [value]); asserts that the sentinels around every job's output
    are untouched."""
    import torch
    blob, jobs, outs, tables, off = bytearray(), [], [], [], 0
    for k, (data, w, h, bps, mode, table) in enumerate(frames):
        skew = 0 if in_skews is None else in_skews[k]
        blob += bytes((-len(blob)) % 16 + skew)
        pitch = K.pitch_elems(w)
        off += GAP
        j = rs.KodakJob()
        j.in_offset, j.in_size, j.width, j.height, j.bps = len(blob), len(data), w, h, bps
        j.table = -1
        if mode != K.NONE:
            j.table = len(tables)
            tables.append(K.device_table(table, mode))
        j.out_offset, j.out_pitch = off * 2, pitch * 2
        jobs.append(j)
        blob += data
        outs.append((off, h, pitch))
        off += pitch * h
    off += GAP
    plan = rs.kodak_plan(ctx, jobs, np.stack(tables) if tables else None)
    d_in = torch.from_numpy(np.frombuffer(bytes(blob) + b"\x5a" * 64, np.uint8).copy()).cuda()
    out = torch.full((off,), FILL, dtype=torch.int32).to(torch.int16).cuda()
    plan.run((d_in.data_ptr(), len(blob)), out)
    torch.cuda.synchronize()
    res = plan.results(check=False)
    vals = plan.kodak_values()
    plan.close()
    o = out.cpu().numpy().view(np.uint16)
    imgs, seen = [], np.zeros(off, bool)
    for p, h, pitch in outs:
        imgs.append(o[p:p + h * pitch].reshape(h, pitch))
        seen[p:p + h * pitch] = True
    assert np.all(o[~seen] == FILL), "a store outside the jobs' images"
    return imgs, res, vals


def host_run(data, w, h, bps, cpp=1, curve=None, dither=False, uncorrected=True):
    """KodakDecompressor(img, data, bps, uncorrected).decompress() through the host mirror ->
    (image, message)."""
    img = np.full((max(h, 1), K.pitch_elems(max(w, 1) * cpp)), FILL, np.uint16)
    try:
        host.kodak(img, w, np.frombuffer(bytes(data), np.uint8).copy(), bps, uncorrected, curve, dither, cpp)
        return img, ""
    except (rs.RawDecoderException, rs.IOException) as e:
        text = re.sub(r"^rsb200 error -?[0-9]+: ", "", str(e))
        assert isinstance(e, rs.IOException) == (K.message_id(text) in K.IOE_MSGS), text
        return img, text


def check(ctx, frames, in_skews=None):
    imgs, res, vals = run_frames(ctx, frames, in_skews)
    for k, ((data, w, h, bps, mode, table), img, got, val) in enumerate(zip(frames, imgs, res, vals)):
        want, rc, r, c, v = K.decompress(data, w, h, bps, mode, table, fill=FILL)
        st = 0 if rc == K.OK else (2 if rc in K.IOE_MSGS else 1)
        assert got == (st, K.consumed(rc, r, c)), (k, got, rc, r, c)
        assert val == (v if rc == K.VALUE else 0), (k, val, v)
        assert np.array_equal(img, want), k


def frame_of(case):
    data, w, h, bps, cpp, curve, dither, uncorrected = case
    mode, table = T.case_table(curve, dither, uncorrected)
    return data, w, h, bps, mode, table


def accepted(case):
    data, w, h, bps, cpp, curve, dither, uncorrected = case
    return T.run_case(*case)[1] < K.CPP


def test_golden_cases_through_mirror(ctx):
    """Every pinned case, one plan each through the C ABI where the constructor accepts it, and through
    the host mirror (constructor rejections included), whose text and image are the reference's."""
    for name, case in T.golden_cases():
        want, rc, _, _, _, msg = T.run_case(*case)
        data, w, h, bps, cpp, curve, dither, uncorrected = case
        if rc < K.CPP:
            check(ctx, [frame_of(case)])
        if w <= 0 or h <= 0:  # (the mirror's RawImage, like the reference's, cannot hold an empty image)
            continue
        himg, text = host_run(data, w, h, bps, cpp, curve, dither, uncorrected)
        assert text == msg, (name, text, msg)
        if cpp == 1:
            assert np.array_equal(himg, want), name


@pytest.mark.parametrize("skew", [0, 1, 2, 3, 5, 7])
def test_golden_cases_one_plan_skewed(ctx, skew):
    """All accepted pinned cases but the full-size ones in one plan (mixed outcomes, widths, depths and
    table modes), every stream at in_offset & 15 == skew."""
    frames = [frame_of(c) for n, c in T.golden_cases() if accepted(c) and not n.startswith("full_")]
    check(ctx, frames, [skew] * len(frames))


def test_full_size_frames(ctx):
    """4500x3000 and 4516x3012 frames, four per plan: clean, with a table, truncated, out of range."""
    v12 = K.natural(4500, 3000, 12, seed=11)
    d12 = K.encode(v12)
    v10 = K.natural(4516, 3012, 10, seed=12)
    v10[2000, 4400] = 1 << 10
    d10 = K.encode(v10)
    dither = K.lookup_table(T.GAMMA, True)
    frames = [(d12, 4500, 3000, 12, K.NONE, None), (d12[:len(d12) * 2 // 3], 4500, 3000, 12, K.DITHER, dither),
              (d10, 4516, 3012, 10, K.PLAIN, K.lookup_table(T.ZIGZAG, False)),
              (d12 + bytes(1000), 4500, 3000, 12, K.PLAIN, K.lookup_table(T.SHORT, False))]
    check(ctx, frames, [3, 0, 2, 1])


def test_every_failure_kind(ctx):
    """An out-of-range pixel (2^bps, -1) and an over-read in every position of a row, in one plan."""
    frames = []
    for bps in (10, 12):
        for x in (1 << bps, -1, (1 << bps) - 1):
            for col in (0, 1, 255, 256, 257, 511, 515):
                v = K.natural(516, 4, bps, seed=col)
                v[2, col] = x
                frames.append((K.encode(v), 516, 4, bps, K.NONE, None))
    v = K.natural(516, 40, 12, seed=1)
    data = K.encode(v)
    segs, _ = T.segment_starts(data, 516, 40)
    for i in (0, 1, 2, 3, 50, 117, len(segs) - 1):
        p = segs[i][2]
        for cut in (p, p + 1, p + 100, p + 131):
            frames.append((data[:max(cut, 516 * 40 // 2)], 516, 40, 12, K.NONE, None))
    check(ctx, frames)


def test_seeded_fuzz(ctx):
    rng = np.random.default_rng(2024)
    for rnd in range(4):
        frames = []
        for k in range(30):
            w, h, bps = 4 * int(rng.integers(1, 300)), int(rng.integers(1, 80)), (10, 12)[k % 2]
            mode = int(rng.integers(0, 3))
            table = None if mode == K.NONE else K.lookup_table(
                rng.integers(0, 65536, int(rng.integers(1, 5000))), mode == K.DITHER)
            kind = k % 3
            if kind == 0:
                data = K.encode(K.random_values(w, h, bps, seed=k + 100 * rnd))
                data = data[:len(data) - int(rng.integers(0, 64))]
            elif kind == 1:
                lens = rng.integers(0, 9, (h, w)).astype(np.uint8)
                codes = rng.integers(0, 1 << 16, (h, w)).astype(np.uint16)
                data = K.write(lens, codes, w, h)
            else:
                data = rng.integers(0, 256, int(rng.integers(w * h // 2, 2 * w * h + 1)), dtype=np.uint8).tobytes()
            if len(data) < w * h // 2:
                data += bytes(w * h // 2 - len(data))
            frames.append((data, w, h, bps, mode, table))
        check(ctx, frames, [int(s) for s in rng.integers(0, 16, len(frames))])


def test_plan_refusals(ctx):
    """Constructor checks with the reference's classes; malformed descriptors with RSB200_ERR_ARG."""
    def job(**kw):
        j = rs.KodakJob()
        j.in_offset, j.in_size, j.width, j.height, j.bps, j.table = 0, 1000, 16, 8, 12, -1
        j.out_offset, j.out_pitch = 0, 32
        for k, v in kw.items():
            setattr(j, k, v)
        return j
    for kw, exc in (({"width": 18}, rs.RawDecoderException), ({"height": 3013}, rs.RawDecoderException),
                    ({"bps": 14}, rs.RawDecoderException), ({"in_size": 63}, rs.IOException)):
        with pytest.raises(exc):
            rs.kodak_plan(ctx, [job(**kw)])
    for kw in ({"out_offset": 2}, {"out_pitch": 30}, {"out_pitch": 34}, {"in_size": (1 << 28) + 1},
               {"reserved": 1}, {"table": 0}):
        with pytest.raises(rs.Rsb200Error) as e:
            rs.kodak_plan(ctx, [job(**kw)])
        assert e.value.code == 4, kw
    rs.kodak_plan(ctx, [job(in_size=64)]).close()


def test_values_refused_for_other_plans(ctx):
    j = rs.KodakJob()
    j.in_size, j.width, j.height, j.bps, j.table, j.out_pitch = 64, 16, 8, 12, -1, 32
    p = rs.kodak_plan(ctx, [j])
    with pytest.raises(rs.Rsb200Error):
        p.kodak_values()  # not run yet
    p.close()


def test_lifecycle(ctx):
    """create / run / results / run again / destroy, the launch count per run."""
    import torch
    v = K.natural(300, 20, 12, seed=3)
    data = K.encode(v)
    j = rs.KodakJob()
    j.in_size, j.width, j.height, j.bps, j.table, j.out_pitch = len(data), 300, 20, 12, -1, 2 * K.pitch_elems(300)
    plan = rs.kodak_plan(ctx, [j])
    d_in = torch.from_numpy(np.frombuffer(data, np.uint8).copy()).cuda()
    for _ in range(2):
        out = torch.zeros(20 * K.pitch_elems(300), dtype=torch.int16).cuda()
        before = ctx.launches
        plan.run((d_in.data_ptr(), len(data)), out)
        assert ctx.launches - before == plan.launches
        assert plan.results() == [(0, 0)]
        assert plan.kodak_values() == [0]
        img = out.cpu().numpy().view(np.uint16).reshape(20, -1)
        assert np.array_equal(img[:, :300], v)
    plan.close()
