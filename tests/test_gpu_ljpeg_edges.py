"""The edges of the LJPEG decode's buffer contract, on every kernel path, against the oracle.

The C ABI asks only for 16-byte aligned input and output buffers, bounds each segment by its
`in_size`, and lets a kernel read the input up to the next 16-byte boundary behind `in_total`.  The
cases here pass buffers at 0 and 16 modulo 32 (pointers into a torch allocation), segments at every
offset modulo 32, segments whose stream goes on behind `in_size`, garbage in the readable slack, and
a batch just above the size at which k2_stream_kernel switches to its full-launch form.  Each case
compares the whole padded output buffer (new_image's 0xA5A5 fill included; only the rows of a
segment that fails are left out) and (status, consumed) of every segment with the oracle."""
import numpy as np
import pytest

import rawspeed_b200 as rs
from oracle import port, synth
from helpers import TableSet, dng_ljpeg_scans
from test_gpu_ljpeg import LJPEG_PATHS, _exact_end_of_stream, set_ljpeg_path
from test_ljpeg_stream_emu import _random_table, inject_bad_code

pytestmark = pytest.mark.gpu


@pytest.fixture(params=LJPEG_PATHS)
def ljpeg_path(request, monkeypatch):
    """The kernel paths of tests/test_gpu_ljpeg.py, stream_wide (the full-launch form) included."""
    set_ljpeg_path(monkeypatch, request.param)
    return request.param


def _huffs(tabs):
    """port.Huff of every table of a TableSet, by table index."""
    return [port.Huff(*k) for k in sorted(tabs.keys, key=tabs.keys.get)]


def _oracle(s, data, huffs, img):
    """The oracle on one segment, decoded into `img` (a whole frame): (status, consumed)."""
    g = s.mcu_w * s.mcu_h
    try:
        c = port.ljpeg_decompress(img, img.shape[1], 1, (s.out_x, s.out_y, s.store_w, s.rows), (s.mcu_w, s.mcu_h),
                                  (s.frame_w, s.rows), [huffs[s.table[c]] for c in range(g)],
                                  [s.init_pred[c] for c in range(g)], s.rows, data)
        return 0, c
    except port.IOException:
        return 2, None
    except port.RawDecoderException:
        return 1, None


def _run(plan, blob, out, in_off=0, out_off=0, in_total=None, slack=None):
    """Run `plan` with d_in = blob at `in_off` bytes into a torch allocation (which starts on a 512-byte
    boundary) and d_out = `out` at `out_off` bytes into another.  The readable bytes behind in_total, up
    to the next 16-byte boundary, hold `slack` (zeros by default).  Returns (output, results); the bytes
    of the output allocation around d_out must stay as they were."""
    import torch
    in_total = blob.size if in_total is None else in_total
    padded = (in_total + 15) & ~15
    host = np.zeros(in_off + padded + 64, np.uint8)
    host[in_off:in_off + in_total] = blob[:in_total]
    if slack is not None:
        host[in_off + in_total:in_off + padded] = slack[:padded - in_total]
    d_in = torch.from_numpy(host).cuda()
    ob = out.view(np.uint8).reshape(-1)
    hout = np.full(out_off + ob.size + 64, 0x5A, np.uint8)
    hout[out_off:out_off + ob.size] = ob
    d_out = torch.from_numpy(hout).cuda()
    plan.run((d_in.data_ptr() + in_off, in_total), (d_out.data_ptr() + out_off, ob.size))
    torch.cuda.synchronize()
    res = plan.results(check=False)
    back = d_out.cpu().numpy()
    assert (back[:out_off] == 0x5A).all() and (back[out_off + ob.size:] == 0x5A).all(), "write outside d_out"
    return back[out_off:out_off + ob.size].copy().view(np.uint16).reshape(out.shape), res


def _rows_of(frame, s):
    return frame[s.out_y:s.out_y + s.rows, s.out_x:s.out_x + s.store_w]


def _check(got, want, scans, wants, res, exact=True):
    """(status, consumed) of every segment, then the whole buffer; the rows of a segment that failed in
    both are left out.  exact=False: k2_fused_kernel's conservative end of stream (an IOException where
    the reference may still decode)."""
    got, want = got.copy(), want.copy()
    for k, (s, (ws, wc), (gs, gc)) in enumerate(zip(scans, wants, res)):
        if not exact and gs == 2 and ws != 2:
            ws = 2
        assert gs == ws, (k, gs, ws)
        if ws == 0:
            assert gc == wc, (k, gc, wc)
        else:
            _rows_of(got, s)[...] = 0
            _rows_of(want, s)[...] = 0
    bad = np.argwhere(got != want)
    assert bad.size == 0, (bad[:5], got[tuple(bad[0])], want[tuple(bad[0])])


def _segments(img, tile_w, tile_h, tabs=None, **kw):
    """Scan descriptors and the entropy-coded data (SOS to EOI) of every tile of `img`."""
    t = synth.make_dng_ljpeg(img, tile_w, tile_h, **kw)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(img.shape[1]), tabs=tabs)
    return tabs, scans, [t.blob[s.in_offset:s.in_offset + s.in_size].copy() for s in scans]


def _lay_out(segs, first, fill=0xFF):
    """One input buffer: segment k at an offset congruent to first + k modulo 32 (the first one at
    `first`, with nothing but `fill` bytes before it), `fill` in the gaps, the buffer ending with the
    last segment.  Returns the buffer and the offsets."""
    offs, pos = [], first
    for k, seg in enumerate(segs):
        pos += (first + k - pos) % 32
        offs.append(pos)
        pos += seg.size
    blob = np.full(pos, fill, np.uint8)
    for o, seg in zip(offs, segs):
        blob[o:o + seg.size] = seg
    return blob, offs


# ---------------------------------------------------------------------------------------------
# 1. Buffer bases: d_in at 0, 16 and 80 bytes into an allocation (80: 16 mod 32, not the start of a
#    128-byte line), d_out at 0 and 16; segments at every offset modulo 32, the first one within the
#    first 16 bytes of the buffer (from d_in at 16 mod 32, the 32-byte boundary below it lies before
#    d_in); pitches of 0 and 16 modulo 32 bytes.
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ncomp,w", [(1, 512), (1, 520), (2, 512), (2, 520), (4, 512), (4, 520)])
def test_buffer_bases_and_segment_offsets(ctx, ljpeg_path, ncomp, w):
    h = 64
    img = synth.image_model(w, h, 300 + w + ncomp)
    tabs, scans, segs = _segments(img, 64, 16, ncomp=ncomp)
    assert len(segs) >= 32
    blob, offs = _lay_out(segs, first=(5 * ncomp + w) % 16)
    huffs = _huffs(tabs)
    want = port.new_image(w, h)
    wants = []
    for s, o in zip(scans, offs):
        s.in_offset = o
        wants.append(_oracle(s, blob[o:o + s.in_size], huffs, want))
    assert all(st == 0 for st, _ in wants)
    assert np.array_equal(want[:, :w], img)
    plan = rs.ljpeg_plan(ctx, tabs.tabs, scans)
    for in_off in (0, 16, 80):
        for out_off in (0, 16):
            got, res = _run(plan, blob, port.new_image(w, h), in_off=in_off, out_off=out_off)
            _check(got, want, scans, wants, res)


# ---------------------------------------------------------------------------------------------
# 2. A segment bounded by in_size inside a longer buffer: the rest of the real stream (or an end
#    marker) lies right behind it and must not be read as part of it.
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("marker", [False, True])
def test_segment_limit_inside_a_longer_buffer(ctx, ljpeg_path, marker):
    img = synth.image_model(256, 32, 53)
    t = synth.make_dng_ljpeg(img, 256, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    huffs = _huffs(tabs)
    for cut in list(range(1, 41)) + [64, 100]:
        s = rs.LJpegScan.from_buffer_copy(scans[0])
        s.in_size = scans[0].in_size - cut
        end = s.in_offset + s.in_size
        blob = np.concatenate([t.blob, np.zeros(2, np.uint8)])
        if marker:
            blob[end:end + 2] = [0xFF, 0xD9]
        want = port.new_image(256, 32)
        wants = [_oracle(s, blob[s.in_offset:end], huffs, want)]
        got, res = _run(rs.ljpeg_plan(ctx, tabs.tabs, [s]), blob, port.new_image(256, 32))
        _check(got, want, [s], wants, res, exact=_exact_end_of_stream(ljpeg_path))


# ---------------------------------------------------------------------------------------------
# 3. Garbage in the readable slack: in_total not a multiple of 16, the last segment ending exactly
#    there, the bytes up to the 16-byte boundary all FF, FF D9, FF 00 or random.
# ---------------------------------------------------------------------------------------------
_SLACK = {"ff": np.full(16, 0xFF, np.uint8), "ffd9": np.tile(np.array([0xFF, 0xD9], np.uint8), 8),
          "ff00": np.tile(np.array([0xFF, 0x00], np.uint8), 8),
          "random": np.random.default_rng(3).integers(0, 256, 16).astype(np.uint8)}


@pytest.mark.parametrize("cut", [0, 1, 2, 3, 5, 8, 13, 16, 17, 18, 19, 24, 31, 40, 100])
def test_garbage_in_the_readable_slack(ctx, ljpeg_path, cut):
    """cut 0: the whole segment; otherwise truncated by `cut` bytes (the cuts of test_streams_that_end_early)."""
    img = synth.image_model(256, 32, 53)
    t = synth.make_dng_ljpeg(img, 256, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    huffs = _huffs(tabs)
    s = rs.LJpegScan.from_buffer_copy(scans[0])
    s.in_size = scans[0].in_size - cut
    end = s.in_offset + s.in_size
    shift = ((1, 7, 15)[cut % 3] - end) % 16        # in_total = 1, 7 or 15 modulo 16
    blob = np.concatenate([np.full(shift, 0xFF, np.uint8), t.blob[:end]])
    s.in_offset += shift
    assert blob.size % 16 != 0 and s.in_offset + s.in_size == blob.size
    want = port.new_image(256, 32)
    wants = [_oracle(s, blob[s.in_offset:], huffs, want)]
    plan = rs.ljpeg_plan(ctx, tabs.tabs, [s])
    got0, res0 = _run(plan, blob, port.new_image(256, 32))
    _check(got0, want, [s], wants, res0, exact=_exact_end_of_stream(ljpeg_path))
    for name, slack in _SLACK.items():
        got, res = _run(plan, blob, port.new_image(256, 32), slack=slack)
        assert res == res0, name
        assert np.array_equal(got, got0), name


# ---------------------------------------------------------------------------------------------
# 3b. An unassigned code inside the data of a segment the tile kernel cannot take (rows of 64 samples,
#     or two tables): the decode goes on behind it out of step and often runs past the end of the
#     data, but the answer stays the reference's RawDecoderException at the code.
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["rows64", "two_tables"])
def test_unassigned_code_in_the_data(ctx, ljpeg_path, layout):
    if layout == "rows64":
        img = synth.image_model(64, 128, 71)
        t = synth.make_dng_ljpeg(img, 64, 128)
    else:
        img = synth.image_model(256, 32, 73)
        t = synth.make_dng_ljpeg(img, 256, 32, tabs=synth.default_tables(2), tab_of_comp=[0, 1])
    h, w = img.shape
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(w))
    huffs = _huffs(tabs)
    rng = np.random.default_rng(77)
    n_rde = 0
    for trial in range(30):
        s = rs.LJpegScan.from_buffer_copy(scans[0])
        data = t.blob[s.in_offset:s.in_offset + s.in_size].copy()
        inject_bad_code(data, rng, int(rng.integers(8, data.size - 8)))
        s.in_offset, s.in_size = 0, data.size
        want = port.new_image(w, h)
        wants = [_oracle(s, data, huffs, want)]
        n_rde += wants[0][0] == 1
        got, res = _run(rs.ljpeg_plan(ctx, tabs.tabs, [s]), data, port.new_image(w, h))
        _check(got, want, [s], wants, res, exact=_exact_end_of_stream(ljpeg_path) or wants[0][0] == 1)
    assert n_rde >= 10


# ---------------------------------------------------------------------------------------------
# 4. A batch at the launch size where the plan switches k2_stream_kernel from its prefetch form to its
#    full-launch form (no L2 prefetch, two units stored as one whole 32-byte sector), without any
#    override: a few hundred distinct segments, each decoded once by the oracle, referenced by N slots
#    in shuffled order (warps mix cheap and expensive streams), every slot with its own output place.
# ---------------------------------------------------------------------------------------------
def _content(kind, w, h, seed):
    if kind == "flat":
        img = np.full((h, w), 2000, np.uint16)
        img[::3, ::5] += 3
        return img
    if kind == "model":
        return synth.image_model(w, h, seed)
    if kind == "wild":
        return synth.image_model(w, h, seed, wild=True)
    if kind == "ssss16":
        img = synth.image_model(w, h, seed, wild=True, bits=16)
        img[0, 0:8] = [0, 0x8000, 0, 0x8000, 0xFFFF, 0x7FFF, 0, 0x8000]
        return img
    assert kind == "ffdense"   # long runs of FF bytes in the stream: stuffing everywhere
    img = np.zeros((h, w), np.uint16)
    img[:, 0::2] = 0x3FFF
    img[::3, 2::4] = 0
    return img


def _pool(tab_list, rng):
    """Distinct segments: (scan template, data, decoded tile, (status, consumed)).  Tables: indices into
    tab_list (the plan's tables, in order)."""
    tabs = TableSet()
    for hf in tab_list:
        tabs.add(hf.ncpl, hf.values)
    ntab = len(tab_list)
    pool = []

    for seed in range(3):
        for kind in ("flat", "model", "wild", "ssss16", "ffdense"):
            for g in (1, 2, 4):
                for rsamp in (64, 72, 128):          # 8, 9, 16 units: even / odd; below / above TileGeom<1>::MIN_RS
                    rows = (2, 4)[(seed + g) % 2]
                    if kind in ("ssss16",) or ntab == 1:
                        toc = [0] * g             # (only the default table codes SSSS = 16)
                    else:
                        toc = [int(v) for v in rng.integers(0, ntab, g)]
                    pool.append(dict(kind=kind, g=g, rs=rsamp, rows=rows, toc=toc, seed=100 * seed + 7 * g + rsamp))
    good = len(pool)
    for k in range(40):     # truncated: the buffer of the segment ends early
        g, rsamp = (1, 2, 4)[k % 3], (64, 72, 128)[k % 3 if k < 30 else 1]
        toc = [0] * g if ntab == 1 or k % 2 else [int(v) for v in rng.integers(0, ntab, g)]
        pool.append(dict(kind="model", g=g, rs=rsamp, rows=4, toc=toc, seed=500 + k, cut=(1, 3, 8, 17, 40)[k % 5]))
    for k in range(30):     # an end marker inside the data (single table, rows the tile kernel takes)
        g = (1, 2, 4)[k % 3]
        pool.append(dict(kind=("model", "wild")[k % 2], g=g, rs=(72, 128)[k % 2], rows=4, toc=[k % ntab] * g,
                         seed=600 + k, marker=(2, 5, 11, 19, 32)[k % 5]))
    for k in range(20):     # an unassigned code of the default table: 39 one-bits at byte 40
        g = (1, 2, 4)[k % 3]
        pool.append(dict(kind="wild", g=g, rs=(64, 72, 128)[k % 3], rows=4, toc=[0] * g, seed=700 + k, badcode=True))
    for k in range(40):     # ... inside the data, with an out-of-step decode behind it, or near its end
        g = (1, 2, 4)[k % 3]
        at = ("mid", "end")[(k // 2) % 2]
        toc = [0] * g if ntab == 1 or g == 1 else [0] + [int(v) for v in rng.integers(0, ntab, g - 1)]
        rsamp = (64, 72, 128)[k % 3]
        if at == "end":     # (a code whose bits reach behind the data: only the tile kernel settles it exactly)
            toc, rsamp = [0] * g, (72, 128)[k % 2]
        pool.append(dict(kind=("model", "wild")[k % 2], g=g, rs=rsamp, rows=4, toc=toc, seed=800 + k, badcode_at=at))
    out = []
    for e in pool:
        g, rsamp, rows = e["g"], e["rs"], e["rows"]
        img = _content(e["kind"], rsamp, rows, e["seed"])
        t = synth.make_dng_ljpeg(img, rsamp, rows, ncomp=g, prec=16 if e["kind"] == "ssss16" else 14,
                                 tabs=tab_list, tab_of_comp=e["toc"])
        _, (s,) = dng_ljpeg_scans(t, port.image_pitch(rsamp), tabs=tabs)
        data = t.blob[s.in_offset:s.in_offset + s.in_size].copy()
        if e.get("cut"):
            data = data[:-e["cut"]]
        if e.get("marker"):
            pos = data.size - 2 - e["marker"]
            if data[pos - 1] == 0xFF:
                pos -= 2
            data[pos:pos + 2] = [0xFF, 0xD9]
        if e.get("badcode"):
            pos = 41 if data[39] == 0xFF else 40   # (not behind an FF: 39 one-bits, stuffed)
            data[pos:pos + 9] = [0xFF, 0, 0xFF, 0, 0xFF, 0, 0xFF, 0, 0xFE]
        if e.get("badcode_at"):
            lo, hi = (8, data.size - 40) if e["badcode_at"] == "mid" else (data.size - 24, data.size - 4)
            inject_bad_code(data, rng, int(rng.integers(lo, hi)))
        s.in_size = data.size
        tile = port.new_image(rsamp, rows)
        outcome = _oracle(s, data, _huffs(tabs), tile)
        if e.get("badcode"):
            assert outcome[0] == 1
        out.append((s, data, tile[:, :rsamp], outcome))
    assert all(o[0] == 0 for _, _, _, o in out[:good])
    assert len(tabs.tabs) == ntab
    return tabs, out, good


def _batch(pool, ngood, nslots, rng):
    """nslots scans over the pool (the last len(pool) - ngood pool segments fill a few hundred slots),
    shuffled, each stored at its own place of one of two frames (pitch 0 and 16 modulo 32 bytes) in one
    output buffer; out_x is 0 or 8 modulo 16 samples, store_w the row, the row less 8 samples, or the row
    less 3.  Returns (scans, pool index and frame per slot, input buffer, frames (byte offset, pitch, rows),
    output bytes)."""
    blob, offs = _lay_out([d for _, d, _, _ in pool], first=9)
    nbad = 360
    which = np.concatenate([ngood + np.arange(nbad) % (len(pool) - ngood),
                            rng.integers(0, ngood, nslots - nbad)])
    rng.shuffle(which)
    frame_w = [4096, 4104]            # samples: pitches of 8192 and 8208 bytes
    cur = [[0, 0], [0, 0]]            # (x, y) of the next place in each frame
    band = 4
    scans = []
    place = rng.integers(0, 2, nslots)
    xs = rng.integers(0, 2, nslots) * 8
    sw = rng.integers(0, 3, nslots)
    for i in range(nslots):
        tpl, data, tile, _ = pool[which[i]]
        f = int(place[i])
        rsamp = tile.shape[1]
        cell = (int(xs[i]) + rsamp + 15) // 16 * 16
        if cur[f][0] + cell > frame_w[f]:
            cur[f] = [0, cur[f][1] + band]
        s = rs.LJpegScan.from_buffer_copy(tpl)
        s.in_offset = offs[which[i]]
        s.out_pitch = 2 * frame_w[f]
        s.out_x = cur[f][0] + int(xs[i])
        s.out_y = cur[f][1]
        s.store_w = (rsamp, rsamp - 8, rsamp - 3)[int(sw[i])]
        cur[f][0] += cell
        scans.append(s)
    rows = [cur[0][1] + band, cur[1][1] + band]
    frames = [(0, 2 * frame_w[0], rows[0]), (2 * frame_w[0] * rows[0], 2 * frame_w[1], rows[1])]
    for s, f in zip(scans, place):
        s.out_offset = frames[f][0]
    return scans, which, place, blob, frames, frames[1][0] + frames[1][1] * frames[1][2]


def _full_launch_batch(ctx, monkeypatch, ntab, paths):
    rng = np.random.default_rng(11 + ntab)
    tab_list = synth.default_tables(1) + [_random_table(rng, 16) for _ in range(ntab - 1)]
    tabs, pool, ngood = _pool(tab_list, rng)
    # k2_stream_kernel's prefetch form up to K2S_PREFETCH_CTAS_PER_SM (3) CTAs of T_NT (128) threads per
    # SM, one thread per segment (rsb200.cu, stream_full_launch)
    n = ctx.sm_count * 3 * 128
    scans, which, place, blob, frames, nbytes = _batch(pool, ngood, n + 1, rng)
    # expected: every slot's tile, cropped to store_w, at its place
    want = np.full(nbytes // 2, 0xA5A5, np.uint16)

    def views(buf):
        return [buf[o // 2:(o + p * r) // 2].reshape(r, p // 2) for o, p, r in frames]

    wv = views(want)
    for s, w, f in zip(scans, which, place):
        _rows_of(wv[f], s)[...] = pool[w][2][:, :s.store_w]
    wants = [pool[w][3] for w in which]

    def check(got, sc, ws, res):
        st = np.array([r[0] for r in res])
        assert np.array_equal(st, np.array([x[0] for x in ws])), np.nonzero(st != np.array([x[0] for x in ws]))[0][:8]
        assert (st == 1).any() and (st == 2).any()
        got, exp = got.copy(), want.copy()
        gv, ev = views(got), views(exp)
        for s, f in zip(scans[len(sc):], place[len(sc):]):   # (slots the plan does not hold)
            _rows_of(ev[f], s)[...] = 0xA5A5
        for k, (s, f, (wst, wc), (gs, gc)) in enumerate(zip(sc, place, ws, res)):
            if wst == 0:
                assert gc == wc, (k, gc, wc)
            else:
                _rows_of(gv[f], s)[...] = 0
                _rows_of(ev[f], s)[...] = 0
        bad = np.argwhere(got != exp)
        assert bad.size == 0, (bad[:5], got[tuple(bad[0])], exp[tuple(bad[0])])

    set_ljpeg_path(monkeypatch, "auto")
    plan_n = rs.ljpeg_plan(ctx, tabs.tabs, scans[:n])
    assert "prefetch form" in plan_n.kernels, plan_n.kernels
    plan = rs.ljpeg_plan(ctx, tabs.tabs, scans)
    assert "full-launch form" in plan.kernels, plan.kernels
    got, res = _run(plan, blob, np.full(nbytes // 2, 0xA5A5, np.uint16))
    check(got, scans, wants, res)
    if "prefetch" in paths:
        got, res = _run(plan_n, blob, np.full(nbytes // 2, 0xA5A5, np.uint16))
        check(got, scans[:n], wants[:n], res)
    if "thread" in paths:
        set_ljpeg_path(monkeypatch, "thread")
        plan_t = rs.ljpeg_plan(ctx, tabs.tabs, scans)
        assert "k2_thread_kernel" in plan_t.kernels, plan_t.kernels
        got, res = _run(plan_t, blob, np.full(nbytes // 2, 0xA5A5, np.uint16))
        check(got, scans, wants, res)


def test_full_launch_batch_one_table(ctx, monkeypatch):
    _full_launch_batch(ctx, monkeypatch, 1, ("prefetch", "thread"))


def test_full_launch_batch_four_tables(ctx, monkeypatch):
    """T_MAXTAB tables: the shared-memory LUTs are reduced to the windows all four resolve."""
    _full_launch_batch(ctx, monkeypatch, 4, ("thread",))
