"""K2+K3 parity: CUDA LJPEG decode vs the oracle through the C ABI (bit-exact)."""
import numpy as np
import pytest

import rawspeed_b200 as rs
from oracle import port, synth
from helpers import dng_ljpeg_scans, gpu_run

pytestmark = pytest.mark.gpu


LJPEG_PATHS = ["auto", "tile2", "fused", "thread", "thread_clean2", "stream", "stream_wide", "par"]


@pytest.fixture(autouse=True, params=LJPEG_PATHS)
def ljpeg_path(request, monkeypatch):
    """Every case runs eight times: with the plan's own choice of kernel (k2_tile_kernel<1> for
    plain single-table tiles, k2_fused_kernel for the rest, at these sizes), with the second
    geometry of the tile kernel (RSB200_TILE_R=2), with the round-1 block-per-segment kernel for
    everything (RSB200_LJPEG_PATH=fused), with the one-thread-per-segment path in its three
    forms (K2C + K2T, K2C2 + K2T, and k2_stream_kernel which unstuffs inside the thread), with
    k2_stream_kernel in the form the plan gives full launches whatever the batch size (no L2
    prefetch, whole-sector stores: RSB200_STREAM_FORM=wide) and with the one-CTA-per-segment
    speculative parse on the clean stream (K2C + k2_par_kernel)."""
    set_ljpeg_path(monkeypatch, request.param)
    return request.param


def set_ljpeg_path(monkeypatch, name):
    """The environment of one of LJPEG_PATHS (tests/test_gpu_ljpeg_edges.py uses it as well)."""
    monkeypatch.delenv("RSB200_LJPEG_PATH", raising=False)
    monkeypatch.delenv("RSB200_TILE_R", raising=False)
    monkeypatch.delenv("RSB200_THREAD_KERNEL", raising=False)
    monkeypatch.delenv("RSB200_STREAM_FORM", raising=False)
    monkeypatch.setenv("RSB200_CLEAN", "1")   # (the plan picks by segment size; here: both, explicitly)
    if name == "tile2":
        monkeypatch.setenv("RSB200_TILE_R", "2")
    elif name == "thread_clean2":
        monkeypatch.setenv("RSB200_LJPEG_PATH", "thread")
        monkeypatch.setenv("RSB200_CLEAN", "2")
    elif name == "stream_wide":
        monkeypatch.setenv("RSB200_LJPEG_PATH", "stream")
        monkeypatch.setenv("RSB200_STREAM_FORM", "wide")
    elif name != "auto":
        monkeypatch.setenv("RSB200_LJPEG_PATH", name)


def _check_tiles(ctx, img, tile_w, tile_h, **kw):
    h, w = img.shape
    cpp = kw.pop("cpp", 1)
    w //= cpp
    t = synth.make_dng_ljpeg(img, tile_w, tile_h, cpp=cpp, **kw)
    want = port.new_image(w, h, cpp)
    got0 = want.copy()
    port.dng_decompress(t.blob, t.offsets, t.lengths, want, w, cpp, tile_w, tile_h, 7,
                        fix_ljpeg=kw.get("fix16", False), nthreads=4)
    tabs, scans = dng_ljpeg_scans(t, got0.shape[1] * 2, fix16=kw.get("fix16", False))
    plan = rs.ljpeg_plan(ctx, tabs.tabs, scans)
    got, res = gpu_run(plan, t.blob, got0)
    assert np.array_equal(got, want)
    assert np.array_equal(got[:, :w * cpp], img)
    return t, res


def test_single_small_tile(ctx):
    img = synth.image_model(64, 32, 1)
    _check_tiles(ctx, img, 64, 32)


def test_tiles_ragged_edges(ctx):
    img = synth.image_model(300, 200, 7)
    _check_tiles(ctx, img, 128, 64)


def test_wild_noise_long_codes(ctx):
    img = synth.image_model(256, 96, 9, wild=True)
    _check_tiles(ctx, img, 128, 32)


def test_sixteen_bit_ssss16(ctx):
    # full 16-bit range: differences of -32768 (SSSS=16) occur
    img = synth.image_model(128, 64, 11, wild=True, bits=16)
    img[0, 0:8] = [0, 0x8000, 0, 0x8000, 0xFFFF, 0x7FFF, 0, 0x8000]
    _check_tiles(ctx, img, 64, 64, prec=16)
    _check_tiles(ctx, img, 64, 64, prec=16, fix16=True)


def test_components_1_3_4_and_2x2(ctx):
    img = synth.image_model(96, 48, 13)
    _check_tiles(ctx, img, 48, 24, ncomp=1)
    _check_tiles(ctx, img, 96, 48, ncomp=4)
    _check_tiles(ctx, img, 48, 48, ncomp=3)
    _check_tiles(ctx, img, 48, 24, ncomp=4, mcu=(2, 2))
    img3 = synth.image_model(96 * 3, 40, 14)
    _check_tiles(ctx, img3, 32, 20, ncomp=3, cpp=3)


def test_two_tables(ctx):
    img = synth.image_model(200, 100, 15)
    tabs = synth.default_tables(2)
    _check_tiles(ctx, img, 100, 50, tabs=tabs, tab_of_comp=[0, 1])
    _check_tiles(ctx, img, 100, 50, ncomp=4, tabs=tabs, tab_of_comp=[1, 0, 0, 1])


def test_two_tables_long_code_of_one_is_a_short_code_of_the_other(ctx):
    """Component 0: wild noise with the default table (codes of 12-14 bits, resolved outside the LUT);
    component 1: a COMPLETE table of eight 3-bit codes, in which every window is a valid code.  A decoder
    that looks a window up again after a miss -- with the next component's table -- must not take the hit."""
    rng = np.random.default_rng(5)
    img = np.zeros((64, 256), np.uint16)
    img[:, 0::2] = rng.integers(0, 1 << 14, (64, 128))
    img[:, 1::2] = 8192 + rng.integers(0, 60, (64, 128))
    tabs = [synth.default_tables(1)[0], port.Huff(bytes([0, 0, 8] + [0] * 13), bytes(range(8)))]
    _check_tiles(ctx, img, 128, 32, tabs=tabs, tab_of_comp=[0, 1])
    _check_tiles(ctx, img, 256, 32, ncomp=4, tabs=tabs, tab_of_comp=[0, 1, 0, 1])


@pytest.mark.parametrize("seed", range(6))
def test_random_tables_and_components(ctx, seed):
    """Differential fuzz (the CPU replays run the same generator, tests/test_ljpeg_stream_emu.py): 1 / 2 / 4
    components, one to four random COMPLETE canonical codes of up to 16 bits, noise from a few bits to the
    full 14-bit range."""
    from test_ljpeg_stream_emu import _random_table
    rng = np.random.default_rng(7000 + seed)
    ncomp = int(rng.choice([1, 2, 4]))
    ntab = int(rng.integers(1, min(ncomp, 4) + 1))
    bits = int(rng.choice([3, 6, 10, 14]))
    h, tw = int(rng.choice([8, 16, 24])), int(rng.choice([64, 128, 256]))
    w = tw * int(rng.integers(1, 3))
    img = (8192 + rng.integers(0, 1 << bits, (h, w)) - (1 << bits) // 2).astype(np.uint16) & 0x3FFF
    tabs = [_random_table(rng, 16) for _ in range(ntab)]
    tab_of_comp = [int(rng.integers(0, ntab)) for _ in range(ncomp)]
    for t in range(ntab):
        if t not in tab_of_comp:
            tab_of_comp[t % ncomp] = t
    _check_tiles(ctx, img, tw, h, ncomp=ncomp, tabs=tabs, tab_of_comp=tab_of_comp)


def test_restart_intervals(ctx):
    img = synth.image_model(160, 96, 17)
    _check_tiles(ctx, img, 80, 48, restart_rows=1)
    _check_tiles(ctx, img, 80, 48, restart_rows=5)


def test_odd_width_trailing_pixels(ctx):
    img = synth.image_model(101, 33, 19)
    _check_tiles(ctx, img, 64, 16)


def test_consumed_matches_reference(ctx):
    img = synth.image_model(128, 64, 21)
    t = synth.make_dng_ljpeg(img, 64, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(128))
    plan = rs.ljpeg_plan(ctx, tabs.tabs, scans)
    got, res = gpu_run(plan, t.blob, port.new_image(128, 64))
    hts = synth.default_tables(1)
    for (status, consumed), s, off, ln in zip(res, scans, t.offsets, t.lengths):
        assert status == 0
        data = t.blob[s.in_offset:off + ln]
        o = port.new_image(128, 64)
        want = port.ljpeg_decompress(o, 128, 1, (s.out_x, s.out_y, s.store_w, s.rows),
                                     (2, 1), (s.frame_w, s.rows), [hts[0], hts[0]],
                                     [1 << 13] * 2, s.rows, data)
        assert consumed == want


def test_c3_45mp_dng(ctx):
    """BASELINE configs[2]: DNG LJPEG predictor 1, 8256x5504, 726 tiles 256x256."""
    img = synth.image_model(8256, 5504, 12345)
    t = synth.make_dng_ljpeg(img, 256, 256)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(8256))
    assert len(scans) == 726
    plan = rs.ljpeg_plan(ctx, tabs.tabs, scans)
    got, res = gpu_run(plan, t.blob, port.new_image(8256, 5504))
    assert all(s == 0 for s, _ in res)
    assert np.array_equal(got[:, :8256], img)   # round trip == the reference's output
    want = port.new_image(8256, 5504)
    port.dng_decompress(t.blob, t.offsets, t.lengths, want, 8256, 1, 256, 256, 7, nthreads=8)
    assert np.array_equal(got, want)


def test_bad_huffman_code_reports_rde(ctx):
    img = synth.image_model(64, 32, 23, wild=True)
    # table without SSSS >= 12: craft a stream with an unassigned all-ones code
    t = synth.make_dng_ljpeg(img, 64, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(64))
    blob = t.blob.copy()
    s = scans[0]
    # 39 consecutive one-bits (FF is stuffed): no code of this table starts with 15 ones
    blob[s.in_offset + 40:s.in_offset + 49] = [0xFF, 0, 0xFF, 0, 0xFF, 0, 0xFF, 0, 0xFE]
    plan = rs.ljpeg_plan(ctx, tabs.tabs, scans)
    import torch
    d_in = torch.from_numpy(np.concatenate([blob, np.zeros(64, np.uint8)])).cuda()
    d_out = torch.zeros(32 * port.image_pitch(64) // 2, dtype=torch.int16, device="cuda")
    plan.run((d_in.data_ptr(), blob.size), d_out)
    with pytest.raises(rs.RawDecoderException):
        plan.results()
    with pytest.raises(port.RawDecoderException):
        port.dng_decompress(blob, t.offsets, t.lengths, port.new_image(64, 32), 64, 1, 64, 32, 7)


def test_big_untiled_strip_multi_cta(ctx):
    """One LJPEG segment far above the multi-CTA threshold (several ranges of 64 KiB):
    count / verify / diffs kernels + K3, single and two-table variants, 2 and 4
    components, with and without restart intervals."""
    img = synth.image_model(2048, 700, 41)
    _check_tiles(ctx, img, 2048, 700)
    _check_tiles(ctx, img, 2048, 700, tabs=synth.default_tables(2), tab_of_comp=[0, 1])
    _check_tiles(ctx, img, 2048, 700, ncomp=4, tabs=synth.default_tables(2),
                 tab_of_comp=[0, 1, 1, 0])
    wild = synth.image_model(1536, 512, 43, wild=True)
    _check_tiles(ctx, wild, 1536, 512)
    _check_tiles(ctx, wild, 768, 512, restart_rows=150)


def test_mixed_small_and_big_segments(ctx):
    img = synth.image_model(2100, 520, 47)
    _check_tiles(ctx, img, 2048, 512)   # tiles: one big (2048x512), small edge tiles


def test_many_segments_take_the_thread_path(ctx, ljpeg_path):
    """>= 16384 segments in one plan: the plan itself picks the one-thread-per-segment path; every
    forced path decodes the same launch-sized batch bit for bit."""
    img = synth.image_model(4096, 4096, 51)
    t = synth.make_dng_ljpeg(img, 32, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(4096))
    assert len(scans) == 16384
    plan = rs.ljpeg_plan(ctx, tabs.tabs, scans)
    if ljpeg_path == "auto":
        # K2C + K2T, or k2_stream_kernel alone (32x32 tiles are below the tile kernel's row size: no second opinion)
        assert plan.launches in (1, 2)
        assert "thread" in plan.kernels or "stream" in plan.kernels, plan.kernels
    got, res = gpu_run(plan, t.blob, port.new_image(4096, 4096))
    assert all(s == 0 for s, _ in res)
    want = port.new_image(4096, 4096)
    port.dng_decompress(t.blob, t.offsets, t.lengths, want, 4096, 1, 32, 32, 7, nthreads=8)
    assert np.array_equal(got, want)
    # consumed of a few segments against the reference restatement
    hts = synth.default_tables(1)
    for k in (0, 1, 8191, 16383):
        s, off, ln = scans[k], t.offsets[k], t.lengths[k]
        o = port.new_image(4096, 4096)
        c = port.ljpeg_decompress(o, 4096, 1, (s.out_x, s.out_y, s.store_w, s.rows), (2, 1),
                                  (s.frame_w, s.rows), [hts[0], hts[0]], [1 << 13] * 2, s.rows,
                                  t.blob[s.in_offset:off + ln])
        assert res[k][1] == c


def test_truncated_and_garbage_tail_segments(ctx):
    """Streams that end early (status 2 -> IOException) and streams followed by garbage
    before EOI (consumed still the reference's) -- same outcome on both kernels."""
    img = synth.image_model(128, 64, 53)
    t = synth.make_dng_ljpeg(img, 64, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(128))
    # cut the first segment short by 40 bytes: its data ends at the buffer end of the segment
    short = [rs.LJpegScan.from_buffer_copy(s) for s in scans]
    short[0].in_size = scans[0].in_size - 40
    plan = rs.ljpeg_plan(ctx, tabs.tabs, short[:1])
    import torch
    d_in = torch.from_numpy(np.concatenate([t.blob, np.zeros(64, np.uint8)])).cuda()
    d_out = torch.zeros(64 * port.image_pitch(128) // 2, dtype=torch.int16, device="cuda")
    plan.run((d_in.data_ptr(), t.blob.size), d_out)
    with pytest.raises(rs.IOException):
        plan.results()


# ---------------------------------------------------------------------------------------------
# The end of the stream (VERDICT r1 item 3): bits behind the last data byte / the end marker read
# as zero, and the segment fails exactly where the reference's pump would have thrown
# (BitStreamer.h:120-127, BitStreamerJPEG.h:155-183, LJpegDecompressor.cpp:334).  The expectation
# comes from the compiled reference where it is present (oracle.ref), else from the restatement.
# ---------------------------------------------------------------------------------------------
def _reference_outcome(s, data, w, h):
    import oracle
    hts = synth.default_tables(1)
    o = port.new_image(w, h)
    try:
        if oracle.HAVE_REF:
            c = oracle.ref.ljpeg_decompress(o, w, 1, (s.out_x, s.out_y, s.store_w, s.rows), (2, 1),
                                            (s.frame_w, s.rows), [hts[0]], [0, 0], [1 << 13] * 2, s.rows, data)
        else:
            c = port.ljpeg_decompress(o, w, 1, (s.out_x, s.out_y, s.store_w, s.rows), (2, 1),
                                      (s.frame_w, s.rows), [hts[0], hts[0]], [1 << 13] * 2, s.rows, data)
        return 0, c, o
    except Exception as e:   # noqa: BLE001
        return (2 if "IOException" in type(e).__name__ or "IOE" in type(e).__name__ else 1), None, o


def _gpu_outcome(ctx, tabs, s, blob, w, h):
    import torch
    plan = rs.ljpeg_plan(ctx, tabs.tabs, [s])
    d_in = torch.from_numpy(np.concatenate([blob, np.zeros(64, np.uint8)])).cuda()
    got0 = port.new_image(w, h)
    d_out = torch.from_numpy(got0.view(np.int16).copy()).cuda()
    plan.run((d_in.data_ptr(), blob.size), d_out)
    torch.cuda.synchronize()
    (status, consumed), = plan.results(check=False)
    return status, consumed, d_out.cpu().numpy().view(np.uint16).reshape(got0.shape)


def _exact_end_of_stream(ljpeg_path):
    # k2_fused_kernel (shapes the tile kernel does not take) keeps the conservative answer
    # "IOException whenever a needed bit is not there" (DESIGN.md, known deviations)
    return ljpeg_path != "fused"


@pytest.mark.parametrize("cut", [1, 2, 3, 5, 8, 13, 16, 17, 18, 19, 24, 31, 40, 100])
def test_streams_that_end_early(ctx, ljpeg_path, cut):
    img = synth.image_model(256, 32, 53)
    t = synth.make_dng_ljpeg(img, 256, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    s = rs.LJpegScan.from_buffer_copy(scans[0])
    s.in_size = scans[0].in_size - cut
    blob = t.blob[:s.in_offset + s.in_size].copy()
    want_status, want_cons, want_img = _reference_outcome(s, blob[s.in_offset:], 256, 32)
    status, consumed, got = _gpu_outcome(ctx, tabs, s, blob, 256, 32)
    assert status == want_status          # (a buffer that ends early is always an IOException)
    if want_status == 0:
        assert consumed == want_cons and np.array_equal(got, want_img)


@pytest.mark.parametrize("cut", [2, 3, 5, 8, 11, 13, 16, 19, 24, 32, 40])
def test_streams_with_an_early_marker(ctx, ljpeg_path, cut):
    img = synth.image_model(256, 32, 57)
    t = synth.make_dng_ljpeg(img, 256, 32)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    s = rs.LJpegScan.from_buffer_copy(scans[0])
    blob = t.blob.copy()
    end = s.in_offset + s.in_size
    pos = end - 2 - cut
    if blob[pos - 1] == 0xFF:
        pos -= 2
    blob[pos] = 0xFF
    blob[pos + 1] = 0xD9
    want_status, want_cons, want_img = _reference_outcome(s, blob[s.in_offset:end], 256, 32)
    status, consumed, got = _gpu_outcome(ctx, tabs, s, blob[:end], 256, 32)
    if not _exact_end_of_stream(ljpeg_path):
        assert status in (want_status, 2)
        return
    assert status == want_status
    if want_status == 0:
        assert consumed == want_cons and np.array_equal(got, want_img)


def test_rows_below_the_crop_are_not_decoded(ctx, ljpeg_path):
    img = synth.image_model(256, 64, 59)
    t = synth.make_dng_ljpeg(img, 256, 64)
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(256))
    s = rs.LJpegScan.from_buffer_copy(scans[0])
    s.rows = 40
    want_status, want_cons, want_img = _reference_outcome(s, t.blob[s.in_offset:], 256, 64)
    status, consumed, got = _gpu_outcome(ctx, tabs, s, t.blob, 256, 64)
    assert (status, consumed) == (want_status, want_cons)
    assert np.array_equal(got, want_img)
