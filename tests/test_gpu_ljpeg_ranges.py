"""The multi-CTA range decoder (ljpeg_ranges.cuh: P1 count, P2 verify, P3 diffs, and the exact redo by
k2_entropy_kernel when a seam fails) against the oracle: CR2 frames, untiled LJPEG strips above
256 KiB, Pentax and Nikon streams.  Bit-exact pixels of the whole padded buffer, the same status and,
for the JPEG pump, the same `consumed`.

rsb200_debug_range_redo (a debug entry of the library, not in the public header) tells which scans
of the last run were redone.  Ordinary streams must verify without a redo.  A redo is forced with a
Huffman table in which every code length plus its extra bits is a multiple of 3 and that has no
unassigned code: a parse that starts at a bit position of another residue mod 3 then never
resynchronises, so P1's guess at the start of a range stays wrong and P2's seam check fails."""
import ctypes as C

import numpy as np
import pytest

import rawspeed_b200 as rs
from oracle import port, synth
from helpers import TableSet, dng_ljpeg_scans, parse_ljpeg
from test_gpu_cr2 import cr2_job

pytestmark = pytest.mark.gpu

RANGE_BYTES = 8 * 8192                     # R_CHUNKS * F_RAW (ljpeg_ranges.cuh)

# Code length of difference category (SSSS) 0..12; length + SSSS is a multiple of 3, Kraft sum 1.
LEN3 = [3, 2, 4, 3, 5, 4, 3, 5, 4, 6, 5, 4, 6]
# Differences of the ordinary redo streams (SSSS 0..6) and of the streams that carry an unassigned
# code (SSSS 0, 1, 3 only: no run of six one-bits anywhere).
RICH = [0, 1, 2, 3, 4, 5, 7, 9, 15, 16, 23, 31, 40, 63]
PLAIN = [0, 1, 4, 5, 6, 7]
HOLE = 1 << 11                             # SSSS 12: the one code (111111) the decode table leaves out


def table_of(lengths):
    """(ncpl[16], values) of the canonical code with these lengths per SSSS."""
    order = sorted(range(len(lengths)), key=lambda s: (lengths[s], s))
    ncpl = [0] * 16
    for s in order:
        ncpl[lengths[s] - 1] += 1
    return ncpl, order


def pentax_meta(lengths):
    """A PEF Huffman-table maker note (PentaxDecompressor::SetupHuffmanTable, big endian) whose
    table is the canonical code with these lengths per SSSS."""
    order = sorted(range(len(lengths)), key=lambda s: (lengths[s], s))
    code, prev, codes = 0, lengths[order[0]], {}
    for s in order:
        code <<= lengths[s] - prev
        prev = lengths[s]
        codes[s] = code
        code += 1
    out = bytearray([0, len(lengths) - 12]) + bytes(12)
    for s in range(len(lengths)):
        out += bytes([(codes[s] << (12 - lengths[s])) >> 8, (codes[s] << (12 - lengths[s])) & 255])
    out += bytes(lengths)
    return bytes(out)


T3 = table_of(LEN3)
T3_HOLE = table_of(LEN3[:12])              # no code for SSSS 12


def _walk(rng, h, w, mags, first, mid, hole_at=None):
    """Values whose differences (per-parity left predictor; columns 0/1 from first(v, r, c)) all have
    magnitudes from `mags`, signed to head for `mid`.  hole_at = (r, c): that difference is HOLE."""
    m = rng.choice(np.array(mags, dtype=np.int64), size=(h, w))
    if hole_at is not None:
        m[hole_at] = HOLE
    v = np.zeros((h, w), np.int64)
    for r in range(h):
        for c in (0, 1):
            p = first(v, r, c)
            v[r, c] = p + (m[r, c] if p < mid else -m[r, c])
    for c in range(2, w):
        p = v[:, c - 2]
        v[:, c] = p + np.where(p < mid, m[:, c], -m[:, c])
    return v


def pentax_image(rng, h, w, mags, hole_at=None):
    v = _walk(rng, h, w, mags, lambda v, r, c: v[r - 2, c] if r >= 2 else 0, 32768, hole_at)
    assert v.min() >= 0 and v.max() <= 65535
    return v.astype(np.uint16)


def ljpeg_image(rng, h, w, mags, hole_at=None):
    """Two components, predictor 1, one MCU row per frame row (a strip or a one-slice CR2)."""
    v = _walk(rng, h, w, mags, lambda v, r, c: v[r - 1, c] if r >= 1 else 1 << 13, 1 << 13, hole_at)
    assert v.min() >= 0 and v.max() < 1 << 14
    return v.astype(np.uint16)


def nikon_diffs(rng, h, w, mags, pup):
    v = _walk(rng, h, w, mags, lambda v, r, c: v[r - 2, c] if r >= 2 else pup[2 * r + c], 1 << 14)
    d = np.zeros((h, w), np.int64)
    d[:, 2:] = v[:, 2:] - v[:, :-2]
    d[2:, :2] = v[2:, :2] - v[:-2, :2]
    for r in range(min(h, 2)):
        d[r, 0], d[r, 1] = v[r, 0] - pup[2 * r], v[r, 1] - pup[2 * r + 1]
    return d


def nikon_expected(d, pup):
    """NikonDecompressor without a curve: pUp[row & 1] + per-parity prefix sums, clampBits(v, 15)."""
    v = d.astype(np.int64).copy()
    for q in (0, 1):
        for c in (0, 1):
            v[q::2, c] = np.cumsum(v[q::2, c]) + pup[2 * q + c]
    v[:, 0::2] = np.cumsum(v[:, 0::2], axis=1)
    v[:, 1::2] = np.cumsum(v[:, 1::2], axis=1)
    return np.clip(v, 0, 32767).astype(np.uint16)


def _outcome(fn):
    try:
        fn()
        return 0
    except port.RawDecoderException:
        return 1
    except port.IOException:
        return 2


def oracle_pentax(data, w, h, meta=None):
    o = port.new_image(w, h)
    st = _outcome(lambda: port.pentax_decompress(o, w, data, meta, True))
    return st, o


def redo_flags(plan):
    f = plan.ctx._lib.rsb200_debug_range_redo
    f.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_int]
    arr = (C.c_uint32 * plan.nunits)()
    plan.ctx.check(f(plan.h, arr, plan.nunits))
    return list(arr)


def run(plan, blob, out_shape, fill=0xFF):
    """Run with the device buffer = blob + 64 bytes of `fill` (bytes behind a segment's in_size must
    not matter) and an output buffer filled like port.new_image's; -> (image, [(status, consumed)],
    [redo flag])."""
    import torch
    d_in = torch.from_numpy(np.concatenate([blob, np.full(64, fill, np.uint8)])).cuda()
    d_out = torch.from_numpy(np.full(int(np.prod(out_shape)), 0xA5A5, np.uint16).view(np.int16)).cuda()
    plan.run((d_in.data_ptr(), blob.size), d_out)
    torch.cuda.synchronize()
    res = plan.results(check=False)
    flags = redo_flags(plan)
    return d_out.cpu().numpy().view(np.uint16).reshape(out_shape), res, flags


def pentax_jobs(sizes, w, h, pitch, table_idx=0):
    """One job per (in_offset, in_size), images stacked vertically."""
    jobs = []
    for k, (o, n) in enumerate(sizes):
        j = rs.PentaxJob()
        j.in_offset, j.in_size, j.table, j.width, j.height = o, n, table_idx, w, h
        j.out_offset, j.out_pitch = k * h * pitch * 2, pitch * 2
        jobs.append(j)
    return jobs


def nikon_jobs(sizes, w, h, pitch, pup, lut=-1):
    jobs = []
    for k, (o, n) in enumerate(sizes):
        j = rs.NikonJob()
        j.in_offset, j.in_size, j.table, j.width, j.height = o, n, 0, w, h
        j.out_offset, j.out_pitch = k * h * pitch * 2, pitch * 2
        j.lut = lut
        for q in range(4):
            j.pup[q] = pup[q]
        jobs.append(j)
    return jobs


def pack(streams, align=64, skews=None):
    """Place streams one after the other, the k-th at an offset = skews[k] mod 16; gaps hold 0xA5."""
    offs, pos = [], 0
    for k, s in enumerate(streams):
        pos = (pos + align - 1) // align * align + (skews[k] if skews else 0)
        offs.append(pos)
        pos += len(s)
    blob = np.full(pos, 0xA5, np.uint8)
    for o, s in zip(offs, streams):
        blob[o:o + len(s)] = s
    return blob, offs


# ------------------------------------------------------------------ 1. ordinary streams: no redo
def _cr2_case(ctx, w, h, fmt, frame, slicing, toc, seed, hts=None, split_tables=False):
    img = port.new_image(w, h)
    img[:, :w] = synth.image_model(w, h, seed)
    hts = hts or synth.default_tables(2)
    blob = port.cr2_encode(img, w, fmt, frame, slicing, 14, hts, toc)
    want = port.new_image(w, h)
    port.cr2_ljpeg_decode(blob, want, w, slicing)
    tabs = TableSet()
    job = cr2_job(blob, w, h, fmt, slicing, want.shape[1] * 2, tabs)
    tables = tabs.tabs
    if split_tables:        # the same table under two indices (TableSet would merge them)
        assert len(tables) == 1
        tables = [tables[0], rs.huff_table(*parse_ljpeg(blob)["tables"][toc[0]])]
        for c in range(fmt[0]):
            job.table[c] = c % 2
    got, res, flags = run(rs.cr2_plan(ctx, tables, [job]), blob, want.shape)
    info = parse_ljpeg(blob)
    cons = port.cr2_decompress(port.new_image(w, h), w, fmt, (job.frame_w, job.frame_h),
                               (job.num_slices, job.slice_w, job.last_slice_w),
                               [hts[t] for t in toc], [1 << 13] * fmt[0], blob[info["data_off"]:])
    assert res[0] == (0, cons)
    assert np.array_equal(got, want)
    return flags[0]


@pytest.mark.parametrize("case", [
    (1440, 960, (2, 1, 1), (720, 960), (3, 480, 480), [0, 1], 5),
    (1440, 960, (4, 1, 1), (360, 960), (3, 480, 480), [0, 1, 0, 1], 6),
    (1440, 960, (2, 1, 1), (720, 960), (3, 480, 480), [0, 0], 7),
    (6720, 4480, (2, 1, 1), (3360, 4480), (3, 2240, 2240), [0, 1], 4),
    (6720, 4480, (4, 1, 1), (1680, 4480), (3, 2240, 2240), [0, 1, 0, 1], 4),
])
def test_cr2_frames_verify_without_a_redo(ctx, case):
    w, h, fmt, frame, slicing, toc, seed = case
    assert _cr2_case(ctx, w, h, fmt, frame, slicing, toc, seed) == 0


def _strip_case(ctx, img, tile_w, tile_h, **kw):
    h, w = img.shape
    t = synth.make_dng_ljpeg(img, tile_w, tile_h, **kw)
    want = port.new_image(w, h)
    port.dng_decompress(t.blob, t.offsets, t.lengths, want, w, 1, tile_w, tile_h, 7, nthreads=4)
    tabs, scans = dng_ljpeg_scans(t, want.shape[1] * 2)
    got, res, flags = run(rs.ljpeg_plan(ctx, tabs.tabs, scans), t.blob, want.shape)
    assert all(s == 0 for s, _ in res)
    assert np.array_equal(got, want)
    big = [k for k, s in enumerate(scans) if s.in_size > 256 << 10]
    assert big
    return [flags[k] for k in big]


def test_big_strips_verify_without_a_redo(ctx):
    """The cases of test_big_untiled_strip_multi_cta."""
    img = synth.image_model(2048, 700, 41)
    assert _strip_case(ctx, img, 2048, 700) == [0]
    assert _strip_case(ctx, img, 2048, 700, tabs=synth.default_tables(2), tab_of_comp=[0, 1]) == [0]
    assert _strip_case(ctx, img, 2048, 700, ncomp=4, tabs=synth.default_tables(2),
                       tab_of_comp=[0, 1, 1, 0]) == [0]
    wild = synth.image_model(1536, 512, 43, wild=True)
    assert _strip_case(ctx, wild, 1536, 512) == [0]
    assert set(_strip_case(ctx, wild, 768, 512, restart_rows=150)) == {0}


@pytest.mark.parametrize("w,h,wild", [(1000, 333, False), (6016, 4000, False), (640, 200, True),
                                      (2048, 1024, True)])
def test_pentax_streams_verify_without_a_redo(ctx, w, h, wild):
    meta = synth.pentax_modern_meta(True) if wild else None
    table = port.pentax_table(meta, True)
    if wild:
        img = np.random.default_rng(3).integers(0, 16384, (h, w), dtype=np.uint16)
    else:
        img = (synth.image_model(w, h, seed=11, bits=12) & 0x0FFF).astype(np.uint16)
    data = synth.make_pentax(img, table)
    pitch = port.image_pitch(w) // 2
    plan = rs.pentax_plan(ctx, [rs.huff_table(*table)], pentax_jobs([(0, data.size)], w, h, pitch))
    got, res, flags = run(plan, data, (h, pitch))
    assert res[0][0] == 0 and flags == [0]
    assert np.array_equal(got[:, :w], img)


@pytest.mark.parametrize("w,h", [(1026, 300), (6032, 4032)])
def test_nikon_streams_verify_without_a_redo(ctx, w, h):
    from test_gpu_nikon import _case
    meta, su, img, data = _case("table", 14, w, h, seed=7)
    want = port.new_image(w, h)
    port.nikon_decompress(want, w, meta, True, 14, data)
    ncpl, values = port.nikon_tree(su["huff_select"])
    pitch = want.shape[1]
    plan = rs.nikon_plan(ctx, [rs.huff_table(ncpl, values)],
                         nikon_jobs([(0, data.size)], w, h, pitch, su["pup"], lut=0),
                         port.build_table(su["curve"], True))
    got, res, flags = run(plan, data, want.shape)
    assert res[0][0] == 0 and flags == [0]
    assert np.array_equal(got, want)


# ------------------------------------------------------------------ 2. forced redo: positions
def test_cr2_forced_redo(ctx):
    """A one-slice two-component CR2 of about 1 MB coded with the mod-3 table."""
    import time
    w, h = 1600, 900
    img = port.new_image(w, h)
    img[:, :w] = ljpeg_image(np.random.default_rng(21), h, w, RICH)
    hts = [port.Huff(*T3), port.Huff(*T3)]
    fmt, frame, slicing = (2, 1, 1), (w // 2, h), (1, 0, w)
    blob = port.cr2_encode(img, w, fmt, frame, slicing, 14, hts, [0, 1])
    assert blob.size > 12 * RANGE_BYTES
    want = port.new_image(w, h)
    port.cr2_ljpeg_decode(blob, want, w, slicing)
    assert np.array_equal(want, img)
    tabs = TableSet()
    job = cr2_job(blob, w, h, fmt, slicing, want.shape[1] * 2, tabs)
    t0 = time.perf_counter()
    got, res, flags = run(rs.cr2_plan(ctx, tabs.tabs, [job]), blob, want.shape)
    print("forced redo, CR2 %d bytes: plan + upload + decode %.1f ms" % (blob.size, 1e3 * (time.perf_counter() - t0)))
    info = parse_ljpeg(blob)
    cons = port.cr2_decompress(port.new_image(w, h), w, fmt, frame, (job.num_slices, job.slice_w,
                               job.last_slice_w), hts, [1 << 13] * 2, blob[info["data_off"]:])
    assert flags == [1]
    assert res[0] == (0, cons)
    assert np.array_equal(got, want)


def _strip_blob(img, tabs, skew=0, pad=0):
    """One LJPEG strip of the whole image whose entropy data starts at an offset = skew mod 16, `pad`
    bytes of 0x5A behind its end."""
    h, w = img.shape
    t = synth.make_dng_ljpeg(img, w, h, tabs=tabs)
    lead = 64 + (skew - t.offsets[0] - parse_ljpeg(t.blob[t.offsets[0]:])["data_off"]) % 16
    blob = np.concatenate([np.zeros(lead, np.uint8), t.blob, np.full(pad, 0x5A, np.uint8)])
    offs = [o + lead for o in t.offsets]
    lens = [n + pad for n in t.lengths]
    return synth.DngTiles(blob, offs, lens, w, h, 1, w, h)


def _strip_outcome(ctx, t):
    """LJpegDecompressor (the oracle) and the plan on the one segment of strip t:
    -> (status, consumed, image), (status, consumed, image), redo flag, scan."""
    h, w = t.h, t.w
    tabs, scans = dng_ljpeg_scans(t, port.image_pitch(w))
    s = scans[0]
    info = parse_ljpeg(t.blob[t.offsets[0]:])
    hts = [port.Huff(*info["tables"][k]) for k in info["table_of_comp"]]
    want = port.new_image(w, h)
    cons = [None]

    def decode():
        cons[0] = port.ljpeg_decompress(want, w, 1, (s.out_x, s.out_y, s.store_w, s.rows), (2, 1),
                                        (s.frame_w, s.rows), hts, [1 << 13] * 2, s.rows,
                                        t.blob[s.in_offset:s.in_offset + s.in_size])
    st = _outcome(decode)
    got, res, flags = run(rs.ljpeg_plan(ctx, tabs.tabs, scans), t.blob, want.shape)
    return (st, cons[0], want), (res[0][0], res[0][1], got), flags[0], s


def test_strip_forced_redo(ctx):
    img = ljpeg_image(np.random.default_rng(22), 700, 1800, RICH)
    t = _strip_blob(img, [port.Huff(*T3)])
    (st, cons, want), (gst, gcons, got), flag, s = _strip_outcome(ctx, t)
    assert s.in_size > 12 * RANGE_BYTES
    assert st == 0 and np.array_equal(want[:, :1800], img)
    assert (gst, gcons, flag) == (0, cons, 1)
    assert np.array_equal(got, want)


def test_pentax_forced_redo(ctx):
    w, h = 1400, 1000
    meta = pentax_meta(LEN3)
    table = port.pentax_table(meta, True)
    assert (table[0], table[1]) == (T3[0], T3[1])
    img = pentax_image(np.random.default_rng(23), h, w, RICH)
    data = synth.make_pentax(img, table)
    assert data.size > 12 * RANGE_BYTES
    pitch = port.image_pitch(w) // 2
    plan = rs.pentax_plan(ctx, [rs.huff_table(*table)], pentax_jobs([(0, data.size)], w, h, pitch))
    got, res, flags = run(plan, data, (h, pitch))
    assert (res[0][0], flags) == (0, [1])
    st, want = oracle_pentax(data, w, h, meta)
    assert st == 0 and np.array_equal(want[:, :w], img)
    assert np.array_equal(got, want)


def test_nikon_forced_redo(ctx):
    w, h = 1400, 1000
    pup = [16000, 16010, 15990, 16020]
    d = nikon_diffs(np.random.default_rng(24), h, w, RICH, pup)
    data = port.encode_diffs_plain(d.reshape(-1), port.Huff(*T3))
    assert data.size > 12 * RANGE_BYTES
    pitch = port.image_pitch(w) // 2
    plan = rs.nikon_plan(ctx, [rs.huff_table(*T3)], nikon_jobs([(0, data.size)], w, h, pitch, pup), None)
    got, res, flags = run(plan, data, (h, pitch))
    assert (res[0][0], flags) == (0, [1])
    assert np.array_equal(got[:, :w], nikon_expected(d, pup))


def test_errors_inside_forced_redo_streams(ctx):
    """An unassigned code (the decode table leaves out SSSS 12, whose code 111111 is the only run of six
    one-bits in the stream) and a stream cut to half: the oracle's error class."""
    w, h = 1400, 1000
    # Pentax
    meta, meta_hole = pentax_meta(LEN3), pentax_meta(LEN3[:12])
    img = pentax_image(np.random.default_rng(25), h, w, PLAIN, hole_at=(900, 333))
    data = synth.make_pentax(img, port.pentax_table(meta, True))
    cut = data[:data.size // 2].copy()
    blob, offs = pack([data, cut, data[:data.size - 3 * RANGE_BYTES]])
    sizes = [(offs[0], data.size), (offs[1], cut.size), (offs[2], data.size - 3 * RANGE_BYTES)]
    pitch = port.image_pitch(w) // 2
    plan = rs.pentax_plan(ctx, [rs.huff_table(*port.pentax_table(meta_hole, True))],
                          pentax_jobs(sizes, w, h, pitch))
    got, res, flags = run(plan, blob, (3 * h, pitch))
    want = [oracle_pentax(blob[o:o + n], w, h, meta_hole)[0] for o, n in sizes]
    assert want == [1, 2, 2]
    assert [s for s, _ in res] == want
    assert flags == [1, 1, 1]
    # strip (JPEG pump): the DHT of the blob is patched so that SSSS 12 has a 16-bit code
    # (111111 0000000000); the stream's 111111 is followed by the extra bits 100000000000
    img = ljpeg_image(np.random.default_rng(26), 700, 1800, PLAIN, hole_at=(600, 1001))
    t = synth.make_dng_ljpeg(img, 1800, 700, tabs=[port.Huff(*T3)])
    blob = t.blob.copy()
    i = bytes(blob).index(bytes(T3[0]))
    assert blob[i + 5] == 2 and blob[i + 15] == 0
    blob[i + 5], blob[i + 15] = 1, 1
    for name, b, length, want in [("unassigned code", blob, t.lengths[0], 1),
                                  ("cut", t.blob, t.lengths[0] // 2, 2)]:
        tt = synth.DngTiles(b, t.offsets, [length], 1800, 700, 1, 1800, 700)
        (st, _, _), (gst, _, _), flag, _ = _strip_outcome(ctx, tt)
        assert (st, gst) == (want, want)
        assert flag == 1, name


# ------------------------------------------------------------------ 3. forced redo: phase only
def test_cr2_phase_only_redo(ctx):
    """Two components coded with the same table, passed under two table ids: every seam's position
    agrees, only P2's phase comparison can see that a range started at the wrong component."""
    assert _cr2_case(ctx, 1440, 960, (2, 1, 1), (720, 960), (3, 480, 480), [0, 0], 7,
                     split_tables=True) == 1


# ------------------------------------------------------------------ 4. range geometry
def _last_range_sizes(skew):
    """Segment sizes (bytes) for which the last of six 64 KiB ranges holds 1, 31, 32, 33 or 65536
    bytes, and the 256 KiB threshold of the multi-CTA path for LJPEG strips."""
    return [5 * RANGE_BYTES + last - skew for last in (1, 31, 32, 33, RANGE_BYTES)] + [256 << 10,
                                                                                        (256 << 10) + 1]


@pytest.mark.parametrize("redo", [False, True])
def test_pentax_range_geometry(ctx, redo):
    w, h = 1024, 256
    meta = pentax_meta(LEN3) if redo else None
    table = port.pentax_table(meta, True)
    if redo:
        img = pentax_image(np.random.default_rng(27), h, w, RICH)
    else:
        img = (synth.image_model(w, h, seed=27, bits=12) & 0x0FFF).astype(np.uint16)
    data = synth.make_pentax(img, table)
    assert 2 * RANGE_BYTES < data.size < 4 * RANGE_BYTES
    streams, skews = [], []
    for skew in range(16):
        for n in [data.size] + _last_range_sizes(skew):
            # garbage behind the stream: the reference never decodes it
            s = np.concatenate([data, np.random.default_rng(n).integers(0, 256, n - data.size, np.uint8)])
            streams.append(s)
            skews.append(skew)
    blob, offs = pack(streams, skews=skews)
    pitch = port.image_pitch(w) // 2
    plan = rs.pentax_plan(ctx, [rs.huff_table(*table)],
                          pentax_jobs([(o, s.size) for o, s in zip(offs, streams)], w, h, pitch))
    got, res, flags = run(plan, blob, (len(streams) * h, pitch))
    st, want = oracle_pentax(data, w, h, meta)
    assert st == 0 and np.array_equal(want[:, :w], img)
    for k, s in enumerate(streams):
        assert offs[k] % 16 == skews[k]
        assert res[k][0] == 0, (k, s.size, skews[k])
        assert np.array_equal(got[k * h:(k + 1) * h], want), (k, s.size, skews[k])
        assert flags[k] == (1 if redo else 0), (k, s.size, skews[k])


@pytest.mark.parametrize("skew", range(16))
def test_strip_range_geometry(ctx, skew):
    """in_offset & 15, last ranges of 1..65536 bytes (garbage behind the end marker), and the end
    marker in the halo chunk of the next range (data ending a few bytes after a range boundary)."""
    img = synth.image_model(1024, 195, 61)
    t0 = synth.make_dng_ljpeg(img, 1024, 195)
    data_len = t0.lengths[0] - parse_ljpeg(t0.blob[t0.offsets[0]:])["data_off"]   # entropy data + FFD9
    # the marker lies in the last chunk of range 2, which range 3 parses as its halo
    assert 3 * RANGE_BYTES - 8192 + 16 < data_len < 3 * RANGE_BYTES - 16
    for n in [data_len] + _last_range_sizes(skew):
        t = _strip_blob(img, None, skew=skew, pad=n - data_len)
        (st, cons, want), (gst, gcons, got), flag, s = _strip_outcome(ctx, t)
        assert (s.in_offset & 15, s.in_size) == (skew, n)
        assert (st, gst, gcons) == (0, 0, cons), n
        assert flag == 0 or s.in_size <= 256 << 10, n
        assert np.array_equal(got, want), n


# ------------------------------------------------------------------ 5. where plain streams end
def _cut_sweep(streams_of_cut, decode_jobs, oracle_of, nh, w, pitch):
    cuts = list(range(41))
    streams = [streams_of_cut(c) for c in cuts]
    blob, offs = pack(streams, skews=[c % 16 for c in cuts])
    plan = decode_jobs([(o, s.size) for o, s in zip(offs, streams)])
    got, res, flags = run(plan, blob, (len(cuts) * nh, pitch))
    summary = []
    for k, c in enumerate(cuts):
        st, want = oracle_of(streams[k])
        summary.append(st)
        assert res[k][0] == st, (c, res[k], st)
        if st == 0:
            assert np.array_equal(got[k * nh:(k + 1) * nh, :w], want[:, :w]), c
    return summary, flags


@pytest.mark.parametrize("w,h,redo", [(640, 64, False), (1000, 333, False), (1000, 333, True)])
def test_pentax_stream_ends(ctx, w, h, redo):
    meta = pentax_meta(LEN3) if redo else None
    table = port.pentax_table(meta, True)
    if redo:
        img = pentax_image(np.random.default_rng(w + h), h, w, RICH)
    else:
        img = (synth.image_model(w, h, seed=w + h, bits=12) & 0x0FFF).astype(np.uint16)
    data = synth.make_pentax(img, table)
    pitch = port.image_pitch(w) // 2
    summary, flags = _cut_sweep(
        lambda c: data[:data.size - c].copy(),
        lambda sizes: rs.pentax_plan(ctx, [rs.huff_table(*table)], pentax_jobs(sizes, w, h, pitch)),
        lambda s: oracle_pentax(s, w, h, meta), h, w, pitch)
    print("Pentax %dx%d: oracle outcome by cut:" % (w, h), summary)
    assert 0 in summary and 2 in summary
    if redo:
        assert set(flags[:summary.index(2)]) == {1}


@pytest.mark.parametrize("w,h,redo", [(640, 64, False), (1026, 300, False), (1000, 333, True)])
def test_nikon_stream_ends(ctx, w, h, redo):
    pitch = port.image_pitch(w) // 2
    if redo:
        # the mod-3 table is no Nikon tree: the expectation is the numpy restatement, the outcome
        # the oracle's MSB pump + Huffman decoder over the cut stream (IOException or every symbol)
        pup = [16000, 16010, 15990, 16020]
        ncpl, values = T3
        d = nikon_diffs(np.random.default_rng(w + h), h, w, RICH, pup)
        data = port.encode_diffs_plain(d.reshape(-1), port.Huff(ncpl, values))
        hu = port.Huff(ncpl, values)

        def oracle_of(s):
            got = []
            st = _outcome(lambda: got.append(hu.decode(s, w * h, port.MSB)))
            o = port.new_image(w, h)
            if st == 0:     # (the last differences of a cut stream may come from zero bits)
                o[:, :w] = nikon_expected(np.array(got[0]).reshape(h, w), pup)
            return st, o
        assert np.array_equal(oracle_of(data)[1][:, :w], nikon_expected(d, pup))
    else:
        from test_gpu_nikon import _case
        meta, su, img, data = _case("table", 14, w, h, seed=w)
        pup = su["pup"]
        ncpl, values = port.nikon_tree(su["huff_select"])

        def oracle_of(s):
            o = port.new_image(w, h)
            return _outcome(lambda: port.nikon_decompress(o, w, meta, True, 14, s, True)), o

    summary, flags = _cut_sweep(
        lambda c: data[:data.size - c].copy(),
        lambda sizes: rs.nikon_plan(ctx, [rs.huff_table(ncpl, values)], nikon_jobs(sizes, w, h, pitch, pup),
                                    None),
        oracle_of, h, w, pitch)
    print("Nikon %dx%d: oracle outcome by cut:" % (w, h), summary)
    assert 0 in summary and 2 in summary


# ------------------------------------------------------------------ 5b. data that ends at a chunk end
# A chunk of the range kernels holds the 8-byte carried tail plus 8192 raw bytes, so a final chunk may hold
# codes that start behind its 256 subsequences of 32 bytes: data (or an end marker) at chunk offsets
# 8176..8192, and for the plain pump the zero bits behind the data.
CHUNK = 8192
ZONE = set(range(CHUNK - 16, CHUNK)) | {0}          # chunk offsets of the end of the data


def _code_lengths(table):
    ncpl, values = table
    ln, k = {}, 0
    for l in range(16):
        for _ in range(ncpl[l]):
            ln[values[k]] = l + 1
            k += 1
    return ln


def _plain_sizes(d, table):
    """Bytes encode_diffs_plain writes for the first h rows of differences d, for every h."""
    ln = _code_lengths(table)
    a = np.abs(d)
    ssss = np.zeros(a.shape, np.int64)
    nz = a > 0
    ssss[nz] = np.floor(np.log2(a[nz])).astype(np.int64) + 1
    lut = np.array([ln.get(k, 0) + k for k in range(17)], np.int64)
    bits = np.cumsum(lut[ssss].sum(axis=1))
    return ((bits + 7) // 8 + 3) // 4 * 4 + 16


def _pentax_diffs(img):
    a = img.astype(np.int64)
    d = np.zeros(a.shape, np.int64)
    d[:, 2:] = a[:, 2:] - a[:, :-2]
    d[2:, :2] = a[2:, :2] - a[:-2, :2]
    d[:2, :2] = a[:2, :2]
    return d


def _nikon_img_diffs(img, pup):
    a = img.astype(np.int64)
    d = np.zeros(a.shape, np.int64)
    d[:, 2:] = a[:, 2:] - a[:, :-2]
    d[2:, :2] = a[2:, :2] - a[:-2, :2]
    for r in range(min(2, a.shape[0])):
        d[r, 0], d[r, 1] = a[r, 0] - pup[2 * r], a[r, 1] - pup[2 * r + 1]
    return d


def _rows_ending_at(sizes_of_w, chunk, lo=CHUNK + 8, hi=CHUNK + 23):
    """(w, h) for which the stream of h rows has chunk * 8192 + lo .. + hi bytes."""
    for w in range(64, 160, 2):
        sizes = sizes_of_w(w)
        hit = np.nonzero((sizes >= chunk * CHUNK + lo) & (sizes <= chunk * CHUNK + hi))[0]
        if hit.size:
            return w, int(hit[0]) + 1
    raise AssertionError("no image size ends in the window")


@pytest.mark.parametrize("codec", ["pentax", "nikon"])
@pytest.mark.parametrize("chunk", [0, 16, 20])     # one chunk; the last range's first chunk; mid range
def test_plain_streams_that_end_at_a_chunk_end(ctx, codec, chunk):
    """Cuts of 0..40 bytes at every in_offset & 15 of a stream of 8200..8215 bytes mod 8192: the data
    ends at every chunk offset around 8192, in a final chunk with a carried tail and without one."""
    h_max = 5000
    if codec == "pentax":
        table = port.pentax_table(None)
        imgs = {}

        def sizes_of_w(w):
            imgs[w] = (synth.image_model(w, h_max, seed=w, bits=12) & 0x0FFF).astype(np.uint16)
            return _plain_sizes(_pentax_diffs(imgs[w]), table)
        w, h = _rows_ending_at(sizes_of_w, chunk)
        img = imgs[w][:h]
        data = synth.make_pentax(img, table)

        def oracle_of(s):
            return oracle_pentax(s, w, h)

        def plan_of(sizes):
            return rs.pentax_plan(ctx, [rs.huff_table(*table)], pentax_jobs(sizes, w, h, pitch))
    else:
        meta, su, _, _ = __import__("test_gpu_nikon")._case("table", 14, 2, 2)
        pup, table = su["pup"], port.nikon_tree(su["huff_select"])
        imgs = {}

        def sizes_of_w(w):
            imgs[w] = (synth.image_model(w, h_max, seed=w, bits=14) & 0x3FFF).astype(np.uint16)
            return _plain_sizes(_nikon_img_diffs(imgs[w], pup), table)
        w, h = _rows_ending_at(sizes_of_w, chunk)
        img = imgs[w][:h]
        data = synth.make_nikon(img, su["huff_select"], pup)

        def oracle_of(s):
            o = port.new_image(w, h)
            return _outcome(lambda: port.nikon_decompress(o, w, meta, True, 14, s, True)), o

        def plan_of(sizes):
            return rs.nikon_plan(ctx, [rs.huff_table(*table)], nikon_jobs(sizes, w, h, pitch, pup), None)
    assert data.size // CHUNK == chunk + 1 and CHUNK + 8 <= data.size % CHUNK + CHUNK <= CHUNK + 23
    pitch = port.image_pitch(w) // 2
    cases = [(c, k) for c in range(41) for k in range(16)]
    streams = [data[:data.size - c].copy() for c, _ in cases]
    blob, offs = pack(streams, skews=[k for _, k in cases])
    got, res, flags = run(plan_of([(o, s.size) for o, s in zip(offs, streams)]), blob,
                          (len(cases) * h, pitch))
    want = {c: oracle_of(data[:data.size - c]) for c in range(41)}
    in_zone = 0
    for i, (c, k) in enumerate(cases):
        st, o = want[c]
        assert res[i][0] == st, (c, k, res[i], st)
        if st == 0:
            assert np.array_equal(got[i * h:(i + 1) * h, :w], o[:, :w]), (c, k)
            in_zone += (k + streams[i].size) % CHUNK in ZONE
    assert in_zone >= 8
    print("%s, %d bytes: outcome by cut" % (codec, data.size), [want[c][0] for c in range(41)])


def _search_rows(length_of, lo_h, hi_h, target_lo, target_hi):
    """First h in lo_h..hi_h whose length_of(h) % 8192 lies in target_lo..target_hi."""
    h = lo_h
    while h <= hi_h:
        n = length_of(h)
        if target_lo <= n % CHUNK <= target_hi:
            return h, n
        h += 1
    raise AssertionError("no image height puts the end marker in the window")


def test_strip_marker_at_a_chunk_end(ctx):
    """An untiled strip above 256 KiB whose end marker lies at chunk offsets 8161..8192 + every
    in_offset & 15: the last codes may start behind the 256 subsequences of the final chunk."""
    # differences of magnitude 1..3 under the default table: no FF byte, so no stuffing shortens the
    # final chunk's clean data (it holds the 8-byte tail + every byte up to the marker)
    w = 96
    img_all = ljpeg_image(np.random.default_rng(63), 12000, w, [1, 2, 3])

    def length_of(h):
        t = synth.make_dng_ljpeg(img_all[:h].copy(), w, h)
        return t.lengths[0] - parse_ljpeg(t.blob[t.offsets[0]:])["data_off"] - 2   # bytes before FFD9
    h0 = int((5 * RANGE_BYTES + CHUNK) / (length_of(2000) / 2000))   # near 5 ranges + 1 chunk
    h, n = _search_rows(length_of, h0 - 40, h0 + 1000, CHUNK - 31, CHUNK - 4)
    img = img_all[:h].copy()
    t = _strip_blob(img, None)
    data = t.blob[t.offsets[0]:t.offsets[0] + t.lengths[0]]
    assert int(np.count_nonzero(data[parse_ljpeg(data)["data_off"]:] == 0xFF)) == 1   # FFD9 only
    hits = 0
    for skew in range(16):
        for pad in (0, 100):
            t = _strip_blob(img, None, skew=skew, pad=pad)
            (st, cons, want), (gst, gcons, got), flag, s = _strip_outcome(ctx, t)
            assert s.in_size > 256 << 10
            assert (st, gst, gcons, flag) == (0, 0, cons, 0), (skew, pad)
            assert np.array_equal(got, want), (skew, pad)
            hits += (skew + n) % CHUNK in ZONE
    assert hits >= 2 * 8


@pytest.mark.parametrize("chunk", [0, 8])
def test_cr2_marker_at_a_chunk_end(ctx, chunk):
    """One-slice CR2 frames whose end marker lies at chunk offsets 8161..8192 + every in_offset & 15
    (a frame in one chunk; the first chunk of a second range)."""
    w = 16                        # about 15 bytes per row: every window of 28 bytes holds a row end
    full = port.new_image(w, 6000)
    full[:, :w] = synth.image_model(w, 6000, 65)
    hts = synth.default_tables(2)
    fmt, slicing = (2, 1, 1), (1, 0, w)

    def blob_of(h):
        img = full[:h].copy()
        return img, port.cr2_encode(img, w, fmt, (w // 2, h), slicing, 14, hts, [0, 1])

    def length_of(h):
        b = blob_of(h)[1]
        return b.size - parse_ljpeg(b)["data_off"] - 2

    per_row = length_of(400) / 400
    h0 = int(chunk * CHUNK / per_row) - 20
    h, n = _search_rows(length_of, max(2, h0), h0 + int(2 * CHUNK / per_row), CHUNK - 31, CHUNK - 4)
    while n // CHUNK < chunk:
        h, n = _search_rows(length_of, h + 1, h + int(2 * CHUNK / per_row), CHUNK - 31, CHUNK - 4)
    assert n // CHUNK == chunk
    img, blob = blob_of(h)
    want = port.new_image(w, h)
    port.cr2_ljpeg_decode(blob, want, w, slicing)
    assert np.array_equal(want, img)
    data_off = parse_ljpeg(blob)["data_off"]
    cons = port.cr2_decompress(port.new_image(w, h), w, fmt, (w // 2, h), slicing, hts, [1 << 13] * 2,
                               blob[data_off:])
    hits = 0
    for skew in range(16):
        lead = 64 + (skew - data_off) % 16
        b = np.concatenate([np.zeros(lead, np.uint8), blob])
        tabs = TableSet()
        job = cr2_job(blob, w, h, fmt, slicing, want.shape[1] * 2, tabs)
        job.in_offset += lead
        got, res, flags = run(rs.cr2_plan(ctx, tabs.tabs, [job]), b, want.shape)
        assert (res[0], flags) == ((0, cons), [0]), skew
        assert np.array_equal(got, want), skew
        hits += (skew + n) % CHUNK in ZONE
    assert hits >= 4


# ------------------------------------------------------------------ 6. small gaps
def test_pentax_out_of_bounds_far_from_range_0(ctx):
    """Values leave 0..65535 in several ranges and rows; the first one in stream order lies far from
    range 0 and must win over a later one that an earlier range holds no part of."""
    w, h = 1024, 512
    table = port.pentax_table(None)
    img = (synth.image_model(w, h, seed=5, bits=12) & 0x0FFF).astype(np.int64)
    d = np.zeros((h, w), np.int64)
    d[:, 2:] = img[:, 2:] - img[:, :-2]
    d[2:, :2] = img[2:, :2] - img[:-2, :2]
    d[:2, :2] = img[:2, :2]
    for (r, c) in [(300, 500), (301, 7), (400, 2), (511, 1000)]:
        d[r, c] = -4000              # values below 3100 minus 4000: below 0 (SSSS 12)
    data = port.encode_diffs_plain(d.reshape(-1), port.Huff(*table))
    assert data.size > 3 * RANGE_BYTES
    with pytest.raises(port.RawDecoderException) as ei:
        port.pentax_decompress(port.new_image(w, h), w, data)
    pitch = port.image_pitch(w) // 2
    plan = rs.pentax_plan(ctx, [rs.huff_table(*table)], pentax_jobs([(0, data.size)], w, h, pitch))
    got, res, flags = run(plan, data, (h, pitch))
    from rawspeed_b200 import _abi
    assert res[0] == (_abi.ERR_RDE, _abi.PENTAX_OOB | (300 << 14) | 500)
    assert "500:300" in ei.value.msg


def test_nikon_two_images_two_luts_unaligned(ctx):
    """Two Nikon images in one plan, each with its own curve, the second at an unaligned in_offset:
    the dither seed is read at in + in_offset."""
    from test_gpu_nikon import _case
    w, h = 1026, 300
    cases = [_case("table", 14, w, h, seed=3), _case("table", 12, w, h, seed=4)]
    blob, offs = pack([c[3] for c in cases], skews=[3, 13])
    wants, jobs, luts = [], [], []
    pitch = port.image_pitch(w) // 2
    for k, (meta, su, img, data) in enumerate(cases):
        want = port.new_image(w, h)
        port.nikon_decompress(want, w, meta, True, 14 if k == 0 else 12, data)
        wants.append(want)
        j = nikon_jobs([(offs[k], data.size)], w, h, pitch, su["pup"], lut=k)[0]
        j.table = k
        j.out_offset = k * h * pitch * 2
        jobs.append(j)
        luts.append(port.build_table(su["curve"], True))
    tables = [rs.huff_table(*port.nikon_tree(c[1]["huff_select"])) for c in cases]
    plan = rs.nikon_plan(ctx, tables, jobs, np.concatenate(luts))
    got, res, flags = run(plan, blob, (2 * h, pitch))
    assert [s for s, _ in res] == [0, 0] and flags == [0, 0]
    assert np.array_equal(got[:h], wants[0]) and np.array_equal(got[h:], wants[1])
