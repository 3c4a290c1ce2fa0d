"""K1 (unpack_fast_kernel / unpack_kernel) and K1b (rawform_kernel) on every path the plan
can dispatch to, against the oracle (port.unpack / port.unpack_form), byte for byte over the
WHOLE output buffer.

The output buffer is filled with random sentinel bytes, each job is placed at a chosen
out_offset / out_pitch / row0 / out_col0, and the expected buffer is the same sentinel
buffer with the oracle's rows copied into each job's footprint.  So a case fails on a wrong
value, on a byte the kernel should have written and did not, and on a byte written outside
the footprint (row padding, the columns before out_col0, the bytes between jobs).

Every case asserts the kernels its plan launches (Plan.kernels, Plan.launches), so a change of
the dispatch rule cannot silently move it off the branch it was written for.  Layouts the
kernels cannot store to (odd output offsets or pitches) are only ever plan-creation refusals;
none is launched."""
import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import formats as F
from oracle import port, synth
from helpers import dng_ljpeg_scans

pytestmark = pytest.mark.gpu

ORDERS = [rs.LSB, rs.MSB, rs.MSB16, rs.MSB32]
ORDER_NAME = {rs.LSB: "LSB", rs.MSB: "MSB", rs.MSB16: "MSB16", rs.MSB32: "MSB32"}
TAIL = 37        # input bytes after the last strip (random: bytes past in_size must read as 0)
OUT_SLACK = 48   # output bytes after the last footprint


@pytest.fixture(scope="module")
def uctx():
    c = rs.Context(0)
    yield c
    c.close()


def _r16(x):
    return (x + 15) // 16 * 16


def _r4(x):
    return (x + 3) // 4 * 4


# ---------------------------------------------------------------------------------------
# harness
# ---------------------------------------------------------------------------------------
class Foot:
    """Where one job's rows land: rows x (samples * sb) bytes at out_offset + (row0 + r) *
    out_pitch + col0 * sb."""

    def __init__(self, out_offset, out_pitch, row0, col0, rows, samples, sb):
        self.out_offset, self.out_pitch, self.row0, self.col0 = out_offset, out_pitch, row0, col0
        self.rows, self.samples, self.sb = rows, samples, sb

    def row_start(self, r):
        return self.out_offset + (self.row0 + r) * self.out_pitch + self.col0 * self.sb

    @property
    def end(self):
        return self.row_start(self.rows - 1) + self.samples * self.sb

    def place(self, buf, rows_u8):
        n = self.samples * self.sb
        for r in range(self.rows):
            a = self.row_start(r)
            buf[a:a + n] = rows_u8[r, :n]

    def mask(self, nbytes):
        m = np.zeros(nbytes, dtype=bool)
        n = self.samples * self.sb
        for r in range(self.rows):
            a = self.row_start(r)
            m[a:a + n] = True
        return m

    def where(self, off):
        rel = off - self.out_offset
        row, cb = divmod(rel, self.out_pitch)
        col = cb // self.sb - self.col0
        inside = (self.row0 <= row < self.row0 + self.rows and 0 <= col < self.samples)
        return row, col, inside


def assert_same(got, want, feet, what, mask=None):
    """Byte compare (optionally only where mask is set); on failure name the first differing
    offset, its row and sample column in the job that owns it, and whether it lies inside
    that job's footprint."""
    diff = got != want
    if mask is not None:
        diff &= mask
    if not diff.any():
        return
    off = int(np.flatnonzero(diff)[0])
    desc = []
    for k, f in enumerate(feet):
        row, col, inside = f.where(off)
        if inside:
            desc = ["job %d row %d col %d, inside the footprint" % (k, row, col)]
            break
        desc.append("job %d: row %d col %d" % (k, row, col))
    else:
        desc.insert(0, "outside every footprint")
    raise AssertionError("%s: %d bytes differ; first at byte %d (got 0x%02x want 0x%02x): %s" % (
        what, int(diff.sum()), off, got[off], want[off], "; ".join(desc)))


def dev_run(plan, in_buf, out_buf):
    """plan.run on device copies of in_buf / out_buf (the input readable 64 bytes past its
    end, as plan_run requires); returns the output buffer."""
    import torch
    d_in = torch.zeros(in_buf.size + 64, dtype=torch.uint8, device="cuda")
    d_in[:in_buf.size] = torch.from_numpy(in_buf)
    d_out = torch.from_numpy(out_buf.copy()).cuda()
    plan.run((d_in.data_ptr(), in_buf.size), d_out)
    torch.cuda.synchronize()
    plan.results()
    return d_out.cpu().numpy()


def sentinel(n, rng):
    return rng.integers(0, 256, n, dtype=np.uint8)


# ---------------------------------------------------------------------------------------
# K1: packed unpack
# ---------------------------------------------------------------------------------------
class U:
    """One unpack job: geometry, input placement (in_res: in_offset mod 16 after the previous
    strip), output layout (out_offset absolute)."""

    def __init__(self, samples, rows, bps, order, in_pitch=None, in_res=0, out_offset=0,
                 out_pitch=None, row0=0, col0=0):
        self.samples, self.rows, self.bps, self.order = samples, rows, bps, order
        self.row_bytes = samples * bps // 8
        assert samples * bps % 8 == 0
        self.in_pitch = in_pitch or self.row_bytes
        self.in_res = in_res
        self.foot = Foot(out_offset, out_pitch or _r16(2 * (col0 + samples)), row0, col0, rows,
                         samples, 2)

    def fast(self):
        return (self.bps in (8, 10, 12, 14, 16) and self.in_offset % 4 == 0 and
                self.in_pitch % 4 == 0 and (self.samples + 15) // 16 >= 64)

    def vec_ok(self):
        f = self.foot
        return f.out_offset % 16 == 0 and f.out_pitch % 16 == 0 and f.col0 % 8 == 0


def _unpack_inputs(specs, rng):
    pos = 0
    strips = []
    for s in specs:
        s.in_offset = _r16(pos) + s.in_res
        s.in_size = s.rows * s.in_pitch
        strips.append((s.in_offset, sentinel(s.in_size, rng)))
        pos = s.in_offset + s.in_size
    buf = sentinel(pos + TAIL, rng)
    for off, st in strips:
        buf[off:off + st.size] = st
    return buf


def _ujob(s):
    j = rs.UnpackJob()
    j.in_offset, j.in_size, j.out_offset = s.in_offset, s.in_size, s.foot.out_offset
    j.out_pitch, j.row0, j.rows, j.samples = s.foot.out_pitch, s.foot.row0, s.rows, s.samples
    j.out_col0, j.in_pitch, j.bps, j.order = s.foot.col0, s.in_pitch, s.bps, s.order
    return j


def _unpack_oracle(s, in_buf):
    strip = in_buf[s.in_offset:s.in_offset + s.in_size]
    img = port.new_image(s.samples, s.rows)
    port.unpack(strip, img, s.samples, 1, (0, 0, s.samples, s.rows), s.in_pitch, s.bps, s.order)
    return img.view(np.uint8)


def unpack_case(ctx, specs, kernels, launches, seed, what):
    """Build, run and check one unpack plan."""
    rng = np.random.default_rng(seed)
    in_buf = _unpack_inputs(specs, rng)
    nout = max(s.foot.end for s in specs) + OUT_SLACK
    out0 = sentinel(nout, rng)
    want = out0.copy()
    for s in specs:
        s.foot.place(want, _unpack_oracle(s, in_buf))
    plan = rs.unpack_plan(ctx, [_ujob(s) for s in specs])
    assert plan.kernels == kernels, (what, plan.kernels)
    assert plan.launches == launches, (what, plan.launches)
    got = dev_run(plan, in_buf, out0)
    assert_same(got, want, [s.foot for s in specs], what)


def _tail_samples(bps):
    # a row length whose last 16-sample item is partial (samples % 16 != 0), 65 items
    return 1036 if bps in (8, 10, 14, 16) else 1034


# name -> (samples(bps), rows, in_pitch(row_bytes), out layout(samples) -> (off, pitch, row0, col0))
FAST_VARIANTS = {
    # 64 items per row (the threshold): a CTA's 512 items are exactly 8 rows; tight input
    "ipr64_tight_vec": (lambda b: 1024, 20, lambda rb: rb,
                        lambda n: (0, _r16(2 * n), 0, 0)),
    # 65 items: a CTA spans 9 rows; padded input pitch, row0 / out_col0 > 0, 128-bit stores
    "ipr65_padded_vec_row0_col0": (lambda b: 1040, 20, lambda rb: rb + 12,
                                   lambda n: (32, _r16(2 * (8 + n)) + 16, 3, 8)),
    # partial last item; padded pitch; only 2-aligned out_offset -> 16-bit stores
    "tail_padded_offset2": (_tail_samples, 19, lambda rb: _r4(rb) + 8,
                            lambda n: (18, _r16(2 * n) + 16, 2, 0)),
    # 16-bit stores because the pitch is only 2-aligned
    "ipr64_tight_pitch2": (lambda b: 1024, 17, lambda rb: rb,
                           lambda n: (16, _r16(2 * n) + 2, 1, 0)),
    # 16-bit stores because out_col0 is odd
    "ipr65_tight_col0_odd": (lambda b: 1040, 18, lambda rb: rb,
                             lambda n: (0, _r16(2 * (5 + n)), 4, 5)),
}


@pytest.mark.parametrize("variant", list(FAST_VARIANTS) + ["ipr63_generic_control"])
@pytest.mark.parametrize("order", ORDERS, ids=[ORDER_NAME[o] for o in ORDERS])
@pytest.mark.parametrize("bps", [8, 10, 12, 14, 16])
def test_fast_kernel_instantiations(uctx, bps, order, variant):
    """Every unpack_fast_kernel<BPS, LSB/MSB-family> instantiation on each condition of its
    body: 8 and 9 rows per CTA, the partial last item, padded input pitch (seg_delta),
    row0 / out_col0 > 0, both store branches; 63 items per row stays on unpack_kernel."""
    if variant == "ipr63_generic_control":
        samples, rows, pitch, lay = 1008, 20, (lambda rb: rb), (lambda n: (16, _r16(2 * n), 1, 0))
    else:
        samples, rows, pitch, lay = FAST_VARIANTS[variant]
        samples = samples(bps)
    off, opitch, row0, col0 = lay(samples)
    rb = samples * bps // 8
    s = U(samples, rows, bps, order, in_pitch=pitch(rb), out_offset=off, out_pitch=opitch,
          row0=row0, col0=col0)
    s.in_offset = 0
    fast = s.fast()
    assert fast == (variant != "ipr63_generic_control")
    if variant in ("ipr64_tight_vec", "ipr65_padded_vec_row0_col0"):
        assert s.vec_ok()
    elif fast:
        assert not s.vec_ok()
    if variant == "tail_padded_offset2":
        assert samples % 16 and s.in_pitch > rb
    unpack_case(uctx, [s], "unpack_fast_kernel" if fast else "unpack_kernel", 1,
                seed=bps * 100 + order * 10 + len(variant), what=(bps, ORDER_NAME[order], variant))


def test_fast_kernel_several_jobs(uctx):
    """Seven jobs in one plan: five fast jobs of different widths, bit depths and orders in
    two fast buckets (<12, MSB family> and <14, LSB>), jobs that end inside their last CTA's
    item range and jobs that end on a CTA boundary, plus two generic jobs.  Every job is
    checked."""
    specs = [
        U(1040, 9, 12, rs.MSB, in_res=0, row0=0),                    # 585 items: ends inside CTA 2
        U(1024, 16, 12, rs.MSB32, in_pitch=1540, in_res=4, row0=9),   # 1024 items: 2 whole CTAs
        U(2000, 7, 12, rs.MSB16, in_res=8, row0=25, col0=8),          # 875 items
        U(1100, 11, 14, rs.LSB, in_pitch=1928, in_res=12, row0=32, col0=3),  # 759 items
        U(1024, 8, 14, rs.LSB, in_res=0, row0=43),                   # 512 items: one whole CTA
        U(1000, 5, 14, rs.LSB, in_res=0, row0=51),                   # 63 items: generic
        U(9000, 2, 13, rs.MSB, in_res=3, row0=56),                   # odd depth, 2 chunks: generic
    ]
    W = 9000
    pitch = _r16(2 * (W + 8))
    for s in specs:
        s.foot.out_pitch = pitch
        s.foot.out_offset = 16
    # one output image, each job on its own rows
    # launches: fast buckets <12, MSB family> and <14, LSB>, generic buckets <14, LSB> and
    # <any depth, MSB>
    unpack_case(uctx, specs, "unpack_fast_kernel + unpack_kernel", 4, seed=7, what="several jobs")
    assert [s.fast() for s in specs] == [True] * 5 + [False] * 2


# generic kernel: (samples, rows, bps, in_pitch(row_bytes), in_res)
GENERIC_CASES = {
    # > 8192 samples: 2 chunks (1025 groups of 8 -> 513 + 512) and 3 chunks (2053 groups ->
    # 685 + 685 + 683); chunk seams at 513 / 685 groups * bps bytes, not word multiples
    "bps13_2chunks": (8200, 3, 13, lambda rb: rb, 0),
    "bps13_3chunks": (16424, 3, 13, lambda rb: rb + 3, 0),
    "bps7_2chunks": (8200, 3, 7, lambda rb: rb, 0),
    "bps7_3chunks": (16424, 2, 7, lambda rb: rb + 1, 0),
    "bps1_2chunks": (8200, 4, 1, lambda rb: rb, 0),
    "bps1_3chunks": (16424, 3, 1, lambda rb: rb + 5, 0),
    # a fast-eligible depth pushed onto the generic kernel by the input layout
    "bps14_odd_in_offset_2chunks": (8204, 3, 14, lambda rb: _r4(rb), 3),
    "bps14_odd_in_pitch_2chunks": (8204, 3, 14, lambda rb: rb + 2, 0),
    "bps14_odd_in_offset_1chunk": (4000, 5, 14, lambda rb: rb, 1),
    "bps14_odd_in_pitch_3chunks": (16420, 2, 14, lambda rb: rb, 0),  # tight: 28735 bytes
}


@pytest.mark.parametrize("layout", ["vec", "offset2_col0"])
@pytest.mark.parametrize("order", ORDERS, ids=[ORDER_NAME[o] for o in ORDERS])
@pytest.mark.parametrize("case", list(GENERIC_CASES))
def test_generic_kernel_wide_rows(uctx, case, order, layout):
    """unpack_kernel on rows of 1, 2 and 3 chunks; in_size is exactly rows * in_pitch, so the
    last words of the strip are zero-filled (the bytes after it in the buffer are random)."""
    samples, rows, bps, pitch, in_res = GENERIC_CASES[case]
    rb = samples * bps // 8
    if layout == "vec":
        off, opitch, row0, col0 = 32, _r16(2 * samples) + 16, 1, 0
    else:
        off, opitch, row0, col0 = 2, _r16(2 * (samples + 3)) + 2, 2, 3
    s = U(samples, rows, bps, order, in_pitch=pitch(rb), in_res=in_res, out_offset=off,
          out_pitch=opitch, row0=row0, col0=col0)
    s.in_offset = in_res
    assert not s.fast()
    if "odd_in_pitch" in case:
        assert s.in_pitch % 2 == 1
    if "odd_in_offset" in case:
        assert s.in_offset % 2 == 1
    assert s.vec_ok() == (layout == "vec")
    groups = (samples + 7) // 8
    nchunks = int(case.split("_")[-1][0])
    assert (groups + 1023) // 1024 == nchunks
    assert nchunks == 1 or ((groups + nchunks - 1) // nchunks * bps) % 4   # seam inside a word
    seed = 1000 * list(GENERIC_CASES).index(case) + 10 * order + (layout == "vec")
    unpack_case(uctx, [s], "unpack_kernel", 1, seed=seed, what=(case, ORDER_NAME[order], layout))


# ---------------------------------------------------------------------------------------
# K1b: raw forms
# ---------------------------------------------------------------------------------------
CURVE = ((np.arange(256, dtype=np.uint32) * 977 + 13) % 65536).astype(np.uint16)
TABLE = port.build_table(CURVE, False)

# format -> (oracle bps, order, form, output sample bytes, samples per item)
FORMS = {
    F.RAW_8BIT: (8, port.LSB, port.FORM_8BIT_UNCORRECTED, 2, 8),
    F.RAW_8BIT_TABLE: (8, port.LSB, port.FORM_8BIT, 2, 8),
    F.RAW_12BIT_CONTROL_BE: (12, port.MSB, port.FORM_12BIT_CONTROL_BE, 2, 10),
    F.RAW_12BIT_CONTROL_LE: (12, port.MSB, port.FORM_12BIT_CONTROL_LE, 2, 10),
    F.RAW_12BIT_LEFT_BE: (16, port.LSB, port.FORM_12BIT_LEFT_BE, 2, 8),
    F.RAW_12BIT_LEFT_LE: (16, port.LSB, port.FORM_12BIT_LEFT_LE, 2, 8),
    F.RAW_FP16_MSB: (16, port.MSB, port.FORM_READ, 4, 4),
    F.RAW_FP16_LSB: (16, port.LSB, port.FORM_READ, 4, 4),
    F.RAW_FP24_MSB: (24, port.MSB, port.FORM_READ, 4, 4),
    F.RAW_FP24_LSB: (24, port.LSB, port.FORM_READ, 4, 4),
    F.RAW_F32_COPY: (32, port.LSB, port.FORM_READ, 4, 4),
}


def _form_pitch(fmt, w):
    """Input bytes between rows: the fixed layouts have one (decode8BitRaw: w, 12-bit control:
    perline, left aligned: 2w); the float forms take any pitch (padded here, odd)."""
    bps = FORMS[fmt][0]
    if fmt in (F.RAW_8BIT, F.RAW_8BIT_TABLE):
        return w
    if fmt in (F.RAW_12BIT_CONTROL_BE, F.RAW_12BIT_CONTROL_LE):
        return 12 * w // 8 + (w + 2) // 10
    if fmt in (F.RAW_12BIT_LEFT_BE, F.RAW_12BIT_LEFT_LE):
        return 2 * w
    return w * bps // 8 + 3


class R:
    def __init__(self, fmt, w, rows, in_res=0, out_offset=0, out_pitch=None, row0=0, col0=0):
        self.fmt, self.samples, self.rows, self.in_res = fmt, w, rows, in_res
        self.in_pitch = _form_pitch(fmt, w)
        sb = FORMS[fmt][3]
        self.foot = Foot(out_offset, out_pitch or _r16(sb * (col0 + w)), row0, col0, rows, w, sb)


def _raw_oracle(s, in_buf):
    bps, order, form, sb, _ = FORMS[s.fmt]
    strip = in_buf[s.in_offset:s.in_offset + s.in_size]
    w = s.samples
    img = port.new_image(w, s.rows) if sb == 2 else port.new_image_f32(w, s.rows)
    port.unpack_form(strip, img, w, 1, (0, 0, w, s.rows), s.in_pitch, bps, order, form,
                     TABLE if s.fmt == F.RAW_8BIT_TABLE else None)
    return img.view(np.uint8)


def _rjob(s):
    j = rs.RawJob()
    j.in_offset, j.in_size, j.out_offset = s.in_offset, s.in_size, s.foot.out_offset
    j.out_pitch, j.row0, j.rows, j.samples = s.foot.out_pitch, s.foot.row0, s.rows, s.samples
    j.out_col0, j.in_pitch, j.format, j.table = s.foot.col0, s.in_pitch, s.fmt, 0
    return j


def raw_build(specs, rng):
    """(in_buf, out0, want, jobs) of one raw-form plan."""
    in_buf = _unpack_inputs(specs, rng)
    nout = max(s.foot.end for s in specs) + OUT_SLACK
    out0 = sentinel(nout, rng)
    want = out0.copy()
    for s in specs:
        s.foot.place(want, _raw_oracle(s, in_buf))
    return in_buf, out0, want, [_rjob(s) for s in specs]


def raw_plan(ctx, jobs):
    uses_table = any(j.format == F.RAW_8BIT_TABLE for j in jobs)
    return rs.raw_plan(ctx, jobs, TABLE if uses_table else None)


# widths with a partial last item: 8-sample items (45, 21), 10-sample items (46, 62: even, as
# the 12-bit control forms need), 4-sample items (23, 22)
FORM_WIDTHS = {8: (45, 21), 10: (46, 62), 4: (23, 22)}


@pytest.mark.parametrize("fmt", list(FORMS), ids=["f%d" % f for f in FORMS])
def test_rawform_store_branches(uctx, fmt):
    """rawform_kernel<FORMAT> with out_offset at every multiple of the output sample size mod 16
    and an out_pitch that is sample size mod 16 (consecutive rows change store branch: 128-bit,
    32-bit words, 16-bit halves), every in_offset & 3, a partial last item per row."""
    sb, K = FORMS[fmt][3], FORMS[fmt][4]
    widths = FORM_WIDTHS[K]
    n = 0
    for wi, w in enumerate(widths):
        assert w % K
        col0, row0 = (0, 0) if wi == 0 else (3, 2)
        for k in range(16 // sb):
            for in_res in range(4):
                out_offset = 16 + k * sb
                pitch = _r16(sb * (col0 + w)) + 16 + sb
                s = R(fmt, w, 5, in_res=in_res, out_offset=out_offset, out_pitch=pitch,
                      row0=row0, col0=col0)
                rng = np.random.default_rng(1000 * fmt + n)
                n += 1
                in_buf, out0, want, jobs = raw_build([s], rng)
                plan = raw_plan(uctx, jobs)
                assert plan.kernels == "rawform_kernel" and plan.launches == 1
                got = dev_run(plan, in_buf, out0)
                assert_same(got, want, [s.foot], ("format", fmt, "w", w, "out_offset", out_offset,
                                                   "in_offset", s.in_offset))


@pytest.mark.parametrize("w", [10, 20, 30, 40, 100, 250])
def test_rawform_12bit_control_item_residues(uctx, w):
    """12-bit control forms: 20-byte items start at every dst & 15 residue (even ones) across
    the rows of one plan; widths of whole items."""
    specs = []
    off = 0
    for fmt in (F.RAW_12BIT_CONTROL_BE, F.RAW_12BIT_CONTROL_LE):
        for k in range(8):
            s = R(fmt, w, 3, in_res=k % 4, out_offset=off + 2 * k,
                  out_pitch=_r16(2 * w) + 16 + 2 * (k | 1))
            specs.append(s)
            off = _r16(s.foot.end) + 32
    rng = np.random.default_rng(w)
    in_buf, out0, want, jobs = raw_build(specs, rng)
    plan = raw_plan(uctx, jobs)
    assert plan.kernels == "rawform_kernel" and plan.launches == 2
    got = dev_run(plan, in_buf, out0)
    assert_same(got, want, [s.foot for s in specs], ("12-bit control", w))


def _all_forms_specs():
    specs = []
    off = 0
    for i, fmt in enumerate(FORMS):
        sb, K = FORMS[fmt][3], FORMS[fmt][4]
        w = FORM_WIDTHS[K][i % 2]
        s = R(fmt, w, 4 + i % 3, in_res=i % 4, out_offset=off + (i * sb) % 16,
              out_pitch=_r16(sb * (w + 2)) + sb, row0=i % 2, col0=2 if i % 3 == 0 else 0)
        specs.append(s)
        off = _r16(s.foot.end) + 16
    return specs


def test_rawform_one_plan_every_format(uctx):
    specs = _all_forms_specs()
    in_buf, out0, want, jobs = raw_build(specs, np.random.default_rng(11))
    plan = raw_plan(uctx, jobs)
    assert plan.kernels == "rawform_kernel" and plan.launches == 11
    got = dev_run(plan, in_buf, out0)
    assert_same(got, want, [s.foot for s in specs], "every format")


# ---------------------------------------------------------------------------------------
# rsb200_plan_run_host: host buffers (pinned and pageable), pipelined and not
# ---------------------------------------------------------------------------------------
def host_buf(arr, pinned):
    """(copy of arr, owner): ordinary (pageable) host memory, or page-locked memory of a pinned
    torch tensor (the owner, to be kept alive while the array is in use)."""
    if not pinned:
        return arr.copy(), None
    import torch
    t = torch.empty(arr.size, dtype=torch.uint8, pin_memory=True)
    h = t.numpy()
    h[:] = arr
    return h, t


def _frames():
    # four 14-bit MSB frames, disjoint increasing input and output spans (one fast bucket):
    # the multi-stream pipeline takes such a plan unless `partial` is set
    specs = []
    off = 0
    for k in range(4):
        s = U(1040 + 16 * k, 10 + k, 14, rs.MSB, in_pitch=(1040 + 16 * k) * 14 // 8 + 16 + 4 * k,
              in_res=0, out_offset=off, out_pitch=_r16(2 * (1040 + 16 * k + 8)) + 16, row0=1,
              col0=8)
        specs.append(s)
        off = _r16(s.foot.out_offset + (s.foot.row0 + s.rows) * s.foot.out_pitch) + 64
    return specs


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_run_host_unpack_pipeline_and_partial(uctx, pinned):
    """The same plan through the multi-stream pipeline (partial=False: one sub-launch per
    frame, each with its own block_base) and through the plain path (partial=True)."""
    specs = _frames()
    rng = np.random.default_rng(21 + pinned)
    in_buf = _unpack_inputs(specs, rng)
    nout = max(s.foot.end for s in specs) + OUT_SLACK
    plan = rs.unpack_plan(uctx, [_ujob(s) for s in specs])
    assert plan.kernels == "unpack_fast_kernel" and plan.launches == 1
    feet = [s.foot for s in specs]
    fp = np.zeros(nout, dtype=bool)
    for f in feet:
        fp |= f.mask(nout)
    for partial in (False, True):
        # fresh input and output bytes for every run: the library's device buffers persist
        # between runs, so whatever a path fails to upload, decode or download there holds
        # the previous run's (different) results and cannot match
        in_buf = _unpack_inputs(specs, rng)
        out0 = sentinel(nout, rng)
        want = out0.copy()
        for s in specs:
            s.foot.place(want, _unpack_oracle(s, in_buf))
        h_in, t_in = host_buf(in_buf, pinned)
        h_out, t_out = host_buf(out0, pinned)
        before = uctx.launches
        plan.run_host(h_in, h_out, partial=partial)
        # the pipeline launches the kernel once per frame, the plain path once per plan
        assert uctx.launches - before == (1 if partial else len(specs)), partial
        # with partial=False the bytes outside the footprint are undefined
        assert_same(h_out, want, feet, ("run_host", "partial" if partial else "pipelined"),
                    mask=None if partial else fp)
        del t_in, t_out


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_run_host_rawforms(uctx, pinned):
    specs = _all_forms_specs()
    rng = np.random.default_rng(31 + pinned)
    in_buf, out0, want, jobs = raw_build(specs, rng)
    plan = raw_plan(uctx, jobs)
    feet = [s.foot for s in specs]
    fp = np.zeros(out0.size, dtype=bool)
    for f in feet:
        fp |= f.mask(out0.size)
    for partial in (False, True):
        if partial:  # fresh bytes: nothing the previous run left on the device can match
            in_buf, out0, want, jobs2 = raw_build(specs, rng)
            assert all(bytes(a) == bytes(b) for a, b in zip(jobs, jobs2))
        h_in, t_in = host_buf(in_buf, pinned)
        h_out, t_out = host_buf(out0, pinned)
        before = uctx.launches
        plan.run_host(h_in, h_out, partial=partial)
        assert uctx.launches - before == 11
        assert_same(h_out, want, feet, ("run_host raw forms", partial),
                    mask=None if partial else fp)
        del t_in, t_out


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_run_host_ljpeg_tile_pipeline(uctx, pinned, monkeypatch):
    """An LJPEG plan of tile-kernel segments in two or more groups (1 MB of output each):
    run_host pipelines the groups (one launch per group) and gives what plan.run gives."""
    import torch
    monkeypatch.setenv("RSB200_GROUP_MB", "1")
    monkeypatch.delenv("RSB200_LJPEG_PATH", raising=False)
    W, H = 1024, 1024
    # a different image per parameter: the library's device buffers persist between runs, so a
    # group the pipeline fails to upload, decode or download there holds the other image
    img = synth.image_model(W, H, 4242 + pinned)
    t = synth.make_dng_ljpeg(img, 256, 256)
    pitch = port.image_pitch(W)
    tabs, scans = dng_ljpeg_scans(t, pitch)
    plan = rs.ljpeg_plan(uctx, tabs.tabs, scans)
    assert plan.kernels.startswith("k2_tile_kernel"), plan.kernels
    out0 = sentinel(pitch * H, np.random.default_rng(5))
    d_in = torch.zeros(t.blob.size + 64, dtype=torch.uint8, device="cuda")
    d_in[:t.blob.size] = torch.from_numpy(t.blob)
    d_out = torch.from_numpy(out0.copy()).cuda()
    plan.run((d_in.data_ptr(), t.blob.size), d_out)
    torch.cuda.synchronize()
    assert all(s == 0 for s, _ in plan.results())
    ref = d_out.cpu().numpy()
    assert np.array_equal(ref.view(np.uint16).reshape(H, -1)[:, :W], img)
    h_in, t_in = host_buf(t.blob, pinned)
    h_out, t_out = host_buf(sentinel(pitch * H, np.random.default_rng(6)), pinned)
    before = uctx.launches
    plan.run_host(h_in, h_out, partial=False)
    assert uctx.launches - before >= 2
    assert all(s == 0 for s, _ in plan.results())
    foot = Foot(0, pitch, 0, 0, H, W, 2)
    assert_same(h_out, ref, [foot], "run_host tile pipeline", mask=foot.mask(ref.size))
    del t_in, t_out


# ---------------------------------------------------------------------------------------
# plan creation refuses output layouts the kernels cannot store to (nothing is launched)
# ---------------------------------------------------------------------------------------
def _refused(ctx, make):
    before = ctx.launches
    with pytest.raises(rs.Rsb200Error) as e:
        make()
    assert e.value.code == F.ERR_ARG
    assert ctx.launches == before


def _accepted(ctx, make):
    before = ctx.launches
    plan = make()
    assert ctx.launches == before
    plan.close()


def _with(job, **kw):
    """A copy of the ctypes descriptor `job` with some fields changed."""
    j = type(job).from_buffer_copy(job)
    for k, v in kw.items():
        setattr(j, k, v)
    return j


def _unpack_base():
    j = rs.UnpackJob()
    j.in_size, j.out_offset, j.out_pitch, j.rows, j.samples = 4096, 16, 2080, 2, 1024
    j.in_pitch, j.bps, j.order = 1792, 14, rs.MSB
    return j


def _ljpeg_base():
    s = rs.LJpegScan()
    s.in_size, s.rows, s.frame_w, s.mcu_w, s.mcu_h = 256, 4, 16, 2, 1
    s.out_offset, s.out_pitch, s.store_w = 16, 64, 32
    return s


def _cr2_base():
    j = rs.Cr2Job()
    j.in_size, j.n_comp, j.x_s_f, j.y_s_f = 256, 2, 1, 1
    j.frame_w, j.frame_h, j.num_slices, j.slice_w, j.last_slice_w = 32, 8, 1, 0, 64
    j.img_w, j.img_h, j.out_offset, j.out_pitch = 64, 8, 16, 128
    return j


def _huff():
    return rs.huff_table(synth.DEFAULT_NCPL, synth.DEFAULT_VALUES)


@pytest.mark.parametrize("field,value", [("out_offset", 17), ("out_pitch", 2081)])
def test_unpack_ljpeg_cr2_refuse_odd_output_layouts(uctx, field, value):
    """unpack jobs, LJPEG scans and CR2 jobs store 16-bit samples: an odd out_offset or
    out_pitch is refused with RSB200_ERR_ARG when the plan is made."""
    u = _unpack_base()
    _accepted(uctx, lambda: rs.unpack_plan(uctx, [u]))
    _refused(uctx, lambda: rs.unpack_plan(uctx, [_with(u, **{field: value})]))
    # the generic path too (odd bit depth)
    g = _with(u, bps=13, in_pitch=1664)
    _accepted(uctx, lambda: rs.unpack_plan(uctx, [g]))
    _refused(uctx, lambda: rs.unpack_plan(uctx, [_with(g, **{field: value})]))

    s = _ljpeg_base()
    lv = value if field == "out_offset" else 65
    _accepted(uctx, lambda: rs.ljpeg_plan(uctx, [_huff()], [s]))
    _refused(uctx, lambda: rs.ljpeg_plan(uctx, [_huff()], [_with(s, **{field: lv})]))

    c = _cr2_base()
    cv = value if field == "out_offset" else 129
    _accepted(uctx, lambda: rs.cr2_plan(uctx, [_huff()], [c]))
    _refused(uctx, lambda: rs.cr2_plan(uctx, [_huff()], [_with(c, **{field: cv})]))


def _other_kinds():
    """kind -> (required alignment, make(job) -> plan, valid job, offset field, pitch field)."""
    H = _huff
    out = {}

    j = rs.PanaJob()
    j.in_size, j.out_offset, j.out_pitch, j.width, j.height = 0x4000, 16, 256, 120, 2
    j.version, j.bps = 5, 12
    out["pana"] = (2, lambda c, x: rs.pana_plan(c, [x]), j, "out_offset", "out_pitch")

    j = rs.Arw1Job()
    j.in_size, j.width, j.height, j.out_offset, j.out_pitch = 1024, 64, 8, 16, 128
    out["arw1"] = (2, lambda c, x: rs.arw1_plan(c, [x]), j, "out_offset", "out_pitch")

    j = rs.BadPixJob()
    j.offset, j.pitch, j.width, j.height, j.is_cfa = 16, 128, 64, 8, 1
    out["badpix"] = (2, lambda c, x: rs.badpix_plan(c, [x], np.zeros(0, np.uint32)), j,
                     "offset", "pitch")

    j = rs.SrawJob()
    j.in_pitch, j.num_mcus, j.in_rows, j.sub_x, j.sub_y, j.version = 64, 8, 2, 2, 1, 1
    j.out_offset, j.out_pitch = 16, 96
    out["sraw"] = (4, lambda c, x: rs.sraw_plan(c, [x]), j, "out_offset", "out_pitch")

    j = rs.PentaxJob()
    j.in_size, j.width, j.height, j.out_offset, j.out_pitch = 1024, 64, 8, 16, 128
    out["pentax"] = (4, lambda c, x: rs.pentax_plan(c, [H()], [x]), j, "out_offset", "out_pitch")

    j = rs.NikonJob()
    j.in_size, j.width, j.height, j.out_offset, j.out_pitch, j.lut = 1024, 64, 8, 16, 128, -1
    out["nikon"] = (4, lambda c, x: rs.nikon_plan(c, [H()], [x]), j, "out_offset", "out_pitch")

    j = rs.HasselbladJob()
    j.in_size, j.width, j.height, j.out_pitch, j.out_offset = 1024, 64, 8, 128, 16
    out["hasselblad"] = (4, lambda c, x: rs.hasselblad_plan(c, [H()], [x]), j, "out_offset",
                         "out_pitch")

    j = rs.PhaseOneJob()
    j.out_offset, j.out_pitch, j.width, j.height, j.first_strip = 16, 128, 64, 2, 0

    def p1(c, x):
        strips = []
        for r in range(2):
            st = rs.PhaseOneStrip()
            st.in_offset, st.in_size, st.row = 64 * r, 64, r
            strips.append(st)
        return rs.phaseone_plan(c, [x], strips)
    out["phaseone"] = (4, p1, j, "out_offset", "out_pitch")

    j = rs.Arw2Job()
    j.out_offset, j.out_pitch, j.width, j.height, j.table = 16, 128, 64, 8, -1
    out["arw2"] = (16, lambda c, x: rs.arw2_plan(c, [x]), j, "out_offset", "out_pitch")

    j = rs.ScaleJob()
    j.offset, j.pitch, j.width, j.height, j.cpp = 16, 128, 64, 8, 1
    j.crop_w, j.crop_h, j.white_point = 64, 8, 4095
    out["scale"] = (16, lambda c, x: rs.scale_plan(c, [x]), j, "offset", "pitch")

    j = rs.LookupJob()
    j.offset, j.pitch, j.width, j.height, j.cpp = 16, 128, 64, 8, 1
    out["lookup"] = (16, lambda c, x: rs.lookup_plan(c, [x], np.arange(65536, dtype=np.uint16)),
                     j, "offset", "pitch")

    j = rs.DngOpJob()
    j.offset, j.pitch, j.width, j.height, j.cpp = 16, 128, 64, 8, 1
    out["dngop"] = (16, lambda c, x: rs.dngop_plan(c, [x], []), j, "offset", "pitch")

    j = rs.RawJob()
    j.in_size, j.out_offset, j.out_pitch, j.rows, j.samples = 1024, 16, 128, 2, 16
    j.in_pitch, j.format = 64, F.RAW_FP16_LSB
    out["rawform_f32"] = (4, lambda c, x: rs.raw_plan(c, [x]), j, "out_offset", "out_pitch")

    j = rs.RawJob()
    j.in_size, j.out_offset, j.out_pitch, j.rows, j.samples = 1024, 16, 128, 2, 16
    j.in_pitch, j.format = 64, F.RAW_8BIT
    out["rawform_u16"] = (2, lambda c, x: rs.raw_plan(c, [x]), j, "out_offset", "out_pitch")
    return out


OTHER_KINDS = ["pana", "arw1", "badpix", "sraw", "pentax", "nikon", "hasselblad", "phaseone",
               "arw2", "scale", "lookup", "dngop", "rawform_f32", "rawform_u16"]


@pytest.mark.parametrize("kind", OTHER_KINDS)
def test_other_plan_kinds_refuse_misaligned_output(uctx, kind):
    """Regression table: every other plan kind refuses an output offset or pitch below the
    alignment its kernels store with (the same descriptor, aligned, is accepted)."""
    align, make, job, off_f, pitch_f = _other_kinds()[kind]
    _accepted(uctx, lambda: make(uctx, job))
    for f in (off_f, pitch_f):
        bad = _with(job, **{f: getattr(job, f) + align // 2})
        _refused(uctx, lambda: make(uctx, bad))
