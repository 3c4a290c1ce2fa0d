"""Python face of the C ABI: contexts and plans.

Device memory, streams and process groups come from PyTorch (plumbing); the
decode itself is the hand-written CUDA in csrc/ reached through ctypes.  If the
CUDA library or a GPU is missing every call raises: no CPU fallback exists."""
import ctypes as C

import numpy as np

from . import _abi
from ._abi import (Arw1Job, Arw2Job, HasselbladJob, NikonJob, PanaJob, ScaleJob, DngOp, DngOpJob, BadPixJob, LookupJob, PhaseOneJob, PhaseOneStrip, SamsungV0Job, SamsungV0Strip, SamsungV1Job, SamsungV2Job, KodakJob, Vc5Code, Vc5Job, Vc5Band, Cr2Job, HuffTable, LJpegScan, PentaxJob, RawJob, ScanResult, SrawJob, UnpackJob,  # noqa: F401
                   LSB, MSB, MSB16, MSB32)


class Rsb200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("rsb200 error %d: %s" % (code, msg))
        self.code = code
        self.msg = msg


class RawDecoderException(Rsb200Error):
    """Mirrors rawspeed::RawDecoderException (decoders/RawDecoderException.h)."""


class IOException(Rsb200Error):
    """Mirrors rawspeed::IOException (io/IOException.h)."""


def _raise(code, msg):
    if code == _abi.ERR_RDE:
        raise RawDecoderException(code, msg)
    if code == _abi.ERR_IOE:
        raise IOException(code, msg)
    raise Rsb200Error(code, msg)


class Context:
    """One per process / GPU (rsb200_create)."""

    def __init__(self, device=0):
        self._lib = _abi.load()
        h = C.c_void_p()
        rc = self._lib.rsb200_create(int(device), C.byref(h))
        if rc != _abi.OK:
            raise Rsb200Error(rc, "rsb200_create(device=%d) failed: no usable CUDA "
                              "device; there is no CPU fallback" % device)
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self._lib.rsb200_destroy(self.h)
            self.h = None

    __del__ = close

    def err(self):
        return self._lib.rsb200_last_error(self.h).decode("utf-8", "replace")

    @property
    def launches(self):
        return int(self._lib.rsb200_kernel_launches(self.h))

    @property
    def sm_count(self):
        return int(self._lib.rsb200_device_sm_count(self.h))

    def check(self, rc):
        if rc != _abi.OK:
            _raise(rc, self.err())


def huff_table(ncpl, values, fix16=False):
    t = HuffTable()
    for i in range(16):
        t.ncodes_per_len[i] = ncpl[i]
    for i, v in enumerate(values):
        t.values[i] = v
    t.nvalues = len(values)
    t.fix_dng16 = 1 if fix16 else 0
    return t


def _ptr_bytes(x):
    """(device pointer, nbytes) of a torch CUDA tensor or (ptr, nbytes) tuple; None = no
    buffer (plans that work in place on the output)."""
    if x is None:
        return 0, 0
    if isinstance(x, tuple):
        return int(x[0]), int(x[1])
    return int(x.data_ptr()), int(x.numel() * x.element_size())


class Plan:
    def __init__(self, ctx, handle, nunits):
        self.ctx = ctx
        self.h = handle
        self.nunits = nunits
        self._keep = None

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.ctx._lib.rsb200_plan_destroy(self.h)
        self.h = None

    __del__ = close

    def run(self, d_in, d_out, stream=None):
        """Enqueue the decode on `stream` (torch.cuda.Stream, raw handle or None
        = torch's current stream).  Asynchronous."""
        ip, ib = _ptr_bytes(d_in)
        op, ob = _ptr_bytes(d_out)
        if stream is None:
            import torch
            stream = torch.cuda.current_stream().cuda_stream
        elif hasattr(stream, "cuda_stream"):
            stream = stream.cuda_stream
        rc = self.ctx._lib.rsb200_plan_run(self.h, ip, ib, op, ob, C.c_void_p(stream))
        self.ctx.check(rc)

    def run_gather(self, comm, d_in, d_out_all, slab_bytes, mode, root=0, stream=None):
        """Decode into this rank's slab of d_out_all and gather the slabs over NVLink
        (rsb200_plan_run_gather: the transfer of a group of segments overlaps the decode of the
        following ones).  mode: GATHER_NONE / GATHER_ALL / GATHER_ROOT.  Asynchronous."""
        ip, ib = _ptr_bytes(d_in)
        op, _ = _ptr_bytes(d_out_all)
        if stream is None:
            import torch
            stream = torch.cuda.current_stream().cuda_stream
        elif hasattr(stream, "cuda_stream"):
            stream = stream.cuda_stream
        rc = self.ctx._lib.rsb200_plan_run_gather(self.h, comm.h, ip, ib, op, slab_bytes, mode, root,
                                                  C.c_void_p(stream))
        self.ctx.check(rc)

    def run_host(self, in_np, out_np, partial=False):
        """Host buffers in, host buffers out (H2D + kernels + D2H, synchronous)."""
        assert in_np.flags.c_contiguous and out_np.flags.c_contiguous
        rc = self.ctx._lib.rsb200_plan_run_host(
            self.h, in_np.ctypes.data, in_np.nbytes, out_np.ctypes.data,
            out_np.nbytes, 1 if partial else 0)
        self.ctx.check(rc)

    def results(self, check=True):
        """Per-segment (status, consumed); waits for the last run."""
        arr = (ScanResult * self.nunits)()
        rc = self.ctx._lib.rsb200_plan_results(self.h, arr, self.nunits)
        if check:
            self.ctx.check(rc)
        return [(r.status, r.consumed) for r in arr]

    def bytes(self):
        a, b, p = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self.ctx._lib.rsb200_plan_bytes(self.h, C.byref(a), C.byref(b), C.byref(p))
        return a.value, b.value, p.value

    def bad_pixels(self, job=0, cap=1 << 20):
        """Panasonic V4 job with zero_is_not_bad == 0: (count, positions[:min(count, cap)]) of
        the pixels the last run decoded as 0, positions = (row << 16) | col, unordered."""
        buf = (C.c_uint32 * cap)()
        n = C.c_uint32(0)
        self.ctx.check(self.ctx._lib.rsb200_plan_bad_pixels(self.h, job, buf, cap, C.byref(n)))
        return n.value, list(buf[:min(n.value, cap)])

    def kodak_values(self):
        """Kodak plan after a run: per job, the value its "Value out of bounds" failure prints (0 for
        a job without one)."""
        buf = (C.c_int32 * self.nunits)()
        self.ctx.check(self.ctx._lib.rsb200_kodak_plan_values(self.h, buf, self.nunits))
        return list(buf)

    @property
    def launches(self):
        return int(self.ctx._lib.rsb200_plan_launches(self.h))

    @property
    def kernels(self):
        """Which kernels one run of this plan launches (a short description)."""
        return self.ctx._lib.rsb200_plan_kernels(self.h).decode()


GATHER_NONE, GATHER_ALL, GATHER_ROOT = 0, 1, 2


def comm_unique_id():
    """128-byte NCCL id (rank 0 makes it, the caller ships it to the other ranks)."""
    from . import _abi
    buf = (C.c_uint8 * 128)()
    if _abi.load().rsb200_comm_unique_id(buf) != 0:
        raise RuntimeError("rsb200_comm_unique_id failed: NCCL (libnccl.so.2) not available")
    return bytes(buf)


class Comm:
    """One rank's communicator for the output gather (rsb200_comm_create)."""

    def __init__(self, ctx, uid, world, rank):
        self.ctx = ctx
        self.world, self.rank = world, rank
        h = C.c_void_p()
        buf = (C.c_uint8 * 128).from_buffer_copy(uid)
        ctx.check(ctx._lib.rsb200_comm_create(ctx.h, buf, world, rank, C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.ctx._lib.rsb200_comm_destroy(self.h)
        self.h = None

    __del__ = close


def unpack_plan(ctx, jobs):
    arr = (UnpackJob * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_unpack_plan_create(ctx.h, arr, len(jobs), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def raw_plan(ctx, jobs, tables=None):
    """Plan over the fixed-layout UncompressedDecompressor forms (RAW_* formats).
    tables: array (ntables, 65536) uint16 for RAW_8BIT_TABLE jobs, or None."""
    arr = (RawJob * len(jobs))(*jobs)
    h = C.c_void_p()
    tp, nt = None, 0
    if tables is not None:
        tables = np.ascontiguousarray(tables, dtype=np.uint16).reshape(-1, 65536)
        tp, nt = tables.ctypes.data_as(C.POINTER(C.c_uint16)), tables.shape[0]
    ctx.check(ctx._lib.rsb200_raw_plan_create(ctx.h, arr, len(jobs), tp, nt, C.byref(h)))
    return Plan(ctx, h, len(jobs))


def sraw_plan(ctx, jobs):
    """Canon sRaw interpolation (Cr2sRawInterpolator) over subsampled uint16 images."""
    arr = (SrawJob * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_sraw_plan_create(ctx.h, arr, len(jobs), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def nikon_plan(ctx, tables, jobs, luts=None):
    """Nikon NEF streams without split (NikonDecompressor::decompress), one job per image.
    luts: dithered TableLookUp storage per curve (2*65536 uint16 each), or None."""
    ta = (HuffTable * len(tables))(*tables)
    ja = (NikonJob * len(jobs))(*jobs)
    h = C.c_void_p()
    lp, nl = None, 0
    if luts is not None:
        luts = np.ascontiguousarray(luts, dtype=np.uint16).reshape(-1, 131072)
        lp, nl = luts.ctypes.data_as(C.POINTER(C.c_uint16)), luts.shape[0]
    ctx.check(ctx._lib.rsb200_nikon_plan_create(ctx.h, ta, len(tables), ja, len(jobs), lp, nl,
                                                C.byref(h)))
    return Plan(ctx, h, len(jobs))


def pana_plan(ctx, jobs):
    """Panasonic RW2 images (PanasonicV5/V6/V7Decompressor::decompress), one job per image."""
    arr = (PanaJob * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_pana_plan_create(ctx.h, arr, len(jobs), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def scale_plan(ctx, jobs):
    """Black / white scaling of decoded images in place (RawImageDataU16::scaleValues); run
    with d_in=None: plan.run(None, d_image)."""
    arr = (ScaleJob * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_scale_plan_create(ctx.h, arr, len(jobs), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def dngop_plan(ctx, jobs, ops, tables=None, deltas=None):
    """A DNG opcode list per image, applied in one pass in place (DngOpcodes::applyOpCodes);
    tables: (n, 65536) uint16, deltas: uint32 words; run with plan.run(None, d_image).
    plan.bad_pixels(k) reads the positions BAD_CONSTANT opcode k collected."""
    ja = (DngOpJob * len(jobs))(*jobs)
    oa = (DngOp * max(1, len(ops)))(*ops)
    tp, nt, dp, nd = None, 0, None, 0
    if tables is not None and len(tables):
        tables = np.ascontiguousarray(tables, dtype=np.uint16).reshape(-1, 65536)
        tp, nt = tables.ctypes.data_as(C.POINTER(C.c_uint16)), tables.shape[0]
    if deltas is not None and len(deltas):
        deltas = np.ascontiguousarray(deltas, dtype=np.uint32)
        dp, nd = deltas.ctypes.data_as(C.POINTER(C.c_uint32)), deltas.size
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_dngop_plan_create(ctx.h, ja, len(jobs), oa, len(ops), tp, nt, dp, nd,
                                                C.byref(h)))
    plan = Plan(ctx, h, len(jobs))
    plan._keep = (tables, deltas)
    return plan


def lookup_plan(ctx, jobs, tables, dither=False):
    """Whole-image table lookup in place (RawImageData::sixteenBitLookup); tables: TableLookUp
    storage per table (65536 uint16, or 2*65536 when dithered); run with plan.run(None, d_image)."""
    ja = (LookupJob * len(jobs))(*jobs)
    tables = np.ascontiguousarray(tables, dtype=np.uint16).reshape(-1, 131072 if dither else 65536)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_lookup_plan_create(ctx.h, ja, len(jobs),
                                                 tables.ctypes.data_as(C.POINTER(C.c_uint16)),
                                                 tables.shape[0], int(dither), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def badpix_plan(ctx, jobs, positions):
    """Bad-pixel interpolation in place (RawImageData::fixBadPixels); positions: uint32
    (y << 16) | x, each job names its slice; run with plan.run(None, d_image)."""
    ja = (BadPixJob * len(jobs))(*jobs)
    pos = np.ascontiguousarray(positions, dtype=np.uint32)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_badpix_plan_create(ctx.h, ja, len(jobs), pos.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                 pos.size, C.byref(h)))
    return Plan(ctx, h, len(jobs))


def phaseone_plan(ctx, jobs, strips):
    """Phase One IIQ images (PhaseOneDecompressor::decompress): one strip per image row."""
    ja = (PhaseOneJob * len(jobs))(*jobs)
    sa = (PhaseOneStrip * len(strips))(*strips)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_phaseone_plan_create(ctx.h, ja, len(jobs), sa, len(strips),
                                                   C.byref(h)))
    return Plan(ctx, h, len(jobs))


def samsung0_plan(ctx, jobs, strips):
    """Samsung SRW V0 row streams (SamsungV0Decompressor::decompress), one job per frame; job.first_strip
    names the first of its `height` strips, rows in order."""
    ja = (SamsungV0Job * len(jobs))(*jobs)
    sa = (SamsungV0Strip * len(strips))(*strips)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_samsung0_plan_create(ctx.h, ja, len(jobs), sa, len(strips), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def hasselblad_plan(ctx, tables, jobs):
    """Hasselblad 3FR frames (HasselbladDecompressor::decompress), one job per frame: one MSB32
    Huffman stream of pixel pairs.  plan.results(): per job (status, consumed)."""
    ta = (HuffTable * len(tables))(*tables)
    ja = (HasselbladJob * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_hasselblad_plan_create(ctx.h, ta, len(tables), ja, len(jobs), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def arw2_plan(ctx, jobs, tables=None, dither=False):
    """Sony ARW2 images (SonyArw2Decompressor::decompress), one job per image.  tables:
    TableLookUp storage per table (65536 uint16, or 2*65536 when dithered), or None."""
    arr = (Arw2Job * len(jobs))(*jobs)
    h = C.c_void_p()
    tp, nt = None, 0
    if tables is not None:
        tables = np.ascontiguousarray(tables, dtype=np.uint16).reshape(-1, 131072 if dither else 65536)
        tp, nt = tables.ctypes.data_as(C.POINTER(C.c_uint16)), tables.shape[0]
    ctx.check(ctx._lib.rsb200_arw2_plan_create(ctx.h, arr, len(jobs), tp, nt, int(dither),
                                               C.byref(h)))
    return Plan(ctx, h, len(jobs))


def pentax_plan(ctx, tables, jobs):
    """Pentax PEF streams (PentaxDecompressor::decompress), one job per image."""
    ta = (HuffTable * len(tables))(*tables)
    ja = (PentaxJob * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_pentax_plan_create(ctx.h, ta, len(tables), ja, len(jobs),
                                                 C.byref(h)))
    return Plan(ctx, h, len(jobs))


def arw1_plan(ctx, jobs):
    """Sony ARW1 streams (SonyArw1Decompressor::decompress), one job per frame."""
    ja = (Arw1Job * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_arw1_plan_create(ctx.h, ja, len(jobs), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def samsung1_plan(ctx, jobs):
    """Samsung SRW V1 streams (SamsungV1Decompressor::decompress), one job per frame."""
    ja = (SamsungV1Job * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_samsung1_plan_create(ctx.h, ja, len(jobs), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def samsung2_plan(ctx, jobs):
    """Samsung SRW V2 strips (SamsungV2Decompressor::decompress), one job per frame; job.header holds
    the strip's first 16 bytes."""
    ja = (SamsungV2Job * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_samsung2_plan_create(ctx.h, ja, len(jobs), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def kodak_plan(ctx, jobs, tables=None):
    """Kodak DCR streams (KodakDecompressor::decompress), one job per frame.  tables: None or a
    (n, 65536) uint16 array (for a dithered RawImage table, its entries 2*v); job.table indexes it
    (-1 = none).  After a run, plan.kodak_values() gives the value each job's "Value out of bounds"
    prints."""
    ja = (KodakJob * len(jobs))(*jobs)
    if tables is None:
        tp, nt = None, 0
    else:
        t = np.ascontiguousarray(tables, dtype=np.uint16).reshape(-1, 65536)
        tp, nt = t.ctypes.data, t.shape[0]
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_kodak_plan_create(ctx.h, ja, len(jobs), tp, nt, C.byref(h)))
    return Plan(ctx, h, len(jobs))


def vc5_plan(ctx, codebook, jobs, bands):
    """GoPro VC-5 frames (VC5Decompressor::decode), one job per frame.  codebook: Vc5Code entries or an
    (n, 4) array of {size, bits, count, value}; bands: the Vc5Band payloads the jobs index (40 per job,
    channel * 10 + subband from job.first_band), as the tag walk cut them."""
    if not (len(codebook) and isinstance(codebook[0], Vc5Code)):
        codebook = [Vc5Code(*(int(x) for x in e)) for e in codebook]
    ca = (Vc5Code * len(codebook))(*codebook)
    ja = (Vc5Job * len(jobs))(*jobs)
    ba = (Vc5Band * len(bands))(*bands)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_vc5_plan_create(ctx.h, ca, len(codebook), ja, len(jobs), ba, len(bands), C.byref(h)))
    return Plan(ctx, h, len(jobs))


def ljpeg_plan(ctx, tables, scans):
    ta = (HuffTable * len(tables))(*tables)
    sa = (LJpegScan * len(scans))(*scans)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_ljpeg_plan_create(ctx.h, ta, len(tables), sa, len(scans),
                                                C.byref(h)))
    return Plan(ctx, h, len(scans))


def cr2_plan(ctx, tables, jobs):
    ta = (HuffTable * len(tables))(*tables)
    ja = (Cr2Job * len(jobs))(*jobs)
    h = C.c_void_p()
    ctx.check(ctx._lib.rsb200_cr2_plan_create(ctx.h, ta, len(tables), ja, len(jobs),
                                              C.byref(h)))
    return Plan(ctx, h, len(jobs))


def image_pitch(w, cpp=1):
    """RawImageData::createData(): pitch = roundUp(w*cpp*2, 16) (RawImage.cpp:80-82)."""
    return (w * cpp * 2 + 15) // 16 * 16


def new_image(w, h, cpp=1, fill=0):
    return np.full((h, image_pitch(w, cpp) // 2), fill, dtype=np.uint16)
