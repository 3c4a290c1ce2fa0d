"""Plan lifecycle through the C ABI, one small valid plan per create entry point: one run adds
exactly plan.launches to the context's launch count, and the plan's device memory (the device's
default memory pool, read through the driver API) goes back to where it was when the plan is closed,
also when a create is refused after it has allocated."""
import ctypes as C
import gc

import numpy as np
import pytest

import rawspeed_b200 as rs
from rawspeed_b200 import formats as F
from rawspeed_b200 import host
from oracle import port, synth
from helpers import TableSet, dng_ljpeg_scans

import arw1_oracle as A1
import samsung0_oracle as S0
import samsung1_oracle as S1
import samsung2_oracle as S2
import test_gpu_arw2
import test_gpu_cr2
import test_gpu_hasselblad
import test_gpu_lookup
import test_gpu_nikon
import test_gpu_panasonic
import test_gpu_pentax
import test_gpu_phaseone
import test_gpu_scale
import test_gpu_sraw
import test_oracle_badpixels
import test_oracle_dngopcodes
import test_oracle_lookup
import test_oracle_panasonic
import test_oracle_sraw
from test_oracle_vs_ref import CR2_CASES
from test_samsung0_emu import strips_of

pytestmark = pytest.mark.gpu

CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7  # cuda.h, CUmemPool_attribute


def pool_used():
    """Bytes in use in device 0's default memory pool, after everything queued has finished."""
    import torch
    torch.cuda.synchronize()
    cu = C.CDLL("libcuda.so.1")
    dev, pool, used = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuInit(0) == 0
    assert cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, C.byref(used)) == 0
    return used.value


# Each builder: ctx -> (plan, its input as bytes or a numpy array, its output buffer as a numpy array).

def _unpack(ctx):
    w, h = 512, 8
    data, pitch = synth.packed_frame(w, h, 14, seed=2)
    out = port.new_image(w, h)
    j = rs.UnpackJob()
    j.in_size, j.out_pitch, j.rows, j.samples = data.size, out.shape[1] * 2, h, w
    j.in_pitch, j.bps, j.order = pitch, 14, rs.MSB
    return rs.unpack_plan(ctx, [j]), data, out


def _raw(ctx):
    w, h = 70, 9
    data = synth.lcg_bytes(w * h, seed=3)
    out = port.new_image(w, h)
    j = rs.RawJob()
    j.in_size, j.out_pitch, j.rows, j.samples, j.in_pitch, j.format = data.size, out.shape[1] * 2, h, w, w, F.RAW_8BIT
    return rs.raw_plan(ctx, [j]), data, out


def _lookup(ctx):
    w, h, cpp, _, ncurve = test_oracle_lookup.CASES[0]
    out = test_oracle_lookup.image(w, h, cpp, 0)
    t = port.build_table(test_oracle_lookup.curve(ncurve, 10), False)
    return rs.lookup_plan(ctx, [test_gpu_lookup._job(0, out, w, cpp)], t, False), np.zeros(0, np.uint8), out


def _badpix(ctx):
    _, w, h, _, cfa, points = test_oracle_badpixels.scenarios()[0]
    out = test_oracle_badpixels.image(w, h, 1, 0)
    j = rs.BadPixJob()
    j.offset, j.pitch, j.width, j.height = 0, out.shape[1] * 2, w, h
    j.is_cfa, j.first_position, j.num_positions, j.prior_map = int(cfa), 0, len(points), None
    return rs.badpix_plan(ctx, [j], test_oracle_badpixels.pos(points)), np.zeros(0, np.uint8), out


def _dngop(ctx):
    _, img, w, cpp, crop, blob = test_oracle_dngopcodes.scenarios()[0]
    low = host.dngop_lower(img, w, cpp, crop, blob)
    j = rs.DngOpJob()
    j.offset, j.pitch, j.width, j.height = 0, img.shape[1] * img.itemsize, w, img.shape[0]
    j.cpp, j.is_f32, j.first_op, j.num_ops = cpp, int(img.dtype == np.uint32), 0, len(low["ops"])
    ops = [rs.DngOp.from_buffer_copy(o) for o in low["ops"]]
    return rs.dngop_plan(ctx, [j], ops, low["tables"], low["deltas"]), np.zeros(0, np.uint8), img.copy()


def _scale(ctx):
    w, h, cpp, crop, black, white = test_gpu_scale.CASES[0]
    out = test_gpu_scale._image(w, h, cpp, 40)
    return rs.scale_plan(ctx, [test_gpu_scale._job(0, out, w, h, cpp, crop, black, white)]), np.zeros(0, np.uint8), out


def _sraw(ctx):
    inp, in_w = test_oracle_sraw.sraw_input(5, 3, 4, seed=1)
    out = port.new_image(10, 3, 3)
    j = test_gpu_sraw.job(inp, in_w, out, (2, 1), (2100, 1024, 1700), 12, 1)
    return rs.sraw_plan(ctx, [j]), inp.view(np.uint8).reshape(-1), out


def _hasselblad(ctx):
    w, h = 66, 9
    img = synth.image_model(w, h, seed=w, bits=14)
    ncpl, vals = test_gpu_hasselblad.NCPL, test_gpu_hasselblad.VALS
    data = synth.make_hasselblad(img, port.Huff(ncpl, vals, full=False), 0x8000)
    tab = rs.huff_table(bytes(ncpl), bytes(vals), False)
    j = test_gpu_hasselblad._job(w, h, 0, len(data), 0, 0x8000)
    return rs.hasselblad_plan(ctx, [tab], [j]), data, port.new_image(w, h)


def _phaseone(ctx):
    w, h = 70, 9
    blob, strips = synth.make_phaseone(synth.image_model(w, h, seed=w, bits=14), shuffle_seed=h, gap=3)
    return test_gpu_phaseone._plan(ctx, w, h, strips), blob, port.new_image(w, h)


def _samsung0(ctx):
    w, h = 32, 4
    bso, bsr, _ = S0.make_frame(S0.natural_values(w, h), S0.dirs_left(w, h))
    strips = []
    for o, n in strips_of(bso, bsr, h):
        s = rs.SamsungV0Strip()
        s.in_offset, s.in_size = o, n
        strips.append(s)
    pitch = S0.pitch_elems(w)
    j = rs.SamsungV0Job()
    j.out_offset, j.out_pitch, j.width, j.height, j.first_strip = 0, pitch * 2, w, h, 0
    return rs.samsung0_plan(ctx, [j], strips), bsr, np.zeros((h, pitch), np.uint16)


def _samsung2(ctx):
    w, h = 32, 4
    data = S2.encode(S2.natural_values(w, h))
    pitch = S2.pitch_elems(w)
    j = rs.SamsungV2Job()
    j.in_offset, j.in_size, j.bits, j.width, j.height = 0, len(data), 12, w, h
    for i, b in enumerate(data[:16]):
        j.header[i] = b
    j.out_offset, j.out_pitch = 0, pitch * 2
    return rs.samsung2_plan(ctx, [j]), data, np.zeros((h, pitch), np.uint16)


def _pana(ctx):
    version, bps, w, h = test_oracle_panasonic.CASES[0]
    data = test_oracle_panasonic.payload(version, w, h, bps, seed=1)
    return rs.pana_plan(ctx, [test_gpu_panasonic._job(version, bps, w, h, data.size)]), data, port.new_image(w, h)


def _arw2(ctx):
    w, h = 64, 5
    data = synth.arw2_frame(w, h, seed=w + 3 * h)
    return rs.arw2_plan(ctx, [test_gpu_arw2._job(w, h)]), data, port.new_image(w, h)


def _pentax(ctx):
    w, h = 64, 9
    table = port.pentax_table(None, True)
    img = (synth.image_model(w, h, seed=w + h, bits=12) & 0x0FFF).astype(np.uint16)
    data = synth.make_pentax(img, table)
    out = port.new_image(w, h)
    return test_gpu_pentax.plan_for(ctx, table, data.size, out, w, h), data, out


def _arw1(ctx):
    w, h = 64, 8
    data = A1.encode_frame(A1.natural_frame(w, h))
    pitch = A1.pitch_elems(w)
    j = rs.Arw1Job()
    j.in_offset, j.in_size, j.width, j.height = 0, len(data), w, h
    j.out_offset, j.out_pitch = 0, pitch * 2
    return rs.arw1_plan(ctx, [j]), data, np.zeros((h, pitch), np.uint16)


def _samsung1(ctx):
    w, h = 64, 4
    data = S1.make_stream(S1.natural_values(w, h))
    pitch = S1.pitch_elems(w)
    j = rs.SamsungV1Job()
    j.in_offset, j.in_size, j.bits, j.width, j.height = 0, len(data), 12, w, h
    j.out_offset, j.out_pitch = 0, pitch * 2
    return rs.samsung1_plan(ctx, [j]), data, np.zeros((h, pitch), np.uint16)


def _nikon(ctx):
    w, h = 64, 9
    _, su, _, data = test_gpu_nikon._case("lossless", 12, w, h)
    ncpl, values = port.nikon_tree(su["huff_select"])
    j = rs.NikonJob()
    j.in_offset, j.in_size, j.table, j.width, j.height = 0, data.size, 0, w, h
    j.out_offset, j.out_pitch, j.lut = 0, port.image_pitch(w), -1
    for k in range(4):
        j.pup[k] = su["pup"][k]
    return rs.nikon_plan(ctx, [rs.huff_table(ncpl, values)], [j]), data, port.new_image(w, h)


def _ljpeg(ctx):
    w, h = 256, 128
    t = synth.make_dng_ljpeg(synth.image_model(w, h, 12345), 128, 64)
    out = port.new_image(w, h)
    tabs, scans = dng_ljpeg_scans(t, out.shape[1] * 2)
    return rs.ljpeg_plan(ctx, tabs.tabs, scans), t.blob, out


def _cr2(ctx):
    w, h, fmt, frame, slicing = CR2_CASES[0]
    img = port.new_image(w, h)
    img[:, :w] = synth.image_model(w, h, 31)
    blob = port.cr2_encode(img, w, fmt, frame, slicing, 14, synth.default_tables(2), [0, 1, 0, 1][:fmt[0]],
                           is_cfa=True)
    tabs = TableSet()
    job = test_gpu_cr2.cr2_job(blob, w, h, fmt, slicing, img.shape[1] * 2, tabs)
    return rs.cr2_plan(ctx, tabs.tabs, [job]), blob, port.new_image(w, h)


BUILDERS = {
    "unpack": _unpack, "raw": _raw, "lookup": _lookup, "badpix": _badpix, "dngop": _dngop, "scale": _scale,
    "sraw": _sraw, "hasselblad": _hasselblad, "phaseone": _phaseone, "samsung0": _samsung0,
    "samsung2": _samsung2, "pana": _pana, "arw2": _arw2, "pentax": _pentax, "arw1": _arw1,
    "samsung1": _samsung1, "nikon": _nikon, "ljpeg": _ljpeg, "cr2": _cr2,
}


@pytest.mark.parametrize("name", list(BUILDERS))
def test_one_run_counts_plan_launches_and_close_frees_the_plan(ctx, name):
    import torch
    gc.collect()
    base = pool_used()
    plan, data, out = BUILDERS[name](ctx)
    assert pool_used() > base, "the plan's memory is not in the default pool"
    data = np.frombuffer(bytes(data), np.uint8) if isinstance(data, (bytes, bytearray)) else \
        np.ascontiguousarray(data).view(np.uint8).reshape(-1)
    d_in = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
    d_in[:data.size] = torch.from_numpy(data.copy())
    d_out = torch.from_numpy(np.ascontiguousarray(out).view(np.uint8).reshape(-1).copy()).cuda()
    n0 = ctx.launches
    plan.run((d_in.data_ptr(), data.size), d_out)
    torch.cuda.synchronize()
    plan.results()
    assert plan.launches > 0
    assert ctx.launches - n0 == plan.launches, plan.kernels
    plan.close()
    assert pool_used() == base


def test_refused_create_frees_what_it_allocated(ctx):
    """The raw-form create uploads the jobs of format 1, then refuses format 5, whose two jobs hold
    2^32 - 2 items together."""
    gc.collect()
    base = pool_used()
    small = rs.RawJob()
    small.in_size, small.out_pitch, small.rows, small.samples, small.in_pitch = 8, 16, 1, 8, 8
    small.format = F.RAW_8BIT
    big = rs.RawJob()
    big.rows, big.samples, big.in_pitch, big.out_pitch = 0x7FFFFFFF, 8, 16, 16
    big.in_size, big.format = 0x7FFFFFFF * 16, F.RAW_12BIT_LEFT_BE
    with pytest.raises(rs.Rsb200Error, match="raw plan: too many items of format 5"):
        rs.raw_plan(ctx, [small, big, big])
    assert pool_used() == base
