"""ctypes binding of the C ABI (include/rawspeed_b200.h).

The product path is the CUDA library; if it cannot be built/loaded this module
raises -- there is no CPU fallback."""
import ctypes as C
import os

from . import build as _build

OK, ERR_RDE, ERR_IOE, ERR_CUDA, ERR_ARG = 0, 1, 2, 3, 4
LSB, MSB, MSB16, MSB32 = 0, 1, 2, 3


class UnpackJob(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint64),
                ("out_offset", C.c_uint64), ("out_pitch", C.c_int32),
                ("row0", C.c_int32), ("rows", C.c_int32), ("samples", C.c_int32),
                ("out_col0", C.c_int32), ("in_pitch", C.c_int32), ("bps", C.c_int32),
                ("order", C.c_int32)]


class RawJob(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint64),
                ("out_offset", C.c_uint64), ("out_pitch", C.c_int32),
                ("row0", C.c_int32), ("rows", C.c_int32), ("samples", C.c_int32),
                ("out_col0", C.c_int32), ("in_pitch", C.c_int32), ("format", C.c_int32),
                ("table", C.c_int32)]


(RAW_8BIT, RAW_8BIT_TABLE, RAW_12BIT_CONTROL_BE, RAW_12BIT_CONTROL_LE, RAW_12BIT_LEFT_BE,
 RAW_12BIT_LEFT_LE, RAW_FP16_MSB, RAW_FP16_LSB, RAW_FP24_MSB, RAW_FP24_LSB,
 RAW_F32_COPY) = range(1, 12)


class SrawJob(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_pitch", C.c_uint32), ("num_mcus", C.c_uint32),
                ("in_rows", C.c_uint32), ("sub_x", C.c_uint8), ("sub_y", C.c_uint8),
                ("version", C.c_uint8), ("reserved", C.c_uint8),
                ("sraw_coeffs", C.c_int32 * 3), ("hue", C.c_int32),
                ("out_offset", C.c_uint64), ("out_pitch", C.c_uint32),
                ("reserved1", C.c_uint32)]


class PentaxJob(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("table", C.c_uint32),
                ("width", C.c_int32), ("height", C.c_int32), ("out_offset", C.c_uint64),
                ("out_pitch", C.c_uint32), ("reserved", C.c_uint32)]


class Arw1Job(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("reserved0", C.c_uint32),
                ("width", C.c_int32), ("height", C.c_int32), ("out_offset", C.c_uint64),
                ("out_pitch", C.c_uint32), ("reserved", C.c_uint32)]


class SamsungV1Job(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("bits", C.c_uint32),
                ("width", C.c_int32), ("height", C.c_int32), ("out_offset", C.c_uint64),
                ("out_pitch", C.c_uint32), ("reserved", C.c_uint32)]


class SamsungV2Job(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("bits", C.c_uint32),
                ("width", C.c_int32), ("height", C.c_int32), ("header", C.c_uint8 * 16),
                ("out_offset", C.c_uint64), ("out_pitch", C.c_uint32), ("reserved", C.c_uint32)]


class KodakJob(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("width", C.c_int32),
                ("height", C.c_int32), ("bps", C.c_int32), ("table", C.c_int32),
                ("out_offset", C.c_uint64), ("out_pitch", C.c_uint32), ("reserved", C.c_uint32)]


class Vc5Code(C.Structure):
    _fields_ = [("size", C.c_uint32), ("bits", C.c_uint32), ("count", C.c_uint32), ("value", C.c_uint32)]


class Vc5Band(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("param", C.c_int32)]


class Vc5Job(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("output_bits", C.c_int32), ("phase", C.c_int32),
                ("prescale", (C.c_uint8 * 3) * 4), ("first_band", C.c_uint32), ("out_offset", C.c_uint64),
                ("out_pitch", C.c_uint32), ("reserved", C.c_uint32)]


class NikonJob(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("table", C.c_uint32),
                ("width", C.c_int32), ("height", C.c_int32), ("out_offset", C.c_uint64),
                ("out_pitch", C.c_uint32), ("lut", C.c_int32), ("pup", C.c_uint16 * 4)]


class PanaJob(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint64), ("out_offset", C.c_uint64),
                ("out_pitch", C.c_uint32), ("width", C.c_uint32), ("height", C.c_uint32),
                ("version", C.c_uint8), ("bps", C.c_uint8), ("zero_is_not_bad", C.c_uint8),
                ("reserved", C.c_uint8), ("section_split_offset", C.c_uint32),
                ("reserved1", C.c_uint32)]


PANA_BAD_CAP = 1 << 22


class ScaleJob(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("pitch", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("cpp", C.c_uint32), ("crop_x", C.c_uint32),
                ("crop_y", C.c_uint32), ("crop_w", C.c_uint32), ("crop_h", C.c_uint32),
                ("black_separate", C.c_int32 * 4), ("white_point", C.c_int32),
                ("dither", C.c_uint8), ("path", C.c_uint8), ("reserved", C.c_uint8 * 2)]


SCALE_AUTO, SCALE_SSE2, SCALE_PLAIN = 0, 1, 2


class DngOp(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("top", C.c_uint32), ("left", C.c_uint32),
                ("bottom", C.c_uint32), ("right", C.c_uint32), ("first_plane", C.c_uint32),
                ("planes", C.c_uint32), ("row_pitch", C.c_uint32), ("col_pitch", C.c_uint32),
                ("table", C.c_uint32), ("value", C.c_uint32), ("reserved", C.c_uint32)]


class DngOpJob(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("pitch", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("cpp", C.c_uint32), ("is_f32", C.c_uint32),
                ("first_op", C.c_uint32), ("num_ops", C.c_uint32), ("reserved", C.c_uint32)]


(DNGOP_LOOKUP, DNGOP_OFFSET_ROW, DNGOP_OFFSET_COL, DNGOP_SCALE_ROW, DNGOP_SCALE_COL,
 DNGOP_BAD_CONSTANT) = range(6)


class LookupJob(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("pitch", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("cpp", C.c_uint32), ("table", C.c_uint32),
                ("reserved", C.c_uint32)]


class BadPixJob(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("pitch", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("is_cfa", C.c_uint32), ("first_position", C.c_uint32),
                ("num_positions", C.c_uint32), ("prior_map", C.c_void_p)]


class SamsungV0Strip(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("reserved", C.c_uint32)]


class SamsungV0Job(C.Structure):
    _fields_ = [("out_offset", C.c_uint64), ("out_pitch", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("first_strip", C.c_uint32)]


class PhaseOneStrip(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("row", C.c_uint32)]


class PhaseOneJob(C.Structure):
    _fields_ = [("out_offset", C.c_uint64), ("out_pitch", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("first_strip", C.c_uint32)]


class HasselbladJob(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32), ("width", C.c_uint32),
                ("height", C.c_uint32), ("out_pitch", C.c_uint32), ("out_offset", C.c_uint64),
                ("init_pred", C.c_uint16), ("table", C.c_uint8), ("reserved", C.c_uint8 * 5)]


class Arw2Job(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("out_offset", C.c_uint64),
                ("out_pitch", C.c_uint32), ("width", C.c_uint32), ("height", C.c_uint32),
                ("table", C.c_int32)]


PENTAX_OOB = 0x80000000


class HuffTable(C.Structure):
    _fields_ = [("ncodes_per_len", C.c_uint8 * 16), ("values", C.c_uint8 * 162),
                ("nvalues", C.c_uint16), ("fix_dng16", C.c_uint8),
                ("reserved", C.c_uint8 * 3)]


class LJpegScan(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32),
                ("rows", C.c_uint32), ("frame_w", C.c_uint32), ("mcu_w", C.c_uint8),
                ("mcu_h", C.c_uint8), ("table", C.c_uint8 * 4),
                ("reserved", C.c_uint8 * 2), ("init_pred", C.c_uint16 * 4),
                ("out_offset", C.c_uint64), ("out_pitch", C.c_uint32),
                ("out_x", C.c_uint32), ("out_y", C.c_uint32), ("store_w", C.c_uint32)]


class ScanResult(C.Structure):
    _fields_ = [("status", C.c_uint32), ("consumed", C.c_uint32)]


class Cr2Job(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("in_size", C.c_uint32),
                ("n_comp", C.c_uint8), ("x_s_f", C.c_uint8), ("y_s_f", C.c_uint8),
                ("reserved0", C.c_uint8), ("table", C.c_uint8 * 4),
                ("init_pred", C.c_uint16 * 4), ("frame_w", C.c_int32),
                ("frame_h", C.c_int32), ("num_slices", C.c_int32),
                ("slice_w", C.c_int32), ("last_slice_w", C.c_int32),
                ("img_w", C.c_int32), ("img_h", C.c_int32), ("out_offset", C.c_uint64),
                ("out_pitch", C.c_uint32), ("reserved1", C.c_uint32)]


EXPORTS = [
    "rsb200_abi_version", "rsb200_create", "rsb200_destroy", "rsb200_last_error",
    "rsb200_kernel_launches", "rsb200_device_sm_count", "rsb200_unpack_plan_create",
    "rsb200_raw_plan_create", "rsb200_sraw_plan_create",
    "rsb200_pentax_plan_create", "rsb200_arw1_plan_create", "rsb200_arw2_plan_create", "rsb200_nikon_plan_create",
    "rsb200_pana_plan_create", "rsb200_phaseone_plan_create", "rsb200_samsung0_plan_create", "rsb200_samsung1_plan_create", "rsb200_samsung2_plan_create", "rsb200_kodak_plan_create", "rsb200_kodak_plan_values", "rsb200_vc5_plan_create", "rsb200_hasselblad_plan_create", "rsb200_scale_plan_create", "rsb200_plan_bad_pixels", "rsb200_dngop_plan_create", "rsb200_badpix_plan_create", "rsb200_lookup_plan_create",
    "rsb200_ljpeg_plan_create", "rsb200_cr2_plan_create", "rsb200_plan_run",
    "rsb200_plan_run_host", "rsb200_plan_run_host_image", "rsb200_plan_results", "rsb200_plan_bytes",
    "rsb200_plan_launches", "rsb200_plan_kernels", "rsb200_plan_destroy",
    "rsb200_comm_unique_id", "rsb200_comm_create", "rsb200_comm_destroy", "rsb200_plan_run_gather",
]

_lib = None


def lib_path():
    return _build.LIB


def load():
    """Load (building if needed) the CUDA library.  Raises if impossible."""
    global _lib
    if _lib is not None:
        return _lib
    # RSB200_LIB: load another build of the same library (profiling variants made by
    # tools/phase_timing.py); still the CUDA library, never a fallback
    path = os.environ.get("RSB200_LIB") or _build.LIB
    if not os.path.exists(path):
        path = _build.build()
    L = C.CDLL(path)
    vp, u64, i32 = C.c_void_p, C.c_uint64, C.c_int
    L.rsb200_abi_version.restype = i32
    L.rsb200_create.argtypes = [i32, C.POINTER(vp)]
    L.rsb200_destroy.argtypes = [vp]
    L.rsb200_destroy.restype = None
    L.rsb200_last_error.argtypes = [vp]
    L.rsb200_last_error.restype = C.c_char_p
    L.rsb200_kernel_launches.argtypes = [vp]
    L.rsb200_kernel_launches.restype = u64
    L.rsb200_device_sm_count.argtypes = [vp]
    L.rsb200_unpack_plan_create.argtypes = [vp, C.POINTER(UnpackJob), i32, C.POINTER(vp)]
    L.rsb200_raw_plan_create.argtypes = [vp, C.POINTER(RawJob), i32, C.POINTER(C.c_uint16),
                                         i32, C.POINTER(vp)]
    L.rsb200_sraw_plan_create.argtypes = [vp, C.POINTER(SrawJob), i32, C.POINTER(vp)]
    L.rsb200_nikon_plan_create.argtypes = [vp, C.POINTER(HuffTable), i32, C.POINTER(NikonJob), i32,
                                           C.POINTER(C.c_uint16), i32, C.POINTER(vp)]
    L.rsb200_pana_plan_create.argtypes = [vp, C.POINTER(PanaJob), i32, C.POINTER(vp)]
    L.rsb200_hasselblad_plan_create.argtypes = [vp, C.POINTER(HuffTable), i32, C.POINTER(HasselbladJob), i32,
                                                C.POINTER(vp)]
    L.rsb200_samsung0_plan_create.argtypes = [vp, C.POINTER(SamsungV0Job), i32,
                                              C.POINTER(SamsungV0Strip), i32, C.POINTER(vp)]
    L.rsb200_phaseone_plan_create.argtypes = [vp, C.POINTER(PhaseOneJob), i32,
                                              C.POINTER(PhaseOneStrip), i32, C.POINTER(vp)]
    L.rsb200_arw2_plan_create.argtypes = [vp, C.POINTER(Arw2Job), i32, C.POINTER(C.c_uint16),
                                          i32, i32, C.POINTER(vp)]
    L.rsb200_pentax_plan_create.argtypes = [vp, C.POINTER(HuffTable), i32,
                                            C.POINTER(PentaxJob), i32, C.POINTER(vp)]
    L.rsb200_arw1_plan_create.argtypes = [vp, C.POINTER(Arw1Job), i32, C.POINTER(vp)]
    L.rsb200_samsung1_plan_create.argtypes = [vp, C.POINTER(SamsungV1Job), i32, C.POINTER(vp)]
    L.rsb200_samsung2_plan_create.argtypes = [vp, C.POINTER(SamsungV2Job), i32, C.POINTER(vp)]
    L.rsb200_kodak_plan_create.argtypes = [vp, C.POINTER(KodakJob), i32, vp, i32, C.POINTER(vp)]
    L.rsb200_kodak_plan_values.argtypes = [vp, C.POINTER(C.c_int32), i32]
    L.rsb200_vc5_plan_create.argtypes = [vp, C.POINTER(Vc5Code), i32, C.POINTER(Vc5Job), i32,
                                         C.POINTER(Vc5Band), i32, C.POINTER(vp)]
    L.rsb200_ljpeg_plan_create.argtypes = [vp, C.POINTER(HuffTable), i32,
                                           C.POINTER(LJpegScan), i32, C.POINTER(vp)]
    L.rsb200_cr2_plan_create.argtypes = [vp, C.POINTER(HuffTable), i32,
                                         C.POINTER(Cr2Job), i32, C.POINTER(vp)]
    L.rsb200_plan_run.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, vp]
    L.rsb200_plan_run_host.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, i32]
    L.rsb200_plan_run_host_image.argtypes = [vp, vp, C.c_size_t, vp, C.c_uint32, C.c_uint32,
                                             C.c_uint32, i32]
    L.rsb200_plan_results.argtypes = [vp, C.POINTER(ScanResult), i32]
    u32p = C.POINTER(C.c_uint32)
    L.rsb200_scale_plan_create.argtypes = [vp, C.POINTER(ScaleJob), i32, C.POINTER(vp)]
    L.rsb200_lookup_plan_create.argtypes = [vp, C.POINTER(LookupJob), i32, C.POINTER(C.c_uint16), i32, i32,
                                            C.POINTER(vp)]
    L.rsb200_dngop_plan_create.argtypes = [vp, C.POINTER(DngOpJob), i32, C.POINTER(DngOp), i32,
                                           C.POINTER(C.c_uint16), i32, u32p, i32, C.POINTER(vp)]
    L.rsb200_badpix_plan_create.argtypes = [vp, C.POINTER(BadPixJob), i32, u32p, C.c_uint32, C.POINTER(vp)]
    L.rsb200_plan_bad_pixels.argtypes = [vp, i32, u32p, C.c_uint32, u32p]
    L.rsb200_plan_bytes.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.rsb200_plan_launches.argtypes = [vp]
    L.rsb200_plan_kernels.argtypes = [vp]
    L.rsb200_plan_kernels.restype = C.c_char_p
    L.rsb200_plan_destroy.argtypes = [vp]
    L.rsb200_plan_destroy.restype = None
    L.rsb200_comm_unique_id.argtypes = [vp]
    L.rsb200_comm_create.argtypes = [vp, vp, i32, i32, C.POINTER(vp)]
    L.rsb200_comm_destroy.argtypes = [vp]
    L.rsb200_comm_destroy.restype = None
    L.rsb200_plan_run_gather.argtypes = [vp, vp, vp, C.c_size_t, vp, C.c_size_t, i32, i32, vp]
    _lib = L
    return L
