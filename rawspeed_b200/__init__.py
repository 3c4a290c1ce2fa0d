"""rawspeed_b200 -- H100-native (sm_90a) RAW decompression engine for the
per-pixel decode hot path of darktable-org/rawspeed.

    csrc/             hand-written CUDA kernels + the extern "C" ABI
                      (include/rawspeed_b200.h) + the C++ host mirror of the
                      reference's decompressor classes (csrc/host/)
    _abi.py / api.py  ctypes face of the ABI (plans, contexts)
    build.py          in-tree nvcc build for sm_90a

Nothing in this package imports oracle/ (the CPU checker).  There is no CPU
fallback: without the CUDA library and a GPU the API raises."""
from .api import (Context, Plan, Rsb200Error, RawDecoderException, IOException,  # noqa: F401
                  huff_table, unpack_plan, raw_plan, sraw_plan, SrawJob, arw2_plan, Arw2Job, nikon_plan, NikonJob, pana_plan, PanaJob, scale_plan, ScaleJob, dngop_plan, DngOp, DngOpJob, badpix_plan, BadPixJob, lookup_plan, LookupJob, phaseone_plan, PhaseOneJob, PhaseOneStrip, samsung0_plan, SamsungV0Job, SamsungV0Strip, samsung1_plan, SamsungV1Job, samsung2_plan, SamsungV2Job, kodak_plan, KodakJob, vc5_plan, Vc5Job, Vc5Band, Vc5Code, hasselblad_plan, HasselbladJob, pentax_plan, PentaxJob, arw1_plan, Arw1Job, ljpeg_plan, cr2_plan, image_pitch,
                  new_image, RawJob, UnpackJob, LJpegScan, Cr2Job, HuffTable, LSB, MSB, MSB16, MSB32,
                  Comm, comm_unique_id, GATHER_NONE, GATHER_ALL, GATHER_ROOT)
from . import _abi as formats  # noqa: F401  (formats.RAW_* constants)
from . import build as _build  # noqa: F401

__all__ = ["Context", "Plan", "Rsb200Error", "RawDecoderException", "IOException",
           "huff_table", "unpack_plan", "raw_plan", "RawJob", "sraw_plan", "SrawJob", "arw2_plan", "Arw2Job", "nikon_plan", "NikonJob", "pana_plan", "PanaJob", "scale_plan", "ScaleJob", "dngop_plan", "DngOp", "DngOpJob", "badpix_plan", "BadPixJob", "lookup_plan", "LookupJob", "phaseone_plan", "PhaseOneJob", "PhaseOneStrip", "samsung0_plan", "SamsungV0Job", "SamsungV0Strip", "samsung1_plan", "SamsungV1Job", "samsung2_plan", "SamsungV2Job", "kodak_plan", "KodakJob", "vc5_plan", "Vc5Job", "Vc5Band", "Vc5Code", "hasselblad_plan", "HasselbladJob", "pentax_plan", "PentaxJob", "arw1_plan", "Arw1Job", "ljpeg_plan", "cr2_plan", "image_pitch",
           "new_image", "UnpackJob", "LJpegScan", "Cr2Job", "HuffTable", "LSB", "MSB",
           "MSB16", "MSB32", "Comm", "comm_unique_id", "GATHER_NONE", "GATHER_ALL", "GATHER_ROOT"]
