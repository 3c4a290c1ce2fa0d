"""ctypes face of librawspeed_b200_host.so -- the C++ mirror of the reference's
decompressor classes (csrc/host/).  Same call shapes as the reference's fuzz
drivers; exceptions come back as RawDecoderException / IOException."""
import ctypes as C
import os

import numpy as np

from . import build as _build
from .api import RawDecoderException, IOException, Rsb200Error


class _Err(C.Structure):
    _fields_ = [("code", C.c_int), ("msg", C.c_char * 240)]

    def check(self, rc):
        if rc == 0:
            return
        msg = self.msg.decode("utf-8", "replace")
        if rc == 2:
            raise IOException(2, msg)
        raise RawDecoderException(1, msg)


class _Huff(C.Structure):
    _fields_ = [("ncpl", C.c_uint8 * 16), ("values", C.c_uint8 * 162), ("nvalues", C.c_int)]


EXPORTS = ["rsb200h_unpack", "rsb200h_ljpeg_decompress", "rsb200h_ljpeg_decode",
           "rsb200h_dng_decompress", "rsb200h_cr2_decompress", "rsb200h_cr2_ljpeg_decode",
           "rsb200h_huff_check", "rsb200h_unpack_form", "rsb200h_pentax_decompress", "rsb200h_sony_arw1_decompress", "rsb200h_samsung_v0", "rsb200h_samsung_v1", "rsb200h_samsung_v2", "rsb200h_kodak", "rsb200h_vc5",
           "rsb200h_sraw_interpolate", "rsb200h_nikon_decompress", "rsb200h_sony_arw2",
           "rsb200h_panasonic", "rsb200h_phaseone", "rsb200h_scale_black_white",
           "rsb200h_panasonic_v4", "rsb200h_dng_opcodes", "rsb200h_dngop_lower",
           "rsb200h_fix_bad_pixels", "rsb200h_sixteen_bit_lookup",
           "rsb200h_dng_ljpeg_host_half", "rsb200h_last_call_ms", "rsb200h_hasselblad_ljpeg_decode"]

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_build.HOST_LIB):
            _build.build()
        _lib = C.CDLL(_build.HOST_LIB)
    return _lib


def _u8(data):
    if isinstance(data, np.ndarray):
        assert data.dtype == np.uint8 and data.flags.c_contiguous
        return data.ctypes.data_as(C.c_char_p), data.size
    b = bytes(data)
    return b, len(b)


def _tabs(tabs):
    arr = (_Huff * len(tabs))()
    for i, (ncpl, values) in enumerate(tabs):
        for k in range(16):
            arr[i].ncpl[k] = ncpl[k]
        for k, v in enumerate(values):
            arr[i].values[k] = v
        arr[i].nvalues = len(values)
    return arr


def huff_check(ncpl, values, full=True, fix16=False):
    e = _Err()
    e.check(lib().rsb200h_huff_check(bytes(ncpl), bytes(values), len(values), int(full),
                                     int(fix16), C.byref(e)))


def unpack(data, img, w, cpp, crop, in_pitch, bps, order):
    p, n = _u8(data)
    e = _Err()
    e.check(lib().rsb200h_unpack(p, C.c_uint32(n), C.c_void_p(img.ctypes.data), w, img.shape[0],
                                 cpp, img.shape[1] * 2, crop[0], crop[1], crop[2], crop[3],
                                 in_pitch, bps, order, C.byref(e)))
    return img


def unpack_form(data, img, w, cpp, crop, in_pitch, bps, order, form, curve=None, dither=False):
    """UncompressedDecompressor: readUncompressedRaw on an F32 image (img uint32) or one of
    the fixed-layout members (form 1..6), via the C++ host mirror."""
    p, n = _u8(data)
    e = _Err()
    cp, nc = None, 0
    if curve is not None:
        curve = np.ascontiguousarray(curve, dtype=np.uint16)
        cp, nc = curve.ctypes.data_as(C.POINTER(C.c_uint16)), curve.size
    L = lib()
    L.rsb200h_unpack_form.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p] + [C.c_int] * 13 + \
        [C.POINTER(C.c_uint16), C.c_int, C.c_int, C.POINTER(_Err)]
    e.check(L.rsb200h_unpack_form(p, C.c_uint32(n), C.c_void_p(img.ctypes.data),
                                  int(img.dtype == np.uint32), w, img.shape[0], cpp,
                                  img.shape[1] * img.itemsize, crop[0], crop[1], crop[2],
                                  crop[3], in_pitch, bps, order, form, cp, nc, int(dither),
                                  C.byref(e)))
    return img


def ljpeg_decompress(img, w, cpp, img_frame, mcu, frame_dim, tabs, tab_of_comp, init_pred,
                     rows_per_restart, data, fix16=False):
    p, n = _u8(data)
    toc = (C.c_int * len(tab_of_comp))(*tab_of_comp)
    ip = (C.c_uint16 * len(init_pred))(*init_pred)
    consumed = C.c_uint32(0)
    e = _Err()
    e.check(lib().rsb200h_ljpeg_decompress(
        C.c_void_p(img.ctypes.data), w, img.shape[0], cpp, img.shape[1] * 2, img_frame[0],
        img_frame[1], img_frame[2], img_frame[3], mcu[0], mcu[1], frame_dim[0], frame_dim[1],
        _tabs(tabs), toc, ip, len(tab_of_comp), int(fix16), rows_per_restart, p, C.c_uint32(n),
        C.byref(consumed), C.byref(e)))
    return consumed.value


def ljpeg_decode(blob, img, w, cpp, off, size, max_dim, fix16=False):
    p, n = _u8(blob)
    e = _Err()
    e.check(lib().rsb200h_ljpeg_decode(p, C.c_uint32(n), C.c_void_p(img.ctypes.data), w,
                                       img.shape[0], cpp, img.shape[1] * 2, off[0], off[1],
                                       size[0], size[1], max_dim[0], max_dim[1], int(fix16),
                                       C.byref(e)))
    return img


def dng_decompress(file_bytes, tile_off, tile_len, img, w, cpp, tile_w, tile_h, compression,
                   fix_ljpeg=False, bps=14, big_endian=False):
    p, n = _u8(file_bytes)
    offs = (C.c_uint64 * len(tile_off))(*tile_off)
    lens = (C.c_uint32 * len(tile_len))(*tile_len)
    e = _Err()
    e.check(lib().rsb200h_dng_decompress(p, C.c_uint64(n), offs, lens, len(tile_off),
                                         C.c_void_p(img.ctypes.data),
                                         int(img.dtype == np.uint32), w, img.shape[0], cpp,
                                         img.shape[1] * img.itemsize, tile_w, tile_h,
                                         compression, int(fix_ljpeg), bps, int(big_endian),
                                         C.byref(e)))
    return img


def hasselblad_ljpeg_decode(data, img, w):
    """HasselbladLJpegDecoder(data, img).decode() of the C++ host mirror into img (uint16, pitch =
    img.shape[1] * 2)."""
    p, n = _u8(data)
    e = _Err()
    L = lib()
    L.rsb200h_hasselblad_ljpeg_decode.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                  C.c_void_p]
    e.check(L.rsb200h_hasselblad_ljpeg_decode(p, C.c_uint32(n), C.c_void_p(img.ctypes.data), w, img.shape[0],
                                              img.shape[1] * 2, C.byref(e)))
    return img


def last_call_ms():
    """Wall time of the decompressor's member call inside the last dng_decompress() of this thread
    (the harness around it allocates a RawImage and copies the numpy array in and out)."""
    L = lib()
    L.rsb200h_last_call_ms.restype = C.c_double
    return float(L.rsb200h_last_call_ms())


def pentax_decompress(img, w, data, meta=None, meta_be=True):
    """PentaxDecompressor(img, meta).decompress(data) via the host mirror."""
    p, n = _u8(data)
    mp, mn = (None, 0) if meta is None else _u8(meta)
    e = _Err()
    L = lib()
    L.rsb200h_pentax_decompress.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p,
                                            C.c_int, C.c_int, C.c_char_p, C.c_uint32,
                                            C.POINTER(_Err)]
    e.check(L.rsb200h_pentax_decompress(C.c_void_p(img.ctypes.data), w, img.shape[0],
                                        img.shape[1] * 2, mp, mn, int(meta_be), p,
                                        C.c_uint32(n), C.byref(e)))
    return img


def arw1_decompress(img, w, data):
    """SonyArw1Decompressor(img).decompress(data) via the host mirror; img is (h, pitch) uint16."""
    p, n = _u8(data)
    e = _Err()
    L = lib()
    L.rsb200h_sony_arw1_decompress.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p,
                                               C.c_uint32, C.POINTER(_Err)]
    e.check(L.rsb200h_sony_arw1_decompress(C.c_void_p(img.ctypes.data), w, img.shape[0],
                                           img.shape[1] * 2, p, C.c_uint32(n), C.byref(e)))
    return img


def samsung_v0(img, w, bso, bsr):
    """SamsungV0Decompressor(img, bso, bsr).decompress() via the host mirror; img is (h, pitch) uint16."""
    op, on = _u8(bso)
    rp, rn = _u8(bsr)
    e = _Err()
    L = lib()
    L.rsb200h_samsung_v0.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_uint32,
                                     C.c_char_p, C.c_uint32, C.POINTER(_Err)]
    e.check(L.rsb200h_samsung_v0(C.c_void_p(img.ctypes.data), w, img.shape[0], img.shape[1] * 2, op,
                                 C.c_uint32(on), rp, C.c_uint32(rn), C.byref(e)))
    return img


def samsung_v1(img, w, data, bit=12, cpp=1):
    """SamsungV1Decompressor(img, data, bit).decompress() via the host mirror; img is (h, pitch) uint16
    holding w pixels of `cpp` components per row."""
    p, n = _u8(data)
    e = _Err()
    L = lib()
    L.rsb200h_samsung_v1.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p,
                                     C.c_uint32, C.c_int, C.POINTER(_Err)]
    e.check(L.rsb200h_samsung_v1(C.c_void_p(img.ctypes.data), w, img.shape[0], cpp, img.shape[1] * 2,
                                 p, C.c_uint32(n), bit, C.byref(e)))
    return img


def samsung_v2(img, w, data, bits=12, cpp=1):
    """SamsungV2Decompressor(img, data, bits).decompress() via the host mirror; img is (h, pitch) uint16
    holding w pixels of `cpp` components per row."""
    p, n = _u8(data)
    e = _Err()
    L = lib()
    L.rsb200h_samsung_v2.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p,
                                     C.c_uint32, C.c_uint, C.POINTER(_Err)]
    e.check(L.rsb200h_samsung_v2(C.c_void_p(img.ctypes.data), w, img.shape[0], cpp, img.shape[1] * 2,
                                 p, C.c_uint32(n), bits, C.byref(e)))
    return img


def kodak(img, w, data, bps=12, uncorrected=False, curve=None, dither=False, cpp=1):
    """KodakDecompressor(img, data, bps, uncorrected).decompress() via the host mirror, after
    img.setTable(curve, dither) when a curve is given; img is (h, pitch) uint16 holding w pixels of
    `cpp` components per row."""
    p, n = _u8(data)
    e = _Err()
    L = lib()
    L.rsb200h_kodak.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_uint32, C.c_int,
                                C.c_int, C.c_void_p, C.c_int, C.c_int, C.POINTER(_Err)]
    cv = None if curve is None else np.ascontiguousarray(curve, np.uint16)
    e.check(L.rsb200h_kodak(C.c_void_p(img.ctypes.data), w, img.shape[0], cpp, img.shape[1] * 2, p, C.c_uint32(n),
                            bps, int(uncorrected), None if cv is None else C.c_void_p(cv.ctypes.data),
                            0 if cv is None else cv.size, int(dither), C.byref(e)))
    return img


def vc5(img, w, data, white, phase, codes):
    """VC5Decompressor(data, img, phase, codes).decode(0, 0, w, h) via the host mirror, on an image of white
    level `white` and Bayer phase `phase` (0..3, -1: not a 2x2 CFA); img is (h, pitch) uint16; codes: the
    codebook as an (n, 4) array of {size, bits, count, value}."""
    p, n = _u8(data)
    e = _Err()
    L = lib()
    L.rsb200h_vc5.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_uint32, C.c_int, C.c_int,
                              C.c_void_p, C.c_int, C.POINTER(_Err)]
    cb = np.ascontiguousarray(codes, np.uint32).reshape(-1, 4)
    e.check(L.rsb200h_vc5(C.c_void_p(img.ctypes.data), w, img.shape[0], img.shape[1] * 2, p, C.c_uint32(n), white,
                          phase, C.c_void_p(cb.ctypes.data), cb.shape[0], C.byref(e)))
    return img


def nikon_decompress(img, w, meta, meta_be, bits, data, uncorrected=False):
    """NikonDecompressor(img, meta, bits).decompress(data, uncorrected) via the host mirror."""
    mp, mn = _u8(meta)
    p, n = _u8(data)
    e = _Err()
    L = lib()
    L.rsb200h_nikon_decompress.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p,
                                           C.c_uint32, C.c_int, C.c_int, C.c_char_p, C.c_uint32,
                                           C.c_int, C.POINTER(_Err)]
    e.check(L.rsb200h_nikon_decompress(C.c_void_p(img.ctypes.data), w, img.shape[0],
                                       img.shape[1] * 2, mp, C.c_uint32(mn), int(meta_be), bits,
                                       p, C.c_uint32(n), int(uncorrected), C.byref(e)))
    return img


def panasonic(version, img, w, data, bps=14):
    """PanasonicV{5,6,7}Decompressor(img, data[, bps]).decompress() via the host mirror."""
    p, n = _u8(data)
    e = _Err()
    L = lib()
    L.rsb200h_panasonic.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p,
                                    C.c_uint32, C.c_int, C.POINTER(_Err)]
    e.check(L.rsb200h_panasonic(version, C.c_void_p(img.ctypes.data), w, img.shape[0],
                                img.shape[1] * 2, p, C.c_uint32(n), bps, C.byref(e)))
    return img


def panasonic_v4(img, w, data, zero_is_not_bad=True, split=0, cap=1 << 20, construct_only=False):
    """PanasonicV4Decompressor(img, data, zero_is_not_bad, split).decompress() via the host
    mirror; returns the sorted bad (zero) pixel positions (row << 16 | col)."""
    p, n = _u8(data)
    z = (C.c_uint32 * cap)()
    nz = C.c_uint32(0)
    e = _Err()
    L = lib()
    L.rsb200h_panasonic_v4.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_uint32,
                                       C.c_int, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32,
                                       C.POINTER(C.c_uint32), C.c_int, C.POINTER(_Err)]
    e.check(L.rsb200h_panasonic_v4(C.c_void_p(img.ctypes.data), w, img.shape[0], img.shape[1] * 2,
                                   p, C.c_uint32(n), int(zero_is_not_bad), split, z, cap,
                                   C.byref(nz), int(construct_only), C.byref(e)))
    return sorted(z[:min(nz.value, cap)])


def phaseone(img, w, file, strips):
    """PhaseOneDecompressor(img, strips).decompress() via the host mirror; strips:
    [(offset, size, row)] into `file`."""
    p, n = _u8(file)
    ns = len(strips)
    off = (C.c_uint64 * ns)(*[s[0] for s in strips])
    ln = (C.c_uint32 * ns)(*[s[1] for s in strips])
    rown = (C.c_int32 * ns)(*[s[2] for s in strips])
    e = _Err()
    L = lib()
    L.rsb200h_phaseone.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_uint64,
                                   C.POINTER(C.c_uint64), C.POINTER(C.c_uint32),
                                   C.POINTER(C.c_int32), C.c_int, C.POINTER(_Err)]
    e.check(L.rsb200h_phaseone(C.c_void_p(img.ctypes.data), w, img.shape[0], img.shape[1] * 2, p,
                               C.c_uint64(n), off, ln, rown, ns, C.byref(e)))
    return img


def sony_arw2(img, w, data, curve=None, dither=False):
    """SonyArw2Decompressor(img, data).decompress() via the host mirror; curve:
    img->setTable(curve, dither) first."""
    p, n = _u8(data)
    cp, nc = None, 0
    if curve is not None:
        curve = np.ascontiguousarray(curve, dtype=np.uint16)
        cp, nc = curve.ctypes.data_as(C.POINTER(C.c_uint16)), curve.size
    e = _Err()
    L = lib()
    L.rsb200h_sony_arw2.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_uint32,
                                    C.POINTER(C.c_uint16), C.c_int, C.c_int, C.POINTER(_Err)]
    e.check(L.rsb200h_sony_arw2(C.c_void_p(img.ctypes.data), w, img.shape[0], img.shape[1] * 2,
                                p, C.c_uint32(n), cp, nc, int(dither), C.byref(e)))
    return img


def dng_ljpeg_host_half(file_bytes, tile_off, tile_len, w, h, cpp, tile_w, tile_h, fix_ljpeg=False,
                        threads=0, reps=3, want_scans=False):
    """AbstractDngDecompressor::prepareLJpeg alone (header walk, validation, restart scan, scan
    descriptors; no GPU): dict(ms=best wall ms, scans, tables, errors, digest of everything it
    produced).  threads: 0 = the library's default."""
    p, n = _u8(file_bytes)
    offs = (C.c_uint64 * len(tile_off))(*tile_off)
    lens = (C.c_uint32 * len(tile_len))(*tile_len)
    ms, ns, nt, ne, dg = C.c_double(0), C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
    e = _Err()
    L = lib()
    L.rsb200h_dng_ljpeg_host_half.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint64),
                                              C.POINTER(C.c_uint32)] + [C.c_int] * 9 + [
        C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
        C.POINTER(C.c_uint64), C.c_void_p, C.c_uint32, C.c_char_p, C.c_int, C.POINTER(_Err)]
    from ._abi import LJpegScan
    first = C.create_string_buffer(512)
    cap = 1 << 18 if want_scans else 0
    buf = (LJpegScan * cap)() if want_scans else None
    e.check(L.rsb200h_dng_ljpeg_host_half(p, C.c_uint64(n), offs, lens, len(tile_off), w, h, cpp,
                                          tile_w, tile_h, int(fix_ljpeg), int(threads), reps,
                                          C.byref(ms), C.byref(ns), C.byref(nt), C.byref(ne),
                                          C.byref(dg), buf, cap, first, 512, C.byref(e)))
    out = dict(ms=ms.value, scans=ns.value, tables=nt.value, errors=ne.value, digest=dg.value,
               first_error=first.value.decode("utf-8", "replace"))
    if want_scans:
        out["scan_list"] = [buf[i] for i in range(min(ns.value, cap))]
    return out


def sixteen_bit_lookup(img, w, cpp, curve, dither):
    """mRaw->setTable(curve, dither); mRaw->sixteenBitLookup() via the host mirror, in place."""
    cp, nc = None, 0
    if curve is not None:
        curve = np.ascontiguousarray(curve, dtype=np.uint16)
        cp, nc = curve.ctypes.data_as(C.POINTER(C.c_uint16)), curve.size
    e = _Err()
    L = lib()
    L.rsb200h_sixteen_bit_lookup.argtypes = [C.c_void_p] + [C.c_int] * 4 + [C.POINTER(C.c_uint16), C.c_int,
                                                                            C.c_int, C.POINTER(_Err)]
    e.check(L.rsb200h_sixteen_bit_lookup(C.c_void_p(img.ctypes.data), w, img.shape[0], cpp,
                                         img.shape[1] * 2, cp, nc, int(dither), C.byref(e)))
    return img


def fix_bad_pixels(img, w, cpp, positions, is_cfa=True, map_only=False):
    """RawImageData::fixBadPixels() via the host mirror, in place; map_only: only
    transferBadPixelsToMap(), returns the bitmap (rows of roundUp(ceil(w / 8), 16) bytes)."""
    pos = np.ascontiguousarray(positions, dtype=np.uint32)
    mp = ((w + 7) // 8 + 15) // 16 * 16
    m = np.zeros((img.shape[0], mp), dtype=np.uint8)
    e = _Err()
    L = lib()
    L.rsb200h_fix_bad_pixels.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_uint32, C.c_int,
                                                                        C.c_void_p, C.POINTER(_Err)]
    e.check(L.rsb200h_fix_bad_pixels(C.c_void_p(img.ctypes.data), w, img.shape[0], cpp,
                                     img.shape[1] * 2, int(is_cfa), pos.ctypes.data, pos.size,
                                     int(map_only), m.ctypes.data, C.byref(e)))
    return m if map_only else img


def dng_opcodes(img, w, cpp, crop, data, cap=1 << 20):
    """DngOpcodes(ri, data) + applyOpCodes(ri) via the host mirror, in place; img: uint16 image or
    uint32 array holding an F32 image; crop = [off_x, off_y, crop_w, crop_h].  Returns (crop,
    mBadPixelPositions); dng_opcodes.stage = which half threw (1 constructor, 2 apply, 0 none)."""
    p, n = _u8(data)
    cr = (C.c_int * 4)(*[int(v) for v in crop])
    bad = (C.c_uint32 * cap)()
    nbad = C.c_uint32(0)
    stage = C.c_int(0)
    e = _Err()
    L = lib()
    is_f32 = img.dtype == np.uint32
    L.rsb200h_dng_opcodes.argtypes = [C.c_void_p] + [C.c_int] * 5 + [
        C.POINTER(C.c_int), C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32,
        C.POINTER(C.c_uint32), C.POINTER(C.c_int), C.POINTER(_Err)]
    rc = L.rsb200h_dng_opcodes(C.c_void_p(img.ctypes.data), int(is_f32), w, img.shape[0], cpp,
                               img.shape[1] * img.itemsize, cr, p, C.c_uint32(n), bad, cap,
                               C.byref(nbad), C.byref(stage), C.byref(e))
    dng_opcodes.stage = stage.value
    dng_opcodes.partial = (list(cr), list(bad[:min(nbad.value, cap)]))
    e.check(rc)
    return list(cr), list(bad[:min(nbad.value, cap)])


def dngop_lower(img, w, cpp, crop, data):
    """DngOpcodes(ri, data).lower(ri): the device form of the list (no GPU needed).  Returns a
    dict(ops=[DngOp], tables=(n,65536) uint16, deltas=uint32[], actions=[(kind, index, list or
    roi)], error=exception or None); a constructor error raises."""
    from ._abi import DngOp
    p, n = _u8(data)
    cr = (C.c_int * 4)(*[int(v) for v in crop])
    ops = (DngOp * 64)()
    tables = np.zeros((16, 65536), dtype=np.uint16)
    deltas = np.zeros(1 << 18, dtype=np.uint32)
    actions = (C.c_uint32 * (4 * 64))()
    rois = (C.c_uint32 * (4 * 64))()
    lists = np.zeros(1 << 20, dtype=np.uint32)
    cnt = (C.c_uint32 * 4)(*([0xFFFFFFFF] * 4))   # still the sentinel = the constructor threw
    e = _Err()
    L = lib()
    L.rsb200h_dngop_lower.argtypes = [C.c_void_p] + [C.c_int] * 5 + [
        C.POINTER(C.c_int), C.c_char_p, C.c_uint32, C.POINTER(DngOp), C.c_uint32, C.c_void_p,
        C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32,
        C.POINTER(C.c_uint32), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(_Err)]
    rc = L.rsb200h_dngop_lower(C.c_void_p(img.ctypes.data), int(img.dtype == np.uint32), w,
                               img.shape[0], cpp, img.shape[1] * img.itemsize, cr, p, C.c_uint32(n),
                               ops, 64, tables.ctypes.data, 16, deltas.ctypes.data, deltas.size,
                               actions, 64, cnt, lists.ctypes.data, lists.size, rois, C.byref(e))
    err = None
    if rc != 0:
        if cnt[0] == 0xFFFFFFFF:
            e.check(rc)
        try:
            e.check(rc)
        except Exception as ex:   # noqa: BLE001
            err = ex
    acts = []
    for i in range(cnt[3]):
        kind, index, a, b = actions[4 * i:4 * i + 4]
        if kind == 0:
            acts.append((0, index, lists[b:b + a].tolist()))
        elif kind == 2:
            acts.append((2, index, tuple(rois[4 * i:4 * i + 4])))
        else:
            acts.append((1, index, None))
    return dict(ops=[DngOp.from_buffer_copy(ops[i]) for i in range(cnt[0])],
                tables=tables[:cnt[1]].copy(), deltas=deltas[:cnt[2]].copy(), actions=acts,
                error=err)


def scale_black_white(img, w, crop, black_level=-1, black_sep=None, white=None, areas=(),
                      dither=True, is_cfa=True, cpp=1, path=0, host_part_only=False):
    """RawImageData::scaleBlackWhite() via the host mirror, in place; crop = (off_x, off_y,
    crop_w, crop_h) applied with subFrame(); areas: [(is_vertical, offset, size)].  Returns
    (blackLevelSeparate or None, whitePoint).  host_part_only: the estimate and the black-area
    medians without the device pass (needs no GPU)."""
    b = (C.c_int * 4)(*([int(v) for v in black_sep] if black_sep is not None else [-7] * 4))
    wh = C.c_int(int(white) if white is not None else 0)
    flat = [int(x) for a in areas for x in a] or [0]
    ar = (C.c_int * len(flat))(*flat)
    sep_set = C.c_int(0)
    e = _Err()
    L = lib()
    L.rsb200h_scale_black_white.argtypes = [C.c_void_p] + [C.c_int] * 10 + [
        C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int)] + \
        [C.c_int] * 4 + [C.POINTER(C.c_int), C.POINTER(_Err)]
    e.check(L.rsb200h_scale_black_white(
        C.c_void_p(img.ctypes.data), w, img.shape[0], cpp, img.shape[1] * 2, int(is_cfa),
        crop[0], crop[1], crop[2], crop[3], int(black_level), b, int(black_sep is not None),
        C.byref(wh), int(white is not None), ar, len(areas), int(dither), int(path),
        1 if host_part_only else 0, C.byref(sep_set), C.byref(e)))
    return (list(b) if sep_set.value else None), wh.value


def sraw_interpolate(inp, in_w, out, out_w, sub, coeffs, hue, version):
    """Cr2sRawInterpolator(out, inp, coeffs, hue).interpolate(version) via the host mirror."""
    k = (C.c_int * 3)(*coeffs)
    e = _Err()
    L = lib()
    L.rsb200h_sraw_interpolate.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p] + \
        [C.c_int] * 5 + [C.POINTER(C.c_int), C.c_int, C.c_int, C.POINTER(_Err)]
    e.check(L.rsb200h_sraw_interpolate(inp.ctypes.data, in_w, inp.shape[0], inp.shape[1] * 2,
                                       out.ctypes.data, out_w, out.shape[0], out.shape[1] * 2,
                                       sub[0], sub[1], k, hue, version, C.byref(e)))
    return out


def cr2_decompress(img, w, fmt, frame, slicing, tabs, tab_of_comp, init_pred, data, is_cfa=True):
    p, n = _u8(data)
    toc = (C.c_int * len(tab_of_comp))(*tab_of_comp)
    ip = (C.c_uint16 * len(init_pred))(*init_pred)
    consumed = C.c_uint32(0)
    e = _Err()
    e.check(lib().rsb200h_cr2_decompress(
        C.c_void_p(img.ctypes.data), w, img.shape[0], img.shape[1] * 2, int(is_cfa), fmt[0],
        fmt[1], fmt[2], frame[0], frame[1], slicing[0], slicing[1], slicing[2], _tabs(tabs), toc,
        ip, len(tab_of_comp), p, C.c_uint32(n), C.byref(consumed), C.byref(e)))
    return consumed.value


def cr2_ljpeg_decode(blob, img, w, slicing, is_cfa=True, sub=(1, 1)):
    p, n = _u8(blob)
    e = _Err()
    e.check(lib().rsb200h_cr2_ljpeg_decode(p, C.c_uint32(n), C.c_void_p(img.ctypes.data), w,
                                           img.shape[0], img.shape[1] * 2, int(is_cfa), sub[0],
                                           sub[1], slicing[0], slicing[1], slicing[2],
                                           C.byref(e)))
    return img
