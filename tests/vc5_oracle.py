"""GoPro VC-5 (VC5Decompressor) for the tests: the CPU restatement and band writer of
tests/emu/vc5_oracle.c, the codebook fixture, a writer of whole VC-5 datablocks, synthetic band content
and the band table the device plans take."""
import ctypes as C
import json
import os
import re

import numpy as np

from helpers import compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "vc5_oracle.c")
OUT = os.path.join(HERE, "emu", "_build", "libvc5_oracle.so")
CODEBOOK = os.path.join(HERE, "golden", "vc5_codebook.json")

# band outcomes: RSB200_VC5_* of the C ABI
OK, QUANT, EARLY_END, OVERRUN, NO_END, SHORT, OVERREAD = range(7)
BAND_MESSAGES = {
    QUANT: "Impossible RLV value given current quantum",
    EARLY_END: "Got EndOfBand marker while looking for next pixel",
    OVERRUN: "Not all pixels consumed?",
    NO_END: "EndOfBand marker not found",
    SHORT: "Bit stream size is smaller than MaxProcessBytes",
    OVERREAD: "Buffer overflow read in BitStreamer",
}
BAND_IOE = {SHORT, OVERREAD}
TOO_MANY = 64
# constructor and tag-walk outcomes (vc5_oracle.c), their messages and exception classes
CTOR_MESSAGES = {
    16: "Bad image dimensions.", 17: "Width %i is not a multiple of %i", 18: "Height %i is not a multiple of %i",
    19: "Image has invalid CFA.", 20: "Unexpected bayer phase, please file a bug.", 21: "Bad white level %i",
    22: "not a valid VC-5 datablock", 23: "Bad channel count %u, expected %i", 24: "Image width mismatch: %u vs %i",
    25: "Image height mismatch: %u vs %i", 26: "Invalid precision %i", 27: "Bad channel number (%u)",
    28: "Image format %i is not 4(RAW)", 29: "Unexpected subband count %u, expected %i",
    30: "Bad bits per componend %u, not %i", 31: "Bad pattern width %u, not %u", 32: "Bad pattern height %u, not %u",
    33: "Bad subband number %u", 34: "Bad component per sample count %u, not %u",
    35: "Unknown (unhandled) non-optional Tag 0x%04x", 36: "Did not see VC5Tag::SubbandNumber yet",
    37: "Band %i for wavelet %i on channel %u was already seen", 38: "Did not see VC5Tag::LowpassPrecision yet",
    39: "Did not see VC5Tag::Quantization yet", 40: "Out of bounds access in ByteStream",
    41: "Buffer overflow: image file may be truncated",
}
CTOR_IOE = {40, 41}
FILL_DEFAULT = 0xABCD
RGGB, GBRG = 0, 2
_lib = None
_codes = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(OUT) or os.path.getmtime(SRC) > os.path.getmtime(OUT):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            compile_shared(["gcc", "-std=c99", "-O2", "-Wall", "-fPIC", "-shared", "-o", OUT, SRC, "-lm"])
        L = C.CDLL(OUT)
        P, i = C.c_void_p, C.c_int
        L.vc_decompress.argtypes = [C.c_char_p, i, i, i, i, i, P, i, P, i, P]
        L.vc_parse.argtypes = [C.c_char_p, i, i, i, i, i, P, P, P, P]
        L.vc_decode_band.argtypes = [C.c_char_p, i, i, i, i, P, i, P]
        L.vc_symbols.argtypes = [P, C.c_int64, i, P, i, P, C.c_int64]
        L.vc_symbols.restype = C.c_int64
        L.vc_pack.argtypes = [P, C.c_int64, P, P, C.c_int64]
        L.vc_pack.restype = C.c_int64
        _lib = L
    return _lib


def codebook():
    """The codebook fixture: an (n, 4) int32 array of {size, bits, count, value}."""
    global _codes
    if _codes is None:
        with open(CODEBOOK) as f:
            _codes = np.ascontiguousarray(json.load(f)["entries"], np.int32)
    return _codes


def decompand(v):
    c = float(v)
    c += (c * c * c * 768) / (255. * 255. * 255.)
    return int(max(-32768.0, min(32767.0, c)))


def pitch_elems(w):
    """RawImageData::createData(): pitch = roundUp(w*2, 16) bytes."""
    return (w * 2 + 15) // 16 * 16 // 2


def band_dims(w, h):
    """[(w, h)] of wavelets 1..3 (index 0: the image's half)."""
    out = []
    for _ in range(4):
        w, h = (w + 1) // 2, (h + 1) // 2
        out.append((w, h))
    return out


def level_of(subband):
    return 3 if subband == 0 else 3 - (subband - 1) // 3


def strip_prefixes(what):
    """A reference message without the "function, line N: " in front of it and of a nested message."""
    return "\n".join(re.sub(r"^.*?, line [0-9]+: ", "", part, count=1) for part in what.split("\n"))


def message(rc, args):
    """The reference's text (prefixes stripped) for outcome rc of vc_decompress."""
    if rc == OK:
        return ""
    if rc > TOO_MANY:
        return "Too many errors encountered. Giving up. First Error:\n" + BAND_MESSAGES[rc - TOO_MANY]
    m = CTOR_MESSAGES[rc]
    n = m.count("%")
    return m.replace("%u", "%d").replace("%i", "%d") % tuple(args[:n]) if n else m


def is_ioe(rc):
    """Whether the reference throws outcome rc as an IOException: constructor / tag-walk outcomes only, since
    a band failure comes out of decode() as "Too many errors ...", a RawDecoderException, whatever the
    band's own class."""
    return rc in CTOR_IOE


# ---------------------------------------------------------------- restatement
def decompress(data, w, h, white, cfa=RGGB, fill=FILL_DEFAULT, codes=None):
    """-> (image (h, pitch) uint16, outcome, args)"""
    cb = codebook() if codes is None else np.ascontiguousarray(codes, np.int32)
    img = np.full((max(h, 1), pitch_elems(max(w, 1))), fill, np.uint16)
    args = np.zeros(4, np.int32)
    data = bytes(data)
    rc = lib().vc_decompress(data, len(data), w, h, white, cfa, cb.ctypes.data, cb.shape[0], img.ctypes.data,
                             img.shape[1], args.ctypes.data)
    assert rc >= 0
    return img, rc, [int(a) for a in args]


def parse(data, w, h, white, cfa=RGGB):
    """-> (outcome, bands (40, 3) [offset, size, param] in channel * 10 + subband order, prescale (4, 3),
    output bits)"""
    bands = np.zeros((40, 3), np.int32)
    pre = np.zeros((4, 3), np.int32)
    bits, args = np.zeros(1, np.int32), np.zeros(4, np.int32)
    data = bytes(data)
    rc = lib().vc_parse(data, len(data), w, h, white, cfa, bands.ctypes.data, pre.ctypes.data, bits.ctypes.data,
                        args.ctypes.data)
    return rc, bands, pre, int(bits[0])


# ---------------------------------------------------------------- writer
def band_symbols(values, quant):
    """(n, 2) [entry, sign] symbols of a high-pass band, end marker included."""
    v = np.ascontiguousarray(values, np.int16).reshape(-1)
    cb = codebook()
    cap = v.size + 2
    syms = np.zeros((cap, 2), np.int32)
    n = lib().vc_symbols(v.ctypes.data, v.size, quant, cb.ctypes.data, cb.shape[0], syms.ctypes.data, cap)
    assert n > 0, n
    return syms[:n].copy()


def pack(syms):
    """Bytes (whole 4-byte words) of a symbol list."""
    s = np.ascontiguousarray(syms, np.int32).reshape(-1, 2)
    cb = codebook()
    cap = 4 * len(s) + 8
    out = np.zeros(cap, np.uint8)
    n = lib().vc_pack(s.ctypes.data, len(s), cb.ctypes.data, out.ctypes.data, cap)
    assert n >= 0
    return out[:n].tobytes()


def entry(count, value):
    """Index of the codebook entry with this run length and (unsigned) value."""
    cb = codebook()
    i = np.nonzero((cb[:, 2] == count) & (cb[:, 3] == value))[0]
    assert i.size, (count, value)
    return int(i[0])


def lowpass_bytes(values, prec):
    """A low-pass band: prec bits per value, MSB first, padded to whole 8-byte chunks."""
    v = np.asarray(values, np.int64).reshape(-1) & ((1 << prec) - 1)
    bits = ((v[:, None] >> np.arange(prec - 1, -1, -1)) & 1).astype(np.uint8).reshape(-1)
    nbytes = 8 * ((v.size * prec + 63) // 64)
    out = np.zeros(nbytes * 8, np.uint8)
    out[:bits.size] = bits
    return np.packbits(out).tobytes()


def tag(t, v):
    return int(t & 0xFFFF).to_bytes(2, "big") + int(v & 0xFFFF).to_bytes(2, "big")


HEADER_TAGS = [(0x000c, 4), (0x0054, 4), (0x000e, 10), (0x0066, 12), (0x006a, 2), (0x006b, 2), (0x006c, 1)]


def chunk(payload):
    """A LargeCodeblock chunk (payload: whole 4-byte words)."""
    assert len(payload) % 4 == 0
    n = len(payload) // 4
    return tag(0x6000 | (n >> 16), n & 0xFFFF) + payload


def datablock(w, h, payloads, params, prescale=None, header=None):
    """A VC-5 datablock: header tags, then per channel ChannelNumber, PrescaleShift and its ten subbands
    (LowpassPrecision or Quantization, SubbandNumber, LargeCodeblock).  payloads[ch][s]: bytes;
    params[ch][s]: precision or quantization; prescale[ch]: three 2-bit shifts (wavelet 1, 2, 3)."""
    out = b"VC-5"
    for t, v in (header if header is not None else [(0x0014, w), (0x0015, h)] + HEADER_TAGS):
        out += tag(t, v)
    for ch in range(4):
        out += tag(0x003e, ch)
        if prescale is not None:
            p = prescale[ch]
            out += tag(0x006d, p[0] << 14 | p[1] << 12 | p[2] << 10)
        for s in range(10):
            out += tag(0x0023 if s == 0 else 0x0035, params[ch][s])
            out += tag(0x0030, s)
            out += chunk(payloads[ch][s])
    return out


def encode(w, h, content, prec=16, quants=None, prescale=None):
    """A datablock of band content: content[ch][s] (bh, bw) int arrays (subband 0: the low-pass values,
    the others multiples of decompand(m) * quant)."""
    dims = band_dims(w, h)
    payloads, params = [], []
    for ch in range(4):
        pl, pa = [], []
        for s in range(10):
            bw, bh = dims[level_of(s)]
            v = np.asarray(content[ch][s]).reshape(bh, bw)
            if s == 0:
                pl.append(lowpass_bytes(v, prec))
                pa.append(prec)
            else:
                q = 1 if quants is None else quants[ch][s]
                pl.append(pack(band_symbols(v, q)))
                pa.append(q)
        payloads.append(pl)
        params.append(pa)
    return datablock(w, h, payloads, params, prescale)


# ---------------------------------------------------------------- content
def magnitudes(quant):
    return np.array([decompand(m) * abs(quant) for m in range(256)], np.int64)


def natural(w, h, seed=0, quant=1, sparsity=0.9, span=4095):
    """Smooth low-pass bands whose reconstruction spans about 0..span, and sparse high-pass bands of
    small magnitudes (mostly zero runs).  Use with prescale 2 at every wavelet (unit gain per level)."""
    rng = np.random.default_rng(seed)
    dims = band_dims(w, h)
    mags = magnitudes(quant)
    out = []
    for ch in range(4):
        bands = []
        for s in range(10):
            bw, bh = dims[level_of(s)]
            if s == 0:
                y, x = np.mgrid[0:bh, 0:bw]
                base = 0.5 * (1 + np.sin(x / (3.0 + ch) + seed) * np.cos(y / 5.0 + ch))
                lo = span * base if ch == 0 else 2048 + (span / 4) * (base - 0.5)
                bands.append(np.clip(lo, 0, 65535).astype(np.int64))
            else:
                m = rng.geometric(0.5, size=(bh, bw)).clip(1, 12)
                sign = rng.choice([-1, 1], size=(bh, bw))
                keep = rng.random((bh, bw)) > sparsity
                bands.append(np.where(keep, sign * mags[m], 0).astype(np.int64) * (1 if quant >= 0 else -1))
        out.append(bands)
    return out


def noise(w, h, seed=0, quant=1, top=255):
    """Dense high-pass bands: every coefficient a random magnitude 0..top (long codes), random low pass."""
    rng = np.random.default_rng(seed)
    dims = band_dims(w, h)
    mags = magnitudes(quant)
    out = []
    for ch in range(4):
        bands = []
        for s in range(10):
            bw, bh = dims[level_of(s)]
            if s == 0:
                bands.append(rng.integers(0, 1 << 16, size=(bh, bw)))
            else:
                m = rng.integers(0, top + 1, size=(bh, bw))
                sign = rng.choice([-1, 1], size=(bh, bw))
                bands.append(sign * mags[m] * (1 if quant >= 0 else -1))
        out.append(bands)
    return out


def flat(w, h, level=1000):
    """Constant low pass, all-zero high-pass bands (one long zero run each)."""
    dims = band_dims(w, h)
    return [[np.full(dims[level_of(s)][::-1], level if s == 0 else 0, np.int64) for s in range(10)]
            for _ in range(4)]


# ---------------------------------------------------------------- device band table
def band_table(data, w, h, white, cfa=RGGB):
    """(job fields, [(offset, size, param)] x 40) of a datablock the tag walk accepts, for the plans."""
    rc, bands, pre, bits = parse(data, w, h, white, cfa)
    assert rc == OK, rc
    return dict(width=w, height=h, output_bits=bits, phase=cfa, prescale=pre), [tuple(int(x) for x in b)
                                                                                for b in bands]


def plan_inputs(frames, skew=0, pitch_extra=0, gap=32):
    """frames: [(data, w, h, white, cfa)] datablocks the tag walk accepts -> (blob, [Vc5Job], [Vc5Band],
    [(element offset, h, pitch in elements)], output elements): the datablocks one after the other (each
    at a 16-byte boundary + skew), 40 bands per job, images `gap` elements apart."""
    import rawspeed_b200 as rs
    blob, jobs, bands, outs, off = bytearray(), [], [], [], gap
    for data, w, h, white, cfa in frames:
        blob += bytes((-len(blob)) % 16 + skew)
        base = len(blob)
        blob += data
        fields, table = band_table(data, w, h, white, cfa)
        j = rs.Vc5Job()
        j.width, j.height, j.output_bits, j.phase = w, h, fields["output_bits"], cfa
        for ch in range(4):
            for k in range(3):
                j.prescale[ch][k] = int(fields["prescale"][ch][k])
        j.first_band = len(bands)
        for o, size, param in table:
            b = rs.Vc5Band()
            b.in_offset, b.in_size, b.param = base + o, size, param
            bands.append(b)
        pitch = pitch_elems(w) + pitch_extra
        j.out_offset, j.out_pitch = 2 * off, 2 * pitch
        jobs.append(j)
        outs.append((off, h, pitch))
        off += h * pitch + gap
    return bytes(blob), jobs, bands, outs, off


def expected(frames, fill=FILL_DEFAULT, pitch_extra=0):
    """Per frame: (image (h, pitch), (status, consumed)) of the restatement, as a plan reports them."""
    out = []
    for data, w, h, white, cfa in frames:
        img, rc, args = decompress(data, w, h, white, cfa, fill)
        if pitch_extra:
            img = np.concatenate([img, np.full((img.shape[0], pitch_extra), fill, np.uint16)], axis=1)
        if rc == OK:
            out.append((img, (0, 0)))
        else:
            assert rc > TOO_MANY, rc
            code = rc - TOO_MANY
            out.append((img, (2 if code in BAND_IOE else 1, code << 28 | args[0] << 4 | args[1])))
    return out
