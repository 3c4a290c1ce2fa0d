"""GoPro VC-5 DNG files (compression 9, one tile covering the image, WhiteLevel set) through the
reference's own consumer API: once through the unmodified reference (oracle/_ref/libref_full.so) and
once through the drop-in (oracle/_ref/libdropin.so), whose AbstractDngDecompressor sends compression 9
to the device with the codebook of the reference checkout it was built against.  CPU: the unmodified
build agrees with the restatement.  GPU: the drop-in gives the same image, and the same message for
corrupt bands and for a VC-5 tile that does not cover the image."""
import numpy as np
import pytest

import dngfile
import test_oracle_vc5 as T
import vc5_oracle as V
from test_dropin import _lib, decode_file

LONG, SHORT = 4, 3


def vc5_dng(data, w, h, white, cfa_pattern=(0, 1, 1, 2), tile=None):
    """A DNG whose raw IFD holds the datablock as one tile of w x h (or `tile`)."""
    tw, th = tile or (w, h)
    n = ((w + tw - 1) // tw) * ((h + th - 1) // th)  # every tile holds the same datablock
    e = [x for x in dngfile.dng_common(w, h, 16, 9) if x[0] != 33422]
    e += [(33422, 1, list(cfa_pattern)), (50717, LONG, [white]),
          (322, LONG, [tw]), (323, LONG, [th]),
          (324, LONG, lambda base: [base + k * len(data) for k in range(n)]),
          (325, LONG, [len(data)] * n)]
    return dngfile.build_tiff(e, bytes(data) * n)


def message(lib, f):
    try:
        decode_file(lib, f, threads=1)
        return ""
    except RuntimeError as e:
        return V.strip_prefixes(str(e).split(": ", 1)[1])


def cases():
    good = [(T.golden_cases_by_name()[n]) for n in ("dims_34_48", "phase_2", "quant_-3", "noise", "flat")]
    out = [("%s" % i, vc5_dng(d, w, h, white, (1, 2, 0, 1) if cfa == V.GBRG else (0, 1, 1, 2)), (d, w, h, white, cfa))
           for i, (d, w, h, white, cfa) in enumerate(good)]
    data, w, h, white, cfa = T.failing_block(46, 38, {(2, 5): V.NO_END}), 46, 38, 4095, V.RGGB
    out.append(("bad_band", vc5_dng(data, w, h, white), (data, w, h, white, cfa)))
    data = T.failing_block(46, 38, {(0, 7): V.SHORT, (3, 1): V.EARLY_END})
    out.append(("two_bad_bands", vc5_dng(data, 46, 38, 4095), (data, 46, 38, 4095, V.RGGB)))
    return out


def test_reference_build_decodes_the_vc5_files():
    ref = _lib("libref_full.so")
    for name, f, (data, w, h, white, cfa) in cases():
        want, rc, _ = V.decompress(data, w, h, white, cfa)
        if rc != V.OK:
            assert "Too many errors" in message(ref, f), name
            continue
        got, (gw, gh, cpp, pitch, nerr) = decode_file(ref, f, threads=1)
        assert (gw, gh, nerr) == (w, h, 0) and np.array_equal(got[:h, :w], want[:h, :w]), name


@pytest.mark.gpu
def test_dropin_matches_the_reference():
    ref, dropin = _lib("libref_full.so"), _lib("libdropin.so")
    for name, f, _ in cases():
        mr, md = message(ref, f), message(dropin, f)
        assert md == mr, (name, md, mr)
        if not mr:
            a, ia = decode_file(ref, f, threads=1)
            b, ib = decode_file(dropin, f, threads=1)
            assert ia == ib and np.array_equal(a, b), name
    # a tile that does not cover the image: the reference's whole-image check
    data, w, h, white, cfa = T.golden_cases_by_name()["dims_34_48"]
    f = vc5_dng(data, w, h, white, tile=(w, h // 2))
    assert message(dropin, f) == message(ref, f) != ""
