"""The host mirror VC5Decompressor (rsb200h_vc5) without a GPU: its constructor runs the reference's
checks and tag walk on the host, so every golden case the reference rejects there is rejected before
anything reaches the device, with the reference's exception class and text, and the image untouched."""
import re

import numpy as np

import rawspeed_b200 as rs
from rawspeed_b200 import host
import test_oracle_vc5 as T
import vc5_oracle as V


def host_run(data, w, h, white, cfa):
    """VC5Decompressor(data, img, phase, codebook).decode(0, 0, w, h) through the host mirror ->
    (image, message without the engine's prefix, is IOException)."""
    img = np.full((h, V.pitch_elems(w)), V.FILL_DEFAULT, np.uint16)
    try:
        host.vc5(img, w, np.frombuffer(bytes(data), np.uint8).copy(), white, cfa if cfa < 4 else -1, V.codebook())
        return img, "", False
    except (rs.RawDecoderException, rs.IOException) as e:
        return img, re.sub(r"^rsb200 error -?[0-9]+: ", "", str(e)), isinstance(e, rs.IOException)


def test_constructor_rejections_match_the_reference():
    n = 0
    for name, (data, w, h, white, cfa) in T.golden_cases():
        want, rc, args = V.decompress(data, w, h, white, cfa)
        if rc == V.OK or rc > V.TOO_MANY or w <= 0 or h <= 0:
            continue  # (decodes, or fails in a band: the device's part, tests/test_gpu_vc5.py)
        img, text, ioe = host_run(data, w, h, white, cfa)
        assert text == V.message(rc, args), (name, text)
        assert ioe == V.is_ioe(rc), name
        assert np.array_equal(img, want[:h]), name
        n += 1
    assert n >= 38
