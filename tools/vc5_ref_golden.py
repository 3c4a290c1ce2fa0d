"""Record the reference's VC-5 codebook and the outcomes of its own VC5Decompressor on the VC-5 test
cases:

    tests/golden/vc5_codebook.json  the entries of src/external/gopro/vc5/table17.inc, as data
    tests/golden/vc5_ref.json       per case, a digest of the message and of the whole padded image

so that tests/test_oracle_vc5.py pins the CPU restatement (tests/emu/vc5_oracle.c) against the
reference wherever it runs.

    python tools/vc5_ref_golden.py REF_SOURCE_TREE [BUILD_DIR] [--order]

REF_SOURCE_TREE is a rawspeed checkout; the decompressor and the units it links against are compiled
from it as they are, with oracle/ref_build/rawspeedconfig.h, into BUILD_DIR (a temporary directory by
default) together with tools/vc5_ref_driver.cpp.  --order prints the order in which the reference
(one worker) meets failing high-pass bands, found by failing them two at a time."""
import concurrent.futures as cf
import ctypes as C
import functools
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

UNITS = ["decompressors/VC5Decompressor", "common/RawImage", "common/RawImageDataU16",
         "common/RawImageDataFloat", "common/Common", "common/ErrorLog", "common/RawspeedException",
         "common/TableLookUp", "common/CpuFeatures", "io/IOException", "decoders/RawDecoderException",
         "metadata/ColorFilterArray", "parsers/TiffParserException", "parsers/RawParserException"]


def build(ref, out):
    """Compile the reference's VC5Decompressor and the driver into out/libvc5ref.so."""
    src = os.path.join(ref, "src", "librawspeed")
    flags = ["g++", "-std=c++20", "-O2", "-fopenmp", "-DNDEBUG", "-fPIC",
             "-I" + os.path.join(ROOT, "oracle", "ref_build"), "-I" + src,
             "-I" + os.path.join(ref, "src", "external")]
    jobs = [(os.path.join(src, u + ".cpp"), os.path.join(out, u.replace("/", "_") + ".o")) for u in UNITS]
    jobs.append((os.path.join(ROOT, "tools", "vc5_ref_driver.cpp"), os.path.join(out, "driver.o")))
    with cf.ThreadPoolExecutor(8) as ex:
        list(ex.map(lambda j: subprocess.check_call(flags + ["-c", j[0], "-o", j[1]]), jobs))
    lib = os.path.join(out, "libvc5ref.so")
    subprocess.check_call(["g++", "-shared", "-fopenmp", "-Wl,--no-undefined", "-o", lib] + [j[1] for j in jobs])
    return lib


def load(path):
    L = C.CDLL(path)
    L.ref_vc5.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                          C.c_char_p, C.c_int]
    return L


def codebook_entries(ref):
    """[[size, bits, count, value]] of table17.inc, in its order."""
    with open(os.path.join(ref, "src", "external", "gopro", "vc5", "table17.inc")) as f:
        text = f.read()
    pat = r"\{\s*([0-9]+)\s*,\s*(0x[0-9a-fA-F]+|[0-9]+)\s*,\s*([0-9]+)\s*,\s*([0-9]+)\s*\}"
    return [[int(a), int(b, 0), int(c), int(d)] for a, b, c, d in re.findall(pat, text)]


def ref_call(L, data, w, h, white, cfa):
    """-> (message without its "function, line" prefixes, image after the call) of the reference."""
    import vc5_oracle as V
    img = np.full((max(h, 1), V.pitch_elems(max(w, 1))), V.FILL_DEFAULT, np.uint16)
    msg = C.create_string_buffer(1024)
    rc = L.ref_vc5(bytes(data), len(data), w, h, white, cfa, img.ctypes.data, img.shape[1] * 2, msg, 1024)
    assert rc in (0, 1, 2), rc
    return ("" if rc == 0 else V.strip_prefixes(msg.value.decode())), img, rc


def band_order(L):
    """The order in which the reference meets the 36 high-pass bands: band a comes before band b iff,
    with a failing one way and b another, the message is a's."""
    import vc5_oracle as V
    w = h = 64
    content = V.flat(w, h)
    good = V.encode(w, h, content)

    def fail_two(a, b):
        dims = V.band_dims(w, h)
        payloads, params = [], []
        for ch in range(4):
            pl, pa = [], []
            for s in range(10):
                bw, bh = dims[V.level_of(s)]
                if s == 0:
                    pl.append(V.lowpass_bytes(content[ch][s], 16))
                    pa.append(16)
                    continue
                if (ch, s) == a:
                    pl.append(b"")  # "Bit stream size is smaller than MaxProcessBytes"
                elif (ch, s) == b:
                    pl.append(V.pack([[V.entry(0, 1), 0]]))  # "Got EndOfBand marker while looking ..."
                else:
                    pl.append(V.pack(V.band_symbols(content[ch][s], 1)))
                pa.append(1)
            payloads.append(pl)
            params.append(pa)
        msg = ref_call(L, V.datablock(w, h, payloads, params), w, h, 4095, 0)[0]
        return -1 if "MaxProcessBytes" in msg else 1

    assert ref_call(L, good, w, h, 4095, 0)[0] == ""
    bands = [(ch, s) for ch in range(4) for s in range(1, 10)]
    order = sorted(bands, key=functools.cmp_to_key(fail_two))
    for i in range(len(order)):  # a total order: every pair agrees
        for j in range(i + 1, len(order)):
            assert fail_two(order[i], order[j]) == -1 and fail_two(order[j], order[i]) == 1, (order[i], order[j])
    return order


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    ref = args[0]
    out = args[1] if len(args) > 1 else tempfile.mkdtemp()
    cpath = os.path.join(ROOT, "tests", "golden", "vc5_codebook.json")
    with open(cpath, "w") as f:
        json.dump({"source": "src/external/gopro/vc5/table17.inc of the reference tree",
                   "fields": ["size", "bits", "count", "value"], "entries": codebook_entries(ref)}, f)
        f.write("\n")
    L = load(build(ref, out))
    if "--order" in sys.argv:
        print(",\n".join("{%d, %d}" % b for b in band_order(L)))
        return
    import test_oracle_vc5 as T
    rec = {}
    for name, case in T.golden_cases():
        msg, img, _ = ref_call(L, *case)
        rec[name] = T.digest(msg, img)
    path = os.path.join(ROOT, "tests", "golden", "vc5_ref.json")
    with open(path, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print("%d cases -> %s" % (len(rec), path))


if __name__ == "__main__":
    main()
