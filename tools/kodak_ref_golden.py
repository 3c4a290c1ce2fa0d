"""Record the outcomes of the reference's own KodakDecompressor on the Kodak DCR test cases into
tests/golden/kodak_ref.json, so that tests/test_oracle_kodak.py pins the CPU restatement
(tests/emu/kodak_oracle.c) against the reference wherever it runs.

    python tools/kodak_ref_golden.py REF_SOURCE_TREE [BUILD_DIR]

REF_SOURCE_TREE is a rawspeed checkout; the decompressor and the units it links against are
compiled from it as they are, with oracle/ref_build/rawspeedconfig.h, into BUILD_DIR (a temporary
directory by default) together with tools/kodak_ref_driver.cpp."""
import concurrent.futures as cf
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

UNITS = ["decompressors/KodakDecompressor", "common/RawImage", "common/RawImageDataU16",
         "common/RawImageDataFloat", "common/Common", "common/ErrorLog", "common/RawspeedException",
         "common/TableLookUp", "common/CpuFeatures", "io/IOException", "decoders/RawDecoderException",
         "metadata/ColorFilterArray", "parsers/TiffParserException", "parsers/RawParserException"]


def build(ref, out):
    """Compile the reference's KodakDecompressor and the driver into out/libkdref.so."""
    src = os.path.join(ref, "src", "librawspeed")
    flags = ["g++", "-std=c++20", "-O2", "-fopenmp", "-DNDEBUG", "-fPIC",
             "-I" + os.path.join(ROOT, "oracle", "ref_build"), "-I" + src,
             "-I" + os.path.join(ref, "src", "external")]
    jobs = [(os.path.join(src, u + ".cpp"), os.path.join(out, u.replace("/", "_") + ".o")) for u in UNITS]
    jobs.append((os.path.join(ROOT, "tools", "kodak_ref_driver.cpp"), os.path.join(out, "driver.o")))
    with cf.ThreadPoolExecutor(8) as ex:
        list(ex.map(lambda j: subprocess.check_call(flags + ["-c", j[0], "-o", j[1]]), jobs))
    lib = os.path.join(out, "libkdref.so")
    subprocess.check_call(["g++", "-shared", "-fopenmp", "-Wl,--no-undefined", "-o", lib] + [j[1] for j in jobs])
    return lib


def load(path):
    L = C.CDLL(path)
    L.ref_kodak.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                            C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_char_p, C.c_int]
    return L


def ref_call(L, data, w, h, bps, cpp=1, curve=None, dither=False, uncorrected=True):
    """-> (message without its "function, line" prefix, image after the call) of the reference on one case."""
    import kodak_oracle as K
    img = np.full((max(h, 1), K.pitch_elems(max(w, 1))), K.FILL_DEFAULT, np.uint16)
    msg = C.create_string_buffer(512)
    cv = None if curve is None else np.ascontiguousarray(curve, np.uint16)
    rc = L.ref_kodak(bytes(data), len(data), w, h, bps, cpp, None if cv is None else cv.ctypes.data,
                     0 if cv is None else cv.size, int(dither), int(uncorrected), img.ctypes.data, img.shape[1] * 2,
                     msg, 512)
    assert rc in (0, 1, 2), rc
    text = "" if rc == 0 else K.strip_prefix(msg.value.decode())
    assert rc == 0 or (rc == 2) == (K.message_id(text) in K.IOE_MSGS), msg.value
    return text, img


def main():
    import test_oracle_kodak as T
    ref = sys.argv[1]
    out = sys.argv[2] if len(sys.argv) > 2 else tempfile.mkdtemp()
    L = load(build(ref, out))
    rec = {}
    for name, case in T.golden_cases():
        rec[name] = T.digest(*ref_call(L, *case))
    path = os.path.join(ROOT, "tests", "golden", "kodak_ref.json")
    with open(path, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print("%d cases -> %s" % (len(rec), path))


if __name__ == "__main__":
    main()
