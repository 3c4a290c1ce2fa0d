"""Build the CUDA extension IN-TREE for sm_90a (H100).  nvcc cross-compiles
without a GPU.  Produces rawspeed_b200/librawspeed_b200.so (the C-ABI library
declared in include/rawspeed_b200.h) and rawspeed_b200/librawspeed_b200_host.so
(the C++ host mirror of the reference's decompressor classes)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "librawspeed_b200.so")
HOST_LIB = os.path.join(HERE, "librawspeed_b200_host.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3",
    "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-fopenmp", "-shared",
]


def _nvcc():
    n = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(n):
        raise RuntimeError("nvcc not found: the CUDA extension cannot be built "
                           "(there is no CPU fallback)")
    return n


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _sources(sub, exts):
    d = os.path.join(HERE, "csrc", sub) if sub else os.path.join(HERE, "csrc")
    out = []
    if os.path.isdir(d):
        for f in sorted(os.listdir(d)):
            if f.endswith(exts):
                out.append(os.path.join(d, f))
    return out


def build(force=False, verbose=False):
    hdr = os.path.join(ROOT, "include", "rawspeed_b200.h")
    dev_src = _sources("", (".cu", ".cuh", ".h")) + [hdr]
    if force or _newer(LIB, dev_src):
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + [
            "-o", LIB, os.path.join(HERE, "csrc", "rsb200.cu"), "-ldl", "-lgomp"]
        subprocess.check_call(cmd, cwd=ROOT)
    host_src = _sources("host", (".cpp", ".h"))
    if host_src and (force or _newer(HOST_LIB, host_src + [hdr, LIB])):
        cpps = [s for s in host_src if s.endswith(".cpp")]
        cmd = ["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall",
               "-I", os.path.join(ROOT, "include"), "-o", HOST_LIB] + cpps + [
                   "-L", HERE, "-l:librawspeed_b200.so", "-Wl,-rpath,$ORIGIN"]
        subprocess.check_call(cmd, cwd=ROOT)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB)
