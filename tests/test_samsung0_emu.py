"""K13 (rawspeed_b200/csrc/samsung0.cuh: Samsung V0 walk, differences, node pointer jumping, column
scans, store) without a GPU: the kernel bodies compiled by g++ against tests/emu/cuda_emu.h and run in
the plan's order, compared with the restatement of SamsungV0Decompressor (tests/emu/samsung0_oracle.c,
pinned against the reference in tests/test_oracle_samsung0.py) -- the whole padded output buffer,
status and the failing row and block.  Parity of the real kernels is tests/test_gpu_samsung0.py's job."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import compile_shared

import samsung0_oracle as S
import test_oracle_samsung0 as T

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "samsung0_emu.cpp")
OUT = os.path.join(HERE, "emu", "_build", "libsamsung0_emu.so")
DEPS = [SRC, os.path.join(HERE, "emu", "cuda_emu.h"),
        os.path.join(HERE, "..", "rawspeed_b200", "csrc", "samsung0.cuh"),
        os.path.join(HERE, "..", "rawspeed_b200", "csrc", "phaseone.cuh")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in DEPS):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            compile_shared(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas",
                            "-Wno-unused-function", "-fPIC", "-shared", "-o", OUT, SRC])
        L = C.CDLL(OUT)
        P = C.c_void_p
        L.s0_emu_run.argtypes = [P, C.c_uint64, C.c_int, P, P, P, P, P, P, P, P, P, C.c_int]
        _lib = L
    return _lib


def strips_of(bso, bsr, h):
    """The rows computeStripes() cuts (valid offset tables only)."""
    offs = list(np.frombuffer(bso[:4 * h], "<u4").astype(np.int64)) + [len(bsr)]
    return [(int(offs[r]), int(offs[r + 1] - offs[r])) for r in range(h)]


FIBERS, FIBERS_REVERSE, PLAIN = 0, 1, 2


def run_emu(frames, mode=FIBERS):
    """frames: list of (bsr, strips, w, h); each job's output is its own padded image, back to back.
    mode: threads as fibers in forward or reverse order, or thread after thread (PLAIN).
    -> (list of images, list of (status, consumed))."""
    blob = b""
    ws, hs, oo, op, first, so, ss = [], [], [], [], [], [], []
    out_off = 0
    for bsr, strips, w, h in frames:
        base = len(blob)
        blob += bsr + bytes((-len(bsr)) % 16 + 3)   # (next frame at another in_offset & 15)
        first.append(len(so))
        for o, n in strips:
            so.append(base + o)
            ss.append(n)
        ws.append(w)
        hs.append(h)
        oo.append(out_off)
        op.append(S.pitch_elems(w) * 2)
        out_off += S.pitch_elems(w) * 2 * h
    out = np.full(out_off // 2, S.FILL_DEFAULT, np.uint16)
    res = np.zeros(2 * len(frames), np.uint32)
    a = lambda v, t: np.ascontiguousarray(v, t)  # noqa: E731
    arrs = [a(ws, np.uint32), a(hs, np.uint32), a(oo, np.uint64), a(op, np.uint32), a(first, np.uint32),
            a(so, np.uint64), a(ss, np.uint32)]
    inb = np.frombuffer(blob + bytes(1), np.uint8)
    lib().s0_emu_run(inb.ctypes.data, len(blob), len(frames), *[x.ctypes.data for x in arrs],
                     out.ctypes.data, res.ctypes.data, mode)
    imgs = []
    for i, (_, _, w, h) in enumerate(frames):
        p = S.pitch_elems(w)
        imgs.append(out[oo[i] // 2: oo[i] // 2 + p * h].reshape(h, p))
    return imgs, [(int(res[2 * i]), int(res[2 * i + 1])) for i in range(len(frames))]


CODE = {S.LEN_NEG: 1, S.LEN_BIG: 2, S.UP_FIRST: 3, S.UP_LAST: 4, S.OVERREAD: 5, S.SHORT: 6}


def expect(rc, where):
    if rc == S.OK:
        return (0, 0)
    return (1 if rc in S.RDE_MSGS else 2, CODE[rc] << 24 | where)


def check(cases, mode=FIBERS):
    frames, want = [], []
    for bso, bsr, w, h in cases:
        img, rc, where = S.decompress(bso, bsr, w, h)
        assert rc not in S.CTOR_MSGS
        frames.append((bsr, strips_of(bso, bsr, h), w, h))
        want.append((img, expect(rc, where)))
    imgs, res = run_emu(frames, mode)
    for i, ((img, r), got, gr) in enumerate(zip(want, imgs, res)):
        assert gr == r, (i, gr, r)
        if not np.array_equal(got, img):
            bad = np.argwhere(got != img)[0]
            raise AssertionError("job %d: first difference at row %d col %d: %d != %d" %
                                 (i, bad[0], bad[1], got[tuple(bad)], img[tuple(bad)]))


def golden_decodable():
    return [(n, c) for n, c in T.golden_cases()
            if S.decompress(*c)[1] not in S.CTOR_MSGS]


@pytest.mark.parametrize("chunk", range(6))
def test_golden_cases(chunk):
    """Every decodable case pinned against the reference, several frames per run."""
    cases = [c for i, (_, c) in enumerate(golden_decodable()) if i % 6 == chunk]
    for i in range(0, len(cases), 8):
        check(cases[i:i + 8], mode=FIBERS_REVERSE if chunk & 1 else FIBERS)


@pytest.mark.parametrize("mode", sorted(S.DIRS))
def test_modes_mid_size(mode):
    w, h = 300, 70
    v = S.natural_values(w, h, seed=len(mode))
    bso, bsr, _ = S.make_frame(v, S.DIRS[mode](w, h))
    check([(bso, bsr, w, h)])


@pytest.mark.parametrize("seed", range(3))
def test_random_payloads(seed):
    """Random directions and bytes behind valid headers: lengths and values of every kind."""
    rng = np.random.default_rng(seed)
    cases = []
    for _ in range(4):
        w, h = int(rng.integers(16, 300)), int(rng.integers(1, 70))
        cases.append(T.length_walk(w, h, int(rng.integers(1 << 30))) + (w, h))
        d, op, setlen, adj = T.script(w, h, int(rng.integers(1 << 30)))
        rows = S.write_rows(d, op, setlen, adj)
        r = int(rng.integers(0, h))
        rows[r] = rng.integers(0, 256, len(rows[r]), dtype=np.uint8).tobytes()
        cases.append(S.pack(rows) + (w, h))
    check(cases)


@pytest.mark.parametrize("mode", ["staircase", "up"])
def test_full_size(mode):
    """5546 x 3714, the constructor's limit: the staircase has the deepest node chains (h + nb)."""
    w, h = 5546, 3714
    v = S.natural_values(w, h, seed=9)
    bso, bsr, _ = S.make_frame(v, S.DIRS[mode](w, h))
    check([(bso, bsr, w, h)], mode=PLAIN)


def test_plain_equals_fibers_on_errors():
    """The thread-after-thread order on the error cases too (the masks of the store's second half)."""
    cases = [c for n, c in golden_decodable() if n.startswith(("viol", "cut_r3"))]
    for i in range(0, len(cases), 16):
        check(cases[i:i + 16], mode=PLAIN)
