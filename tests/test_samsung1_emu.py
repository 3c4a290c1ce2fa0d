"""Samsung V1 reconstruction (rawspeed_b200/csrc/samsung1.cuh: column, row, scan and store kernels)
without a GPU: the kernel bodies compiled by g++ against tests/emu/cuda_emu.h and run in the plan's
order, with every CTA's threads as fibers in forward and in reverse order, compared with the
restatement of SamsungV1Decompressor (tests/emu/samsung1_oracle.c, pinned against the reference in
tests/test_oracle_samsung1.py): the whole output buffer with sentinels around every frame, status and
the reported pixel.  Their input is the difference scratch the range decoder leaves: the symbols it
parses (it reads zero bits behind the data up to 8 bytes + 10 bits) and garbage behind them.  Also
samsung1_run_phase, the flat-run alignment of the range decoder's speculative starts.  Parity of the
real kernels is tests/test_gpu_samsung1.py's job."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import compile_shared

import samsung1_oracle as S
import test_oracle_samsung1 as T

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "samsung1_emu.cpp")
OUT = os.path.join(HERE, "emu", "_build", "libsamsung1_emu.so")
DEPS = [SRC, os.path.join(HERE, "emu", "cuda_emu.h"),
        os.path.join(HERE, "..", "rawspeed_b200", "csrc", "samsung1.cuh"),
        os.path.join(HERE, "..", "rawspeed_b200", "csrc", "ljpeg_types.h")]
FILL = S.FILL_DEFAULT
GAP = 32  # sentinel pixels before every frame and behind the last
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
        L.s1_emu_run.argtypes = [C.c_int, P, P, P, P, P, C.c_uint64, P, P, P, P, C.c_int]
        L.s1_emu_run_phase.argtypes = [C.c_uint32, C.c_uint32]
        L.s1_emu_run_phase.restype = C.c_uint32
        _lib = L
    return _lib


def scratch(data, n, seed):
    """The n differences the range decoder leaves for `data`: parsed up to 8 bytes + 10 bits behind the
    data, garbage (any int16) behind that."""
    d = np.zeros(n, np.int16)
    st = np.zeros(n, np.uint64)
    S.lib().s1_parse.argtypes = [C.c_char_p, C.c_uint32, C.c_int64, C.c_void_p, C.c_void_p]
    S.lib().s1_parse(bytes(data), len(data), n, d.ctypes.data, st.ctypes.data)
    behind = st >= 8 * len(data) + 74
    d[behind] = np.random.default_rng(seed).integers(-32768, 32768, int(behind.sum())).astype(np.int16)
    return d


def run_emu(frames, reverse):
    """frames: [(data, w, h)] -> (out buffer, [(offset, h, pitch)], [(status, consumed)])."""
    n = len(frames)
    w = np.array([f[1] for f in frames], np.uint32)
    h = np.array([f[2] for f in frames], np.uint32)
    ts = np.array([S.tstar(len(f[0])) for f in frames], np.uint32)
    doff, parts, off = [], [], 0
    for k, (data, fw, fh) in enumerate(frames):
        doff.append(off)
        parts.append(scratch(data, fw * fh, k))
        off += fw * fh   # (a multiple of 64)
    diffs = np.ascontiguousarray(np.concatenate(parts).view(np.uint16))
    oo, op, layout, pos = [], [], [], 0
    for data, fw, fh in frames:
        pitch = S.pitch_elems(fw)
        pos += GAP
        oo.append(2 * pos)
        op.append(2 * pitch)
        layout.append((pos, fh, pitch))
        pos += fh * pitch
    pos += GAP
    out = np.full(pos, FILL, np.uint16)
    res = np.zeros(2 * n, np.uint32)
    doff = np.array(doff, np.uint64)
    oo = np.array(oo, np.uint64)
    op = np.array(op, np.uint32)
    lib().s1_emu_run(n, w.ctypes.data, h.ctypes.data, ts.ctypes.data, doff.ctypes.data, diffs.ctypes.data,
                     diffs.size, oo.ctypes.data, op.ctypes.data, out.ctypes.data, res.ctypes.data,
                     int(reverse))
    return out, layout, [(int(res[2 * i]), int(res[2 * i + 1])) for i in range(n)]


def check(frames, reverse):
    out, layout, res = run_emu(frames, reverse)
    seen = np.zeros(out.size, bool)
    for k, ((data, w, h), (p, fh, pitch), got) in enumerate(zip(frames, layout, res)):
        want, rc, where = S.decompress(data, w, h, fill=FILL)
        st = {S.OK: 0, S.OOB: 1, S.OVERREAD: 2, S.SHORT: 2}[rc]
        cons = (0x80000000 | where) if rc == S.OOB else (where if rc == S.OVERREAD else 0)
        assert got == (st, cons), (k, got, st, cons)
        assert np.array_equal(out[p:p + fh * pitch].reshape(fh, pitch), want), k
        seen[p:p + fh * pitch] = True
    assert np.all(out[~seen] == FILL), "a store outside the frames"
    return res


def pinned():
    return [(d, w, h) for _, (d, w, h, bit, cpp) in T.golden_cases()
            if bit == 12 and cpp == 1 and w > 0 and h > 0 and w % 32 == 0 and h % 2 == 0
            and w <= 5664 and h <= 3714]


def pinned_sample():
    """Every outcome class of the pinned cases (each fiber runs on its own stack, so not all of them):
    symbols, widths, violations, sizes, random payloads, ties, and every fourth cut."""
    out = []
    for name, (d, w, h, bit, cpp) in T.golden_cases():
        if not (bit == 12 and cpp == 1 and w > 0 and h > 0 and w % 32 == 0 and h % 2 == 0
                and w <= 5664 and h <= 3714):
            continue
        if name.startswith("cut") and int(name[-2:]) % 4:
            continue
        if name.startswith("sym_") and not name.endswith("max"):
            continue
        out.append((d, w, h))
    return out


@pytest.mark.parametrize("reverse", [False, True])
def test_pinned_cases_one_plan(reverse):
    res = check(pinned_sample(), reverse)
    assert {r[0] for r in res} == {0, 1, 2}


@pytest.mark.parametrize("reverse", [False, True])
def test_multi_frame_plan(reverse):
    """Frames of several sizes and outcomes in one plan: CTAs of the row kernels past a short frame's
    rows, frames after a failing one."""
    rng = np.random.default_rng(3)
    frames = []
    for k, (w, h) in enumerate([(64, 40), (32, 6), (96, 18), (5664, 2)]):
        data = S.make_stream(S.natural_values(w, h, seed=k))
        frames += [(data, w, h), (data[:len(data) * 2 // 3], w, h)]
    frames.append((rng.integers(0, 256, 300, dtype=np.uint8).tobytes(), 64, 20))
    res = check(frames, reverse)
    assert [r[0] for r in res[:8:2]] == [0] * 4 and [r[0] for r in res[1:8:2]] == [2] * 4


@pytest.mark.parametrize("reverse", [False, True])
def test_scan_past_1024_rows(reverse):
    """The scan kernel finds the failing row after its first step of 1024 rows; the violation there
    comes first, the cut after it."""
    w, h = 32, 1040
    d = S.diffs_of(S.natural_values(w, h, seed=9))
    d[1030, 17] += 5000
    data = S.encode(d)
    cut = S.encode(S.diffs_of(S.natural_values(w, h, seed=9)))
    cut = cut[:len(cut) - 40]
    res = check([(data + bytes(8), w, h), (cut, w, h)], reverse)
    assert res[0] == (1, 0x80000000 | (1030 << 14) | 17)
    assert res[1][0] == 2 and (res[1][1] >> 14) >= 1024


def test_tie_cases_report_the_refill():
    frames = [(d, w, h) for n, (d, w, h, bit, cpp) in T.golden_cases() if n.startswith("tie_")]
    assert frames
    for rev in (False, True):
        res = check(frames, rev)
        assert all(r[0] == 2 for r in res)


def _bits_of(words):
    return "".join(format(int(x), "032b") for x in words)


def _ref_phase(x0, x1):
    s = _bits_of([x0, x1])
    for o in range(6):
        if s[o:o + 32] == ("110100" * 7)[:32]:
            return o
    return 0


def test_run_phase_every_offset():
    run = "110100" * 30
    for q in range(6):
        s = run[q:q + 64]
        x0, x1 = int(s[:32], 2), int(s[32:], 2)
        assert lib().s1_emu_run_phase(x0, x1) == (6 - q) % 6, q


def test_run_phase_other_windows():
    rng = np.random.default_rng(1)
    cases = [(0, 0), (0xFFFFFFFF, 0xFFFFFFFF), (0xD34D34D3, 0)]
    run = "110100" * 30
    for q in range(6):   # a run that breaks inside the window
        s = list(run[q:q + 64])
        s[20] = "1" if s[20] == "0" else "0"
        s = "".join(s)
        cases.append((int(s[:32], 2), int(s[32:], 2)))
    cases += [(int(a), int(b)) for a, b in rng.integers(0, 1 << 32, (200, 2), dtype=np.uint64)]
    for x0, x1 in cases:
        assert lib().s1_emu_run_phase(x0, x1) == _ref_phase(x0, x1), (hex(x0), hex(x1))
    assert _ref_phase(0xD34D34D3, 0) == 0 and lib().s1_emu_run_phase(0x34D34D34, 0xD34D34D3) == 2
