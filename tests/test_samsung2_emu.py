"""Samsung V2 kernels (rawspeed_b200/csrc/samsung2.cuh) without a GPU: the kernel bodies compiled by g++
against tests/emu/cuda_emu.h and run in the plan's order and layout, with every CTA's threads as fibers
in forward and in reverse order, compared with the restatement of SamsungV2Decompressor
(tests/emu/samsung2_oracle.c, pinned against the reference in tests/test_oracle_samsung2.py): the whole
output buffer with sentinels around every frame, status and `consumed`.  The scratch tables are
checked directly: every candidate and pair-step entry is a failure or a candidate within 0..ncand, the
row classes' entries on the true chain lead from each row start to the next, and the resolved row
starts are the restatement's.  Parity of the real kernels is tests/test_gpu_samsung2.py's job."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import compile_shared

import samsung2_oracle as S
import test_oracle_samsung2 as T

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "samsung2_emu.cpp")
OUT = os.path.join(HERE, "emu", "_build", "libsamsung2_emu.so")
DEPS = [SRC, os.path.join(HERE, "emu", "cuda_emu.h"),
        os.path.join(HERE, "..", "rawspeed_b200", "csrc", "samsung2.cuh"),
        os.path.join(HERE, "..", "rawspeed_b200", "csrc", "phaseone.cuh")]
FILL = S.FILL_DEFAULT
GAP = 32  # sentinel pixels before every frame and behind the last
FAIL = 1 << 31
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
        L.s2_emu_run.argtypes = [P, C.c_uint64, C.c_int, P, P, P, P, P, P, P, P, P, C.c_int,
                                 P, C.c_uint64, P, C.c_uint64, P, C.c_uint64, P, P]
        L.s2_emu_run.restype = C.c_uint64
        _lib = L
    return _lib


def run_emu(frames, reverse, skew=0):
    """frames: [(data, w, h, bits)] -> (images, results, tables), asserting the sentinels and that no
    load left the input."""
    n = len(frames)
    blob, ioff = bytearray(), []
    for data, w, h, bits in frames:
        blob += bytes((-len(blob)) % 16 + skew)
        ioff.append(len(blob))
        blob += data
    isz = np.array([len(f[0]) for f in frames], np.uint32)
    bits = np.array([f[3] for f in frames], np.uint32)
    w = np.array([f[1] for f in frames], np.uint32)
    h = np.array([f[2] for f in frames], np.uint32)
    oo, op, layout, pos = [], [], [], 0
    for data, fw, fh, _ in frames:
        pitch = S.pitch_elems(fw)
        pos += GAP
        oo.append(2 * pos)
        op.append(2 * pitch)
        layout.append((pos, fh, pitch))
        pos += fh * pitch
    pos += GAP
    out = np.full(pos, FILL, np.uint16)
    res = np.zeros(2 * n, np.uint32)
    fail = np.zeros(2 * n, np.uint32)
    counts = np.zeros(3, np.uint64)
    ntab = sum(3 * (((len(f[0]) - 16) // 16 + 2)) + 1 for f in frames)
    njump = sum((len(f[0]) - 16) // 16 + 2 for f in frames)
    tab = np.zeros(ntab, np.uint32)
    jump = np.zeros(njump, np.uint32)
    rows = np.zeros(int(h.sum()), np.uint32)
    ioff = np.array(ioff, np.uint64)
    oo, op = np.array(oo, np.uint64), np.array(op, np.uint32)
    b = bytes(blob)
    outside = lib().s2_emu_run(b, len(b), n, ioff.ctypes.data, isz.ctypes.data, bits.ctypes.data, w.ctypes.data,
                               h.ctypes.data, oo.ctypes.data, op.ctypes.data, out.ctypes.data, res.ctypes.data,
                               int(reverse), tab.ctypes.data, ntab, jump.ctypes.data, njump, rows.ctypes.data,
                               rows.size, fail.ctypes.data, counts.ctypes.data)
    assert outside == 0, "loads outside the input"
    assert list(counts) == [ntab, njump, rows.size]
    imgs, seen = [], np.zeros(pos, bool)
    for p, fh, pitch in layout:
        imgs.append(out[p:p + fh * pitch].reshape(fh, pitch))
        seen[p:p + fh * pitch] = True
    assert np.all(out[~seen] == FILL), "a store outside the frames' images"
    return imgs, [(int(res[2 * i]), int(res[2 * i + 1])) for i in range(n)], (tab, jump, rows, fail)


def check_tables(frames, tables):
    """Candidate and pair-step entries bounded; on the true chain they follow the restatement."""
    tab, jump, rows, fail = tables
    t0 = j0 = r0 = 0
    for k, (data, w, h, bits) in enumerate(frames):
        ncand = (len(data) - 16) // 16 + 1
        n1 = ncand + 1
        ft = tab[t0:t0 + 3 * n1 + 1]
        fj = jump[j0:j0 + n1]
        for e in list(ft) + list(fj):
            assert (e & FAIL) or e <= ncand, (k, hex(int(e)))
        ends = np.zeros(h, np.uint32)
        _, rc, where, _ = S.decompress(data, w, h, bits, ends=ends)
        frow = (where >> 9) & 0x1FFF if rc != S.OK else h
        assert int(fail[2 * k]) == frow, k
        # the restatement's row starts: 0, then the next multiple of 16 behind each row
        starts = [0] + [(int(e) + 15) // 16 for e in ends[:frow]]
        for r in range(min(frow + 1, h)):
            assert rows[r0 + r] == starts[r], (k, r)
            cls = 3 if r == 0 else (2 if r == 1 else r & 1)
            e = int(ft[cls * n1 + starts[r]] if cls < 3 else ft[3 * n1])
            if r < frow:
                assert e == starts[r + 1], (k, r, hex(e))
            else:  # the failing row's entry is the failure itself (rows 0 and 1; later ones by class)
                assert e & FAIL and (e & 0x7FFFFFFF) >> 27 == rc and e & 511 == where & 511, (k, r, hex(e))
                assert (int(fail[2 * k + 1]) >> 27) & 15 == rc
        t0 += 3 * n1 + 1
        j0 += n1
        r0 += h


def check(frames, reverse, skew=0):
    imgs, res, tables = run_emu(frames, reverse, skew)
    for k, ((data, w, h, bits), img, got) in enumerate(zip(frames, imgs, res)):
        want, rc, where, _ = S.decompress(data, w, h, bits, fill=FILL)
        st = 0 if rc == S.OK else (2 if rc in S.IOE_MSGS else 1)
        assert got == (st, S.consumed(rc, where)), (k, got, rc, where)
        assert np.array_equal(img, want), k
    check_tables(frames, tables)


def decodable(cases):
    out = []
    for _, (d, w, h, bits, cpp) in cases:
        if cpp == 1 and len(d) >= 16 and S.decompress(d, w, h, bits)[1] < S.CPP and w * h <= 96 * 8:
            out.append((d, w, h, bits))
    return out


@pytest.mark.parametrize("reverse", [False, True])
def test_pinned_cases_one_plan(reverse):
    """The pinned cases that fit the replay, all in one plan (mixed outcomes)."""
    check(decodable(T.golden_cases()), reverse)


@pytest.mark.parametrize("reverse", [False, True])
def test_tall_frames_failing_past_checkpoints(reverse):
    """Frames of 200 rows (four checkpoints) failing at chosen rows, every failure kind, in one plan."""
    tall = [fr for name, fr in T.tall_cases() if name.endswith(("_66_+0", "_130_+1", "_65_next_0", "_129_next_3"))
            or name.startswith(("tall_motion", "tall_underflow"))]
    check([(d, w, h, bits) for d, w, h, bits, _ in tall], reverse, skew=5)


@pytest.mark.parametrize("reverse", [False, True])
def test_random_payloads(reverse):
    rng = np.random.default_rng(23)
    frames = []
    for k in range(24):
        w, h, bits = 16 * int(rng.integers(1, 8)), int(rng.integers(1, 12)), (12, 14)[k % 2]
        if k % 2:
            data = S.encode(S.random_values(w, h, bits, seed=k), bits, int(rng.integers(0, 8)),
                            int(rng.integers(0, 1 << bits)), int(k % 5), k)
            data = data[:len(data) - int(rng.integers(0, 40))]
        else:
            data = S.header(w, h, bits, int(rng.integers(0, 8)), int(rng.integers(0, 1 << 14))) + \
                rng.integers(0, 256, int(rng.integers(0, 40 * w)), dtype=np.uint8).tobytes()
        frames.append((data, w, h, bits))
    check(frames, reverse)


def test_multi_frame_plan_at_every_skew():
    frames = [(T.natural(w, h, (12, 14)[f % 2], f % 8, init=9, policy=f % 5, seed=f), w, h, (12, 14)[f % 2])
              for f, (w, h) in enumerate([(16, 1), (48, 70), (96, 3), (32, 131), (208, 4)])]
    for skew in (3, 14):
        check(frames, skew == 3, skew)
