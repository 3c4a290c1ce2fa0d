"""VC-5 kernels (rawspeed_b200/csrc/vc5.cuh) without a GPU: the kernel bodies compiled by g++ against
tests/emu/cuda_emu.h and run in the plan's order and layout, threads in forward and reverse order,
against the CPU restatement (tests/emu/vc5_oracle.c, pinned against the reference): every golden case
the tag walk accepts, mixed batches, segment entries that fall at every bit offset of a 26-bit code
and of its sign bit, bands shorter than a segment, and streams whose candidate walks synchronise late."""
import ctypes as C
import os

import numpy as np
import pytest

import rawspeed_b200 as rs
import test_oracle_vc5 as T
import vc5_oracle as V
from helpers import compile_shared

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "emu", "vc5_emu.cpp")
DEPS = [SRC, os.path.join(HERE, "emu", "cuda_emu.h"), os.path.join(ROOT, "rawspeed_b200", "csrc", "vc5.cuh"),
        os.path.join(ROOT, "include", "rawspeed_b200.h")]
OUT = os.path.join(HERE, "emu", "_build", "libvc5_emu.so")
SEG, CAND = 1024, 27
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(OUT) or max(os.path.getmtime(d) for d in DEPS) > os.path.getmtime(OUT):
            os.makedirs(os.path.dirname(OUT), exist_ok=True)
            compile_shared(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-fPIC", "-shared",
                            "-o", OUT, SRC])
        L = C.CDLL(OUT)
        P = C.c_void_p
        L.vc5_emu_run.argtypes = [C.c_char_p, C.c_uint64, P, C.c_int, P, C.c_int, P, C.c_int, P, P, C.c_int, P,
                                  C.c_uint64, P]
        _lib = L
    return _lib


def emu_run(frames, reverse=False, skew=0, pitch_extra=0):
    """-> ([image], [(status, consumed)], scanned maps (nsegs, 27, 2), counts) of the replay."""
    blob, jobs, bands, outs, total = V.plan_inputs(frames, skew, pitch_extra)
    cb = [rs.Vc5Code(*(int(x) for x in e)) for e in V.codebook()]
    ca = (rs.Vc5Code * len(cb))(*cb)
    ja = (rs.Vc5Job * len(jobs))(*jobs)
    ba = (rs.Vc5Band * len(bands))(*bands)
    out = np.full(total, V.FILL_DEFAULT, np.uint16)
    res = np.zeros(2 * len(jobs), np.uint32)
    cap = 8 * len(blob) * CAND // SEG + 64 * CAND * len(bands)
    maps = np.zeros(2 * cap, np.uint32)
    counts = np.zeros(2, np.uint32)
    rc = lib().vc5_emu_run(blob, len(blob), C.cast(ca, C.c_void_p), len(cb), C.cast(ja, C.c_void_p), len(jobs),
                           C.cast(ba, C.c_void_p), len(bands), out.ctypes.data, res.ctypes.data, int(reverse),
                           maps.ctypes.data, cap, counts.ctypes.data)
    assert rc == -1, rc
    imgs, seen = [], np.zeros(total, bool)
    for o, h, pitch in outs:
        imgs.append(out[o:o + h * pitch].reshape(h, pitch))
        seen[o:o + h * pitch] = True
    assert np.all(out[~seen] == V.FILL_DEFAULT), "a store outside the jobs' images"
    n = int(counts[0])
    return imgs, [tuple(int(x) for x in res[2 * i:2 * i + 2]) for i in range(len(jobs))], \
        maps[:2 * n * CAND].reshape(n, CAND, 2), counts


def check(frames, **kw):
    imgs, res, _, _ = emu_run(frames, **kw)
    for k, ((want, wres), img, got) in enumerate(zip(V.expected(frames, pitch_extra=kw.get("pitch_extra", 0)),
                                                     imgs, res)):
        assert got == wres, (k, got, wres)
        assert np.array_equal(img, want), k


def accepted():
    return [(n, c) for n, c in T.golden_cases() if V.parse(*c)[0] == V.OK]


@pytest.mark.parametrize("reverse", [False, True])
def test_golden_cases_one_by_one(reverse):
    for name, case in accepted():
        check([case], reverse=reverse)


def test_golden_cases_one_plan():
    """All accepted cases in one plan: mixed dims, outcomes, phases and depths; odd skews and pitches."""
    frames = [c for n, c in accepted() if not n.startswith("bits_")]
    check(frames, skew=3, pitch_extra=2)


def one_band_frame(w, h, syms, ch=1, sb=8):
    """A natural datablock whose band (ch, sb) is the symbol list `syms`."""
    content = V.natural(w, h, seed=1)
    payloads, params = T.parts(w, h, content)
    payloads[ch][sb] = V.pack(syms)
    return (V.datablock(w, h, payloads, params, T.PS2), w, h, 4095, V.RGGB)


def true_maps(syms, nseg):
    """(exit offset into segment k + 1, coefficients in front of it) of every segment k of a band whose
    stream is the symbol list `syms`, zero-filled behind it (one-bit zero symbols of count 1); the count
    saturates at the first count-0 symbol, as the walks record it."""
    cb = V.codebook()
    starts, counts, p, n = [], [], 0, 0
    for e, _ in syms:
        starts.append(p)
        counts.append(n)
        size, _, count, value = (int(x) for x in cb[e])
        p += size + (value != 0)
        n = n + count if count and n != 0xFFFFFFFF else 0xFFFFFFFF
    while p <= nseg * SEG + 27:
        starts.append(p)
        counts.append(n)
        p += 1
        n = n + 1 if n != 0xFFFFFFFF else n
    out, j = [], 0
    for k in range(nseg):
        end = (k + 1) * SEG
        while starts[j] < end:
            j += 1
        out.append((starts[j] - end, counts[j]))
    return out


def band_maps(frame, maps, ch, sb):
    """The scanned maps' entry 0 of every segment of band (ch, sb) of a one-frame plan."""
    _, table = V.band_table(*frame)
    first = 0
    for b, (_, size, _) in enumerate(table):
        nseg = (8 * size + 65 + SEG - 1) // SEG if b % 10 and size >= 4 else 0
        if b == ch * 10 + sb:
            return [tuple(int(x) for x in maps[first + k][0]) for k in range(nseg)]
        first += nseg


def long_symbol_band(w, h, entry, shift, sign=lambda i: i & 1):
    """Symbols of a level-1 band: `shift` one-bit zero symbols, then `entry` (count 1) back to back to
    the band's end, then the end marker."""
    bw, bh = V.band_dims(w, h)[1]
    syms = [[V.entry(1, 0), 0]] * shift
    while len(syms) < bw * bh:
        syms.append([entry, sign(len(syms))])
    return syms + [[V.entry(0, 1), 0]]


def test_segment_entries_at_every_offset():
    """The longest symbols back to back: a 26-bit code with its sign bit (27 bits, the most a symbol
    can take) and a 26-bit code without one, behind 0..27 leading one-bit symbols.  1024 = 37 * 27 + 25
    and gcd(25, 27) = 1, so a band's segment boundaries fall at every bit offset 0..26 of a 27-bit
    symbol, sign bit included: every candidate entry 0..26 is the true entry of some segment, and the
    scanned maps equal the true symbol boundaries and counts."""
    w, h = 200, 136
    cb = V.codebook()
    long27 = int(np.nonzero((cb[:, 0] == 26) & (cb[:, 2] == 1) & (cb[:, 3] != 0))[0][0])
    long26 = int(np.nonzero((cb[:, 0] == 25) & (cb[:, 2] == 1))[0][0])  # 25 bits + sign
    seen = set()
    frames = []
    for entry in (long27, long26):
        for shift in (0, 1, 13, 26, 27):
            syms = long_symbol_band(w, h, entry, shift)
            fr = one_band_frame(w, h, syms)
            frames.append(fr)
            _, res, maps, _ = emu_run([fr])
            got = band_maps(fr, maps, 1, 8)
            assert got == true_maps(syms, len(got)), (entry, shift)
            seen |= {x for x, _ in got[:-1]}
    assert seen == set(range(27))
    check(frames)


def test_short_bands_and_late_synchronisation():
    """Bands shorter than a segment (the smallest legal image), and walks that synchronise late: a
    band of 27-bit symbols with alternating signs, where the 27 candidate walks of a segment run in
    step through many symbols before they meet; the scanned maps against the true boundaries."""
    check([(V.encode(34, 34, V.natural(34, 34, seed=2), prescale=T.PS2), 34, 34, 4095, V.RGGB),
           (V.encode(120, 90, V.noise(120, 90, seed=4), prescale=T.PS2), 120, 90, 4095, V.GBRG)])
    w, h = 160, 120
    cb = V.codebook()
    long27 = [int(i) for i in np.nonzero((cb[:, 0] == 26) & (cb[:, 2] == 1) & (cb[:, 3] != 0))[0]]
    for entry in long27:
        syms = long_symbol_band(w, h, entry, 3, sign=lambda i: (i // 3) & 1)
        fr = one_band_frame(w, h, syms, ch=2, sb=7)
        _, res, maps, counts = emu_run([fr])
        got = band_maps(fr, maps, 2, 7)
        assert len(got) > 30 and counts[1] >= 5
        assert got == true_maps(syms, len(got))
        check([fr])
