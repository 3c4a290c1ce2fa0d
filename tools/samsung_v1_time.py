"""Time Samsung V1 decoding (rsb200_samsung1_plan_create) on batches of frames at the constructor's
limit (5664x3714) and at a mid size (3008x2000): natural content, flat (every difference 0 but the
first two of row 0), a clipped band (rows of 4095 over far more than a range's halo) and long codes
(differences of 12 and 13 bits).  CUDA events around plan.run after warm-up; prints MPix/s per batch
and the number of frames the exact single-CTA decoder redid, with the GPU name, power limit and SM
clock read in the same run (the card's maximum, and the clock right after each timed loop), and with --profile a per-kernel breakdown (torch.profiler, CUDA
activities) of one batch per content.  With --ref-lib (a build of the reference's
SamsungV1Decompressor by tools/samsung1_ref_golden.py), also the reference's single-thread rate.

    python tools/samsung_v1_time.py [--frames-full 4] [--frames-mid 8] [--iters 10] [--profile]
                                    [--ref-lib PATH]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import samsung1_oracle as S  # noqa: E402

CONTENTS = ("natural", "flat", "clipped", "longcode")


def gpu_info(fields="name,power.limit,clocks.max.sm"):
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=" + fields,
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def ref_rate(path, data, w, h, reps):
    """Single-thread MPix/s of the reference's own SamsungV1Decompressor (constructor + decompress)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import samsung1_ref_golden as G
    L = G.load(path)
    best = None
    for _ in range(reps):
        t0 = time.perf_counter()
        mid, _ = G.ref_call(L, data, w, h)
        dt = time.perf_counter() - t0
        assert mid == S.OK
        best = dt if best is None else min(best, dt)
    return w * h / best / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames-full", type=int, default=4)
    ap.add_argument("--frames-mid", type=int, default=8)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--ref-lib", default=None)
    ap.add_argument("--no-gpu", action="store_true", help="only the reference's rate")
    a = ap.parse_args()
    out = {}
    sizes = [((5664, 3714), a.frames_full), ((3008, 2000), a.frames_mid)]
    values = {(n, wh): S.CONTENT[n](*wh, seed=1) for wh, _ in sizes for n in CONTENTS}
    frames = {k: S.make_stream(v) for k, v in values.items()}
    if a.ref_lib:
        out["reference_single_thread_mpix_s"] = {
            "%s_%dx%d" % (n, wh[0], wh[1]): round(ref_rate(a.ref_lib, frames[(n, wh)], *wh, 3), 1)
            for (n, wh) in frames}
    if a.no_gpu:
        print(json.dumps(out))
        return
    import torch
    import rawspeed_b200 as rs
    out["gpu"] = gpu_info()
    ctx = rs.Context(0)
    for (w, h), nf in sizes:
        for name in CONTENTS:
            data = frames[(name, (w, h))]
            blob, jobs = bytearray(), []
            pitch = S.pitch_elems(w) * 2
            for k in range(nf):
                blob += bytes((-len(blob)) % 16)
                j = rs.SamsungV1Job()
                j.in_offset, j.in_size, j.bits, j.width, j.height = len(blob), len(data), 12, w, h
                j.out_offset, j.out_pitch = k * pitch * h, pitch
                blob += data
                jobs.append(j)
            plan = rs.samsung1_plan(ctx, jobs)
            d_in = torch.from_numpy(np.frombuffer(bytes(blob) + bytes(64), np.uint8).copy()).cuda()
            d_out = torch.zeros(nf * pitch * h // 2 + 64, dtype=torch.int16, device="cuda")
            for _ in range(a.warmup):
                plan.run((d_in.data_ptr(), len(blob)), d_out)
            torch.cuda.synchronize()
            assert all(r == (0, 0) for r in plan.results())
            f = ctx._lib.rsb200_debug_range_redo
            f.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_int]
            redo = (C.c_uint32 * nf)()
            ctx.check(f(plan.h, redo, nf))
            got = d_out[:nf * pitch * h // 2].cpu().numpy().view(np.uint16).reshape(nf, h, pitch // 2)
            assert all(np.array_equal(got[k, :, :w], values[(name, (w, h))]) for k in range(nf)), \
                "output differs from the frame encoded"
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            times = []
            for _ in range(a.iters):
                e0.record()
                plan.run((d_in.data_ptr(), len(blob)), d_out)
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            sm_clock = gpu_info("clocks.sm")   # right after the timed loop
            med = float(np.median(times))
            rec = {"frames": nf, "sm_clock_after": sm_clock, "ms_median": round(med, 3), "ms_min": round(min(times), 3),
                   "mpix_s": round(nf * w * h / med / 1e3, 1), "redone": int(sum(redo)),
                   "mb_per_frame": round(len(data) / 1e6, 2)}
            if a.profile:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    plan.run((d_in.data_ptr(), len(blob)), d_out)
                    torch.cuda.synchronize()
                per = {}
                for ev in prof.key_averages():
                    if "_kernel" in ev.key and ("s1_" in ev.key or "k2_" in ev.key):
                        k = ev.key.split("(")[0].split("::")[-1]
                        per[k] = round(getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0)) / 1e3, 3)
                rec["kernel_ms"] = per
            out["%s_%dx%d" % (name, w, h)] = rec
            del plan, d_in, d_out
    print(json.dumps(out))


if __name__ == "__main__":
    main()
