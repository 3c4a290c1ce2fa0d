"""Time Samsung V2 decoding (rsb200_samsung2_plan_create) on plans of 1 and 4 frames of 6496x4336 (the
constructor's limit) and 5472x3648, at 12 and 14 bits: natural content (the writer's cheapest motion
per block), all motion 7 (left), all up (motion 3) and averaging (motions 2 / 4).  CUDA events around
plan.run after warm-up; prints MPix/s per plan with the GPU name, power limit and SM clock read in the
same run, and the split between the candidate walk, the row-start resolution (pair, doubling, coarse,
fine), the descriptor walk plus difference decode, and the reconstruction (torch.profiler, CUDA
activities, one run per plan).  With --ref-lib (a build of the reference's SamsungV2Decompressor by
tools/samsung2_ref_golden.py), also the reference's single-thread rate on the same content.

    python tools/samsung_v2_time.py [--iters 5] [--frames 1 4] [--ref-lib PATH] [--no-gpu]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import samsung2_oracle as S  # noqa: E402

CONTENTS = {"natural": 0, "left": 1, "up": 2, "average": 3}
STAGES = {"walk": ("s2_cand",), "resolve": ("s2_pair", "s2_double", "s2_coarse", "s2_fine"),
          "decode": ("s2_desc", "s2_diff"), "reconstruct": ("s2_recon",)}


def gpu_info(fields="name,power.limit,clocks.max.sm"):
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=" + fields,
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def ref_rate(path, data, w, h, bits, reps):
    """Single-thread MPix/s of the reference's own SamsungV2Decompressor (constructor + decompress)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import samsung2_ref_golden as G
    L = G.load(path)
    best = None
    for _ in range(reps):
        t0 = time.perf_counter()
        text, _ = G.ref_call(L, data, w, h, bits)
        dt = time.perf_counter() - t0
        assert text == "", text
        best = dt if best is None else min(best, dt)
    return w * h / best / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ref-lib", default=None)
    ap.add_argument("--no-gpu", action="store_true", help="only the reference's rate")
    a = ap.parse_args()
    out = {}
    cases = {}
    for (w, h) in ((6496, 4336), (5472, 3648)):
        for bits in (12, 14):
            v = S.natural_values(w, h, bits, seed=w + bits)
            for name, pol in CONTENTS.items():
                cases[(name, w, h, bits)] = (v, S.encode(v, bits, 0, 77, pol, seed=bits))
    if a.ref_lib:
        out["reference_single_thread_mpix_s"] = {
            "%s_%dx%d_%d" % k: round(ref_rate(a.ref_lib, data, k[1], k[2], k[3], 2), 1)
            for k, (_, data) in cases.items()}
    if a.no_gpu:
        print(json.dumps(out))
        return
    import torch
    from torch.profiler import ProfilerActivity, profile
    import rawspeed_b200 as rs
    out["gpu"] = gpu_info()
    ctx = rs.Context(0)
    for (name, w, h, bits), (v, data) in cases.items():
        for nf in a.frames:
            blob, jobs = bytearray(), []
            pitch = S.pitch_elems(w) * 2
            for k in range(nf):
                blob += bytes((-len(blob)) % 16)
                j = rs.SamsungV2Job()
                j.in_offset, j.in_size, j.bits, j.width, j.height = len(blob), len(data), bits, w, h
                for i in range(16):
                    j.header[i] = data[i]
                j.out_offset, j.out_pitch = k * pitch * h, pitch
                blob += data
                jobs.append(j)
            plan = rs.samsung2_plan(ctx, jobs)
            d_in = torch.from_numpy(np.frombuffer(bytes(blob) + bytes(64), np.uint8).copy()).cuda()
            d_out = torch.zeros(nf * pitch * h // 2 + 64, dtype=torch.int16, device="cuda")
            for _ in range(a.warmup):
                plan.run((d_in.data_ptr(), len(blob)), d_out)
            torch.cuda.synchronize()
            assert all(r == (0, 0) for r in plan.results())
            got = d_out[:nf * pitch * h // 2].cpu().numpy().view(np.uint16).reshape(nf, h, pitch // 2)
            assert all(np.array_equal(got[k, :, :w], v) for k in range(nf)), "output differs from the frame encoded"
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            times = []
            for _ in range(a.iters):
                e0.record()
                plan.run((d_in.data_ptr(), len(blob)), d_out)
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            sm_clock = gpu_info("clocks.sm")  # right after the timed loop
            med = float(np.median(times))
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                plan.run((d_in.data_ptr(), len(blob)), d_out)
                torch.cuda.synchronize()
            split = {s: 0.0 for s in STAGES}
            for ev in prof.key_averages():
                for s, names in STAGES.items():
                    if any(n + "_kernel" in ev.key for n in names):
                        split[s] += getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0)) / 1e3
            out["%s_%dx%d_%d_x%d" % (name, w, h, bits, nf)] = {
                "sm_clock_after": sm_clock, "ms_median": round(med, 3), "ms_min": round(min(times), 3),
                "mpix_s": round(nf * w * h / med / 1e3, 1), "mb_per_frame": round(len(data) / 1e6, 2),
                "split_ms": {s: round(t, 3) for s, t in split.items()}}
            del plan, d_in, d_out
    print(json.dumps(out))


if __name__ == "__main__":
    main()
