"""Time Kodak DCR decoding (rsb200_kodak_plan_create) on plans of 1 and 4 frames of 4500x3000 at 12
bits (the real sensor size) with natural content, flat content (every difference 0 bits) and noisy
content (long differences, about 30 MB per frame).  CUDA events around plan.run after warm-up; prints
MPix/s per plan with the GPU name, power limit and SM clock read in the same run, and the split
between the nibble-sum prefix (tile sums, scan, prefix), the candidate walk, the row-start resolution
(doubling, coarse, fine) and the decode (check, store), from torch.profiler with CUDA activities, one
run per plan.

    python tools/kodak_time.py [--iters 10] [--frames 1 4]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import kodak_oracle as K  # noqa: E402

STAGES = {"prefix": ("kd_tsum", "kd_tscan", "kd_prefix"), "candidates": ("kd_cand",),
          "resolve": ("kd_double", "kd_coarse", "kd_fine"), "decode": ("kd_check", "kd_store")}


def gpu_info(fields="name,power.limit,clocks.max.sm"):
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=" + fields,
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def contents(w, h, bps):
    rng = np.random.default_rng(5)
    top = (1 << bps) - 1
    return {"natural": K.natural(w, h, bps, seed=1),
            "flat": np.full((h, w), top // 2, np.int64),
            "noisy": rng.integers(0, top + 1, size=(h, w))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import rawspeed_b200 as rs
    out = {"gpu": gpu_info()}
    ctx = rs.Context(0)
    w, h, bps = 4500, 3000, 12
    for name, v in contents(w, h, bps).items():
        data = K.encode(v)
        for nf in a.frames:
            blob, jobs = bytearray(), []
            pitch = K.pitch_elems(w) * 2
            for k in range(nf):
                blob += bytes((-len(blob)) % 16)
                j = rs.KodakJob()
                j.in_offset, j.in_size, j.width, j.height, j.bps, j.table = len(blob), len(data), w, h, bps, -1
                j.out_offset, j.out_pitch = k * pitch * h, pitch
                blob += data
                jobs.append(j)
            plan = rs.kodak_plan(ctx, jobs)
            d_in = torch.from_numpy(np.frombuffer(bytes(blob), np.uint8).copy()).cuda()
            d_out = torch.zeros(nf * pitch * h // 2, dtype=torch.int16, device="cuda")
            for _ in range(a.warmup):
                plan.run((d_in.data_ptr(), len(blob)), d_out)
            torch.cuda.synchronize()
            assert all(r == (0, 0) for r in plan.results())
            got = d_out.cpu().numpy().view(np.uint16).reshape(nf, h, pitch // 2)
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
            out["%s_%dx%d_%d_x%d" % (name, w, h, bps, nf)] = {
                "sm_clock_after": sm_clock, "ms_median": round(med, 3), "ms_min": round(min(times), 3),
                "mpix_s": round(nf * w * h / med / 1e3, 1), "mb_per_frame": round(len(data) / 1e6, 2),
                "split_ms": {s: round(t, 3) for s, t in split.items()}}
            plan.close()
            del d_in, d_out
    print(json.dumps(out))


if __name__ == "__main__":
    main()
