"""Time Sony ARW1 decoding (rsb200_arw1_plan_create) on batches of 3872x2592 frames (DSLR-A100
size): natural, uniform and clipped-band content.  CUDA events around plan.run after warm-up;
prints MPix/s per batch with the GPU name and power limit read in the same run, and how many frames
the exact single-CTA decoder had to redo.

    python tools/arw1_time.py [--frames 8] [--iters 20]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import rawspeed_b200 as rs  # noqa: E402
import arw1_oracle as A  # noqa: E402


def gpu_info():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit",
                                     "--format=csv,noheader"], text=True).strip().splitlines()[0]
        return q
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    w, h = 3872, 2592
    ctx = rs.Context(0)
    out = {"gpu": gpu_info(), "frame": [w, h], "frames": a.frames}
    kinds = {"natural": lambda k: A.natural_frame(w, h, k),
             "uniform": lambda k: A.uniform_frame(w, h, 300 + k),
             "clipped": lambda k: A.clipped_frame(w, h, 1000 + 37 * k, 16, seed=k)}
    for name, make in kinds.items():
        streams = [A.encode_frame(make(k)) for k in range(a.frames)]
        blob, jobs = bytearray(), []
        pitch = A.pitch_elems(w)
        for k, s in enumerate(streams):
            blob += bytes((-len(blob)) % 16)
            j = rs.Arw1Job()
            j.in_offset, j.in_size, j.width, j.height = len(blob), len(s), w, h
            j.out_offset, j.out_pitch = k * pitch * 2 * h, pitch * 2
            blob += s
            jobs.append(j)
        plan = rs.arw1_plan(ctx, jobs)
        d_in = torch.from_numpy(np.frombuffer(bytes(blob) + bytes(64), np.uint8).copy()).cuda()
        d_out = torch.zeros(a.frames * pitch * h + 64, dtype=torch.int16, device="cuda")
        for _ in range(a.warmup):
            plan.run((d_in.data_ptr(), len(blob)), d_out)
        torch.cuda.synchronize()
        assert all(r[0] == 0 for r in plan.results())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(a.iters):
            e0.record()
            plan.run((d_in.data_ptr(), len(blob)), d_out)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        f = ctx._lib.rsb200_debug_range_redo
        f.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_int]
        arr = (C.c_uint32 * a.frames)()
        ctx.check(f(plan.h, arr, a.frames))
        med = float(np.median(times))
        out[name] = {"ms_median": round(med, 3), "ms_min": round(min(times), 3),
                     "mpix_s": round(a.frames * w * h / med / 1e3, 1),
                     "mb_per_frame": round(len(blob) / a.frames / 1e6, 2), "redone": int(sum(arr))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
