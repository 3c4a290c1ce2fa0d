"""Time Samsung V0 decoding (rsb200_samsung0_plan_create) on batches of frames at the constructor's
limit (5546x3714) and at a mid size (3000x2000): natural content with mixed directions, all up, all
left and the staircase (the deepest dependency chains).  CUDA events around plan.run after warm-up;
prints MPix/s per batch with the GPU name and power limit read in the same run, and with --profile a
per-kernel breakdown (torch.profiler, CUDA activities) of one batch per content.  With --ref-lib (a
build of the reference's SamsungV0Decompressor by tools/samsung0_ref_golden.py), also the reference's
single-thread rate on the same host.

    python tools/samsung_v0_time.py [--frames-full 4] [--frames-mid 8] [--iters 10] [--profile]
                                    [--ref-lib PATH]"""
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

import samsung0_oracle as S  # noqa: E402


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def content(name, w, h):
    v = S.natural_values(w, h, seed=w + h)
    d = {"natural": S.dirs_random(w, h, seed=1), "up": S.dirs_up(w, h), "left": S.dirs_left(w, h),
         "staircase": S.dirs_staircase(w, h)}[name]
    bso, bsr, _ = S.make_frame(v, d)
    return bso, bsr


def ref_rate(path, bso, bsr, w, h, reps):
    """Single-thread MPix/s of the reference's own SamsungV0Decompressor (constructor + decompress)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import samsung0_ref_golden as G
    L = G.load(path)
    best = None
    for _ in range(reps):
        t0 = time.perf_counter()
        mid, _ = G.ref_call(L, bso, bsr, w, h)
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
    sizes = [((5546, 3714), a.frames_full), ((3000, 2000), a.frames_mid)]
    frames = {(name, wh): content(name, *wh) for wh, _ in sizes
              for name in ("natural", "up", "left", "staircase")}
    if a.ref_lib:
        out["reference_single_thread_mpix_s"] = {
            "%s_%dx%d" % (n, wh[0], wh[1]): round(ref_rate(a.ref_lib, *frames[(n, wh)], *wh, 3), 1)
            for (n, wh) in frames}
    if a.no_gpu:
        print(json.dumps(out))
        return
    import torch
    import rawspeed_b200 as rs
    out["gpu"] = gpu_info()
    ctx = rs.Context(0)
    for (w, h), nf in sizes:
        for name in ("natural", "up", "left", "staircase"):
            bso, bsr = frames[(name, (w, h))]
            offs = list(np.frombuffer(bso, "<u4").astype(np.int64)) + [len(bsr)]
            blob, jobs, strips = bytearray(), [], []
            pitch = S.pitch_elems(w) * 2
            for k in range(nf):
                blob += bytes((-len(blob)) % 16)
                base = len(blob)
                blob += bsr
                j = rs.SamsungV0Job()
                j.out_offset, j.out_pitch, j.width, j.height, j.first_strip = k * pitch * h, pitch, w, h, len(strips)
                jobs.append(j)
                for r in range(h):
                    s = rs.SamsungV0Strip()
                    s.in_offset, s.in_size = base + int(offs[r]), int(offs[r + 1] - offs[r])
                    strips.append(s)
            plan = rs.samsung0_plan(ctx, jobs, strips)
            d_in = torch.from_numpy(np.frombuffer(bytes(blob) + bytes(64), np.uint8).copy()).cuda()
            d_out = torch.zeros(nf * pitch * h // 2 + 64, dtype=torch.int16, device="cuda")
            for _ in range(a.warmup):
                plan.run((d_in.data_ptr(), len(blob)), d_out)
            torch.cuda.synchronize()
            assert all(r == (0, 0) for r in plan.results())
            want = S.decompress(bso, bsr, w, h)[0]
            got = d_out[:pitch * h // 2].cpu().numpy().view(np.uint16).reshape(h, pitch // 2)
            assert np.array_equal(got[:, :w], want[:, :w]), "output differs from the restatement"
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            times = []
            for _ in range(a.iters):
                e0.record()
                plan.run((d_in.data_ptr(), len(blob)), d_out)
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            med = float(np.median(times))
            rec = {"frames": nf, "ms_median": round(med, 3), "ms_min": round(min(times), 3),
                   "mpix_s": round(nf * w * h / med / 1e3, 1),
                   "mb_per_frame": round(len(bsr) / 1e6, 2)}
            if a.profile:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    plan.run((d_in.data_ptr(), len(blob)), d_out)
                    torch.cuda.synchronize()
                per = {}
                for ev in prof.key_averages():
                    if "s0_" in ev.key and "_kernel" in ev.key:
                        k = ev.key.split("s0_")[1].split("_kernel")[0]
                        per[k] = round(getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0)) / 1e3, 3)
                rec["kernel_ms"] = per
            out["%s_%dx%d" % (name, w, h)] = rec
            del plan, d_in, d_out
    print(json.dumps(out))


if __name__ == "__main__":
    main()
