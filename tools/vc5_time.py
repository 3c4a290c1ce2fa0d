"""Time GoPro VC-5 decoding (rsb200_vc5_plan_create) on GoPro-sized frames, 4000x3000 (12 MP) and
5568x4176 (23 MP), in plans of 1 and 16 frames, with natural content (sparse high-pass bands), noisy
content (every coefficient a random magnitude up to 40: dense, longer codes) and flat content (one zero
run per band).  CUDA events around plan.run after warm-up; prints MPix/s per plan with the GPU name, power
limit and maximum SM clock, and the SM clock read right after each timed loop (sm_clock_after), all
read in the same run.  The split between the stages (low pass, segment resolution =
candidate walks + scan rounds, store, each reconstruction level, final combine) comes from
torch.profiler with CUDA activities in a separate run per plan, beside the bytes each stage moves,
computed from the shapes, and what that is against the H100 SXM data sheet's 3.35 TB/s.

    python tools/vc5_time.py [--iters 10] [--frames 1 16] [--sizes 4000x3000 5568x4176]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import vc5_oracle as V  # noqa: E402

PS2 = [[2, 2, 2]] * 4
STAGES = {"lowpass": ("vc5_lowpass",), "resolve": ("vc5_walk", "vc5_scan"), "store": ("vc5_store",),
          "result": ("vc5_result",), "levels_3_2": ("vc5_recon",), "final": ("vc5_final",)}
SEG, CAND = 1024, 27


def gpu_info(fields="name,power.limit,clocks.max.sm"):
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=" + fields,
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def stage_bytes(w, h, high_bytes, rounds, nf):
    """Least bytes each stage must move for nf frames: payload reads, map and band writes, plane reads."""
    dims = V.band_dims(w, h)
    segs = sum(8 * b + 65 for b in high_bytes) // SEG + len(high_bytes)
    coefs = sum(4 * 3 * dims[k][0] * dims[k][1] for k in (1, 2, 3))
    low = 4 * dims[3][0] * dims[3][1]
    rec = [4 * 4 * dims[3][0] * dims[3][1], 4 * 4 * dims[2][0] * dims[2][1]]
    return {k: v * nf for k, v in {
        "lowpass": low * 4,  # 16-bit fields in, int16 out
        "resolve": sum(high_bytes) * CAND + segs * CAND * 8 * (1 + 2 * rounds),
        "store": sum(high_bytes) + segs * 8 + 2 * coefs,
        "result": 0,
        "levels_3_2": 2 * (rec[0] + rec[1]) * 2,  # bands in (as many as out), planes out
        "final": 2 * (4 * 3 * dims[1][0] * dims[1][1] + rec[1]) + 2 * w * h,
    }.items()}


def content(w, h, kind):
    return {"natural": lambda: V.natural(w, h, seed=1),
            "noisy": lambda: V.noise(w, h, seed=2, top=40),
            "flat": lambda: V.flat(w, h, 1000)}[kind]()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--sizes", nargs="+", default=["4000x3000", "5568x4176"])
    ap.add_argument("--kinds", nargs="+", default=["natural", "noisy", "flat"])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import rawspeed_b200 as rs
    out = {"gpu_name_power_limit_max_sm_clock": gpu_info()}
    ctx = rs.Context(0)
    for size in a.sizes:
        w, h = (int(x) for x in size.split("x"))
        for kind in a.kinds:
            data = V.encode(w, h, content(w, h, kind), prescale=PS2)
            want, rc, _ = V.decompress(data, w, h, 4095)
            assert rc == V.OK
            fields, table = V.band_table(data, w, h, 4095)
            high = [b[1] for i, b in enumerate(table) if i % 10]
            for nf in a.frames:
                blob, jobs, bands, outs, total = V.plan_inputs([(data, w, h, 4095, V.RGGB)] * nf)
                plan = rs.vc5_plan(ctx, V.codebook(), jobs, bands)
                d_in = torch.from_numpy(np.frombuffer(blob, np.uint8).copy()).cuda()
                d_out = torch.zeros(total, dtype=torch.int16, device="cuda")
                for _ in range(a.warmup):
                    plan.run((d_in.data_ptr(), len(blob)), d_out)
                torch.cuda.synchronize()
                assert all(tuple(r) == (0, 0) for r in plan.results())
                o = d_out.cpu().numpy().view(np.uint16)
                for off, hh, pitch in outs:
                    assert np.array_equal(o[off:off + hh * pitch].reshape(hh, pitch)[:, :w], want[:h, :w]), \
                        "output differs from the restatement"
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
                rounds = plan.launches - 7
                nb = stage_bytes(w, h, high, rounds, nf)
                out["%s_%s_x%d" % (kind, size, nf)] = {
                    "sm_clock_after": sm_clock, "ms_median": round(med, 3), "ms_min": round(min(times), 3),
                    "mpix_s": round(nf * w * h / med / 1e3, 1), "mb_per_frame": round(len(data) / 1e6, 2),
                    "segments_per_frame": sum((8 * b + 65 + SEG - 1) // SEG for b in high),
                    "largest_band_segments": max((8 * b + 65 + SEG - 1) // SEG for b in high),
                    "scan_rounds": rounds,
                    "split_ms": {s: round(t, 3) for s, t in split.items()},
                    "split_gb_s": {s: round(nb[s] / (t * 1e6), 1) if t else None for s, t in split.items()},
                    "split_share_of_3350_gb_s": {s: round(nb[s] / (t * 1e6) / 3350, 3) if t else None
                                                 for s, t in split.items()}}
                plan.close()
                del d_in, d_out
    print(json.dumps(out))


if __name__ == "__main__":
    main()
