"""How many 64-byte runs k2_stream_kernel's output stage stores by whole warps, and how many lane by lane
(profiling only).

    python tools/ab_ljpeg.py build NAME -DRSB200_FLUSH_COUNT       # here: tools/_ab/NAME.so
    python tools/flush_count.py tools/_ab/NAME.so [FRAMES ...]      # on the GPU box (default: 128 256)

The workload is the one bench.py times: frames of the 8256x5504 DNG (256 x 256 LJPEG tiles) in one plan,
device-resident.  One run per batch size; the output is checked bit for bit against the encoder's input."""
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    lib = os.path.abspath(sys.argv[1])
    frames = [int(x) for x in sys.argv[2:]] or [128, 256]
    os.environ["RSB200_LIB"] = lib
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import numpy as np
    import torch
    import rawspeed_b200 as rs
    from rawspeed_b200 import _abi
    from oracle import synth
    from helpers import dng_ljpeg_scans

    L = _abi.load()
    L.rsb200_debug_flush_runs.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    ctx = rs.Context(0)
    W, H = 8256, 5504
    img = synth.image_model(W, H, 12345)
    t = synth.make_dng_ljpeg(img, 256, 256)
    pitch = rs.image_pitch(W)
    tabs, scans = dng_ljpeg_scans(t, pitch)
    fb = (t.blob.size + 255) // 256 * 256
    ob = (H * pitch + 255) // 256 * 256
    buf = (ctypes.c_ulonglong * 2)()
    for nb in frames:
        d_in = torch.zeros(nb * fb + 64, dtype=torch.uint8, device="cuda")
        blob = torch.from_numpy(t.blob).cuda()
        batch = []
        for f in range(nb):
            d_in[f * fb:f * fb + t.blob.size] = blob
            for s0 in scans:
                s1 = rs.LJpegScan.from_buffer_copy(s0)
                s1.in_offset = s0.in_offset + f * fb
                s1.out_offset = s0.out_offset + f * ob
                batch.append(s1)
        d_out = torch.zeros(nb * ob, dtype=torch.uint8, device="cuda")
        plan = rs.ljpeg_plan(ctx, tabs.tabs, batch)
        L.rsb200_debug_flush_runs(buf, 1)
        plan.run((d_in.data_ptr(), nb * fb), d_out)
        L.rsb200_debug_flush_runs(buf, 1)
        exact = all(s == 0 for s, _ in plan.results())
        for f in (0, nb - 1):
            got = d_out[f * ob:f * ob + H * pitch].cpu().numpy().view(np.uint16).reshape(H, pitch // 2)
            exact = exact and bool(np.array_equal(got[:, :W], img))
        whole, lane = int(buf[0]), int(buf[1])
        print("FLUSH " + json.dumps({"lib": os.path.basename(lib), "frames": nb, "kernel": plan.kernels,
                                     "runs_whole_warp": whole, "runs_single_lane": lane,
                                     "whole_share": round(whole / max(1, whole + lane), 4), "exact": exact}))
        del plan, d_in, d_out


if __name__ == "__main__":
    main()
