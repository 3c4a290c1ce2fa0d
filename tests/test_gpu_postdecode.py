"""The post-decode kernels (K9 scaling, K10 DNG opcodes, K11 bad pixels, K12 table lookup) and
Panasonic V4 on the GPU: the two torch-free scripts under tools/, run as a user would run them.

 * tools/quick_validate.py -- every scenario of their test files through the C++ host mirror
   (-> C ABI -> kernel), compared with the oracle: pixels, crops, bad-pixel lists in order,
   error class after a partially applied opcode list (54 cases);
 * tools/quick_time.py -- full 8256x5504 frames through the C ABI with device-resident buffers,
   first run of every leg compared bit for bit with the oracle.

The per-kernel pytest files (test_gpu_scale / _lookup / _dngopcodes / _badpixels /
_panasonic_v4) cover the same ground through torch-owned buffers (un-gated in round 2)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_scenario_through_the_host_mirror():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "quick_validate.py")],
                       capture_output=True, text=True, timeout=600)
    tail = "\n".join(r.stdout.splitlines()[-60:])
    assert r.returncode == 0, tail + r.stderr[-2000:]
    assert "54 passed, 0 failed" in r.stdout, tail


def test_full_frames_through_the_c_abi_are_bit_exact():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "quick_time.py")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("QUICK_TIME ")][-1]
    legs = json.loads(line[len("QUICK_TIME "):])["legs"]
    assert len(legs) == 7
    assert all(v["bit_exact"] for v in legs.values()), legs
