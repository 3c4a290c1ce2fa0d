"""The Kodak DCR struct of include/rawspeed_b200.h against its ctypes mirror, and the new entry points
in the export lists."""
import ctypes as C
import os
import subprocess

import rawspeed_b200 as rs
from rawspeed_b200 import _abi, host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_struct_layout_matches_header(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(r'''
#include <stdio.h>
#include <stddef.h>
#include "rawspeed_b200.h"
int main(void){
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %u %u\n", sizeof(rsb200_kodak_job),
         offsetof(rsb200_kodak_job, in_offset), offsetof(rsb200_kodak_job, in_size),
         offsetof(rsb200_kodak_job, width), offsetof(rsb200_kodak_job, height),
         offsetof(rsb200_kodak_job, bps), offsetof(rsb200_kodak_job, table),
         offsetof(rsb200_kodak_job, out_offset), offsetof(rsb200_kodak_job, out_pitch),
         offsetof(rsb200_kodak_job, reserved), RSB200_KODAK_VALUE, RSB200_KODAK_OVERFLOW);
  return 0;
}
''')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(prog)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    J = _abi.KodakJob
    want = [C.sizeof(J), J.in_offset.offset, J.in_size.offset, J.width.offset, J.height.offset, J.bps.offset,
            J.table.offset, J.out_offset.offset, J.out_pitch.offset, J.reserved.offset, 1, 2]
    assert got == want


def test_entry_points_listed():
    assert "rsb200_kodak_plan_create" in _abi.EXPORTS
    assert "rsb200_kodak_plan_values" in _abi.EXPORTS
    assert "rsb200h_kodak" in host.EXPORTS
    assert "kodak_plan" in rs.__all__ and "KodakJob" in rs.__all__
