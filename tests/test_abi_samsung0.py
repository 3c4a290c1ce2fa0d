"""The Samsung V0 structs of include/rawspeed_b200.h against their ctypes mirrors, and the new entry
points in the export lists."""
import ctypes as C
import os
import subprocess

from rawspeed_b200 import _abi, host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_struct_layouts_match_header(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(r'''
#include <stdio.h>
#include <stddef.h>
#include "rawspeed_b200.h"
int main(void){
  printf("%zu %zu %zu %zu\n", sizeof(rsb200_samsung0_strip), offsetof(rsb200_samsung0_strip, in_offset),
         offsetof(rsb200_samsung0_strip, in_size), offsetof(rsb200_samsung0_strip, reserved));
  printf("%zu %zu %zu %zu %zu %zu\n", sizeof(rsb200_samsung0_job), offsetof(rsb200_samsung0_job, out_offset),
         offsetof(rsb200_samsung0_job, out_pitch), offsetof(rsb200_samsung0_job, width),
         offsetof(rsb200_samsung0_job, height), offsetof(rsb200_samsung0_job, first_strip));
  printf("%u %u %u %u %u %u\n", RSB200_S0_LEN_NEG, RSB200_S0_LEN_BIG, RSB200_S0_UP_FIRST, RSB200_S0_UP_LAST,
         RSB200_S0_OVERREAD, RSB200_S0_SHORT);
  return 0;
}
''')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(prog)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    S, J = _abi.SamsungV0Strip, _abi.SamsungV0Job
    want = [C.sizeof(S), S.in_offset.offset, S.in_size.offset, S.reserved.offset,
            C.sizeof(J), J.out_offset.offset, J.out_pitch.offset, J.width.offset, J.height.offset,
            J.first_strip.offset, 1, 2, 3, 4, 5, 6]
    assert got == want


def test_entry_points_listed():
    assert "rsb200_samsung0_plan_create" in _abi.EXPORTS
    assert "rsb200h_samsung_v0" in host.EXPORTS
