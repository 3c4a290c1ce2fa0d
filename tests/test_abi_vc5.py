"""The VC-5 structs of include/rawspeed_b200.h against their ctypes mirrors, the new entry point in the
export lists, and the codebook kept out of the product: it reaches a plan only as an argument."""
import ctypes as C
import os
import subprocess

import rawspeed_b200 as rs
from rawspeed_b200 import _abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_struct_layout_matches_header(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(r'''
#include <stdio.h>
#include <stddef.h>
#include "rawspeed_b200.h"
#define O(t, f) (unsigned)offsetof(t, f)
int main(void){
  printf("%u %u %u %u %u  %u %u %u %u  %u %u %u %u %u %u %u %u %u %u  %u %u %u %u %u %u %u %u %u %u\n",
         (unsigned)sizeof(rsb200_vc5_code), O(rsb200_vc5_code, bits), O(rsb200_vc5_code, count),
         O(rsb200_vc5_code, value), 0u,
         (unsigned)sizeof(rsb200_vc5_band), O(rsb200_vc5_band, in_offset), O(rsb200_vc5_band, in_size),
         O(rsb200_vc5_band, param),
         (unsigned)sizeof(rsb200_vc5_job), O(rsb200_vc5_job, width), O(rsb200_vc5_job, height),
         O(rsb200_vc5_job, output_bits), O(rsb200_vc5_job, phase), O(rsb200_vc5_job, prescale),
         O(rsb200_vc5_job, first_band), O(rsb200_vc5_job, out_offset), O(rsb200_vc5_job, out_pitch),
         O(rsb200_vc5_job, reserved),
         RSB200_VC5_RGGB, RSB200_VC5_GBRG, RSB200_VC5_QUANT, RSB200_VC5_EARLY_END, RSB200_VC5_OVERRUN,
         RSB200_VC5_NO_END, RSB200_VC5_SHORT, RSB200_VC5_OVERREAD, 0u, 0u);
  return 0;
}
''')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(prog)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    K, B, J = _abi.Vc5Code, _abi.Vc5Band, _abi.Vc5Job
    want = [C.sizeof(K), K.bits.offset, K.count.offset, K.value.offset, 0,
            C.sizeof(B), B.in_offset.offset, B.in_size.offset, B.param.offset,
            C.sizeof(J), J.width.offset, J.height.offset, J.output_bits.offset, J.phase.offset, J.prescale.offset,
            J.first_band.offset, J.out_offset.offset, J.out_pitch.offset, J.reserved.offset,
            0, 2, 1, 2, 3, 4, 5, 6, 0, 0]
    assert got == want


def test_entry_points_listed():
    assert "rsb200_vc5_plan_create" in _abi.EXPORTS
    for name in ("vc5_plan", "Vc5Job", "Vc5Band", "Vc5Code"):
        assert name in rs.__all__


def test_codebook_only_in_the_fixture():
    """The end marker's 26-bit code word (taken from the fixture) appears in no product, header or test
    source."""
    import vc5_oracle as V
    end = int(V.codebook()[V.entry(0, 1)][1])
    words = ("0x%08x" % end, "0x%x" % end, "%d" % end)
    for top in ("rawspeed_b200", "include", "tests", "tools"):
        for d, _, files in os.walk(os.path.join(ROOT, top)):
            if os.path.relpath(d, ROOT).startswith(os.path.join("tests", "golden")) or "_build" in d or \
                    "__pycache__" in d:
                continue
            for f in files:
                if not f.endswith((".py", ".c", ".cpp", ".h", ".cuh", ".cu", ".json", ".inc")):
                    continue
                text = open(os.path.join(d, f), encoding="utf-8", errors="replace").read().lower()
                assert not any(w.lower() in text for w in words), os.path.join(d, f)
