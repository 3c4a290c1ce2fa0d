// samsung2_emu.cpp -- CPU replay of the Samsung V2 kernels (rawspeed_b200/csrc/samsung2.cuh: candidate
// walk, pair step, doubling, coarse and fine row-start resolution, descriptor walk, differences,
// reconstruction), compiled by g++ against tests/emu/cuda_emu.h and run in the plan's order with the
// plan's layout (s2_place_frame), every CTA's threads as fibers in forward or reverse order.  The
// scratch tables are handed back for direct checks.  Test infrastructure (no GPU needed); parity of
// the real kernels is the GPU tests' job.
#include "cuda_emu.h"

#include "../../rawspeed_b200/csrc/samsung2.cuh"

#include <functional>
#include <vector>

using namespace rsb200;

namespace {
void cta(unsigned b, unsigned nb, int nthreads, size_t smem_bytes, bool reverse,
         const std::function<void(uint8_t*)>& body) {
  cuemu::run_cta(b, nb, nthreads, smem_bytes, reverse, body);
}
// Kernels without barriers or warp collectives (all but the reconstruction): the threads of a CTA one
// after the other, in forward or reverse order -- any interleaving is equivalent to one of these.
void plain(unsigned b, unsigned nb, int nthreads, bool reverse, const std::function<void()>& body) {
  blockIdx.x = b;
  gridDim.x = nb;
  blockDim.x = (unsigned)nthreads;
  for (int k = 0; k < nthreads; ++k) {
    threadIdx.x = (unsigned)(reverse ? nthreads - 1 - k : k);
    body();
  }
}
// scratch that no kernel should read before writing
constexpr uint32_t GARBAGE = 0xCDCDCDCDu;
} // namespace

// Frames (strips with their header in `in`): in_offset, in_size, bits, w, h, out_offset, out_pitch.
// results: (status, consumed) per frame.  The tables the kernels leave go to tab (ntab entries),
// jump (njump: the pair step after S2_JUMP doublings), rowstart (nrows) and fail (2 per frame), when
// their capacities allow; counts: ntab, njump, nrows.  Returns the loads outside `in` (rounded up to
// a whole 32-bit word).
extern "C" uint64_t s2_emu_run(const uint8_t* in, uint64_t in_total, int n, const uint64_t* in_offset,
                               const uint32_t* in_size, const uint32_t* bits, const uint32_t* w, const uint32_t* h,
                               const uint64_t* out_offset, const uint32_t* out_pitch, uint8_t* out, uint32_t* results,
                               int reverse, uint32_t* tab_out, uint64_t tab_cap, uint32_t* jump_out,
                               uint64_t jump_cap, uint32_t* rows_out, uint64_t rows_cap, uint32_t* fail_out,
                               uint64_t* counts) {
  std::vector<uint8_t> buf((size_t)in_total + 512);
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(buf.data()) + 255) & ~(uintptr_t)255);
  memcpy(base, in, (size_t)in_total);
  const uint32_t nf = (uint32_t)n;
  std::vector<S2FrameDev> fr(nf);
  std::vector<uint32_t> starts(4 * (size_t)nf);
  S2Totals t;
  for (uint32_t i = 0; i < nf; ++i)
    s2_place_frame(fr[i], t, starts.data(), nf, i, in_offset[i], in_size[i], in + in_offset[i], bits[i], w[i], h[i],
                   out_offset[i], out_pitch[i]);
  const uint32_t ntab = (uint32_t)t.tab, njump = (uint32_t)t.jump, nrows = (uint32_t)t.rows, ncps = (uint32_t)t.cps;
  std::vector<uint32_t> tab(ntab, GARBAGE), jump(2 * (size_t)njump, GARBAGE), rowstart(nrows, GARBAGE),
      cp(ncps, GARBAGE), ncp(nf, GARBAGE);
  std::vector<uint2> fail(nf, make_uint2(GARBAGE, GARBAGE)), desc((size_t)t.desc, make_uint2(GARBAGE, GARBAGE)),
      res(nf, make_uint2(GARBAGE, GARBAGE));
  std::vector<int16_t> px((size_t)t.px, (int16_t)0x5A5A);
  const bool rev = reverse != 0;
  const uint32_t* s = starts.data();
  cuemu::ldg_lo = base;
  cuemu::ldg_hi = base + ((in_total + 3) & ~3ull); // (a 32-bit load never leaves its aligned word)
  cuemu::ldg_outside = 0;

  unsigned g = (ntab + S2W_NT - 1) / S2W_NT;
  for (unsigned b = 0; b < g; ++b)
    plain(b, g, S2W_NT, rev, [&]() { s2_cand_entry(base, fr.data(), s, nf, ntab, tab.data()); });
  uint32_t* src = jump.data();
  uint32_t* dst = jump.data() + njump;
  g = (njump + S2J_NT - 1) / S2J_NT;
  for (unsigned b = 0; b < g; ++b)
    plain(b, g, S2J_NT, rev, [&]() { s2_pair_entry(fr.data(), s + nf, nf, njump, tab.data(), src); });
  for (int r = 0; r < S2_JUMP; ++r) {
    for (unsigned b = 0; b < g; ++b)
      plain(b, g, S2J_NT, rev, [&]() { s2_double_entry(fr.data(), s + nf, nf, njump, src, dst); });
    std::swap(src, dst);
  }
  g = (nf + S2J_NT - 1) / S2J_NT;
  for (unsigned b = 0; b < g; ++b)
    plain(b, g, S2J_NT, rev, [&]() {
      s2_coarse_entry(fr.data(), nf, tab.data(), src, rowstart.data(), cp.data(), ncp.data(), fail.data());
    });
  g = (ncps + S2J_NT - 1) / S2J_NT;
  for (unsigned b = 0; b < g; ++b)
    plain(b, g, S2J_NT, rev, [&]() {
      s2_fine_entry(fr.data(), s + 3 * nf, nf, ncps, tab.data(), cp.data(), ncp.data(), rowstart.data(),
                     fail.data());
    });
  g = (nrows + S2W_NT - 1) / S2W_NT;
  for (unsigned b = 0; b < g; ++b)
    plain(b, g, S2W_NT, rev, [&]() {
      s2_desc_entry(base, fr.data(), s + 2 * nf, nf, nrows, rowstart.data(), fail.data(), desc.data());
    });
  for (unsigned b = 0; b < nrows; ++b)
    plain(b, nrows, S2X_NT, rev, [&]() {
      s2_diff_entry(base, fr.data(), s + 2 * nf, nf, fail.data(), desc.data(), px.data());
    });
  for (unsigned b = 0; b < nf; ++b)
    cta(b, nf, S2R_NT, sizeof(S2Smem), rev, [&](uint8_t* smem) {
      s2_recon_entry(fr.data(), fail.data(), desc.data(), px.data(), out, res.data(), *reinterpret_cast<S2Smem*>(smem));
    });
  cuemu::ldg_lo = cuemu::ldg_hi = nullptr;

  for (uint32_t i = 0; i < nf; ++i) {
    results[2 * i] = res[i].x;
    results[2 * i + 1] = res[i].y;
    fail_out[2 * i] = fail[i].x;
    fail_out[2 * i + 1] = fail[i].y;
  }
  if (ntab <= tab_cap)
    memcpy(tab_out, tab.data(), sizeof(uint32_t) * ntab);
  if (njump <= jump_cap)
    memcpy(jump_out, src, sizeof(uint32_t) * njump);
  if (nrows <= rows_cap)
    memcpy(rows_out, rowstart.data(), sizeof(uint32_t) * nrows);
  counts[0] = ntab;
  counts[1] = njump;
  counts[2] = nrows;
  return cuemu::ldg_outside;
}
