// vc5_emu.cpp -- CPU replay of the VC-5 kernels (rawspeed_b200/csrc/vc5.cuh: low pass, segment walks,
// scan rounds, store, per-frame result, the two reconstruction levels and the final combine), compiled
// by g++ against tests/emu/cuda_emu.h and run in the plan's order with the plan's layout (vc5_layout)
// and decode table (vc5_build_code), each CTA's threads in forward or reverse order.  Test
// infrastructure (no GPU needed); parity of the real kernels is the GPU tests' job.
#include "cuda_emu.h"

#define __constant__
static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  const unsigned long long o = *p;
  if (v < o)
    *p = v;
  return o;
}

#include "../../rawspeed_b200/csrc/vc5.cuh"

#include <functional>
#include <vector>

namespace {
// kernels without barriers or warp collectives: the threads of a CTA one after the other
void grid(unsigned gx, unsigned gy, bool reverse, const std::function<void()>& body) {
  gridDim.x = gx, gridDim.y = gy;
  blockDim.x = VC5_NT;
  for (unsigned y = 0; y < gy; ++y)
    for (unsigned x = 0; x < gx; ++x) {
      blockIdx.x = x, blockIdx.y = y;
      for (unsigned k = 0; k < VC5_NT; ++k) {
        threadIdx.x = reverse ? VC5_NT - 1 - k : k;
        body();
      }
    }
}
unsigned blocks(uint64_t n) { return (unsigned)std::max<uint64_t>(1, (n + VC5_NT - 1) / VC5_NT); }
} // namespace

// A plan's run on the CPU.  codes: ncodes x {size, bits, count, value}; results: (status, consumed) per
// job; map_out (nsegs * VC5_CAND x 2, if not null): the scanned maps.  Returns -2 for a codebook the
// plan refuses, the refused job's index, or -1 with counts[0] = segments, counts[1] = scan rounds.
extern "C" int vc5_emu_run(const uint8_t* in, uint64_t in_total, const rsb200_vc5_code* codes, int ncodes,
                           const rsb200_vc5_job* jobs, int njobs, const rsb200_vc5_band* bands, int nbands,
                           uint8_t* out, uint32_t* results, int reverse, uint32_t* map_out, uint64_t map_cap,
                           uint32_t* counts) {
  std::vector<uint32_t> code;
  if (!vc5_build_code(codes, ncodes, code))
    return -2;
  Vc5Layout L;
  const char* why = nullptr;
  const int bad = vc5_layout(jobs, njobs, bands, nbands, L, &why);
  if (bad >= 0)
    return bad;
  std::vector<uint8_t> buf((size_t)in_total + 64, 0);
  memcpy(buf.data(), in, (size_t)in_total);
  const uint32_t nf = (uint32_t)njobs, nsegs = (uint32_t)L.seg_band.size();
  std::vector<int16_t> coef((size_t)L.ncoef, 0);  // the run's memset
  std::vector<uint2> map(2 * (size_t)nsegs * VC5_CAND + 1);
  std::vector<unsigned long long> err(L.bands.size(), ~0ull);
  std::vector<uint2> res(nf);
  const std::vector<uint16_t> luts = vc5_luts();
  const Vc5FrameDev* fr = L.frames.data();
  const Vc5BandDev* bd = L.bands.data();
  const bool rev = reverse != 0;
  grid(blocks(L.max_low), 4 * nf, rev, [&] { vc5_lowpass_kernel(buf.data(), bd, coef.data()); });
  uint2* a = map.data();
  uint2* b = a + (size_t)nsegs * VC5_CAND;
  const unsigned gm = blocks((uint64_t)nsegs * VC5_CAND);
  grid(gm, 1, rev, [&] { vc5_walk_kernel(buf.data(), bd, L.seg_band.data(), nsegs, code.data(), a); });
  for (uint32_t r = 0; r < L.rounds; ++r) {
    grid(gm, 1, rev, [&] { vc5_scan_kernel(bd, L.seg_band.data(), nsegs, r, a, b); });
    std::swap(a, b);
  }
  grid(blocks(nsegs), 1, rev, [&] {
    vc5_store_kernel(buf.data(), bd, L.seg_band.data(), nsegs, code.data(), a, err.data(), coef.data());
  });
  grid(blocks(nf), 1, rev, [&] { vc5_result_kernel(fr, nf, bd, err.data(), res.data()); });
  for (uint32_t lvl = 0; lvl < 2; ++lvl)
    grid(blocks(L.max_rec[lvl]), 4 * nf, rev, [&] { vc5_recon_kernel(fr, bd, lvl, coef.data()); });
  grid(blocks(L.max_quads), nf, rev,
       [&] { vc5_final_kernel(fr, bd, coef.data(), luts.data(), res.data(), out); });
  for (uint32_t i = 0; i < nf; ++i)
    results[2 * i] = res[i].x, results[2 * i + 1] = res[i].y;
  for (uint64_t t = 0; map_out && t < (uint64_t)nsegs * VC5_CAND && t < map_cap; ++t)
    map_out[2 * t] = a[t].x, map_out[2 * t + 1] = a[t].y;
  counts[0] = nsegs;
  counts[1] = L.rounds;
  return -1;
}
