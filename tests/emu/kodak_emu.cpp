// kodak_emu.cpp -- CPU replay of the Kodak DCR kernels (rawspeed_b200/csrc/kodak.cuh: nibble-sum
// prefix, candidate walk, doubling, coarse and fine row-start resolution, check and store), compiled by
// g++ against tests/emu/cuda_emu.h and run in the plan's order with the plan's layout (kd_place_frame),
// every CTA's threads as fibers in forward or reverse order.  The candidate entries, the row starts and
// the failures are handed back for direct checks.  Test infrastructure (no GPU needed); parity of the
// real kernels is the GPU tests' job.
#include "cuda_emu.h"

#include "../../rawspeed_b200/csrc/kodak.cuh"

#include <functional>
#include <vector>

using namespace rsb200;

namespace {
void cta(unsigned b, unsigned nb, int nthreads, size_t smem_bytes, bool reverse,
         const std::function<void(uint8_t*)>& body) {
  cuemu::run_cta(b, nb, nthreads, smem_bytes, reverse, body);
}
// Kernels without barriers or warp collectives: the threads of a CTA one after the other, in forward
// or reverse order -- any interleaving is equivalent to one of these.
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

// Frames in `in`: in_offset, in_size, w, h, bps, table (first entry in `tables`, or ~0u), out_offset,
// out_pitch.  results: (status, consumed) per frame, values: the printed value per frame.  The
// candidate entries go to tab (cap entries), the row starts to rows (cap), the failures to fail (2 per
// frame); counts: candidates, rows.  Returns the loads outside `in`.
extern "C" uint64_t kd_emu_run(const uint8_t* in, uint64_t in_total, int n, const uint64_t* in_offset,
                               const uint32_t* in_size, const uint32_t* w, const uint32_t* h, const uint32_t* bps,
                               const uint32_t* table, const uint16_t* tables, const uint64_t* out_offset,
                               const uint32_t* out_pitch, uint8_t* out, uint32_t* results, int32_t* values,
                               int reverse, uint32_t* tab_out, uint64_t tab_cap, uint32_t* rows_out,
                               uint64_t rows_cap, uint32_t* fail_out, uint64_t* counts) {
  std::vector<uint8_t> buf((size_t)in_total + 512);
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(buf.data()) + 255) & ~(uintptr_t)255);
  memcpy(base, in, (size_t)in_total);
  const uint32_t nf = (uint32_t)n;
  std::vector<KdFrameDev> fr(nf);
  std::vector<uint32_t> starts(4 * (size_t)nf);
  KdTotals t;
  for (uint32_t i = 0; i < nf; ++i)
    kd_place_frame(fr[i], t, starts.data(), nf, i, in_offset[i], in_size[i], w[i], h[i], bps[i], table[i],
                   out_offset[i], out_pitch[i]);
  const uint32_t ntiles = (uint32_t)t.tiles, ncand = (uint32_t)t.cand, ncps = (uint32_t)t.cps,
                 nsegs = (uint32_t)t.segs;
  std::vector<uint32_t> tsum(ntiles, GARBAGE), q((size_t)t.q, GARBAGE), tab(ncand, GARBAGE),
      jump(2 * (size_t)ncand, GARBAGE), rowstart((size_t)t.rows, GARBAGE), cp(ncps, GARBAGE), ncp(nf, GARBAGE),
      key(nf, GARBAGE);
  std::vector<uint2> fail(nf, make_uint2(GARBAGE, GARBAGE)), res(nf, make_uint2(GARBAGE, GARBAGE));
  std::vector<int32_t> val(nf, (int32_t)GARBAGE);
  const bool rev = reverse != 0;
  const uint32_t* s = starts.data();
  cuemu::ldg_lo = base;
  cuemu::ldg_hi = base + in_total;
  cuemu::ldg_outside = 0;

  const size_t ws = sizeof(uint32_t) * (KD_NT / 32);
  for (unsigned b = 0; b < ntiles; ++b)
    cta(b, ntiles, KD_NT, ws, rev, [&](uint8_t* sm) {
      kd_tsum_entry(base, fr.data(), s, nf, tsum.data(), reinterpret_cast<uint32_t*>(sm));
    });
  for (unsigned b = 0; b < nf; ++b)
    cta(b, nf, KD_NT, ws, rev,
        [&](uint8_t* sm) { kd_tscan_entry(fr.data(), tsum.data(), reinterpret_cast<uint32_t*>(sm)); });
  for (unsigned b = 0; b < ntiles; ++b)
    cta(b, ntiles, KD_NT, ws, rev, [&](uint8_t* sm) {
      kd_prefix_entry(base, fr.data(), s, nf, tsum.data(), q.data(), reinterpret_cast<uint32_t*>(sm));
    });
  unsigned g = (ncand + KD_NT - 1) / KD_NT;
  for (unsigned b = 0; b < g; ++b)
    plain(b, g, KD_NT, rev, [&]() { kd_cand_entry(fr.data(), s + nf, nf, ncand, q.data(), tab.data()); });
  const uint32_t* src = tab.data();
  uint32_t* dst = jump.data();
  for (int r = 0; r < KD_JUMP; ++r) {
    for (unsigned b = 0; b < g; ++b)
      plain(b, g, KD_NT, rev, [&]() { kd_double_entry(fr.data(), s + nf, nf, ncand, src, dst); });
    src = dst;
    dst = dst == jump.data() ? jump.data() + ncand : jump.data();
  }
  g = (nf + KD_NT - 1) / KD_NT;
  for (unsigned b = 0; b < g; ++b)
    plain(b, g, KD_NT, rev,
          [&]() { kd_coarse_entry(fr.data(), nf, src, cp.data(), ncp.data(), fail.data(), key.data()); });
  g = (ncps + KD_NT - 1) / KD_NT;
  for (unsigned b = 0; b < g; ++b)
    plain(b, g, KD_NT, rev, [&]() {
      kd_fine_entry(fr.data(), s + 2 * nf, nf, ncps, tab.data(), cp.data(), ncp.data(), rowstart.data(), fail.data());
    });
  g = (nsegs + KD_NT / 32 - 1) / (KD_NT / 32);
  for (unsigned b = 0; b < g; ++b)
    cta(b, g, KD_NT, 0, rev, [&](uint8_t*) {
      kd_check_entry(base, fr.data(), s + 3 * nf, nf, nsegs, q.data(), rowstart.data(), fail.data(), key.data());
    });
  for (unsigned b = 0; b < g; ++b)
    cta(b, g, KD_NT, 0, rev, [&](uint8_t*) {
      kd_store_entry(base, fr.data(), s + 3 * nf, nf, nsegs, q.data(), rowstart.data(), fail.data(), key.data(),
                     tables, out, res.data(), val.data());
    });
  cuemu::ldg_lo = cuemu::ldg_hi = nullptr;

  for (uint32_t i = 0; i < nf; ++i) {
    results[2 * i] = res[i].x;
    results[2 * i + 1] = res[i].y;
    values[i] = val[i];
    fail_out[2 * i] = fail[i].x;
    fail_out[2 * i + 1] = fail[i].y;
  }
  if (ncand <= tab_cap)
    memcpy(tab_out, tab.data(), sizeof(uint32_t) * ncand);
  if (t.rows <= rows_cap)
    memcpy(rows_out, rowstart.data(), sizeof(uint32_t) * t.rows);
  counts[0] = ncand;
  counts[1] = t.rows;
  return cuemu::ldg_outside;
}
