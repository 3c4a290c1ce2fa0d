// samsung1_emu.cpp -- CPU replay of the Samsung V1 reconstruction (rawspeed_b200/csrc/samsung1.cuh:
// s1_column_kernel, s1_row_kernel, s1_scan_kernel, s1_store_kernel), compiled by g++ against
// tests/emu/cuda_emu.h and run in the plan's order with the plan's layout, every CTA's threads as
// fibers in forward or reverse order.  Its input is the difference scratch the range decoder leaves
// (given by the caller), and samsung1_run_phase, the flat-run alignment of the range decoder's
// speculative starts, is exposed for a direct test.  Test infrastructure (no GPU needed); parity of
// the real kernels is the GPU tests' job.
#include "cuda_emu.h"

// (the one warp collective the kernels use that cuda_emu.h does not provide)
static inline uint32_t __shfl_xor_sync(uint32_t mask, uint32_t v, int m) {
  uint32_t pr;
  const uint32_t* r = cuemu::warp_exchange(mask, v, &pr);
  return r[((int)threadIdx.x & 31) ^ (m & 31)];
}

#include "../../rawspeed_b200/csrc/samsung1.cuh"

#include <functional>
#include <vector>

using namespace rsb200;

namespace {
void cta(unsigned b, unsigned nb, int nthreads, size_t smem_bytes, bool reverse,
         const std::function<void(uint8_t*)>& body) {
  cuemu::run_cta(b, nb, nthreads, smem_bytes, reverse, body);
}
} // namespace

extern "C" uint32_t s1_emu_run_phase(uint32_t x0, uint32_t x1) { return samsung1_run_phase(x0, x1); }

// Frames: w, h, T*, first difference (elements, a multiple of 8) in `diffs`, output offset and pitch
// (bytes) in `out`.  results: (status, consumed) per frame.
extern "C" void s1_emu_run(int n, const uint32_t* w, const uint32_t* h, const uint32_t* tstar,
                           const uint64_t* diff_off, const uint16_t* diffs, uint64_t ndiffs,
                           const uint64_t* out_off, const uint32_t* out_pitch, uint8_t* out,
                           uint32_t* results, int reverse) {
  std::vector<DevS1> fr((size_t)n);
  uint32_t rows = 0, maxh = 0;
  for (int i = 0; i < n; ++i) {
    DevS1& f = fr[(size_t)i];
    memset(&f, 0, sizeof f);
    f.diff_offset = diff_off[i];
    f.out_offset = out_off[i];
    f.w = w[i];
    f.h = h[i];
    f.out_pitch = out_pitch[i];
    f.tstar = tstar[i];
    f.scan = (uint32_t)i;
    f.row_base = rows;
    rows += h[i];
    maxh = std::max(maxh, h[i]);
  }
  // 16-byte aligned copy of the scratch (the row walk reads it as uint4)
  std::vector<uint4> dbuf((size_t)(ndiffs + 7) / 8 + 1);
  memcpy(dbuf.data(), diffs, (size_t)ndiffs * 2);
  const uint16_t* d = reinterpret_cast<const uint16_t*>(dbuf.data());
  std::vector<uint16_t> colvals(2 * (size_t)rows, 0xCDCD);
  std::vector<uint2> rowbits((size_t)rows, make_uint2(0xCDCDCDCDu, 0xCDCDCDCDu));
  std::vector<uint32_t> oob((size_t)n, 0xFFFFFFFFu), lim((size_t)n, 0xCDCDCDCDu);
  std::vector<DevResult> res((size_t)n);
  const bool rev = reverse != 0;
  const unsigned ncol = (unsigned)(n * 4 * 32 + 127) / 128;
  for (unsigned b = 0; b < ncol; ++b)
    cta(b, ncol, 128, 0, rev, [&](uint8_t*) { s1_column_kernel(fr.data(), n, d, colvals.data(), oob.data()); });
  const uint32_t rb = (maxh + S1_ROWS_PER_CTA - 1) / S1_ROWS_PER_CTA;
  for (unsigned b = 0; b < rb * (uint32_t)n; ++b)
    cta(b, rb * (uint32_t)n, S1_NT, 0, rev,
        [&](uint8_t*) { s1_row_kernel(fr.data(), rb, d, colvals.data(), rowbits.data(), oob.data()); });
  for (unsigned b = 0; b < (unsigned)n; ++b)
    cta(b, (unsigned)n, S1_SCAN_NT, sizeof(S1ScanShared), rev, [&](uint8_t* smem) {
      s1_scan_body(fr.data(), d, rowbits.data(), oob.data(), lim.data(), res.data(),
                   *reinterpret_cast<S1ScanShared*>(smem));
    });
  for (unsigned b = 0; b < rb * (uint32_t)n; ++b)
    cta(b, rb * (uint32_t)n, S1_NT, 0, rev,
        [&](uint8_t*) { s1_store_kernel(fr.data(), rb, d, colvals.data(), lim.data(), out); });
  for (int i = 0; i < n; ++i) {
    results[2 * i] = res[(size_t)i].status;
    results[2 * i + 1] = res[(size_t)i].consumed;
  }
}
