// badpix.cuh -- K11: bad-pixel interpolation in place (sm_90a).
// Reference: RawImageData::fixBadPixels / fixBadPixelsThread (common/RawImage.cpp:231-239,
// :297-323) + RawImageDataU16::fixBadPixel (common/RawImageDataU16.cpp:399-485); the
// per-pixel arithmetic is in badpix_core.h (shared with the CPU replay in tests/emu).
//
// One thread = one bad pixel of the plan's de-duplicated list (built on the host from
// mBadPixelPositions, with the reference's (w + 15) / 32 block rule applied); the bitmap it
// consults is the reference's mBadPixelMap.  Work is proportional to the number of bad
// pixels, not to the image: a latency-bound scatter of a few thousand threads.
//
// Developed against a CPU replay of the thread program (tests/test_badpix_emu.py).
#pragma once

#include "badpix_core.h"
#include "common.cuh"

namespace rsb200 {

constexpr int BADPIX_NT = 128;

__global__ void __launch_bounds__(BADPIX_NT)
    badpix_kernel(uint8_t* __restrict__ img, const BadPixJobDev* __restrict__ jobs, int njobs,
                  const uint32_t* __restrict__ list, uint32_t total, const uint8_t* __restrict__ maps) {
  const uint32_t i = blockIdx.x * BADPIX_NT + threadIdx.x;
  if (i >= total)
    return;
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].first <= i)
      lo = mid;
    else
      hi = mid - 1;
  }
  const BadPixJobDev jb = jobs[lo];
  const uint32_t pos = list[i];
  const int x = (int)(pos & 0xFFFFu), y = (int)(pos >> 16);
  const uint32_t v = badpix_value(img, jb, maps + jb.map_offset, x, y);
  reinterpret_cast<uint16_t*>(img + jb.offset + (size_t)y * jb.pitch)[x] = (uint16_t)v;
}

} // namespace rsb200
