// sraw.cuh -- K5: Canon sRaw chroma interpolation + YCbCr -> RGB (sm_90a).
// Reference: interpolators/Cr2sRawInterpolator.cpp (paths relative to
// /root/reference/src/librawspeed):
//   YCbCr::process (sign-extend by 16384, add hue)            :66-86
//   interpolate_422_row / interpolate_422                      :96-187
//   interpolate_420_row / interpolate_420 (edge rows/columns)  :189-453
//   YUV_TO_RGB<0|1|2>, STORE_RGB (clampBits(x >> 8, 16))       :455-497
//
// A pure streaming map (HBM bound): one thread = one MCU of the subsampled image
// (4:2:2: Y1 Y2 Cb Cr -> 2 RGB pixels; 4:2:0: Y1..Y4 Cb Cr -> 2x2 RGB pixels).
// The MCU and the chroma of its right / lower / lower-right neighbours are read
// as aligned 32-bit words (neighbouring threads read neighbouring words); each
// output row of the MCU is 12 bytes = three 32-bit stores.
#pragma once

#include "common.cuh"

namespace rsb200 {

struct SrawJobDev {
  uint64_t in_offset, out_offset;
  uint32_t in_pitch, out_pitch;
  uint32_t num_mcus, in_rows;
  int32_t k0, k1, k2, hue;
  uint32_t mcu_begin; // first global MCU of this job
  uint32_t pad;
};

constexpr int SRAW_NT = 256;

struct SrawC {
  int cb, cr;
};

__device__ __forceinline__ SrawC sraw_chroma(uint32_t w, int hue) {
  SrawC c;
  c.cb = (int)(w & 0xFFFFu) - 16384 + hue;
  c.cr = (int)(w >> 16) - 16384 + hue;
  return c;
}

__device__ __forceinline__ uint32_t sraw_clamp16(int x) {
  return (uint32_t)min(max(x, 0), 65535);
}

template <int VERSION>
__device__ __forceinline__ void sraw_rgb(int Y, SrawC c, int k0, int k1, int k2, uint32_t& r,
                                         uint32_t& g, uint32_t& b) {
  int ri, gi, bi;
  if (VERSION == 0) { // EOS 40D
    ri = k0 * (Y + c.cr - 512);
    gi = k1 * (Y + ((-778 * c.cb - (c.cr * 2048)) >> 12) - 512);
    bi = k2 * (Y + (c.cb - 512));
  } else if (VERSION == 1) {
    ri = k0 * (Y + ((50 * c.cb + 22929 * c.cr) >> 12));
    gi = k1 * (Y + ((-5640 * c.cb - 11751 * c.cr) >> 12));
    bi = k2 * (Y + ((29040 * c.cb - 101 * c.cr) >> 12));
  } else { // EOS 5D Mk III
    ri = k0 * (Y + c.cr);
    gi = k1 * (Y + ((-778 * c.cb - (c.cr * 2048)) >> 12));
    bi = k2 * (Y + c.cb);
  }
  r = sraw_clamp16(ri >> 8);
  g = sraw_clamp16(gi >> 8);
  b = sraw_clamp16(bi >> 8);
}

// two RGB pixels (6 uint16) -> three words
template <int VERSION>
__device__ __forceinline__ void sraw_store2(uint8_t* dst, int Ya, SrawC ca, int Yb, SrawC cb,
                                            const SrawJobDev& j) {
  uint32_t r0, g0, b0, r1, g1, b1;
  sraw_rgb<VERSION>(Ya, ca, j.k0, j.k1, j.k2, r0, g0, b0);
  sraw_rgb<VERSION>(Yb, cb, j.k0, j.k1, j.k2, r1, g1, b1);
  uint32_t* o = reinterpret_cast<uint32_t*>(dst);
  o[0] = r0 | (g0 << 16);
  o[1] = b0 | (r1 << 16);
  o[2] = g1 | (b1 << 16);
}

__device__ __forceinline__ SrawC sraw_avg2(SrawC a, SrawC b) {
  SrawC c;
  c.cb = (a.cb + b.cb) >> 1;
  c.cr = (a.cr + b.cr) >> 1;
  return c;
}

template <int VERSION, bool IS420>
__global__ void __launch_bounds__(SRAW_NT)
    sraw_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                const SrawJobDev* __restrict__ jobs, int njobs, uint32_t total_mcus) {
  const uint32_t gm = blockIdx.x * SRAW_NT + threadIdx.x;
  if (gm >= total_mcus)
    return;
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].mcu_begin <= gm)
      lo = mid;
    else
      hi = mid - 1;
  }
  const SrawJobDev j = jobs[lo];
  const uint32_t local = gm - j.mcu_begin;
  const uint32_t row = local / j.num_mcus, m = local - row * j.num_mcus;
  const bool lastCol = m + 1 == j.num_mcus;
  const uint32_t* r0 =
      reinterpret_cast<const uint32_t*>(in + j.in_offset + (uint64_t)row * j.in_pitch);
  if (!IS420) {
    // [Y1 Y2 | Cb Cr] = words 2m, 2m+1
    const uint32_t wy = __ldg(r0 + 2 * m);
    const SrawC c0 = sraw_chroma(__ldg(r0 + 2 * m + 1), j.hue);
    SrawC c1 = c0; // last pixel of the line keeps the previous chroma
    if (!lastCol)
      c1 = sraw_avg2(c0, sraw_chroma(__ldg(r0 + 2 * m + 3), j.hue));
    uint8_t* dst = out + j.out_offset + (uint64_t)row * j.out_pitch + 12ull * m;
    sraw_store2<VERSION>(dst, (int)(wy & 0xFFFFu), c0, (int)(wy >> 16), c1, j);
  } else {
    // [Y1 Y2 | Y3 Y4 | Cb Cr] = words 3m .. 3m+2
    const bool lastRow = row + 1 == j.in_rows;
    const uint32_t* r1 = reinterpret_cast<const uint32_t*>(
        reinterpret_cast<const uint8_t*>(r0) + j.in_pitch);
    const uint32_t wy0 = __ldg(r0 + 3 * m), wy1 = __ldg(r0 + 3 * m + 1);
    const SrawC c00 = sraw_chroma(__ldg(r0 + 3 * m + 2), j.hue);
    SrawC p01 = c00, p10 = c00, p11 = c00;
    if (!lastRow && !lastCol) {
      const SrawC c01 = sraw_chroma(__ldg(r0 + 3 * m + 5), j.hue);
      const SrawC c10 = sraw_chroma(__ldg(r1 + 3 * m + 2), j.hue);
      const SrawC c11 = sraw_chroma(__ldg(r1 + 3 * m + 5), j.hue);
      p01 = sraw_avg2(c00, c01);
      p10 = sraw_avg2(c00, c10);
      p11.cb = (c00.cb + c01.cb + c10.cb + c11.cb) >> 2;
      p11.cr = (c00.cr + c01.cr + c10.cr + c11.cr) >> 2;
    } else if (!lastRow) { // last MCU of the line
      p10 = sraw_avg2(c00, sraw_chroma(__ldg(r1 + 3 * m + 2), j.hue));
      p11 = p10;
    } else if (!lastCol) { // last line
      p01 = sraw_avg2(c00, sraw_chroma(__ldg(r0 + 3 * m + 5), j.hue));
      p11 = p01;
    }
    uint8_t* dst = out + j.out_offset + (uint64_t)(2 * row) * j.out_pitch + 12ull * m;
    sraw_store2<VERSION>(dst, (int)(wy0 & 0xFFFFu), c00, (int)(wy0 >> 16), p01, j);
    sraw_store2<VERSION>(dst + j.out_pitch, (int)(wy1 & 0xFFFFu), p10, (int)(wy1 >> 16), p11, j);
  }
}

} // namespace rsb200
