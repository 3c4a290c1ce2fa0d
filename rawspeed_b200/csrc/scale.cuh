// scale.cuh -- K9: black/white level scaling of a decoded uint16 image, in place (sm_90a).
// Reference: RawImageDataU16::scaleValues (common/RawImageDataU16.cpp:185-399); the
// per-lane arithmetic is in scale_core.h (shared with the CPU replay in tests/emu).
//
// A streaming map: 2 B read + 2 B written per sample (HBM bound).  One warp = one quad of
// four crop rows; per iteration it moves 4 x 512 B (one LDG.128 / STG.128 per lane and
// row, the four loads issued before any arithmetic).  The dither of the SSE2 semantics is
// sequential along a row, so every iteration starts with the 32 lanes advancing the 4 x 8
// generators of the quad by 32 steps into the warp's private 1 KB of shared memory.
//
// Developed against a CPU replay of this loop (tests/test_scale_emu.py).
#pragma once

#include "common.cuh"
#include "scale_core.h"

namespace rsb200 {

constexpr int SCALE_WARPS = 8; // warps per CTA
constexpr int SCALE_NT = 32 * SCALE_WARPS;

__device__ __forceinline__ ScaleVec scale_ld(const uint8_t* p) {
  const uint4 v = *reinterpret_cast<const uint4*>(p);
  ScaleVec r;
  r.w[0] = v.x;
  r.w[1] = v.y;
  r.w[2] = v.z;
  r.w[3] = v.w;
  return r;
}
__device__ __forceinline__ void scale_st(uint8_t* p, const ScaleVec& v) {
  stg_cs_v4(p, make_uint4(v.w[0], v.w[1], v.w[2], v.w[3]));
}

// job of global row quad `quad` (jobs sorted by quad_begin)
__device__ __forceinline__ int scale_find_job(const ScaleJobDev* jobs, int njobs, uint32_t quad) {
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].quad_begin <= quad)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}

// MODE 0: scaleValues_SSE2 semantics, MODE 1: scaleValues_plain semantics
template <int MODE>
__global__ void __launch_bounds__(SCALE_NT)
    scale_kernel(uint8_t* __restrict__ img, const ScaleJobDev* __restrict__ jobs, int njobs,
                 uint32_t total_quads, uint32_t nseg) {
  // MODE 1: a warp = four rows x one of nseg column segments (the plain loop's generator can be
  // started at any sample, scale_mwc_state); MODE 0: nseg = 1 (the SSE2 loop's 16-bit generator
  // has no jump, a row is walked from its first sample)
  __shared__ __align__(16) uint8_t s_rnd[MODE == 0 ? SCALE_WARPS : 1][SCALE_ROWS * SCALE_RND_STRIDE];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t item = blockIdx.x * SCALE_WARPS + warp;
  const uint32_t quad = MODE == 0 ? item : item / nseg, seg = MODE == 0 ? 0u : item - quad * nseg;
  if (quad >= total_quads)
    return;
  const ScaleJobDev j = jobs[scale_find_job(jobs, njobs, quad)];
  const uint32_t y0 = (quad - j.quad_begin) * SCALE_ROWS;
  uint8_t* const base = img + j.offset + (uint64_t)(j.off_y + y0) * j.pitch + (uint64_t)j.group0 * 16;
  const uint32_t gps = MODE == 0 ? j.ngroups : ((((j.ngroups + nseg - 1) / nseg) + 31u) & ~31u);
  const uint32_t g0 = seg * gps, g1 = min(g0 + gps, j.ngroups);
  if (g0 >= g1)
    return;
  const uint32_t iters = (g1 - g0 + 31) / 32;

  if (MODE == 0) {
    uint8_t* const rnd = s_rnd[MODE == 0 ? warp : 0];
    int32_t state = j.dither ? scale_sse2_seed(j.crop_w, y0 + (lane >> 3), lane & 7) : 0;
    for (uint32_t it = 0; it < iters; ++it) {
      if (j.dither) {
        scale_sse2_advance(state, lane, rnd);
        __syncwarp();
      }
      const uint32_t g = it * 32 + lane;
      if (g < j.ngroups) {
        ScaleVec v[SCALE_ROWS];
#pragma unroll
        for (int r = 0; r < SCALE_ROWS; ++r)
          if (y0 + r < j.crop_h)
            v[r] = scale_ld(base + (uint64_t)r * j.pitch + (uint64_t)g * 16);
#pragma unroll
        for (int r = 0; r < SCALE_ROWS; ++r) {
          if (y0 + r < j.crop_h) {
            uint2 rb = make_uint2(0u, 0u);
            if (j.dither)
              rb = *reinterpret_cast<const uint2*>(rnd + r * SCALE_RND_STRIDE + lane * 8);
            const ScaleVec o = scale_sse2_group(v[r], j, (j.off_y + y0 + r) & 1u, rb.x, rb.y);
            scale_st(base + (uint64_t)r * j.pitch + (uint64_t)g * 16, o);
          }
        }
      }
      if (j.dither)
        __syncwarp();
    }
  } else {
    // state before the first sample of this lane's first group, per row; the jump from the end
    // of one group to the start of the lane's next one is 31 groups = 248 samples
    const uint32_t jump = scale_powmod(248u);
    const int32_t x_first = (int32_t)(8u * (g0 + (uint32_t)lane)) - (int32_t)j.skip;
    uint32_t st[SCALE_ROWS];
#pragma unroll
    for (int r = 0; r < SCALE_ROWS; ++r)
      st[r] = j.dither ? scale_mwc_state(j.crop_w, y0 + r, (uint32_t)max(x_first, 0)) : 0u;
    for (uint32_t it = 0; it < iters; ++it) {
      const uint32_t g = g0 + it * 32 + lane;
      if (g < g1) {
        ScaleVec v[SCALE_ROWS];
#pragma unroll
        for (int r = 0; r < SCALE_ROWS; ++r)
          if (y0 + r < j.crop_h)
            v[r] = scale_ld(base + (uint64_t)r * j.pitch + (uint64_t)g * 16);
        const int32_t x0 = (int32_t)(8u * g) - (int32_t)j.skip;
#pragma unroll
        for (int r = 0; r < SCALE_ROWS; ++r) {
          if (y0 + r < j.crop_h) {
            const ScaleVec o = scale_plain_group(v[r], j, y0 + r, x0, st[r]);
            scale_st(base + (uint64_t)r * j.pitch + (uint64_t)g * 16, o);
            if (j.dither)
              st[r] = scale_mwc_jump(st[r], 248u, jump);
          }
        }
      }
    }
  }
}

} // namespace rsb200
