// lookup.cuh -- K12: 16-bit table lookup (curve, optionally dithered) of a whole image, in
// place (sm_90a).  Reference: RawImageDataU16::doLookup (common/RawImageDataU16.cpp:487-520);
// the per-lane arithmetic is in lookup_core.h (shared with the CPU replay in tests/emu).
//
// A streaming map, 2 B read + 2 B written per sample; the 128 KB (256 KB dithered) table is read
// through L1/L2.  Same decomposition as K9: one warp = four rows, a lane owns one aligned group
// of eight samples per row and iteration (4 x LDG.128 issued before the arithmetic), and jumps
// the 248 samples to its next group with one modular multiplication.
//
// Developed against a CPU replay of this loop (tests/test_lookup_emu.py); the plain lookup is
// bound by the table gather (one 2-byte load per sample) -- staging the 128 KB table in shared memory is the lever.
#pragma once

#include "common.cuh"
#include "lookup_core.h"
#include "scale.cuh" // scale_ld / scale_st, SCALE_ROWS

namespace rsb200 {

constexpr int LUT_WARPS = 8;
constexpr int LUT_NT = 32 * LUT_WARPS;

template <bool DITHER>
__global__ void __launch_bounds__(LUT_NT)
    lookup_kernel(uint8_t* __restrict__ img, const LookupJobDev* __restrict__ jobs, int njobs,
                  uint32_t total_quads, const uint16_t* __restrict__ tables, uint32_t nseg) {
  // a warp = four rows x one of nseg column segments (the dither generator can be started at any
  // sample, lut_mwc_state: rows need not be walked from their first sample; with
  // whole rows per warp a 45 MP frame leaves most warp slots of an SM empty)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t item = blockIdx.x * LUT_WARPS + warp;
  const uint32_t quad = item / nseg, seg = item - quad * nseg;
  if (quad >= total_quads)
    return;
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].quad_begin <= quad)
      lo = mid;
    else
      hi = mid - 1;
  }
  const LookupJobDev j = jobs[lo];
  const uint32_t y0 = (quad - j.quad_begin) * SCALE_ROWS;
  uint8_t* const base = img + j.offset + (uint64_t)y0 * j.pitch;
  const uint16_t* const table = tables + (size_t)j.table * (DITHER ? 131072u : 65536u);
  const uint32_t gps = (((j.ngroups + nseg - 1) / nseg) + 31u) & ~31u; // groups per segment
  const uint32_t g0 = seg * gps, g1 = min(g0 + gps, j.ngroups);
  if (g0 >= g1)
    return;
  const uint32_t iters = (g1 - g0 + 31) / 32;
  const uint32_t jump = DITHER ? lut_powmod(248u) : 0u;
  uint32_t st[SCALE_ROWS];
#pragma unroll
  for (int r = 0; r < SCALE_ROWS; ++r)
    st[r] = DITHER ? lut_mwc_state(j.width, y0 + r, 8u * (g0 + (uint32_t)lane)) : 0u;
  for (uint32_t it = 0; it < iters; ++it) {
    const uint32_t g = g0 + it * 32 + lane;
    if (g < g1) {
      ScaleVec v[SCALE_ROWS];
#pragma unroll
      for (int r = 0; r < SCALE_ROWS; ++r)
        if (y0 + r < j.height)
          v[r] = scale_ld(base + (uint64_t)r * j.pitch + (uint64_t)g * 16);
#pragma unroll
      for (int r = 0; r < SCALE_ROWS; ++r) {
        if (y0 + r < j.height) {
          const ScaleVec o = lut_group<DITHER>(v[r], table, j.ncols, 8u * g, st[r]);
          scale_st(base + (uint64_t)r * j.pitch + (uint64_t)g * 16, o);
          if (DITHER)
            st[r] = lut_mwc_jump(st[r], 248u, jump);
        }
      }
    }
  }
}

// ---- A/B candidate (RSB200_LUT_SMEM=1; plain lookup, plans with ONE table) -------------------
// With the table in global memory the random 2-byte table reads go through L1 one sector per lane.
// Here the 128 KB table is staged once per CTA in shared memory (opt-in dynamic size) and the
// CTAs are persistent (one per SM, 32 warps), walking the row quads with a grid stride.  Same
// per-lane arithmetic (lut_group<false>), not yet run on a GPU, hence not the default.
constexpr int LUT_SMEM_NT = 1024;
constexpr int LUT_SMEM_BYTES = 65536 * 2;

__global__ void __launch_bounds__(LUT_SMEM_NT, 1)
    lookup_smem_kernel(uint8_t* __restrict__ img, const LookupJobDev* __restrict__ jobs, int njobs,
                       uint32_t total_quads, const uint16_t* __restrict__ tables) {
  extern __shared__ __align__(16) uint8_t s_lut_raw[];
  uint16_t* const s_table = reinterpret_cast<uint16_t*>(s_lut_raw);
  {
    const uint4* src = reinterpret_cast<const uint4*>(tables);
    uint4* dst = reinterpret_cast<uint4*>(s_lut_raw);
    for (uint32_t i = threadIdx.x; i < LUT_SMEM_BYTES / 16; i += LUT_SMEM_NT)
      dst[i] = src[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t warps_per_cta = LUT_SMEM_NT / 32;
  for (uint32_t quad = blockIdx.x * warps_per_cta + warp; quad < total_quads;
       quad += gridDim.x * warps_per_cta) {
    int lo = 0, hi = njobs - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (jobs[mid].quad_begin <= quad)
        lo = mid;
      else
        hi = mid - 1;
    }
    const LookupJobDev j = jobs[lo];
    const uint32_t y0 = (quad - j.quad_begin) * SCALE_ROWS;
    uint8_t* const base = img + j.offset + (uint64_t)y0 * j.pitch;
    const uint32_t iters = (j.ngroups + 31) / 32;
    uint32_t unused = 0;
    for (uint32_t it = 0; it < iters; ++it) {
      const uint32_t g = it * 32 + lane;
      if (g < j.ngroups) {
        ScaleVec v[SCALE_ROWS];
#pragma unroll
        for (int r = 0; r < SCALE_ROWS; ++r)
          if (y0 + r < j.height)
            v[r] = scale_ld(base + (uint64_t)r * j.pitch + (uint64_t)g * 16);
#pragma unroll
        for (int r = 0; r < SCALE_ROWS; ++r)
          if (y0 + r < j.height)
            scale_st(base + (uint64_t)r * j.pitch + (uint64_t)g * 16,
                     lut_group<false>(v[r], s_table, j.ncols, 8u * g, unused));
      }
    }
  }
}

} // namespace rsb200
