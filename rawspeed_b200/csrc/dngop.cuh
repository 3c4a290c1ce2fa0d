// dngop.cuh -- K10: a DNG opcode list applied to a decoded image in ONE pass, in place (sm_90a).
// Reference: DngOpcodes::applyOpCodes (common/DngOpcodes.cpp:730-735), one pass over the image
// per opcode (:390-409); the per-sample arithmetic is in dngop_core.h (shared with the CPU
// replay in tests/emu).
//
// One thread = eight consecutive samples of a row (uint16: one LDG.128 / STG.128; float: two of
// each); the opcode list is walked once per thread with the samples in registers and the group
// is written back only if a sample changed.  2 (or 4) bytes read and at most as many written
// per sample regardless of the length of the list: HBM bound.  Lookup tables (128 KB each)
// and delta arrays stay in L2.
//
// Developed against a CPU replay of the thread program (tests/test_dngop_emu.py); issue bound
// (the per-sample lattice tests).
#pragma once

#include "common.cuh"
#include "dngop_core.h"

namespace rsb200 {

constexpr int DNGOP_NT = 256;
constexpr uint32_t DNGOP_BAD_CAP = 1u << 22; // positions kept per FixBadPixelsConstant and run

struct DngOpSinkDev {
  uint32_t* count;
  uint32_t* list;
  __device__ __forceinline__ void hit(uint32_t slot, uint32_t row, uint32_t col) {
    const uint32_t at = atomicAdd(count + slot, 1u);
    if (at < DNGOP_BAD_CAP)
      list[(uint64_t)slot * DNGOP_BAD_CAP + at] = (row << 16) | col;
  }
};

__global__ void __launch_bounds__(DNGOP_NT)
    dngop_kernel(uint8_t* __restrict__ img, const DngOpJobDev* __restrict__ jobs, int njobs,
                 uint32_t total_units, const DngOpDev* __restrict__ ops,
                 const uint16_t* __restrict__ tables, const uint32_t* __restrict__ deltas,
                 uint32_t* __restrict__ bad_count, uint32_t* __restrict__ bad_list) {
  const uint32_t u = blockIdx.x * DNGOP_NT + threadIdx.x;
  if (u >= total_units)
    return;
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].unit_begin <= u)
      lo = mid;
    else
      hi = mid - 1;
  }
  const DngOpJobDev jb = jobs[lo];
  const uint32_t ul = u - jb.unit_begin;
  const uint32_t r = jb.row0 + ul / jb.groups, g = ul % jb.groups;
  const uint32_t s0 = g * 8u;
  uint8_t* const rowp = img + jb.offset + (uint64_t)r * jb.pitch;
  uint32_t v[8], old[8];
  if (jb.is_f32) {
    // (rows are padded to 16 bytes = 4 floats: the second half of the last group may lie
    // beyond the row; samples past jb.samples are neither used nor written)
    const uint4 a = *reinterpret_cast<const uint4*>(rowp + (uint64_t)s0 * 4u);
    uint4 b = make_uint4(0u, 0u, 0u, 0u);
    const bool second = s0 + 4u < jb.samples;
    if (second)
      b = *reinterpret_cast<const uint4*>(rowp + (uint64_t)s0 * 4u + 16u);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    const uint4 a = *reinterpret_cast<const uint4*>(rowp + (uint64_t)s0 * 2u);
    v[0] = a.x & 0xFFFFu; v[1] = a.x >> 16; v[2] = a.y & 0xFFFFu; v[3] = a.y >> 16;
    v[4] = a.z & 0xFFFFu; v[5] = a.z >> 16; v[6] = a.w & 0xFFFFu; v[7] = a.w >> 16;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
    old[i] = v[i];
  DngOpSinkDev sink{bad_count, bad_list};
  dngop_apply_group(ops + jb.first_op, jb.num_ops, tables, deltas, jb, r, s0, v, sink);
  bool lo_changed = false, hi_changed = false;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    lo_changed |= v[i] != old[i];
    hi_changed |= v[i + 4] != old[i + 4];
  }
  if (jb.is_f32) {
    if (lo_changed)
      *reinterpret_cast<uint4*>(rowp + (uint64_t)s0 * 4u) = make_uint4(v[0], v[1], v[2], v[3]);
    if (hi_changed)
      *reinterpret_cast<uint4*>(rowp + (uint64_t)s0 * 4u + 16u) = make_uint4(v[4], v[5], v[6], v[7]);
  } else if (lo_changed || hi_changed) {
    *reinterpret_cast<uint4*>(rowp + (uint64_t)s0 * 2u) =
        make_uint4(v[0] | (v[1] << 16), v[2] | (v[3] << 16), v[4] | (v[5] << 16), v[6] | (v[7] << 16));
  }
}

} // namespace rsb200
