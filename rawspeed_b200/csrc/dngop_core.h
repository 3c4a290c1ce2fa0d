// dngop_core.h -- the per-thread program of K10 (fused DNG opcode pass), written so that the
// same source compiles as device code (dngop.cuh) and as plain C++ (tests/emu/dngop_emu.cpp).
//
// Reference: DngOpcodes::PixelOpcode::applyOP and the opcodes built on it
//   common/DngOpcodes.cpp:390-409 (lattice walk), LookupOpcode :417-438, OffsetPerRowOrCol
//   :591-623, ScalePerRowOrCol :625-662, FixBadPixelsConstant::apply :172-183.
//
// The reference makes one pass over the image per opcode.  Every opcode here is a map of one
// sample (its result depends on the sample's own value and position only), and opcodes are
// applied in list order, so the list can be evaluated per sample in registers: one read and
// one write of the image for the whole list.  A thread owns eight consecutive samples of a
// row and walks the opcode list once.
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define RSD_HD __host__ __device__ __forceinline__
#else
#define RSD_HD inline
#endif

namespace rsb200 {

enum : uint32_t {
  DNGOP_LOOKUP = 0,      // MapTable / MapPolynomial: v = table[v]
  DNGOP_OFFSET_ROW = 1,  // DeltaPerRow:    v = clamp16(delta[row index] + v)   | float: d + v
  DNGOP_OFFSET_COL = 2,  // DeltaPerColumn
  DNGOP_SCALE_ROW = 3,   // ScalePerRow:    v = clamp16((delta * v + 512) >> 10) | float: d * v
  DNGOP_SCALE_COL = 4,   // ScalePerColumn
  DNGOP_BAD_CONSTANT = 5 // FixBadPixelsConstant: report samples equal to `value`
};

struct DngOpDev {
  uint32_t kind;
  uint32_t top, left, bottom, right; // ROI in uncropped pixel coordinates
  uint32_t first_plane, planes;
  uint32_t row_pitch, col_pitch;
  uint32_t table; // LOOKUP: table index; OFFSET / SCALE: first element in `deltas`
  uint32_t value; // BAD_CONSTANT
  uint32_t slot;  // BAD_CONSTANT: index of its position list
};

struct DngOpJobDev {
  uint64_t offset;    // byte offset of row 0 of the uncropped image (multiple of 16)
  uint32_t pitch;     // bytes between rows (multiple of 16)
  uint32_t cpp;
  uint32_t is_f32;    // samples are floats (4 bytes) instead of uint16
  uint32_t row0;      // first / one-past-last row any opcode touches
  uint32_t row1;
  uint32_t groups;    // 8-sample groups per row = ceil(width * cpp / 8)
  uint32_t samples;   // width * cpp
  uint32_t first_op, num_ops;
  uint32_t unit_begin; // first (row, group) unit of this job
};

RSD_HD uint32_t dngop_clamp16(int32_t v) { return (uint32_t)(v < 0 ? 0 : (v > 65535 ? 65535 : v)); }

// v[8]: samples s0 .. s0+7 of row r (uint16 values, or float bit patterns); Sink::hit(slot,
// row, col) receives FixBadPixelsConstant matches.
template <class Sink>
RSD_HD void dngop_apply_group_v1(const DngOpDev* ops, uint32_t nops, const uint16_t* tables,
                              const uint32_t* deltas, const DngOpJobDev& jb, uint32_t r,
                              uint32_t s0, uint32_t (&v)[8], Sink& sink) {
  for (uint32_t k = 0; k < nops; ++k) {
    const DngOpDev op = ops[k];
    // row lattice: rows top, top + row_pitch, ... below bottom
    if (r < op.top || r >= op.bottom)
      continue;
    const uint32_t ry = r - op.top;
    const uint32_t yi = ry / op.row_pitch;
    if (yi * op.row_pitch != ry)
      continue;
    const bool by_row = op.kind == DNGOP_OFFSET_ROW || op.kind == DNGOP_SCALE_ROW;
    uint32_t col = s0 / jb.cpp, plane = s0 - col * jb.cpp;
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int i = 0; i < 8; ++i) {
      const bool in_planes = plane - op.first_plane < op.planes; // (unsigned wrap: plane >= first)
      if (s0 + i < jb.samples && in_planes && col >= op.left && col < op.right) {
        const uint32_t cx = col - op.left;
        const uint32_t xi = op.col_pitch == 1 ? cx : cx / op.col_pitch;
        if (xi * op.col_pitch == cx) {
          const uint32_t sel = by_row ? yi : xi;
          switch (op.kind) {
          case DNGOP_LOOKUP:
            v[i] = tables[(size_t)op.table * 65536u + v[i]];
            break;
          case DNGOP_OFFSET_ROW:
          case DNGOP_OFFSET_COL:
            if (jb.is_f32) {
              union { uint32_t u; float f; } a, d;
              a.u = v[i];
              d.u = deltas[op.table + sel];
              a.f = d.f + a.f;
              v[i] = a.u;
            } else {
              v[i] = dngop_clamp16((int32_t)deltas[op.table + sel] + (int32_t)v[i]);
            }
            break;
          case DNGOP_SCALE_ROW:
          case DNGOP_SCALE_COL:
            if (jb.is_f32) {
              union { uint32_t u; float f; } a, d;
              a.u = v[i];
              d.u = deltas[op.table + sel];
              a.f = d.f * a.f;
              v[i] = a.u;
            } else {
              v[i] = dngop_clamp16(((int32_t)deltas[op.table + sel] * (int32_t)v[i] + 512) >> 10);
            }
            break;
          default: // DNGOP_BAD_CONSTANT (uint16, cpp == 1: checked by the plan)
            if (v[i] == op.value)
              sink.hit(op.slot, r, col);
            break;
          }
        }
      }
      if (++plane == jb.cpp) {
        plane = 0;
        ++col;
      }
    }
  }
}

// ---- second version of the walk (the default; -DRSB200_DNGOP_V1 selects the first) ----
// The first version pays, per opcode and SAMPLE, a division by the run-time column pitch and a
// switch on the opcode kind.  Here the lattice position of the group's first column is computed
// once per opcode (one division) and stepped incrementally as the column advances, and the
// kind is dispatched once per opcode, outside the sample loop (the first version is issue bound).
template <class Sink>
RSD_HD void dngop_apply_group_v2(const DngOpDev* ops, uint32_t nops, const uint16_t* tables,
                                 const uint32_t* deltas, const DngOpJobDev& jb, uint32_t r,
                                 uint32_t s0, uint32_t (&v)[8], Sink& sink) {
  const uint32_t col0 = s0 / jb.cpp, plane0 = s0 - col0 * jb.cpp;
  const uint32_t nvalid = jb.samples - s0 < 8u ? jb.samples - s0 : 8u;
  for (uint32_t k = 0; k < nops; ++k) {
    const DngOpDev op = ops[k];
    if (r < op.top || r >= op.bottom)
      continue;
    const uint32_t ry = r - op.top;
    const uint32_t yi = op.row_pitch == 1 ? ry : ry / op.row_pitch;
    if (yi * op.row_pitch != ry)
      continue;
    // the group's columns: col0 .. col0 + 7 / cpp; nothing to do if they miss [left, right)
    if (col0 >= op.right || col0 + 8u <= op.left)
      continue;
    // lattice phase of col0 relative to `left`: d = col0 - left (may be negative),
    // xi = floor(d / pitch), rem = d mod pitch in [0, pitch)
    const int32_t d = (int32_t)col0 - (int32_t)op.left, pit = (int32_t)op.col_pitch;
    int32_t xi, rem;
    if (d >= 0) {
      xi = pit == 1 ? d : d / pit;
      rem = d - xi * pit;
    } else {
      const int32_t q = (-d + pit - 1) / pit; // ceil(-d / pit)
      xi = -q;
      rem = d + q * pit;
    }
    const bool by_row = op.kind == DNGOP_OFFSET_ROW || op.kind == DNGOP_SCALE_ROW;
    // which of the eight samples this opcode touches, and with which delta index
    uint32_t hit = 0;
    uint32_t col = col0, plane = plane0;
    int32_t sel[8];
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int i = 0; i < 8; ++i) {
      const bool in = (uint32_t)i < nvalid && rem == 0 && col >= op.left && col < op.right &&
                      plane - op.first_plane < op.planes;
      hit |= (in ? 1u : 0u) << i;
      sel[i] = by_row ? (int32_t)yi : xi;
      if (++plane == jb.cpp) {
        plane = 0;
        ++col;
        if (++rem == pit) {
          rem = 0;
          ++xi;
        }
      }
    }
    if (!hit)
      continue;
    if (op.kind == DNGOP_LOOKUP) {
      const uint16_t* t = tables + (size_t)op.table * 65536u;
#if defined(__CUDACC__)
#pragma unroll
#endif
      for (int i = 0; i < 8; ++i)
        if ((hit >> i) & 1u)
          v[i] = t[v[i]];
    } else if (op.kind == DNGOP_BAD_CONSTANT) {
#if defined(__CUDACC__)
#pragma unroll
#endif
      for (int i = 0; i < 8; ++i)
        if (((hit >> i) & 1u) && v[i] == op.value)
          sink.hit(op.slot, r, (s0 + (uint32_t)i) / jb.cpp);
    } else {
      const bool scale = op.kind == DNGOP_SCALE_ROW || op.kind == DNGOP_SCALE_COL;
      const uint32_t* dl = deltas + op.table;
#if defined(__CUDACC__)
#pragma unroll
#endif
      for (int i = 0; i < 8; ++i) {
        if (!((hit >> i) & 1u))
          continue;
        const uint32_t dv = dl[sel[i]];
        if (jb.is_f32) {
          union { uint32_t u; float f; } a, dd;
          a.u = v[i];
          dd.u = dv;
          a.f = scale ? dd.f * a.f : dd.f + a.f;
          v[i] = a.u;
        } else if (scale) {
          v[i] = dngop_clamp16(((int32_t)dv * (int32_t)v[i] + 512) >> 10);
        } else {
          v[i] = dngop_clamp16((int32_t)dv + (int32_t)v[i]);
        }
      }
    }
  }
}

// ---- third version of the walk: one sample per pixel (cpp = 1, every CFA image) ----
// The second version is issue bound at ~300 thread-instructions
// per opcode and group -- eight rounds of range / lattice / plane tests, eight delta indices, and
// twelve scalar loads of the opcode.  With one sample per pixel the eight samples of a group are
// eight consecutive columns, so the opcode's footprint in the group is a bit mask with a closed
// form: columns [lo, hi) of the group lie in [left, right), and inside that range every
// col_pitch-th one from the first lattice column on.  The mask is built once per opcode (no
// division for pitch 1, one otherwise), the delta index of a hit is the index of the first hit
// plus the number of hits before it, and the opcode is read with three 128-bit loads.

template <class Sink>
RSD_HD void dngop_apply_group_v3(const DngOpDev* ops, uint32_t nops, const uint16_t* tables,
                                 const uint32_t* deltas, const DngOpJobDev& jb, uint32_t r,
                                 uint32_t s0, uint32_t (&v)[8], Sink& sink) {
  const uint32_t col0 = s0; // cpp == 1
  const uint32_t nvalid = jb.samples - s0 < 8u ? jb.samples - s0 : 8u;
  for (uint32_t k = 0; k < nops; ++k) {
    DngOpDev op;
#if defined(__CUDA_ARCH__)
    {
      static_assert(sizeof(DngOpDev) == 48, "three 16-byte loads");
      const uint4* q = reinterpret_cast<const uint4*>(ops + k); // (the array is 16-byte aligned: plan allocation)
      const uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2);
      op.kind = a.x; op.top = a.y; op.left = a.z; op.bottom = a.w;
      op.right = b.x; op.first_plane = b.y; op.planes = b.z; op.row_pitch = b.w;
      op.col_pitch = c.x; op.table = c.y; op.value = c.z; op.slot = c.w;
    }
#else
    op = ops[k];
#endif
    if (r < op.top || r >= op.bottom || op.first_plane != 0u || op.planes == 0u)
      continue; // (plane 0 is the only plane)
    const uint32_t ry = r - op.top;
    const uint32_t yi = op.row_pitch == 1 ? ry : ry / op.row_pitch;
    if (yi * op.row_pitch != ry)
      continue;
    // samples [lo, hi) of the group lie in [left, right)
    const uint32_t lo = op.left > col0 ? op.left - col0 : 0u;
    uint32_t hi = op.right > col0 ? op.right - col0 : 0u;
    hi = hi < nvalid ? hi : nvalid;
    if (lo >= hi)
      continue;
    // first lattice column at or behind col0 + lo, its index on the lattice
    const uint32_t pit = op.col_pitch;
    const uint32_t d = col0 + lo - op.left;
    uint32_t xi0 = d, i0 = lo, hit;
    if (pit == 1u) {
      hit = ((1u << hi) - 1u) & ~((1u << lo) - 1u);
    } else {
      xi0 = d / pit;
      const uint32_t rem = d - xi0 * pit;
      if (rem) {
        i0 += pit - rem;
        ++xi0;
      }
      hit = 0;
      for (uint32_t i = i0; i < hi; i += pit)
        hit |= 1u << i;
      if (!hit)
        continue;
    }
    if (op.kind == DNGOP_LOOKUP) {
      const uint16_t* t = tables + (size_t)op.table * 65536u;
#if defined(__CUDACC__)
#pragma unroll
#endif
      for (int i = 0; i < 8; ++i)
        if ((hit >> i) & 1u)
          v[i] = t[v[i]];
    } else if (op.kind == DNGOP_BAD_CONSTANT) {
#if defined(__CUDACC__)
#pragma unroll
#endif
      for (int i = 0; i < 8; ++i)
        if (((hit >> i) & 1u) && v[i] == op.value)
          sink.hit(op.slot, r, s0 + (uint32_t)i);
    } else {
      const bool by_row = op.kind == DNGOP_OFFSET_ROW || op.kind == DNGOP_SCALE_ROW;
      const bool scale = op.kind == DNGOP_SCALE_ROW || op.kind == DNGOP_SCALE_COL;
      const uint32_t* dl = deltas + op.table + (by_row ? yi : xi0);
      const uint32_t row_dv = dl[0]; // a row delta is the same for every hit
      uint32_t nth = 0;              // hits before sample i: the column delta of a hit is dl[nth]
#if defined(__CUDACC__)
#pragma unroll
#endif
      for (int i = 0; i < 8; ++i) {
        if (!((hit >> i) & 1u))
          continue;
        const uint32_t dv = by_row ? row_dv : dl[nth];
        ++nth;
        if (jb.is_f32) {
          union { uint32_t u; float f; } a, dd;
          a.u = v[i];
          dd.u = dv;
          a.f = scale ? dd.f * a.f : dd.f + a.f;
          v[i] = a.u;
        } else if (scale) {
          v[i] = dngop_clamp16(((int32_t)dv * (int32_t)v[i] + 512) >> 10);
        } else {
          v[i] = dngop_clamp16((int32_t)dv + (int32_t)v[i]);
        }
      }
    }
  }
}

// the walk the kernel (and its CPU replay) uses
template <class Sink>
RSD_HD void dngop_apply_group(const DngOpDev* ops, uint32_t nops, const uint16_t* tables,
                              const uint32_t* deltas, const DngOpJobDev& jb, uint32_t r,
                              uint32_t s0, uint32_t (&v)[8], Sink& sink) {
#if defined(RSB200_DNGOP_V1)
  dngop_apply_group_v1(ops, nops, tables, deltas, jb, r, s0, v, sink);
#elif defined(RSB200_DNGOP_V2)
  dngop_apply_group_v2(ops, nops, tables, deltas, jb, r, s0, v, sink);
#else
  if (jb.cpp == 1u)
    dngop_apply_group_v3(ops, nops, tables, deltas, jb, r, s0, v, sink);
  else
    dngop_apply_group_v2(ops, nops, tables, deltas, jb, r, s0, v, sink);
#endif
}

} // namespace rsb200
