// ljpeg_lane.cuh -- what the two one-thread-per-segment LJPEG kernels share (K2T, ljpeg_thread.cuh:
// clean data from the K2C pre-pass; K2S, ljpeg_stream.cuh: raw data, unstuffed by the thread):
// the per-thread ring geometry in shared memory and the decode of one difference.  Usable from
// nvcc and from the CPU replay (tests/emu/).
#pragma once

#ifdef RSB200_EMU
#include "ljpeg_types.h"
#else
#include "common.cuh"
#include "ljpeg_types.h"
#endif

namespace rsb200 {

constexpr int T_NT = 128;      // threads (= segments) per CTA
constexpr int T_MAXTAB = 4;    // plan tables staged in shared memory

// Per-thread ring of clean data in shared memory (word w of the stream at
// ring[w % T_RING][thread]: conflict free while the lanes of a warp are in step).  A warp runs
// 32 unrelated streams, and the scoreboard that guards a load's destination register
// is per WARP: a per-lane "load the next word when I cross into a new one" makes
// every lane wait for whatever load another lane issued a moment ago.  So global
// loads happen only at the start of a unit, the same instruction for all lanes,
// land in the ring at the end of that unit, and are first needed in the next one;
// inside a unit lanes only touch their ring.
constexpr int T_RING = 32;       // words per thread (8 blocks of 16 bytes)
constexpr uint32_t T_AHEAD = 96; // bytes kept requested ahead of the read position
constexpr uint32_t T_WSTRIDE = 4u * T_NT;             // bytes between consecutive words of a stream
constexpr uint32_t T_RMASK = T_RING * T_WSTRIDE - 1u; // ring size in bytes - 1

// symbols the LUT does not resolve (T.81 F.16 walk); .x = difference, .y = bits
// consumed | bad-code flag << 31
__device__ __noinline__ uint2 t_slow_symbol(const DevTable* t, uint32_t x) {
  const SymLen s = decode_sym(t, x);
  return make_uint2((uint32_t)sym_diff(s, x),
                    (uint32_t)s.total | (s.codelen == 0 ? 0x80000000u : 0u));
}

// The reference stops at the first unassigned code (RawDecoderException); the kernels decode on
// behind it (one bit per such code) and keep the bit position where the first one began, bad_at
// (T_NOBAD: none).  A code whose 16 bits lie wholly in the data is that verdict whatever follows.
// One that reaches behind the end may be made of bits that are not the stream's (the reference
// reads zeros there): then reading past the end decides, as for a segment without a bad code.
constexpr uint32_t T_NOBAD = 0xFFFFFFFFu;
__device__ __forceinline__ bool t_bad_in_data(uint32_t bad_at, uint32_t data_bits) {
  return bad_at != T_NOBAD && bad_at + 16u <= data_bits;
}

// One difference at bit p, the top of window x, with the LUT at shared address lutb (slow path:
// table t).  Same arithmetic as f_decode_diff.
__device__ __forceinline__ uint32_t t_decode_diff(const DevTable* t, uint32_t lutb, uint32_t x, uint32_t p,
                                                  uint32_t& tl, uint32_t& bad_at) {
  const uint32_t e =
      lds_u16<0>(mad_hi(x & ~((1u << (32 - LUT_BITS)) - 1u), 1u << (LUT_BITS + 1), lutb));
  tl = e >> 10;
  if (e == 0) { // code longer than the LUT, SSSS = 16, or corrupt
    const uint2 r = t_slow_symbol(t, x);
    tl = r.y & 0xFFu;
    if (r.y >> 31)
      bad_at = min(bad_at, p);
    return r.x;
  }
  const uint32_t tt = __funnelshift_l(0u, x, e);
  const uint32_t f = (uint32_t)((int32_t)~tt >> 31);
  return __funnelshift_l(tt, f, e >> 5) - f;
}

} // namespace rsb200
