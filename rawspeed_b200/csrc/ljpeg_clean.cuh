// ljpeg_clean.cuh -- K2C: unstuffing pre-pass of the one-thread-per-segment LJPEG
// path (K2T, ljpeg_thread.cuh), sm_90a.
//
// One WARP per entropy-coded segment streams its raw bytes in pieces of 512 bytes
// (one coalesced 128-bit load per lane, the next piece already in flight) and
// applies the JPEG bit source's byte rules (BitStreamerJPEG.h:106-183 -- FF00 ->
// FF, the first FFxx ends the data, bytes past the buffer read as zero / do not
// exist).  It writes
//   * the clean data as big-endian 32-bit words (the serial decoders then need
//     no stuffing / marker / bounds logic at all), zero padded behind the end;
//   * one "anchor" per 256 raw bytes: the number of clean bytes that precede that
//     raw offset (lets a decoder map a clean offset back to a raw position for
//     `consumed`, the reference's BitStreamerJPEG::getStreamPosition());
//   * the clean length and whether an end marker was found.
// Everything is warp-synchronous: ballots / shuffles for the FF00 pairing across
// lanes, a shuffle prefix sum for the destination offsets, and a 132-word staging
// buffer in shared memory where lanes OR their (byte-shifted) 16 bytes together so
// that the global stores are whole, coalesced words.
#pragma once

#include "ljpeg.cuh"

namespace rsb200 {

// per thread-path segment, written by the host at plan creation
struct DevTScan {
  uint64_t clean_off;   // first word of this segment's clean data (in words, multiple of 4)
  uint32_t cap_words;   // words that may be read (data + zero padding)
  uint32_t anchor_off;  // first anchor of this segment
  uint32_t n_anchor;    // anchors (one per 256 raw bytes from the 16-byte aligned base)
  uint32_t pad;
};
// ... and by K2C
struct DevTInfo {
  uint32_t clean_len; // data bytes of the segment
  uint32_t marker;    // 1: an end marker was found; 0: the data ran to the end of the buffer
};

constexpr uint32_t T_ANCHOR_SHIFT = 8; // one anchor per 256 raw bytes
constexpr uint32_t T_PAD_WORDS = 8;    // zero words behind the data
constexpr int C_WARPS = 4;             // segments per CTA
constexpr int C_STAGE = 160;           // staging words per warp (3 + 512 bytes + padding, 5 x 32)

// bit i (0..3) = byte i of w is 0xFF / 0x00 (exact per byte: no carries between bytes)
__device__ __forceinline__ uint32_t c_ff_mask4(uint32_t w) {
  const uint32_t t = ((w & 0x7F7F7F7Fu) + 0x01010101u) & w & 0x80808080u; // bit 7 of each FF byte
  return ((t >> 7) * 0x00204081u) >> 21 & 0xFu;                            // gather bits 0,8,16,24
}
__device__ __forceinline__ uint32_t c_zero_mask4(uint32_t w) {
  const uint32_t t = ~(((w & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | w) & 0x80808080u; // bit 7 of each 00 byte
  return ((t >> 7) * 0x00204081u) >> 21 & 0xFu;
}
__device__ __forceinline__ uint32_t c_ff_mask16(const uint4& q) {
  return c_ff_mask4(q.x) | (c_ff_mask4(q.y) << 4) | (c_ff_mask4(q.z) << 8) | (c_ff_mask4(q.w) << 12);
}
__device__ __forceinline__ uint32_t c_zero_mask16(const uint4& q) {
  return c_zero_mask4(q.x) | (c_zero_mask4(q.y) << 4) | (c_zero_mask4(q.z) << 8) |
         (c_zero_mask4(q.w) << 12);
}

// remove byte i (0..15) of the little-endian 128-bit value q (upper bytes move down):
// word k keeps its bytes below i and takes the others one position up (byte permute
// over the pair (q[k], q[k+1]))
__device__ __forceinline__ void c_remove_byte(uint4& q, uint32_t i) {
  auto sel = [&](int k) -> uint32_t {
    // byte j of word k comes from position j (below the removed byte) or j + 1 (at / above
    // it): selector 0x3210 with 1 added to the nibbles j >= r, r = i - 4k clamped to 0..4
    const int r = min(max((int)i - 4 * k, 0), 4);
    return 0x3210u + (0x1111u & ((0xFFFFu << (4 * r)) & 0xFFFFu));
  };
  const uint32_t a = __byte_perm(q.x, q.y, sel(0)), b = __byte_perm(q.y, q.z, sel(1)),
                 c = __byte_perm(q.z, q.w, sel(2)), d = __byte_perm(q.w, 0u, sel(3));
  q = make_uint4(a, b, c, d);
}

__global__ void __launch_bounds__(32 * C_WARPS)
    k2_clean_kernel(const uint8_t* __restrict__ in, uint64_t in_total,
                    const DevScan* __restrict__ scans, const uint32_t* __restrict__ scan_ids,
                    uint32_t nids, const DevTScan* __restrict__ tscans,
                    uint32_t* __restrict__ clean, uint32_t* __restrict__ anchors,
                    DevTInfo* __restrict__ infos) {
  __shared__ uint32_t stage_all[C_WARPS][C_STAGE];
  const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  const uint32_t id = blockIdx.x * C_WARPS + wid;
  if (id >= nids)
    return;
  uint32_t* stage = stage_all[wid];
  const DevScan* scp = scans + scan_ids[id];
  const DevTScan ts = tscans[id];
  const uint64_t in_offset = scp->in_offset;
  const uint64_t abase = in_offset & ~15ull;
  const uint32_t skew = (uint32_t)(in_offset - abase);
  const uint32_t limit = skew + scp->in_size;
  const uint64_t readable = ((in_total + 15) & ~15ull) - abase;
  const uint4* blocks = reinterpret_cast<const uint4*>(in + abase);
  const uint32_t nblk = (uint32_t)min(readable >> 4, (uint64_t)0xFFFFFFFFu);
  uint32_t* cw = clean + ts.clean_off;
  uint32_t* anc = anchors + ts.anchor_off;
  const uint32_t npieces = (limit + 511u) >> 9;

  auto load = [&](uint32_t piece) {
    const uint32_t b = piece * 32u + lane;
    uint4 q = make_uint4(0, 0, 0, 0);
    if (piece < npieces && b < nblk)
      q = ldg_nc_v4(blocks + b);
    return q;
  };

  for (int i = lane; i < C_STAGE; i += 32)
    stage[i] = 0;
  __syncwarp();
  uint32_t co = 0;      // clean bytes produced so far
  uint32_t wout = 0;    // words written so far (co - wout*4 = bytes waiting in stage[0])
  uint32_t pff = 0;     // the last byte of the previous piece is a data FF
  uint32_t ended = 0, marker = 0;
  uint32_t piece = 0;
  // one piece: q = my 16 raw bytes, nq_first = first byte of the next piece
  auto step = [&](uint4 q, uint32_t nq_first) {
    const uint32_t raw0 = piece * 512u + lane * 16u; // raw offset of my first byte
    // bytes that belong to the segment: [skew, limit); bytes past the limit read as zero
    uint32_t lim = 0xFFFFu;
    if (raw0 + 16u > limit)
      lim = (raw0 >= limit) ? 0u : (0xFFFFu >> (16u - (limit - raw0)));
    uint32_t v = lim;
    if (raw0 < skew)
      v &= (skew - raw0 >= 16u) ? 0u : (0xFFFFu << (skew - raw0)) & 0xFFFFu;
    if (lim != 0xFFFFu) {
      auto bm = [&](uint32_t m4) {
        return ((m4 & 1u) ? 0xFFu : 0u) | ((m4 & 2u) ? 0xFF00u : 0u) |
               ((m4 & 4u) ? 0xFF0000u : 0u) | ((m4 & 8u) ? 0xFF000000u : 0u);
      };
      q.x &= bm(lim & 15u);
      q.y &= bm((lim >> 4) & 15u);
      q.z &= bm((lim >> 8) & 15u);
      q.w &= bm((lim >> 12) & 15u);
    }
    const uint32_t ffm = c_ff_mask16(q) & v;
    // (one ballot tells whether this piece needs any of the FF logic at all)
    const uint32_t any_ff = __ballot_sync(0xFFFFFFFFu, ffm != 0u);
    const uint32_t last_ff = __shfl_up_sync(0xFFFFFFFFu, ffm >> 15, 1);
    const uint32_t prev_ff = lane == 0 ? pff : last_ff;
    uint32_t stuff = 0, mk = 0;
    if (any_ff | pff) {
      const uint32_t zm = c_zero_mask16(q);
      // first byte of the next lane / next piece (past the limit: zero)
      uint32_t nb = __shfl_down_sync(0xFFFFFFFFu, q.x & 0xFFu, 1);
      if (lane == 31)
        nb = (raw0 + 16u < limit) ? nq_first : 0u;
      stuff = zm & ((ffm << 1) | prev_ff) & v;
      mk = ffm & ~((zm >> 1) | ((nb == 0u ? 1u : 0u) << 15));
    }
    // the first marker ends the data
    const uint32_t mk_lanes = __ballot_sync(0xFFFFFFFFu, mk != 0u);
    uint32_t emit = v & ~stuff;
    if (mk_lanes) {
      const uint32_t ml = __ffs(mk_lanes) - 1u;
      if (lane > ml)
        emit = 0;
      else if (lane == ml)
        emit &= (1u << (__ffs(mk) - 1u)) - 1u;
      ended = 1;
      marker = 1;
    }
    const uint32_t n = __popc(emit);
    uint32_t incl = n;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
      if (lane >= (uint32_t)d)
        incl += t;
    }
    const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
    const uint32_t dst = co + incl - n; // clean offset of my first byte
    if ((lane & 15u) == 0u) {
      const uint32_t a = raw0 >> T_ANCHOR_SHIFT;
      if (a < ts.n_anchor)
        anc[a] = dst;
    }
    // ---- my clean bytes, compacted to the low end of q (little endian) ----
    if (emit != 0xFFFFu) {
      uint32_t drop = ~emit & 0xFFFFu; // bytes that are not delivered
      // bytes above the highest delivered one just fall off the end (n says so);
      // remove the others from the top down so that positions stay valid
      const uint32_t top = emit ? 32u - __clz(emit) : 0u; // one past the highest delivered byte
      drop &= (1u << top) - 1u;
      while (drop) {
        const uint32_t i = 31u - __clz(drop);
        c_remove_byte(q, i);
        drop &= ~(1u << i);
      }
      // zero what lies behind the n delivered bytes (the staging buffer is OR-ed)
      auto keepn = [&](int k) {
        const int t = 8 * (int)n - 32 * k;
        uint32_t m = 0xFFFFFFFFu;
        asm("shl.b32 %0, %0, %1;" : "+r"(m) : "r"((uint32_t)max(t, 0)));
        return ~m;
      };
      q.x &= keepn(0);
      q.y &= keepn(1);
      q.z &= keepn(2);
      q.w &= keepn(3);
    }
    // ---- big-endian words, shifted to the byte position in the staging buffer ----
    {
      const uint32_t c0 = __byte_perm(q.x, 0, 0x0123), c1 = __byte_perm(q.y, 0, 0x0123),
                     c2 = __byte_perm(q.z, 0, 0x0123), c3 = __byte_perm(q.w, 0, 0x0123);
      const uint32_t so = dst - wout * 4u; // byte offset in the staging buffer
      const uint32_t sh = 8u * (so & 3u);
      uint32_t* s = stage + (so >> 2);
      if (n) {
        atomicOr(s + 0, c0 >> sh);
        atomicOr(s + 1, __funnelshift_r(c1, c0, sh));
        atomicOr(s + 2, __funnelshift_r(c2, c1, sh));
        atomicOr(s + 3, __funnelshift_r(c3, c2, sh));
        if (sh)
          atomicOr(s + 4, __funnelshift_r(0u, c3, sh));
      }
    }
    pff = __shfl_sync(0xFFFFFFFFu, (ffm >> 15) & 1u, 31);
    co += total;
    if ((piece + 1) * 512u >= limit)
      ended = 1;
    __syncwarp();
    // ---- whole words out; at the end also the partial word and the zero padding ----
    const uint32_t have = co - wout * 4u; // bytes in the staging buffer
    uint32_t nw = have >> 2;
    if (ended)
      nw = ((have + 3u) >> 2) + T_PAD_WORDS;
    const uint32_t part = (have & 3u) && !ended ? stage[have >> 2] : 0u; // carried to the next piece
    __syncwarp();
    {
      // (nw <= 129 + T_PAD_WORDS < C_STAGE = 5 x 32; the segment's capacity covers data + padding)
      uint32_t* cwp = cw + wout + lane;
#pragma unroll
      for (int it = 0; it < C_STAGE / 32; ++it) {
        const uint32_t i = lane + 32u * it;
        const uint32_t w = stage[i];
        stage[i] = (it == 0 && lane == 0) ? part : 0u; // clean again for the next piece
        if (i < nw)
          cwp[32 * it] = w;
      }
    }
    __syncwarp();
    wout += have >> 2;
    ++piece;
  };
  // Four pieces (2 KiB per warp) are requested together: the loads of a group are
  // in flight at once and none is pending across the loop edge.
  while (piece < npieces && !ended) {
    const uint32_t p0 = piece;
    const uint4 q0 = load(p0), q1 = load(p0 + 1), q2 = load(p0 + 2), q3 = load(p0 + 3);
    uint32_t f4 = 0; // first byte of the piece after the group
    if ((p0 + 4u) * 512u < limit)
      f4 = __ldg(in + abase + (uint64_t)(p0 + 4u) * 512u);
    const uint32_t f1 = __shfl_sync(0xFFFFFFFFu, q1.x & 0xFFu, 0);
    const uint32_t f2 = __shfl_sync(0xFFFFFFFFu, q2.x & 0xFFu, 0);
    const uint32_t f3 = __shfl_sync(0xFFFFFFFFu, q3.x & 0xFFu, 0);
    step(q0, f1);
    if (piece < npieces && !ended)
      step(q1, f2);
    if (piece < npieces && !ended)
      step(q2, f3);
    if (piece < npieces && !ended)
      step(q3, f4);
  }
  if (npieces == 0) // (empty segment: nothing but the zero padding)
    for (uint32_t i = lane; i < T_PAD_WORDS && i < ts.cap_words; i += 32)
      cw[i] = 0;
  // anchors of raw blocks behind the last processed piece (the data ended at a marker
  // before them): no clean offset maps there
  for (uint32_t a = ((piece * 512u) >> T_ANCHOR_SHIFT) + lane; a < ts.n_anchor; a += 32)
    anc[a] = 0xFFFFFFFFu;
  if (lane == 0) {
    infos[id].clean_len = co;
    infos[id].marker = marker;
  }
}

} // namespace rsb200
