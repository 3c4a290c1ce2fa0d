// ljpeg_stream.cuh -- K2S: LJPEG tile decode for LARGE batches, one THREAD per entropy-coded
// segment, reading the RAW bytes (no unstuffing pre-pass), sm_90a.
//
// Same results as k2_thread_kernel / k2_fused_kernel (reference: PrefixCodeLUTDecoder.h:172-216,
// AbstractPrefixCodeDecoder.h:43-76, LJpegDecompressor.cpp:184-339; the byte rules of the bit
// source: BitStreamerJPEG.h:106-183).
//
// K2T (ljpeg_thread.cuh) needs a cooperative pre-pass (K2C) that writes an unstuffed copy of
// every segment: ~15 thread-instructions per byte for the cross-lane compaction, 27 % of the
// 256-frame step, plus 1 B/px written and read again.  A thread that walks its own stream can
// drop the stuffed zeros with a running write pointer instead -- ~22 instructions per 32-bit
// word, branch free:
//   * FF flags of the word (bit 7 of every FF byte), shifted by one byte (the flag of the last
//     byte of the previous word carried in) = the bytes to remove;
//   * a 16-entry table gives the PRMT selector that packs the kept bytes big-endian and
//     their number; the packed bytes are appended to a left-aligned accumulator and whole
//     words go to the thread's ring in shared memory (the ring K2T already reads from);
//   * a removed byte that is not 00 is a marker: rare, found afterwards (the OR of the removed
//     bytes of a 16-byte block is tested once), handled bytewise by a function off the hot path;
//     so are the first block (bytes before the segment), the block that holds the end of the
//     buffer, and everything behind the end (zero data, like the reference).
// This work is independent of the symbol chain (window -> LUT -> length -> window), so it issues
// in the slots the chain leaves empty.
//
// A warp runs 32 streams at different byte rates; a fill step costs the warp the same whether
// 1 or 32 lanes take part.  Lanes therefore fill TOGETHER: when any lane of the warp runs low,
// every lane that has room in its ring takes a block in that step, and the steps a warp
// executes follow its fastest lane instead of the sum of everybody's thresholds.
//
// `consumed` (BitStreamerJPEG::getStreamPosition()) needs the raw offset of a clean byte
// count: found from the fill position by walking back over whole blocks (stuffed zeros are the
// 00 bytes behind an FF) and forward bytewise, once per segment.
#pragma once

#include "ljpeg_lane.cuh"

namespace rsb200 {

constexpr uint32_t S_OPEN = 0x1FFFFFFFu; // clean_len while the end of the data has not been seen
constexpr uint32_t S_MIN = 44;   // whole clean words (bytes) that a unit needs ahead of its first bit
constexpr uint32_t S_LOW = 64;   // a lane below this asks the warp for a fill step
constexpr uint32_t S_ROOM = 88;  // a lane at or below this takes part: two blocks (ring: 128 bytes; see s_ring_note)
// idx*4 of the 4 "remove" flags (bits 7, 15, 23, 31) in bits 2..5 of the high product word
constexpr uint32_t S_IDXMUL = (1u << 27) | (1u << 20) | (1u << 13) | (1u << 6);

#ifndef RSB200_S_LUT32
#define RSB200_S_LUT32 0 // 32-bit LUT entries laid out for IMAD.HI field extraction (A/B)
#endif

#ifndef RSB200_S_LB
#define RSB200_S_LB 6 // CTAs per SM the kernel is compiled for (__launch_bounds__)
#endif

struct StreamShared {
  uint32_t sel[16];            // [remove flags of a word] -> PRMT selector | 8 * kept bytes << 16
  uint32_t endinfo[2][T_NT];   // per thread: block where the data ended, clean bytes before that block
  uint32_t ring[T_RING][T_NT]; // word w of a stream at ring[w % T_RING][thread]
  DevTable tab[T_MAXTAB];
  // (RSB200_S_LUT32: behind the tables in use, uint32_t lut32[ntab][1 << LUT_BITS])
  // (where it fits, behind those: the output stage, S_STAGE bytes per thread, see s_flush)
};

// Output staged per thread: 4 units = 32 samples = 64 bytes, which leave together as two whole sectors.
constexpr uint32_t S_STAGE = 64;
constexpr uint32_t H100_SMEM_PER_SM = 228u << 10;  // shared memory of an SM
constexpr uint32_t H100_SMEM_PER_CTA_RESERVED = 1u << 10; // of it, reserved by the system per CTA

// shared memory in front of the output stage: ring, tables (and the 32-bit LUTs)
__host__ __device__ inline size_t stream_stage_offset(int ntab) {
  return sizeof(uint32_t) * (16 + 2 * T_NT + T_RING * T_NT) + sizeof(DevTable) * (size_t)ntab +
         (RSB200_S_LUT32 ? sizeof(uint32_t) * (size_t)ntab * (1u << LUT_BITS) : 0);
}
// The stage is there only when RSB200_S_LB CTAs with it still fit an SM (one or two tables); with more
// tables a lane stores its units directly.
__host__ __device__ inline bool stream_staged(int ntab) {
  return (stream_stage_offset(ntab) + S_STAGE * T_NT + H100_SMEM_PER_CTA_RESERVED) * RSB200_S_LB <=
         H100_SMEM_PER_SM;
}
__host__ __device__ inline size_t stream_smem_bytes(int ntab) {
  return stream_stage_offset(ntab) + (stream_staged(ntab) ? S_STAGE * T_NT : 0);
}
// LUT entry for the straight-line decode: [4:0] code length, [12:8] SSSS, bit 16 = 1 (a hit; eight
// of them add up in a counter without touching the other fields' sums), [31:26] bits of code +
// mantissa.  The fields a symbol needs come out with IMAD.HI (FMA pipe): e >> 8 as a shift amount
// (SHF takes it modulo 32), p + (e >> 26).
__host__ __device__ inline uint32_t s_lut32_entry(uint32_t e16) {
  return e16 ? ((e16 & 31u) | (((e16 >> 5) & 31u) << 8) | (1u << 16) | ((e16 >> 10) << 26)) : 0u;
}

// entry of the selector table for remove-mask m (bit i = byte i of the little-endian word, i.e.
// the i-th byte of the stream, is dropped): kept bytes in stream order from the top byte down
__host__ __device__ inline uint32_t s_sel_entry(uint32_t m) {
  uint32_t sel = 0, k = 0;
  for (uint32_t i = 0; i < 4; ++i)
    if (!(m & (1u << i))) {
      sel |= i << (4 * (3 - k));
      ++k;
    }
  for (uint32_t j = k; j < 4; ++j)
    sel |= 4u << (4 * (3 - j)); // a byte of the zero operand
  return sel | ((8u * k) << 16);
}

// the unstuffer of one thread (registers)
struct SFill {
  uint32_t acc;       // clean bytes not yet in the ring, left aligned
  uint32_t sh;        // 8 * their number (0, 8, 16, 24)
  uint32_t wo;        // T_WSTRIDE * whole words stored so far (ring byte offset, unwrapped)
  uint32_t pffm;      // FF flags of the previous raw word (bit 31: the byte before the next word is FF)
  uint32_t nblk;      // next raw block (16 bytes, from the aligned base of the segment)
  uint32_t slow_from; // blocks >= this go the bytewise way (end of the buffer; 0 once the data ended)
  uint32_t clean_len; // data bytes of the segment once its end (marker / buffer) was seen, else S_OPEN
};

__device__ __forceinline__ uint32_t s_clean_count(const SFill& f) { return (f.wo >> 7) + (f.sh >> 3); }
static_assert(T_WSTRIDE == 512, "s_clean_count: wo / T_WSTRIDE * 4");

__device__ __forceinline__ void s_put_byte(SFill& f, uint32_t ringb, uint32_t b) {
  f.acc |= b << (24u - f.sh);
  f.sh += 8u;
  if (f.sh == 32u) {
    sts_u32<0>(ringb + (f.wo & T_RMASK), f.acc);
    f.wo += T_WSTRIDE;
    f.acc = 0;
    f.sh = 0;
  }
}

// Once the data has ended, the ring bytes from data byte `clean_len` on become zero data, as the
// reference reads them: the fast way puts a whole block into the ring, the bytes behind a marker too,
// and the bytewise way has put the FF of a marker in as a data byte.
// Otherwise a code that starts before the marker and reaches behind it could decode as unassigned
// without its bits counting as missing.
__device__ __noinline__ SFill s_zero_behind(SFill f, uint32_t ringb, uint32_t clean_len) {
  const uint32_t stored = f.wo >> 7; // bytes in whole ring words
  if (clean_len < stored) {
#pragma unroll 1
    for (uint32_t w = clean_len >> 2; w < (stored >> 2); ++w) {
      const uint32_t keep = w == (clean_len >> 2) ? (clean_len & 3u) : 0u; // data bytes of the word
      const uint32_t a = ringb + ((w * T_WSTRIDE) & T_RMASK);
      sts_u32<0>(a, keep ? lds_u32<0>(a) & (~0u << (32u - 8u * keep)) : 0u);
    }
    f.acc = 0;
  } else {
    const uint32_t keep = clean_len - stored; // data bytes of the accumulator (left aligned)
    f.acc = keep ? f.acc & (~0u << (32u - 8u * keep)) : 0u;
  }
  return f;
}

// One block the bytewise way: block 0 (the bytes before `skew` are not the segment's), the block
// that holds raw offset `limit` (end of the buffer: what lies behind reads as zero data) and all
// blocks once the data has ended.  The first marker ends the data (the FF before it was appended
// as a data byte and is taken back from the count).
__device__ __noinline__ SFill s_slow_block(SFill f, uint32_t ringb, uint32_t einfo, uint4 q,
                                           uint32_t blk, uint32_t skew, uint32_t limit) {
  if (f.clean_len != S_OPEN) { // behind the end: 16 zero bytes
#pragma unroll 1
    for (int k = 0; k < 4; ++k) {
      sts_u32<0>(ringb + (f.wo & T_RMASK), f.acc);
      f.wo += T_WSTRIDE;
      f.acc = 0;
    }
    return f;
  }
  const uint32_t cc0 = s_clean_count(f);
  bool carry = (f.pffm >> 31) != 0u;
#pragma unroll 1
  for (uint32_t i = 0; i < 16; ++i) {
    const uint32_t raw = 16u * blk + i;
    if (raw < skew)
      continue;
    const uint32_t w = i < 4 ? q.x : (i < 8 ? q.y : (i < 12 ? q.z : q.w));
    uint32_t b = (w >> (8u * (i & 3u))) & 0xFFu;
    if (f.clean_len == S_OPEN) {
      if (raw >= limit) {
        f.clean_len = s_clean_count(f);
      } else if (carry) {
        carry = false;
        if (b == 0u)
          continue; // stuffing
        f.clean_len = s_clean_count(f) - 1u; // marker
      } else {
        carry = b == 0xFFu;
      }
    }
    if (f.clean_len != S_OPEN)
      b = 0;
    s_put_byte(f, ringb, b);
  }
  f.pffm = carry ? 0x80000000u : 0u;
  if (f.clean_len != S_OPEN) {
    f = s_zero_behind(f, ringb, f.clean_len); // (the FF of a marker went in as a data byte)
    f.slow_from = 0;
    f.pffm = 0;
    sts_u32<0>(einfo, blk);
    sts_u32<(int)(4 * T_NT)>(einfo, cc0);
  }
  return f;
}

// After a fast block whose removed bytes were not all zero: the marker's second byte lies in
// block `blk` (>= 1, wholly inside the segment).  .x = data bytes before the marker, .y = clean
// bytes counted before the block (cc_end counts every byte that does not follow an FF).
__device__ __noinline__ uint2 s_find_marker(const uint8_t* __restrict__ gbase, uint32_t blk,
                                            uint32_t cc_end, uint32_t skew) {
  const uint8_t* bp = gbase + 16ull * blk;
  const bool carry0 = (16u * blk - 1u) >= skew && __ldg(bp - 1) == 0xFFu;
  uint32_t kept = 0;
  {
    bool c = carry0;
#pragma unroll 1
    for (int i = 0; i < 16; ++i) {
      const uint32_t b = __ldg(bp + i);
      kept += c ? 0u : 1u;
      c = b == 0xFFu;
    }
  }
  const uint32_t cc0 = cc_end - kept;
  uint32_t c = cc0;
  bool carry = carry0;
#pragma unroll 1
  for (int i = 0; i < 16; ++i) {
    const uint32_t b = __ldg(bp + i);
    if (carry) {
      carry = false;
      if (b == 0u)
        continue;
      return make_uint2(c - 1u, cc0);
    }
    ++c;
    carry = b == 0xFFu;
  }
  return make_uint2(c, cc0); // (not reached: the caller saw a non-zero removed byte)
}

// multipliers ptxas cannot see (constant bank): see RSB200_S_PIPE below
#ifdef RSB200_EMU
static const uint32_t s_pipe_k[4] = {2u, 1u, 1u << 22, 1u << 27};
__device__ __forceinline__ uint32_t s_mad_lo(uint32_t a, uint32_t b, uint32_t c) { return a * b + c; }
#else
__constant__ uint32_t s_pipe_k[4] = {2u, 1u, 1u << 22, 1u << 27};
__device__ __forceinline__ uint32_t s_mad_lo(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t r;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
  return r;
}
#endif

// One block the fast way (4 words); returns the OR of the removed bytes (non-zero: a marker).
// RSB200_S_FILL2 (A/B): the add of the FF test on the FMA pipe, and the byte count of the
// accumulator kept unwrapped inside the block (the shifts take it modulo 32 by themselves, "a word is
// full" is a change of bit 5) and wrapped once at the end.
#ifndef RSB200_S_FILL2
#define RSB200_S_FILL2 0
#endif
__device__ __forceinline__ uint32_t s_fast_block(SFill& f, uint32_t ringb, uint32_t selb, const uint4& q) {
  uint32_t chk = 0;
#if RSB200_S_FILL2
  uint32_t u = f.sh;
#define S_WORD(w)                                                                        \
  do {                                                                                   \
    const uint32_t ffm_ = s_mad_lo((w) & 0x7F7F7F7Fu, s_pipe_k[1], 0x01010101u) & (w) & 0x80808080u; \
    const uint32_t rem_ = __funnelshift_l(f.pffm, ffm_, 8);                              \
    f.pffm = ffm_;                                                                       \
    chk |= (w) & prmt(rem_, 0u, 0xBA98u); /* sign replication: FF where a flag is */     \
    const uint32_t e_ = lds_u32<0>((mad_hi(rem_, S_IDXMUL, 0u) & 0x3Cu) | selb);         \
    const uint32_t out_ = prmt((w), 0u, e_);                                             \
    const uint32_t hi_ = f.acc | __funnelshift_r(out_, 0u, u);                           \
    const uint32_t lo_ = __funnelshift_r(0u, out_, u);                                   \
    const uint32_t tot_ = u + (e_ >> 16);                                                \
    if ((tot_ ^ u) & 32u) {                                                              \
      sts_u32<0>(ringb + (f.wo & T_RMASK), hi_);                                         \
      f.wo += T_WSTRIDE;                                                                 \
      f.acc = lo_;                                                                       \
    } else {                                                                             \
      f.acc = hi_;                                                                       \
    }                                                                                    \
    u = tot_;                                                                            \
  } while (0)
#else
#define S_WORD(w)                                                                        \
  do {                                                                                   \
    const uint32_t ffm_ = (((w) & 0x7F7F7F7Fu) + 0x01010101u) & (w) & 0x80808080u;       \
    const uint32_t rem_ = __funnelshift_l(f.pffm, ffm_, 8);                              \
    f.pffm = ffm_;                                                                       \
    chk |= (w) & prmt(rem_, 0u, 0xBA98u); /* sign replication: FF where a flag is */     \
    const uint32_t e_ = lds_u32<0>((mad_hi(rem_, S_IDXMUL, 0u) & 0x3Cu) | selb);         \
    const uint32_t out_ = prmt((w), 0u, e_);                                             \
    const uint32_t hi_ = f.acc | (out_ >> f.sh);                                         \
    const uint32_t lo_ = __funnelshift_r(0u, out_, f.sh);                                \
    const uint32_t tot_ = f.sh + (e_ >> 16);                                             \
    if (tot_ >= 32u) {                                                                   \
      sts_u32<0>(ringb + (f.wo & T_RMASK), hi_);                                         \
      f.wo += T_WSTRIDE;                                                                 \
      f.acc = lo_;                                                                       \
    } else {                                                                             \
      f.acc = hi_;                                                                       \
    }                                                                                    \
    f.sh = tot_ & 31u;                                                                   \
  } while (0)
#endif
  S_WORD(q.x);
  S_WORD(q.y);
  S_WORD(q.z);
  S_WORD(q.w);
#undef S_WORD
#if RSB200_S_FILL2
  f.sh = u & 31u;
#endif
  return chk;
}

// block `blk` (already loaded) into the ring
__device__ __forceinline__ void s_block(SFill& f, uint32_t ringb, uint32_t selb, uint32_t einfo,
                                        const uint4& q, uint32_t blk, const uint8_t* __restrict__ gbase,
                                        uint32_t skew, uint32_t limit) {
  if (blk >= f.slow_from) {
    f = s_slow_block(f, ringb, einfo, q, blk, skew, limit);
  } else {
    const uint32_t chk = s_fast_block(f, ringb, selb, q);
    if (chk != 0u) {
      const uint2 m = s_find_marker(gbase, blk, s_clean_count(f), skew);
      f = s_zero_behind(f, ringb, m.x);
      f.clean_len = m.x;
      f.slow_from = 0;
      f.pffm = 0;
      sts_u32<0>(einfo, blk);
      sts_u32<(int)(4 * T_NT)>(einfo, m.y);
    }
  }
}

// load + process one block now (start of a segment; a lane that ran dry)
__device__ __noinline__ SFill s_fill_now(SFill f, uint32_t ringb, uint32_t selb, uint32_t einfo,
                                         const uint8_t* __restrict__ gbase, uint32_t bmax, uint32_t skew,
                                         uint32_t limit) {
  const uint32_t blk = f.nblk;
  uint4 q = make_uint4(0, 0, 0, 0);
  if (16u * (blk + 1u) > skew) // (a block wholly before the segment is not read)
    q = __ldg(reinterpret_cast<const uint4*>(gbase) + min(blk, bmax));
  f.nblk = blk + 1u;
  if (16u * blk < skew || blk >= f.slow_from) { // bytes before the segment (skew <= 31) / the end
    f = s_slow_block(f, ringb, einfo, q, blk, skew, limit);
  } else {
    s_block(f, ringb, selb, einfo, q, blk, gbase, skew, limit);
  }
  return f;
}

// BitStreamerJPEG::getStreamPosition() of the reference after the last symbol (see
// t_stream_position in ljpeg_thread.cuh for the cadence): the raw offset behind `need` data
// bytes, or the end marker if that comes first; past the end of the buffer the bytes read as
// zero data.  (blk, c): c bytes that do not follow an FF lie in [skew, 16 blk).
__device__ __noinline__ uint32_t s_stream_position(const uint8_t* __restrict__ gbase, uint32_t limit,
                                                   uint32_t skew, uint32_t T, uint32_t blk, uint32_t c) {
  const uint32_t R = (T >> 5) + 1u + ((T & 31u) ? 1u : 0u);
  const uint32_t need = 4u * R;
  auto byte_at = [&](uint32_t q) { return q < limit ? (uint32_t)__ldg(gbase + q) : 0u; };
  // back over whole blocks until no more than `need` bytes precede the block
  while (blk > 0u && c > need) {
    --blk;
    uint32_t kept = 0;
#pragma unroll 1
    for (uint32_t i = 0; i < 16; ++i) {
      const uint32_t raw = 16u * blk + i;
      if (raw >= skew && !(raw > skew && byte_at(raw - 1u) == 0xFFu))
        ++kept;
    }
    c -= kept;
  }
  uint32_t rawp = max(16u * blk, skew);
  if (blk == 0u)
    c = 0;
  if (rawp > skew && byte_at(rawp - 1u) == 0xFFu) {
    if (byte_at(rawp) != 0u)
      return rawp - 1u - skew; // a marker whose FF ended the previous block
    rawp += 1u;                // the stuffing byte of that FF
  }
  while (c < need) {
    if (byte_at(rawp) == 0xFFu) {
      if (byte_at(rawp + 1u) != 0u)
        break; // marker: the position stays on it
      rawp += 2u;
    } else {
      rawp += 1u;
    }
    ++c;
  }
  return rawp - skew;
}

// The straight-line unit stopped at bit p1 (its first miss; every symbol before it was a hit and is
// done): how many symbols lie between p0, where the unit began, and p1.  The words from p0 >> 5 on
// are still in the ring: nothing is written inside a unit, and a fill step at the end of the unit
// before (taken with at most S_ROOM bytes ahead) leaves the ring starting 8 bytes or more BEHIND
// the read position.  Rare path (codes longer than LUT_BITS, SSSS = 16, corrupt data).
__device__ __noinline__ uint32_t s_count_hits(uint32_t ringb, uint32_t l0, uint32_t l1, uint32_t l2, uint32_t l3,
                                              uint32_t gm1, uint32_t p0, uint32_t p1) {
  uint32_t k = 0, q = p0;
  while (q != p1 && k < 8u) {
    const uint32_t w = (q >> 5) * T_WSTRIDE;
    const uint32_t a = lds_u32<0>(ringb + (w & T_RMASK));
    const uint32_t b = lds_u32<0>(ringb + ((w + T_WSTRIDE) & T_RMASK));
    const uint32_t x = __funnelshift_l(b, a, q);
    const uint32_t c = k & gm1; // component of sample k (G = 1, 2 or 4)
    const uint32_t lutb = c == 0u ? l0 : (c == 1u ? l1 : (c == 2u ? l2 : l3));
    const uint32_t e = lds_u16<0>(mad_hi(x & ~((1u << (32 - LUT_BITS)) - 1u), 1u << (LUT_BITS + 1), lutb));
#ifdef RSB200_EMU
    if (e == 0u || q > p1)
      abort(); // the re-walk left the path of the unit: the ring no longer held its words
#endif
    if (e == 0u)
      break;
    q += e >> 10;
    ++k;
  }
  return k;
}

// "does any lane that is here with me want a fill step" -- a scheduling hint only: results do
// not depend on it (a lane that runs dry fills on its own, s_fill_now)
#ifdef RSB200_EMU
inline int g_emu_any_mode = 0; // 0: the lane's own wish; 1: always
__device__ __forceinline__ bool s_any(bool want) { return g_emu_any_mode ? true : want; }
#else
__device__ __forceinline__ bool s_any(bool want) { return __any_sync(__activemask(), want); }
#endif

// one sample of component c: Huffman code + mantissa at bit position p of the window
#define S_SYM(c, val)                                                           \
  do {                                                                          \
    const uint32_t x_ = __funnelshift_l(nxt, cur, p);                           \
    const uint32_t d_ = t_decode_diff(tabp[c], lutb[c], x_, p, last_tl, bad_at); \
    const uint32_t pn_ = p + last_tl;                                           \
    if ((pn_ ^ p) & 32u) { /* into the next word (a symbol is <= 32 bits) */    \
      cur = nxt;                                                                \
      nxt = nn;                                                                 \
      nn = lds_u32<0>(ringb + (wv & T_RMASK)); /* word wv / T_WSTRIDE */        \
      wv += T_WSTRIDE;                                                          \
    }                                                                           \
    p = pn_;                                                                    \
    pred[c] += d_;                                                              \
    val = pred[c];                                                              \
  } while (0)

// The same without control flow, for the straight-line unit: a code the LUT does not resolve
// (longer than LUT_BITS, SSSS = 16, corrupt) leaves p where it is, so every later symbol of the
// unit sees the same window and -- LOOKING IT UP IN THE SAME TABLE -- misses too: the unit is
// complete iff its last symbol hit; otherwise the symbols before the first miss are counted
// (s_count_hits) and the unit is finished symbol by symbol (S_SYM) from there.
// Without a branch per symbol the eight decodes are one basic block: the difference arithmetic of
// symbol k is scheduled into the latency of symbol k+1's LUT load.  With SEVERAL tables a window
// that starts with a long code of one can be a short code of another and the miss would not stick
// (the kernel of run 23 decoded garbage there): the shared-memory copies of a plan's LUTs are
// therefore reduced to the windows that ALL of them resolve (stream_entry); a window dropped from
// a LUT just takes the symbol-by-symbol path, which walks the code lengths.
// RSB200_S_PIPE (A/B): the unit is bound by the ALU pipe (SHF / LOP3 / LEA / IADD3: one warp
// instruction every two cycles).  ptxas turns every multiply by a constant power of two back into ALU
// forms, so the multipliers come from the constant bank (s_pipe_k), where it cannot see them:
//   1: LUT address = (x >> 21) * 2 + base as SHF + IMAD (was LOP3 + LEA.HI); the sign mask from
//      tt + 0x80000000 (IMAD) instead of ~tt (LOP3)
//   2: + p + (e >> 10) and e >> 5 as IMAD.HI (were LEA.HI, SHF)
// 1 is the default (IMAD.HI with a 64-bit addend costs two FMA-pipe instructions, which makes 2 the
// slower form); not re-measured on H100.
#ifndef RSB200_S_PIPE
#define RSB200_S_PIPE 1
#endif
#if RSB200_S_PIPE >= 1
#define S_LUT_ADDR(x, base) s_mad_lo((x) >> (32 - LUT_BITS), s_pipe_k[0], (base))
#define S_SIGN_MASK(tt) ((uint32_t)((int32_t)s_mad_lo((tt), s_pipe_k[1], 0x80000000u) >> 31))
#else
#define S_LUT_ADDR(x, base) mad_hi((x) & ~((1u << (32 - LUT_BITS)) - 1u), 1u << (LUT_BITS + 1), (base))
#define S_SIGN_MASK(tt) ((uint32_t)((int32_t)~(tt) >> 31))
#endif
#if RSB200_S_PIPE >= 2
#define S_ADD_TOTAL(e, p) mad_hi((e), s_pipe_k[2], (p))
#define S_SSSS(e) mad_hi((e), s_pipe_k[3], 0u)
#else
#define S_ADD_TOTAL(e, p) ((p) + ((e) >> 10))
#define S_SSSS(e) ((e) >> 5)
#endif
#define S_SYMF(c, val)                                                          \
  do {                                                                          \
    const uint32_t x_ = __funnelshift_l(nxt, cur, p);                           \
    const uint32_t e_ = lds_u16<0>(S_LUT_ADDR(x_, lutb[c]));                    \
    elast = e_;                                                                 \
    const uint32_t tt_ = __funnelshift_l(0u, x_, e_);                           \
    const uint32_t f_ = S_SIGN_MASK(tt_);                                       \
    /* a miss (e_ = 0) needs no select: both shifts are by 0, d_ = f_ - f_ */   \
    const uint32_t d_ = __funnelshift_l(tt_, f_, S_SSSS(e_)) - f_;              \
    const uint32_t pn_ = S_ADD_TOTAL(e_, p);                                    \
    last_tl = pn_ - p;                                                          \
    if ((pn_ ^ p) & 32u) {                                                      \
      cur = nxt;                                                                \
      nxt = nn;                                                                 \
      nn = lds_u32<0>(ringb + (wv & T_RMASK));                                  \
      wv += T_WSTRIDE;                                                          \
    }                                                                           \
    p = pn_;                                                                    \
    pred[c] += d_;                                                              \
    val = pred[c];                                                              \
  } while (0)

#if RSB200_S_LUT32
#undef S_SYMF
#define S_SYMF(c, val)                                                          \
  do {                                                                          \
    const uint32_t x_ = __funnelshift_l(nxt, cur, p);                           \
    const uint32_t e_ = lds_u32<0>(                                             \
        mad_hi(x_ & ~((1u << (32 - LUT_BITS)) - 1u), 1u << (LUT_BITS + 2), lut32b[c])); \
    elast += e_; /* hits in bits 19:16 */                                       \
    const uint32_t tt_ = __funnelshift_l(0u, x_, e_);                           \
    const uint32_t f_ = (uint32_t)((int32_t)~tt_ >> 31);                        \
    const uint32_t d_ = __funnelshift_l(tt_, f_, mad_hi(e_, 1u << 24, 0u)) - f_; \
    const uint32_t pn_ = mad_hi(e_, 1u << 6, p);                                \
    last_tl = pn_ - p;                                                          \
    if ((pn_ ^ p) & 32u) {                                                      \
      cur = nxt;                                                                \
      nxt = nn;                                                                 \
      nn = lds_u32<0>(ringb + (wv & T_RMASK));                                  \
      wv += T_WSTRIDE;                                                          \
    }                                                                           \
    p = pn_;                                                                    \
    pred[c] += d_;                                                              \
    val = pred[c];                                                              \
  } while (0)
#endif

#ifndef RSB200_S_STRAIGHT
#define RSB200_S_STRAIGHT 1
#endif
#ifndef RSB200_S_PREFETCH
#define RSB200_S_PREFETCH 8 // blocks ahead of a requested sector that are pulled into L2 when the launch is small
#endif
// 128 bits of output with the default L2 policy.  A lane writes a 128-byte line of its output row
// over two to eight store steps, microseconds apart; with evict-first stores (st.global.cs) the
// kernel was about 2 % slower on H100 (DESIGN.md, K2S), presumably because L2 let such lines go
// before they were whole.
__device__ __forceinline__ void s_stg_v4(void* p, const uint4& v) {
#ifdef RSB200_EMU
  memcpy(p, &v, 16);
#else
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
#endif
}

// Unit j (0..3) of a group sits at 16 * (j ^ ((lane >> 1) & 3)) in the lane's 64-byte stage: the
// 128-bit shared accesses of a quarter warp (8 lanes) then hit 8 different 16-byte bank groups, both
// when each lane writes one unit of its own stage and when four lanes read one stage (s_flush).
__device__ __forceinline__ uint32_t s_stage_unit(uint32_t lane, uint32_t j) {
  return 16u * ((j ^ (lane >> 1)) & 3u);
}

// One whole 32-byte sector of output: Hopper's widest store is 128 bits, so the two halves leave
// back to back from the same lane.
#ifdef RSB200_EMU
// (CPU replay: whole 32-byte sectors of segments whose rows are 32-byte aligned, stored by this branch
//  or as a staged run)
inline unsigned long long g_emu_sector_stores = 0;
#endif
__device__ __forceinline__ void s_stg_sector(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d,
                                             uint32_t e, uint32_t f, uint32_t g, uint32_t h) {
#ifdef RSB200_EMU
  ++g_emu_sector_stores;
#endif
  s_stg_v4(p, make_uint4(a, b, c, d));
  s_stg_v4(static_cast<uint8_t*>(p) + 16, make_uint4(e, f, g, h));
}

// "every lane of my warp is here" -- a hint only: results do not depend on it (s_flush).  `at` names the
// flush (G, row, unit): lanes meet only at the same one, the GPU's lanes at the same program point.
#ifdef RSB200_EMU
inline unsigned long long g_emu_runs_shared = 0; // (CPU replay: 64-byte runs stored by the whole warp)
inline unsigned long long g_emu_runs_own = 0;    // (... by the lane whose run it is)
// a replay that gathers the lanes of a warp defines one of these: RSB200_EMU_WHOLE_WARP_AT(at) where the
// place of the flush matters to it, RSB200_EMU_WHOLE_WARP() where it does not; otherwise every lane is alone
#ifndef RSB200_EMU_WHOLE_WARP
#define RSB200_EMU_WHOLE_WARP() false
#endif
#ifndef RSB200_EMU_WHOLE_WARP_AT
#define RSB200_EMU_WHOLE_WARP_AT(at) ((void)(at), RSB200_EMU_WHOLE_WARP())
#endif
__device__ __forceinline__ bool s_whole_warp(uint64_t at) { return RSB200_EMU_WHOLE_WARP_AT(at); }
#else
__device__ __forceinline__ bool s_whole_warp(uint64_t) { return __activemask() == 0xFFFFFFFFu; }
#endif
#if defined(RSB200_FLUSH_COUNT) && !defined(RSB200_EMU)
// profiling builds only (-DRSB200_FLUSH_COUNT, tools/flush_count.py): 64-byte runs stored by whole warps
// [0] and by single lanes [1], read by rsb200_debug_flush_runs
__device__ unsigned long long g_flush_runs[2];
#endif
// The lane's last four units (its stage) go to `dst` (16-byte aligned).  Where the whole warp is here,
// the lanes store each other's stages: lane l writes 16 bytes of the run of lane 8k + l / 4 in step
// k, so a store instruction carries eight whole 64-byte runs -- 8 requests of two sectors instead of
// 32 requests of 16 bytes to 32 lines.  Every warp that decodes tiles of one shape gets here at the
// same unit; results do not depend on it: a lane of a partial warp, or of a warp whose lanes are
// elsewhere (other tile shapes, row tails), stores its own run.
__device__ __forceinline__ void s_flush(uint32_t stage, uint32_t lane, uint8_t* dst, uint64_t at) {
  if (s_whole_warp(at)) {
#ifdef RSB200_EMU
    ++g_emu_runs_shared;
#elif defined(RSB200_FLUSH_COUNT)
    if (lane == 0u)
      atomicAdd(&g_flush_runs[0], 32ull);
#endif
    __syncwarp(); // the stages are written
    const uint32_t lo = (uint32_t)reinterpret_cast<uintptr_t>(dst);
    const uint32_t hi = (uint32_t)(reinterpret_cast<uintptr_t>(dst) >> 32);
    const uint32_t c = lane & 3u;
#pragma unroll 1
    for (uint32_t k = 0; k < 4; ++k) {
      const uint32_t src = 8u * k + (lane >> 2);
      const uintptr_t d = ((uintptr_t)__shfl_sync(0xFFFFFFFFu, hi, (int)src) << 32) |
                          __shfl_sync(0xFFFFFFFFu, lo, (int)src);
      const uint4 v = lds_v4<0>(stage + S_STAGE * (src - lane) + s_stage_unit(src, c));
      s_stg_v4(reinterpret_cast<uint8_t*>(d) + 16u * c, v);
    }
    __syncwarp(); // the stages are read before they are written again
  } else {
#ifdef RSB200_EMU
    ++g_emu_runs_own;
#elif defined(RSB200_FLUSH_COUNT)
    {
      const uint32_t m = __activemask();
      if (lane == (uint32_t)(__ffs(m) - 1))
        atomicAdd(&g_flush_runs[1], (unsigned long long)__popc(m));
    }
#endif
#pragma unroll 1
    for (uint32_t j = 0; j < 4; ++j)
      s_stg_v4(dst + 16u * j, lds_v4<0>(stage + s_stage_unit(lane, j)));
  }
}

__device__ __forceinline__ void s_prefetch_l2(const void* p) {
#ifndef RSB200_EMU
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#else
  (void)p;
#endif
}

// 128 bits of input through the read-only path, with an L2 fetch-size hint of 128 bytes: a miss
// brings the rest of the 128-byte line into L2 with the sector asked for, and the lane reads it in
// its next fill steps.  The hint adds no request (the explicit L2 prefetches of the small-launch form
// make large launches more than twice as slow).
__device__ __forceinline__ uint4 s_ldg_l2_128b(const uint4* p) {
#ifdef RSB200_EMU
  return __ldg(p);
#else
  uint4 r;
  asm volatile("ld.global.nc.L2::128B.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
#endif
}
// A lane's next two 16-byte blocks = one 32-byte sector (blk even, cb 32-byte aligned): both
// 128-bit loads are issued together, before the unit's decode that hides their latency.  113 k
// streams of lane-private requests are bound by the number of requests the memory system serves,
// so a lane asks for whole sectors and never for a block twice.
__device__ __forceinline__ void s_ldg_sector(const uint4* cb, uint32_t blk, uint32_t bmax, uint4& a,
                                             uint4& b) {
  a = s_ldg_l2_128b(cb + min(blk, bmax));
  b = s_ldg_l2_128b(cb + min(blk + 1u, bmax));
}

template <int G, bool WIDE, bool STAGED>
__device__ __forceinline__ void
stream_body(StreamShared& sh, const int ntab_sh, const DevScan* __restrict__ scp, const bool may_redo, const bool prefetch,
            const uint8_t* __restrict__ in, uint64_t in_total, uint8_t* __restrict__ out,
            DevResult* __restrict__ res, uint32_t* __restrict__ redo) {
  // raw offsets count from the 32-byte boundary at or before the segment's first byte
  const uint8_t* first = in + scp->in_offset;
  const uint32_t skew = (uint32_t)(reinterpret_cast<uintptr_t>(first) & 31u);
  const uint32_t limit = skew + scp->in_size;
  const uint8_t* gbase = first - skew;
  const uint4* cb = reinterpret_cast<const uint4*>(gbase);
  // the caller's buffer is readable up to the next 16-byte boundary behind in_total; a block that
  // lies wholly before the segment (skew >= 16) is never loaded, so nothing before `in` is touched
  const uint64_t nreadable = (uint64_t)((in + ((in_total + 15ull) & ~15ull)) - gbase) >> 4;
  const uint32_t bmax = (nreadable > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)nreadable) - 1u;
  const uint32_t ringb = smem_u32(&sh.ring[0][threadIdx.x]);
  const uint32_t selb = smem_u32(sh.sel);
#if RSB200_S_LUT32
  const uint32_t* lut32 = reinterpret_cast<const uint32_t*>(&sh.tab[ntab_sh]);
#endif
  const uint32_t einfo = smem_u32(&sh.endinfo[0][threadIdx.x]);

  SFill f;
  f.acc = 0;
  f.sh = 0;
  f.wo = 0;
  f.pffm = 0;
  f.nblk = 0;
  f.slow_from = limit >> 4;
  f.clean_len = S_OPEN;
  // prefill
  while ((f.wo >> 7) < S_LOW || (f.nblk & 1u)) // (sectors are taken whole from here on: nblk stays even)
    f = s_fill_now(f, ringb, selb, einfo, gbase, bmax, skew, limit);
  uint32_t cur = sh.ring[0][threadIdx.x], nxt = sh.ring[1][threadIdx.x],
           nn = sh.ring[2][threadIdx.x];
  uint32_t wv = 3u * T_WSTRIDE, p = 0; // wv: ring byte offset of the next word to fetch (unwrapped)

  uint32_t lutb[G];
#if RSB200_S_LUT32
  uint32_t lut32b[G];
#endif
  const DevTable* tabp[G];
  uint32_t rowstart[G], pred[G];
#pragma unroll
  for (int c = 0; c < G; ++c) {
    tabp[c] = &sh.tab[scp->table_idx[scp->table_of[c]]];
    lutb[c] = smem_u32(tabp[c]->lut);
#if RSB200_S_LUT32
    lut32b[c] = smem_u32(lut32 + (size_t)scp->table_idx[scp->table_of[c]] * (1u << LUT_BITS));
#endif
    rowstart[c] = scp->init_pred[c];
  }
  // (the straight-line unit relies on "a miss repeats": the LUTs of a plan with several tables are made
  //  to miss on the same windows, see stream_entry)
  const uint32_t rows = scp->rows;
  const uint32_t units = scp->row_samples >> 3; // row_samples is a multiple of 8
  const uint32_t store_w = scp->store_w;
  const uint32_t out_pitch = scp->out_pitch;
  uint8_t* orow = out + scp->out_offset + (uint64_t)scp->out_y * out_pitch + 2ull * scp->out_x;
  uint32_t bad_at = T_NOBAD, last_tl = 0;
  // WIDE: the whole groups of 4 units of a row in front of store_w (<= row_samples) go through the
  // stage, the rest directly.  (The small-launch form measured the same with the stage as without,
  // and keeps direct stores: its registers spill less.)  A plan whose tables leave no room for the
  // stage stores pairs of units as one 32-byte sector where the rows allow it.
  static_assert(WIDE || !STAGED, "the stage is the full-launch form's");
  const bool staged = STAGED;
  const bool aligned32 = ((reinterpret_cast<uintptr_t>(orow) | out_pitch) & 31u) == 0u;
  const bool pairs = WIDE && !staged && aligned32;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t stage = smem_u32(reinterpret_cast<const uint8_t*>(&sh) + stream_stage_offset(ntab_sh)) +
                         S_STAGE * threadIdx.x;
  const uint32_t groups = staged ? store_w >> 5 : 0u;
  uint32_t h0 = 0, h1 = 0, h2 = 0, h3 = 0;
#ifndef RSB200_EMU
  (void)aligned32;
#endif

  for (uint32_t r = 0; r < rows; ++r) {
#pragma unroll
    for (int c = 0; c < G; ++c)
      pred[c] = rowstart[c];
    for (uint32_t u = 0; u < units; ++u) {
      // ---- start of the unit (s_ring_note): a unit reads at most 8 x 32 bits and the window is
      //      three words long, so the words up to (p >> 5) + 10 must be in the ring: S_MIN = 44
      //      bytes of whole words ahead of byte p >> 3.  A block adds at most 4 words (two: 8);
      //      word W may replace word W - T_RING once that one was fetched (< (p >> 5) + 3):
      //      ahead <= 121 (two blocks: 105) before the step. ----
      uint32_t ahead = (f.wo >> 7) - (p >> 3);
      while (ahead < S_MIN) { // ran dry (more than 32 bytes per unit for a while): fill on my own
        f = s_fill_now(f, ringb, selb, einfo, gbase, bmax, skew, limit);
        f = s_fill_now(f, ringb, selb, einfo, gbase, bmax, skew, limit);
        ahead = (f.wo >> 7) - (p >> 3);
      }
      // blocks requested here go into the ring at the END of the unit: no load is in flight
      // across the loop edge and the decode of the unit hides their latency
      uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
      bool pend = false;
      if (s_any(ahead < S_LOW) && ahead <= S_ROOM) {
        s_ldg_sector(cb, f.nblk, bmax, q0, q1);
        pend = true;
        if (RSB200_S_PREFETCH && prefetch)
          s_prefetch_l2(cb + min(f.nblk + (uint32_t)RSB200_S_PREFETCH, bmax));
      }
      // 8 samples, straight line (component of sample k = k % G)
      uint32_t v0, v1, v2, v3, v4, v5, v6, v7;
#if RSB200_S_STRAIGHT
      uint32_t k_ = 0; // samples of the unit that are done
      {
        // a miss repeats (same window; every LUT of the plan misses on it): complete iff the LAST symbol hit
        const uint32_t p0 = p;
        uint32_t elast = 0;
        S_SYMF(0 % G, v0);
        S_SYMF(1 % G, v1);
        S_SYMF(2 % G, v2);
        S_SYMF(3 % G, v3);
        S_SYMF(4 % G, v4);
        S_SYMF(5 % G, v5);
        S_SYMF(6 % G, v6);
        S_SYMF(7 % G, v7);
#if RSB200_S_LUT32
        k_ = (elast >> 16) & 15u; // (hit flags added up)
#else
        k_ = 8u;
        if (elast == 0u)
          k_ = s_count_hits(ringb, lutb[0], lutb[1 % G], lutb[2 % G], lutb[3 % G], (uint32_t)G - 1u, p0, p);
#endif
      }
      if (k_ != 8u) { // rare: the symbols from the first miss on, one by one
        if (k_ <= 0u)
          S_SYM(0 % G, v0);
        if (k_ <= 1u)
          S_SYM(1 % G, v1);
        if (k_ <= 2u)
          S_SYM(2 % G, v2);
        if (k_ <= 3u)
          S_SYM(3 % G, v3);
        if (k_ <= 4u)
          S_SYM(4 % G, v4);
        if (k_ <= 5u)
          S_SYM(5 % G, v5);
        if (k_ <= 6u)
          S_SYM(6 % G, v6);
        S_SYM(7 % G, v7);
      }
#else
      S_SYM(0 % G, v0);
      S_SYM(1 % G, v1);
      S_SYM(2 % G, v2);
      S_SYM(3 % G, v3);
      S_SYM(4 % G, v4);
      S_SYM(5 % G, v5);
      S_SYM(6 % G, v6);
      S_SYM(7 % G, v7);
#endif
      const uint32_t o0 = __byte_perm(v0, v1, 0x5410), o1 = __byte_perm(v2, v3, 0x5410),
                     o2 = __byte_perm(v4, v5, 0x5410), o3 = __byte_perm(v6, v7, 0x5410);
      if (u == 0) { // the first MCU of the row predicts the first MCU of the next row
        rowstart[0] = v0;
        if (G >= 2)
          rowstart[1] = v1;
        if (G == 4) {
          rowstart[2] = v2;
          rowstart[3] = v3;
        }
      }
      // ---- end of the unit: the requested blocks are unstuffed into the ring ----
      if (pend) {
        s_block(f, ringb, selb, einfo, q0, f.nblk, gbase, skew, limit);
        s_block(f, ringb, selb, einfo, q1, f.nblk + 1u, gbase, skew, limit);
        f.nblk += 2u;
      }
      const uint32_t s = u << 3;
      if (WIDE && (u >> 2) < groups) {
        sts_v4<0>(stage + s_stage_unit(lane, u), make_uint4(o0, o1, o2, o3));
        if ((u & 3u) == 3u) {
          s_flush(stage, lane, orow + 16ull * (u - 3u), ((uint64_t)r << 32) | (u << 3) | (uint32_t)G);
#ifdef RSB200_EMU
          g_emu_sector_stores += aligned32 ? 2u : 0u;
#endif
        }
      } else if (pairs && !(u & 1u) && s + 16u <= store_w) { // the even unit waits for the odd one
        h0 = o0;
        h1 = o1;
        h2 = o2;
        h3 = o3;
      } else if (pairs && (u & 1u) && s + 8u <= store_w) {
        s_stg_sector(orow + 16ull * (u - 1u), h0, h1, h2, h3, o0, o1, o2, o3);
      } else if (s + 8 <= store_w) {
        s_stg_v4(orow + 16ull * u, make_uint4(o0, o1, o2, o3));
      } else if (s < store_w) {
        uint16_t* o16 = reinterpret_cast<uint16_t*>(orow) + s;
        const uint32_t ow[4] = {o0, o1, o2, o3};
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (s + k < store_w)
            o16[k] = (uint16_t)(ow[k >> 1] >> (16 * (k & 1)));
      }
    }
    orow += out_pitch;
  }
  // A needed symbol used bits that are not there.  Whether the reference reads them as zero bits
  // or throws depends on the refill cadence of its pump (BitStreamer.h:120-127,
  // BitStreamerJPEG.h:155-183): segments the tile kernel can take are flagged and decoded again
  // by it (exact, tl_replay in ljpeg_tile.cuh); for the others the answer stays IOException
  // (DESIGN.md "known deviations").
  const bool over = p > 8u * f.clean_len;
  // (an unassigned code wholly in the data is the answer; one that reaches behind it is not, see
  //  t_bad_in_data)
  const bool bad_in = t_bad_in_data(bad_at, 8u * f.clean_len);
  const bool again = over && !bad_in && redo && may_redo;
  if (redo)
    *redo = again ? 1u : 0u;
  res->status = bad_in ? 1u : (over ? (again ? 0u : 2u) : (bad_at != T_NOBAD ? 1u : 0u));
  {
    uint32_t ablk = f.nblk, acc = s_clean_count(f);
    if (f.clean_len != S_OPEN) {
      ablk = lds_u32<0>(einfo);
      acc = lds_u32<(int)(4 * T_NT)>(einfo);
    }
    const uint32_t consumed = s_stream_position(gbase, limit, skew, p - last_tl, ablk, acc);
    res->consumed = consumed;
    // the reference skips `consumed` bytes of its input when the scan is done and throws when the
    // buffer is shorter (LJpegDecompressor.cpp:339 -> ByteStream::skipBytes): a buffer that ends
    // inside the last refill is an IOException even when every symbol was there
    if (res->status != 1u && !again && consumed > scp->in_size)
      res->status = 2u;
  }
}
#undef S_SYM
#undef S_SYMF

// entry: one CTA of T_NT threads (the GPU kernel below; tests/emu replays it on the CPU).  STAGE: 1 =
// the full-launch form with its output stage, 0 = without, -1 = whichever the plan's tables allow
// (stream_staged).  The GPU launches a kernel per choice: a kernel holding both bodies spills more.
template <bool WIDE, int STAGE = -1>
__device__ __forceinline__ void
stream_entry(StreamShared& sh, const uint8_t* __restrict__ in, uint64_t in_total,
             const DevScan* __restrict__ scans, const DevTable* __restrict__ tables, int ntab,
             uint8_t* __restrict__ out, DevResult* __restrict__ results,
             const uint32_t* __restrict__ scan_ids, uint32_t nids, uint32_t* __restrict__ redo,
             const bool prefetch) {
  const int tid = threadIdx.x;
  {
    const uint4* src = reinterpret_cast<const uint4*>(tables);
    uint4* dst = reinterpret_cast<uint4*>(sh.tab);
    const int n = ntab * (int)(sizeof(DevTable) / 16);
    for (int i = tid; i < n; i += T_NT)
      dst[i] = src[i];
    if (tid < 16)
      sh.sel[tid] = s_sel_entry((uint32_t)tid);
  }
  __syncthreads();
  if (ntab > 1) { // a window is a hit only if every table of the plan resolves it (see S_SYMF)
    for (int i = tid; i < (1 << LUT_BITS); i += T_NT) {
      bool all = true;
      for (int t = 0; t < ntab; ++t)
        all = all && sh.tab[t].lut[i] != 0;
      if (!all)
        for (int t = 0; t < ntab; ++t)
          sh.tab[t].lut[i] = 0;
    }
    __syncthreads();
  }
#if RSB200_S_LUT32
  {
    uint32_t* l32 = reinterpret_cast<uint32_t*>(&sh.tab[ntab]);
    for (int i = tid; i < ntab * (1 << LUT_BITS); i += T_NT)
      l32[i] = s_lut32_entry(sh.tab[i >> LUT_BITS].lut[i & ((1 << LUT_BITS) - 1)]);
  }
  __syncthreads();
#endif
  const uint32_t id = blockIdx.x * T_NT + tid;
  if (id >= nids)
    return;
  // bit 31 of an id: the tile kernel can give this segment a second opinion at its end of stream
  const uint32_t sid = scan_ids[id];
  const uint32_t scan_idx = sid & 0x7FFFFFFFu;
  const bool may_redo = (sid >> 31) != 0u;
  const DevScan* scp = scans + scan_idx;
  DevResult* res = results + scan_idx;
  const uint32_t G = scp->group;
  uint32_t* rd = redo ? redo + id : nullptr;
  if (WIDE && (STAGE == 1 || (STAGE < 0 && stream_staged(ntab)))) {
    if (G == 1)
      stream_body<1, WIDE, WIDE>(sh, ntab, scp, may_redo, prefetch, in, in_total, out, res, rd);
    else if (G == 2)
      stream_body<2, WIDE, WIDE>(sh, ntab, scp, may_redo, prefetch, in, in_total, out, res, rd);
    else
      stream_body<4, WIDE, WIDE>(sh, ntab, scp, may_redo, prefetch, in, in_total, out, res, rd);
  } else if (G == 1) {
    stream_body<1, WIDE, false>(sh, ntab, scp, may_redo, prefetch, in, in_total, out, res, rd);
  } else if (G == 2) {
    stream_body<2, WIDE, false>(sh, ntab, scp, may_redo, prefetch, in, in_total, out, res, rd);
  } else {
    stream_body<4, WIDE, false>(sh, ntab, scp, may_redo, prefetch, in, in_total, out, res, rd);
  }
}

#ifndef RSB200_EMU
template <bool WIDE, bool STAGED>
__global__ void __launch_bounds__(T_NT, RSB200_S_LB)
    k2_stream_kernel(const uint8_t* __restrict__ in, uint64_t in_total, const DevScan* __restrict__ scans,
                     const DevTable* __restrict__ tables, int ntab, uint8_t* __restrict__ out,
                     DevResult* __restrict__ results, const uint32_t* __restrict__ scan_ids,
                     uint32_t nids, uint32_t* __restrict__ redo, int prefetch) {
  extern __shared__ __align__(128) uint8_t s_smem_raw[];
  StreamShared& sh = *reinterpret_cast<StreamShared*>(s_smem_raw);
  static_assert(WIDE || !STAGED, "the stage is the full-launch form's");
  stream_entry<WIDE, STAGED ? 1 : 0>(sh, in, in_total, scans, tables, ntab, out, results, scan_ids, nids, redo,
                                     prefetch != 0);
}
#endif

} // namespace rsb200
