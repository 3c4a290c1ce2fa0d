// phaseone.cuh -- K8: Phase One IIQ row codec (SURVEY 8(f)4), sm_90a.
//
// Replaces the body of PhaseOneDecompressor::decompressStrip
// (decompressors/PhaseOneDecompressor.cpp:85-135) and the OpenMP loop over strips
// (:137-150).  One strip = one image row = one MSB32 bit stream (32-bit
// little-endian chunks consumed MSB first, BitStreamMSB32.h): every 8 pixels two
// code lengths are read (up to 5 zero bits, then one bit, into
// {8,7,6,9,11,10,5,12,14,13}; at column 0 any 1 bit in the prefix is an error), then
// each pixel is either a raw 16-bit value (length 14; always for the last width % 8
// pixels) or a difference to its same-parity predecessor.  Rows are independent,
// pixels of a row are not: one thread per row, 64-bit cache in registers,
// fill(32) before every pixel exactly like the reference (the over-read rule of
// BitStreamer.h:100-131 -- zero padding up to 8 bytes past the end, error beyond --
// is part of the result).
#pragma once

#ifndef RSB200_EMU
#include "common.cuh"
#endif
#include <stdint.h>

namespace rsb200 {

constexpr int P1_NT = 64;

struct P1StripDev {
  uint64_t in_offset;
  uint32_t in_size;
  uint32_t row;
  uint32_t job;
  uint32_t pad;
};
struct P1JobDev {
  uint64_t out_offset;
  uint32_t out_pitch;
  uint32_t width;
};

// 4 bytes at byte position pos of a strip, little endian, zero padded past its end
__device__ __forceinline__ uint32_t p1_chunk(const uint8_t* __restrict__ base, uint32_t size,
                                             uint32_t pos) {
  if (pos + 4u <= size) {
    const uint8_t* p = base + pos;
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u);
    const uint32_t* pw = reinterpret_cast<const uint32_t*>(p - mis);
    const uint32_t a = __ldg(pw), b = mis ? __ldg(pw + 1) : 0u;
    return __funnelshift_r(a, b, 8u * mis);
  }
  uint32_t v = 0;
  for (uint32_t k = 0; k < 4; ++k)
    if (pos + k < size)
      v |= (uint32_t)__ldg(base + pos + k) << (8 * k);
  return v;
}

#ifndef RSB200_EMU
__global__ void __launch_bounds__(P1_NT)
    p1_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
              const P1StripDev* __restrict__ strips, uint32_t nstrips,
              const P1JobDev* __restrict__ jobs, uint32_t* __restrict__ bad_jobs) {
  const uint32_t s = blockIdx.x * P1_NT + threadIdx.x;
  if (s >= nstrips)
    return;
  const P1StripDev st = strips[s];
  const P1JobDev jb = jobs[st.job];
  const uint8_t* base = in + st.in_offset;
  const uint32_t size = st.in_size, w = jb.width;
  uint32_t* o32 = reinterpret_cast<uint32_t*>(out + jb.out_offset + (uint64_t)st.row * jb.out_pitch);
  if (size < 4u) { // BitStreamer ctor: "Bit stream size is smaller than MaxProcessBytes"
    atomicOr(bad_jobs + st.job, 1u);
    return;
  }
  uint32_t hi = 0, lo = 0, pos = 0;
  int nbits = 0;
  int32_t pred0 = 0, pred1 = 0;
  uint32_t len0 = 0, len1 = 0, even = 0;
  bool bad = false;
  auto getbits = [&](uint32_t n) { // 1 <= n <= 16, n <= nbits
    const uint32_t v = hi >> (32u - n);
    hi = __funnelshift_l(lo, hi, n);
    lo <<= n;
    nbits -= (int)n;
    return v;
  };
  const uint32_t lim = w & ~7u;
  for (uint32_t col = 0; col < w && !bad; ++col) {
    // pump.fill(32)
    if (nbits < 32) {
      if (pos > size + 8u) { // "Buffer overflow read in BitStreamer"
        bad = true;
        break;
      }
      const uint32_t ch = p1_chunk(base, size, pos);
      hi |= __funnelshift_rc(ch, 0u, (uint32_t)nbits);
      lo = __funnelshift_lc(0u, ch, 32u - (uint32_t)nbits);
      nbits += 32;
      pos += 4;
    }
    if (col >= lim) {
      len0 = len1 = 14;
    } else if ((col & 7u) == 0u) {
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        uint32_t j = 0;
        for (; j < 5; ++j) {
          if (getbits(1) != 0u) {
            if (col == 0)
              bad = true; // "Can not initialize lengths. Data is corrupt."
            break;
          }
        }
        if (j > 0) {
          // length[2 * (j - 1) + bit] of {8, 7, 6, 9, 11, 10, 5, 12, 14, 13}, packed in nibbles
          const uint32_t idx = 2u * (j - 1u) + getbits(1);
          const uint32_t l = (uint32_t)((0xDEC5AB9678ull >> (4u * idx)) & 15u);
          if (t == 0)
            len0 = l;
          else
            len1 = l;
        }
      }
      if (bad)
        break;
    }
    const uint32_t i = (col & 1u) ? len1 : len0;
    int32_t& pred = (col & 1u) ? pred1 : pred0;
    if (i == 14u)
      pred = (int32_t)getbits(16);
    else
      pred += (int32_t)getbits(i) + 1 - (1 << (i - 1u));
    if (col & 1u)
      o32[col >> 1] = even | ((uint32_t)pred << 16);
    else
      even = (uint32_t)pred & 0xFFFFu;
  }
  if (bad)
    atomicOr(bad_jobs + st.job, 1u);
}

// ---- second version: no loads inside a group of 8 pixels ----
// All rows of a warp are at the same column at the same time; only their bit positions
// differ.  A per-lane "refill when my cache runs low" therefore issues a load at almost
// every pixel for SOME lane, and the warp-wide scoreboard of the destination register makes
// every lane wait for it (the lesson of K2T).  A group of 8 pixels consumes at most 14 + 8*16
// = 142 bits, so the 7 chunks from the one that holds the group's first bit are fetched at
// the group boundary -- the same instructions for all lanes -- and the group is decoded from
// registers: window (cur, nxt) + a 5-deep register queue shifted at chunk crossings.
// The reference's over-read rule (BitStreamer.h:100-131) in closed form: refill k reads at
// byte 4k and fails when 4k > size + 8; the pixel that starts at bit T needs refills
// 0 .. T/32 + (T % 32 ? 1 : 0), so the row fails iff some pixel starts at a bit
// T > 32 * (K - 1) with K = (size + 8) / 4 + 1.
__global__ void __launch_bounds__(P1_NT)
    p1_kernel_v2(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                 const P1StripDev* __restrict__ strips, uint32_t nstrips,
                 const P1JobDev* __restrict__ jobs, uint32_t* __restrict__ bad_jobs) {
  const uint32_t s_raw = blockIdx.x * P1_NT + threadIdx.x;
  const bool live = s_raw < nstrips;
  const P1StripDev st = strips[live ? s_raw : nstrips - 1u];
  const P1JobDev jb = jobs[st.job];
  const uint8_t* base = in + st.in_offset;
  const uint32_t size = st.in_size, w = jb.width;
  uint32_t* o32 = reinterpret_cast<uint32_t*>(out + jb.out_offset + (uint64_t)st.row * jb.out_pitch);
  bool bad = size < 4u; // BitStreamer ctor: "Bit stream size is smaller than MaxProcessBytes"
  const uint32_t tmax = 32u * ((size + 8u) / 4u); // a pixel may start at bit T <= tmax
  uint32_t p = 0; // bit position in the row's stream
  uint32_t cur = 0, nxt = 0, q0 = 0, q1 = 0, q2 = 0, q3 = 0, q4 = 0;
  int32_t pred0 = 0, pred1 = 0;
  uint32_t len0 = 0, len1 = 0, even = 0;
  auto getbits = [&](uint32_t n) { // 1 <= n <= 16
    const uint32_t v = __funnelshift_l(nxt, cur, p) >> (32u - n);
    const uint32_t pn = p + n;
    if ((pn ^ p) & 32u) { // into the next chunk
      cur = nxt;
      nxt = q0;
      q0 = q1;
      q1 = q2;
      q2 = q3;
      q3 = q4;
    }
    p = pn;
    return v;
  };
  const uint32_t lim = w & ~7u;
  for (uint32_t col = 0; col < w; ++col) {
    if ((col & 7u) == 0u) { // group boundary: chunks p/32 .. p/32 + 6, for every lane
      const uint32_t c0 = p >> 5;
      cur = p1_chunk(base, size, 4u * c0);
      nxt = p1_chunk(base, size, 4u * c0 + 4u);
      q0 = p1_chunk(base, size, 4u * c0 + 8u);
      q1 = p1_chunk(base, size, 4u * c0 + 12u);
      q2 = p1_chunk(base, size, 4u * c0 + 16u);
      q3 = p1_chunk(base, size, 4u * c0 + 20u);
      q4 = p1_chunk(base, size, 4u * c0 + 24u);
    }
    if (p > tmax) // pump.fill(32) of this pixel would read past size + 8
      bad = true;
    if (col >= lim) {
      len0 = len1 = 14;
    } else if ((col & 7u) == 0u) {
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        uint32_t j = 0;
        for (; j < 5; ++j) {
          if (getbits(1) != 0u) {
            if (col == 0)
              bad = true; // "Can not initialize lengths. Data is corrupt."
            break;
          }
        }
        if (j > 0) {
          const uint32_t idx = 2u * (j - 1u) + getbits(1);
          const uint32_t l = (uint32_t)((0xDEC5AB9678ull >> (4u * idx)) & 15u);
          if (t == 0)
            len0 = l;
          else
            len1 = l;
        }
      }
    }
    uint32_t i = (col & 1u) ? len1 : len0;
    if (i == 0u) // (only after an error at column 0: keep the arithmetic defined)
      i = 14u;
    int32_t& pred = (col & 1u) ? pred1 : pred0;
    if (i == 14u)
      pred = (int32_t)getbits(16);
    else
      pred += (int32_t)getbits(i) + 1 - (1 << (i - 1u));
    if (col & 1u) {
      if (live && !bad)
        o32[col >> 1] = even | ((uint32_t)pred << 16);
    } else {
      even = (uint32_t)pred & 0xFFFFu;
    }
  }
  if (bad && live)
    atomicOr(bad_jobs + st.job, 1u);
}

#endif // !RSB200_EMU (the first two versions have no CPU replay; the third is developed against one)

// ---- third version (round 2): the pixels of a row in parallel ----
// One thread per row leaves the machine almost empty (a 101 MP frame has 8708 rows: 272 warps on 148
// SMs, every one walking 11608 pixels one after the other: 3.9 ms, 26 GPix/s).  What is serial in a
// row is only WHERE its groups of 8 pixels start: the two length codes in front of a group (2 .. 12
// bits) say how long it is.  So the row is decoded in two steps:
//   p1_walk_kernel    one thread per row reads nothing but the group headers and writes, per group,
//                     one word: bit position of its first pixel | len0 | len1 | header bits
//                     (1451 short steps per row instead of 11608 long ones);
//   p1_decode_kernel  one warp per row, 32 groups per step: the bytes of the 32 groups are staged in
//                     shared memory with coalesced loads, a lane extracts the 8 fields of its group,
//                     and the predictors -- "pred += difference" per column parity, restarted by every
//                     group whose length is 14 (raw 16-bit values) -- become a segmented warp scan over
//                     (restarts, sum) pairs with a carry from step to step; a lane stores its 8 pixels.
// The over-read rule in closed form as in the second version: a pixel may start at bit T <= tmax = 32 *
// ((size + 8) / 4) (the group's first pixel is checked where its header starts); positions grow along
// the row, so a pair is stored iff its second pixel passes, and the row has failed iff its last pixel
// does not.  A 1 bit in the length prefixes at column 0, or a strip below 4 bytes, fails the row before
// anything is stored.
constexpr int P1W_NT = 64;          // walk: rows per CTA
constexpr int P1D_NT = 128;         // decode: 4 warps = 4 rows per CTA
constexpr int P1_STAGE_WORDS = 148; // 32 groups x (12 + 8 x 16) bits = 140 words, + the funnel's second word
constexpr uint32_t P1_POS_MASK = 0xFFFFFu; // a row has < 2^20 bits (width <= 11976: 209 580)

// 32 bits of the strip from bit p (MSB32 order: 32-bit little-endian chunks, most significant bit first)
__device__ __forceinline__ uint32_t p1_window(const uint8_t* __restrict__ base, uint32_t size, uint32_t p) {
  const uint32_t c = p >> 5;
  return __funnelshift_l(p1_chunk(base, size, 4u * c + 4u), p1_chunk(base, size, 4u * c), p);
}
__device__ __forceinline__ uint32_t p1_bits_of_len(uint32_t len) { return (len == 14u || len == 0u) ? 16u : len; }

// one length code at the top of x: .x = bits used, .y = new length (0: keep), .z = a 1 bit was met
// before five zeros (fatal at column 0).  PhaseOneDecompressor.cpp:104-118
__device__ __forceinline__ void p1_len_code(uint32_t x, uint32_t& used, uint32_t& len, bool& one) {
  const uint32_t j = (uint32_t)min(__clz((int)x), 5);
  one = j < 5u;
  if (j == 0u) {
    used = 1u;
    return;
  }
  // j zeros, (the 1 that ended them when j < 5), one more bit: length[2 * (j - 1) + bit]
  used = j < 5u ? j + 2u : 6u;
  const uint32_t bit = (x >> (32u - used)) & 1u;
  const uint32_t idx = 2u * (j - 1u) + bit;
  len = (uint32_t)((0xDEC5AB9678ull >> (4u * idx)) & 15u);
}

// the same without control flow (the walk is one dependent chain per row with about two warps per SM:
// every branch and every instruction on the chain is paid in full)
__device__ __forceinline__ void p1_len_code_bf(uint32_t x, uint32_t& used, uint32_t& len, bool& one) {
  const uint32_t j = (uint32_t)min(__clz((int)x), 5);
  one = j < 5u;
  used = j == 0u ? 1u : (j < 5u ? j + 2u : 6u);
  const uint32_t bit = (x >> (32u - used)) & 1u;
  const uint32_t idx = j == 0u ? 0u : 2u * (j - 1u) + bit;
  const uint32_t nl = (uint32_t)((0xDEC5AB9678ull >> (4u * idx)) & 15u);
  len = j == 0u ? len : nl;
}

// FAST: the window comes from three aligned words where they lie wholly inside the strip (all but the last
// groups of a row), and the length codes are decoded without branches; !FAST: the first form of the walk
// (generic chunk loads, branches), kept for A/B runs (RSB200_P1W=1).  The first form needs about 170
// instructions per group on a chain nobody hides.
// A length code is decided by the 6 bits at the top of the window: 64 entries, bits used | a 1 bit came
// before five zeros << 3 | new length << 4 (0: keep) -- one shared-memory load instead of a dozen
// dependent instructions.
constexpr int P1W_RING = 64;   // words per row in shared memory: two lines of 128 bytes (form "lines")
constexpr int P1W_RING4 = 128; // ... four lines (form "cadence"; rows 16-byte aligned for 128-bit stores)
struct P1WalkShared {
  uint32_t code6[64];
  union {
    uint32_t ring[P1W_NT][P1W_RING + 1]; // (+1: the rows of a warp start in different banks)
    uint4 ring4[P1W_NT][P1W_RING4 / 4 + 1];
  };
};

// TOUCH: every step also loads one word 192 bytes further down the row and uses it a step later (an XOR
// into a value nobody needs): L1 is filled sector by sector on demand, and a row advances about half a
// sector per group, so without it every second step waits for L2 and every fourth for DRAM, with nothing
// else on the SM to run meanwhile.  The touch is ten steps ahead.
__device__ __forceinline__ void p1_prefetch(const void* q, int level) {
#ifndef RSB200_EMU
  if (level == 1)
    asm volatile("prefetch.global.L1 [%0];" ::"l"(q));
  else
    asm volatile("prefetch.global.L2 [%0];" ::"l"(q));
#else
  (void)q;
  (void)level;
#endif
}

// TOUCH: 0 nothing, 1 the look-ahead load described above, 2 prefetch.global.L1 192 bytes ahead, 3
// prefetch.global.L2 512 bytes ahead + prefetch.global.L1 128 bytes ahead (no register waits for either),
// 4 "blocks": form 3 spends most of its cycles waiting for the three
// lane-private window loads of every step although most of their sectors hit L1.  So the row is read in
// aligned 16-byte blocks, two of them cached in registers (one 128-bit load every three to four steps, a
// prefetch 192 bytes ahead at the same moment), the window's three words are selected from the eight
// cached ones, and four descriptor words leave with one 128-bit store.  5 "lines": the row is read in
// aligned lines of 128 bytes (eight 128-bit loads issued together, consumed a whole line -- about seven
// steps -- later), two lines per row wait in shared memory and the window comes from there: the walk's
// chain holds shared-memory loads only.  6 "cadence": in "lines" the rows of a warp cross
// their line boundaries at different steps, so SOME lane refills at nearly every step, the whole warp runs
// the refill code (twice the instructions) and -- the scoreboard of a load's destination register being
// per warp -- every store of a pending line waits for the loads another lane issued a step ago.  So every
// lane refills at the SAME steps, every fourth (a row advances at most 70 bytes in four steps, a refill
// brings 128): a ring of four lines per row, the line loaded at one refill point is stored at the next.
template <bool FAST, int TOUCH>
__device__ __forceinline__ void
p1_walk_entry(P1WalkShared& sh, const uint8_t* __restrict__ in, const P1StripDev* __restrict__ strips,
              uint32_t nstrips, const P1JobDev* __restrict__ jobs, uint32_t gstride,
              uint32_t* __restrict__ gdesc, uint32_t* __restrict__ rowflag) {
  if (FAST) {
    for (uint32_t i = threadIdx.x; i < 64u; i += blockDim.x) {
      uint32_t used, len = 0;
      bool one;
      p1_len_code_bf(i << 26, used, len, one);
      sh.code6[i] = used | (one ? 8u : 0u) | (len << 4);
    }
    __syncthreads();
  }
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nstrips)
    return;
  const P1StripDev st = strips[s];
  const P1JobDev jb = jobs[st.job];
  const uint8_t* base = in + st.in_offset;
  const uint32_t size = st.in_size;
  const uint32_t ngroups = jb.width >> 3;
  uint32_t* desc = gdesc + (uint64_t)s * gstride;
  if (size < 4u) { // BitStreamer ctor: "Bit stream size is smaller than MaxProcessBytes"
    rowflag[s] = 1u;
    return;
  }
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(base) & 3u);
  const uint32_t* aw = reinterpret_cast<const uint32_t*>(base - mis); // (inside the caller's buffer: its start is aligned)
  const uint32_t sh8 = 8u * mis;
  uint32_t p = 0, len0 = 0, len1 = 0;
  bool fatal = false;
  const uint32_t wlast = (size - 1u + mis) >> 2; // the last aligned word that holds a byte of the strip
  uint32_t touched = 0, sink = 0;
  // TOUCH == 4: blocks of 16 bytes from the 16-byte boundary at or before the strip
  const uint32_t mis16 = (uint32_t)(reinterpret_cast<uintptr_t>(base) & 15u);
  const uint4* a16 = reinterpret_cast<const uint4*>(base - mis16);
  const uint32_t woff = mis16 >> 2;                   // aligned word of byte 0, counted from a16
  const uint32_t blast = (mis16 + size - 1u) >> 4;    // the last block that holds a byte of the strip
  uint32_t B = 0;                                     // b0 .. b3 = blocks B .. B + 3 (where they exist)
  uint4 b0 = make_uint4(0, 0, 0, 0), b1 = b0, b2 = b0, b3 = b0;
  uint32_t q0 = 0, q1 = 0, q2 = 0;                    // descriptor words waiting for the fourth
  // TOUCH == 5: lines of 128 bytes from the 128-byte boundary at or before the strip
  const uint32_t mis128 = (uint32_t)(reinterpret_cast<uintptr_t>(base) & 127u);
  const uint4* a128 = reinterpret_cast<const uint4*>(base - mis128);
  const uint32_t woff128 = mis128 >> 2;
  const uint32_t blast128 = (mis128 + size - 1u) >> 4; // the last 16-byte block (from a128) with a byte of the strip
  uint32_t* ring = sh.ring[threadIdx.x];
  uint32_t L = 0;                                      // ring: lines L and L + 1; pend: line L + 2
  uint4 pend[8];
  if (TOUCH == 5) {
#pragma unroll
    for (uint32_t i = 0; i < 16u; ++i) {
      const uint4 v = __ldg(a128 + min(i, blast128));
      ring[4u * i] = v.x;
      ring[4u * i + 1u] = v.y;
      ring[4u * i + 2u] = v.z;
      ring[4u * i + 3u] = v.w;
    }
#pragma unroll
    for (uint32_t i = 0; i < 8u; ++i)
      pend[i] = __ldg(a128 + min(16u + i, blast128));
  }
  // TOUCH == 6: ring4 = lines [Lc, Lf) of the row, pend = line Lf (asked for at the last refill point)
  uint4* ring4 = sh.ring4[threadIdx.x];
  uint32_t Lf = 0;
  if (TOUCH == 6) {
#pragma unroll
    for (uint32_t i = 0; i < 24u; ++i) // three lines to start with
      ring4[i] = __ldg(a128 + min(i, blast128));
    Lf = 3;
#pragma unroll
    for (uint32_t i = 0; i < 8u; ++i)
      pend[i] = __ldg(a128 + min(24u + i, blast128));
  }
  if (TOUCH == 4) {
    b0 = __ldg(a16);
    b1 = __ldg(a16 + min(1u, blast));
    b2 = __ldg(a16 + min(2u, blast));
    b3 = __ldg(a16 + min(3u, blast));
  }
  for (uint32_t g = 0; g < ngroups; ++g) {
    uint32_t x;
    const uint32_t c = p >> 5;
    const uint32_t ca = c + woff, k = ca & 3u;
    if (TOUCH == 4) {
      // (a group is at most 140 bits: one or two blocks further.  The block loaded here is used two
      //  blocks -- about seven steps -- later: run 30 showed that a block fetched one step before its use
      //  is waited for just like the window loads of the other forms)
      while (B < (ca >> 2)) {
        ++B;
        b0 = b1;
        b1 = b2;
        b2 = b3;
        b3 = __ldg(a16 + min(B + 3u, blast));
        p1_prefetch(a16 + min(B + 16u, blast), 2);
      }
    }
    if (TOUCH == 1) {
      sink ^= touched;
      touched = __ldg(aw + min(c + 48u, wlast));
    } else if (TOUCH == 2) {
      p1_prefetch(aw + min(c + 48u, wlast), 1);
    } else if (TOUCH == 3) {
      p1_prefetch(aw + min(c + 128u, wlast), 2);
      p1_prefetch(aw + min(c + 32u, wlast), 1);
    }
    if (TOUCH == 5) {
      const uint32_t cl = c + woff128;
      if ((cl >> 5) > L) { // into line L + 1: line L + 2 replaces line L, line L + 3 is asked for
        ++L;
        uint32_t* slot = ring + 32u * ((L + 1u) & 1u);
#pragma unroll
        for (uint32_t i = 0; i < 8u; ++i) {
          slot[4u * i] = pend[i].x;
          slot[4u * i + 1u] = pend[i].y;
          slot[4u * i + 2u] = pend[i].z;
          slot[4u * i + 3u] = pend[i].w;
        }
#pragma unroll
        for (uint32_t i = 0; i < 8u; ++i)
          pend[i] = __ldg(a128 + min(8u * (L + 2u) + i, blast128));
        p1_prefetch(a128 + min(8u * (L + 6u), blast128), 2);
      }
    }
    if (TOUCH == 6 && (g & 3u) == 0u && g != 0u) { // refill point (the same step for every row of the warp)
      const uint32_t Lc = (c + woff128) >> 5;
      if (Lf - Lc < 4u) { // the slot of line Lf is free (it held line Lf - 4 < Lc)
        uint4* slot = ring4 + 8u * (Lf & 3u);
#pragma unroll
        for (uint32_t i = 0; i < 8u; ++i)
          slot[i] = pend[i];
        ++Lf;
#pragma unroll
        for (uint32_t i = 0; i < 8u; ++i)
          pend[i] = __ldg(a128 + min(8u * Lf + i, blast128));
        p1_prefetch(a128 + min(8u * (Lf + 4u), blast128), 2);
      }
    }
    if (FAST && TOUCH == 6 && 4u * c + 16u <= size) {
      // (the window's words hold strip bytes only; their lines are in the ring: a row is at most 70 bytes
      //  further at the next refill point, and at least two whole lines lie ahead of it after each)
      const uint32_t cl = c + woff128;
      const uint32_t* r32 = reinterpret_cast<const uint32_t*>(ring4);
      const uint32_t a0 = r32[cl & 127u], a1 = r32[(cl + 1u) & 127u], a2 = r32[(cl + 2u) & 127u];
      x = __funnelshift_l(__funnelshift_r(a1, a2, sh8), __funnelshift_r(a0, a1, sh8), p);
    } else if (FAST && TOUCH == 5 && 4u * c + 16u <= size) {
      // (the three words hold strip bytes only: their lines are L or L + 1, loaded without clamping)
      const uint32_t cl = c + woff128;
      const uint32_t a0 = ring[cl & 63u], a1 = ring[(cl + 1u) & 63u], a2 = ring[(cl + 2u) & 63u];
      x = __funnelshift_l(__funnelshift_r(a1, a2, sh8), __funnelshift_r(a0, a1, sh8), p);
    } else if (FAST && TOUCH == 4 && 4u * c + 16u <= size) {
      // (the three words hold strip bytes only, so their blocks exist: b1 is block B + 1 if it is needed)
      const uint32_t a0 = k == 0u ? b0.x : (k == 1u ? b0.y : (k == 2u ? b0.z : b0.w));
      const uint32_t a1 = k == 0u ? b0.y : (k == 1u ? b0.z : (k == 2u ? b0.w : b1.x));
      const uint32_t a2 = k == 0u ? b0.z : (k == 1u ? b0.w : (k == 2u ? b1.x : b1.y));
      x = __funnelshift_l(__funnelshift_r(a1, a2, sh8), __funnelshift_r(a0, a1, sh8), p);
    } else if (FAST && 4u * c + 16u <= size) { // the bytes [4c - mis, 4c - mis + 12) lie inside the strip
      const uint32_t a0 = __ldg(aw + c), a1 = __ldg(aw + c + 1u), a2 = __ldg(aw + c + 2u);
      x = __funnelshift_l(__funnelshift_r(a1, a2, sh8), __funnelshift_r(a0, a1, sh8), p);
    } else {
      x = p1_window(base, size, p);
    }
    uint32_t u0, u1;
    bool o0, o1;
    if (FAST) {
      const uint32_t e0 = sh.code6[x >> 26];
      u0 = e0 & 7u;
      const uint32_t e1 = sh.code6[(x << u0) >> 26];
      u1 = e1 & 7u;
      o0 = (e0 & 8u) != 0u;
      o1 = (e1 & 8u) != 0u;
      len0 = (e0 >> 4) ? (e0 >> 4) : len0;
      len1 = (e1 >> 4) ? (e1 >> 4) : len1;
    } else {
      p1_len_code(x, u0, len0, o0);
      p1_len_code(x << u0, u1, len1, o1);
    }
    if (g == 0u && (o0 || o1))
      fatal = true; // "Can not initialize lengths. Data is corrupt."
    const uint32_t hdr = u0 + u1, p0 = p + hdr;
    const uint32_t dv = (p0 & P1_POS_MASK) | (len0 << 20) | (len1 << 24) | (hdr << 28);
    if (TOUCH == 4) { // (rows of descriptors start at multiples of 16 bytes: gstride is a multiple of 4)
      const uint32_t gk = g & 3u;
      if (gk == 3u)
        *reinterpret_cast<uint4*>(desc + g - 3u) = make_uint4(q0, q1, q2, dv);
      q0 = gk == 0u ? dv : q0;
      q1 = gk == 1u ? dv : q1;
      q2 = gk == 2u ? dv : q2;
    } else {
      desc[g] = dv;
    }
    p = p0 + 4u * (p1_bits_of_len(len0) + p1_bits_of_len(len1));
  }
  if (TOUCH == 4) { // the descriptors of the last ngroups % 4 groups
    const uint32_t rest = ngroups & 3u, g4 = ngroups & ~3u;
    if (rest >= 1u)
      desc[g4] = q0;
    if (rest >= 2u)
      desc[g4 + 1u] = q1;
    if (rest >= 3u)
      desc[g4 + 2u] = q2;
  }
  desc[ngroups] = p; // where the last width % 8 pixels (raw) start
  // (bit 1 is never set: the touched words only have to be used by something)
  rowflag[s] = (fatal ? 1u : 0u) | (TOUCH == 1 && (sink ^ touched) == 0x5EC7095Eu && p == 0xFFFFFFFFu ? 2u : 0u);
}

struct P1DecodeShared {
  uint32_t stage[P1D_NT / 32][P1_STAGE_WORDS];
};

// 1 <= n <= 16 bits at bit `rel` of the staged words
__device__ __forceinline__ uint32_t p1_field(const uint32_t* stage, uint32_t rel, uint32_t n) {
  const uint32_t wi = rel >> 5;
  return __funnelshift_l(stage[wi + 1u], stage[wi], rel) >> (32u - n);
}

// inclusive segmented scan over the lanes of (restart, value): a lane's result is absolute when some
// lane at or before it restarted, else a sum still to be added to the carry of the step before
__device__ __forceinline__ void p1_seg_scan(uint32_t& r, uint32_t& a, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t ru = __shfl_up_sync(0xFFFFFFFFu, r, d);
    const uint32_t au = __shfl_up_sync(0xFFFFFFFFu, a, d);
    if (lane >= d) {
      if (!r)
        a += au;
      r |= ru;
    }
  }
}

__device__ __forceinline__ void
p1_decode_entry(P1DecodeShared& sh, const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                const P1StripDev* __restrict__ strips, uint32_t nstrips, const P1JobDev* __restrict__ jobs,
                uint32_t gstride, const uint32_t* __restrict__ gdesc, const uint32_t* __restrict__ rowflag,
                uint32_t* __restrict__ bad_jobs) {
  const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = (int)(threadIdx.x & 31u);
  if (s >= nstrips)
    return;
  const P1StripDev st = strips[s];
  const P1JobDev jb = jobs[st.job];
  if (rowflag[s]) {
    if (lane == 0)
      atomicOr(bad_jobs + st.job, 1u);
    return;
  }
  const uint8_t* base = in + st.in_offset;
  const uint32_t size = st.in_size, w = jb.width;
  const uint32_t ngroups = w >> 3;
  const uint32_t tmax = 32u * ((size + 8u) / 4u);
  const uint32_t* desc = gdesc + (uint64_t)s * gstride;
  uint32_t* o32 = reinterpret_cast<uint32_t*>(out + jb.out_offset + (uint64_t)st.row * jb.out_pitch);
  uint32_t* stage = sh.stage[threadIdx.x >> 5];
  uint32_t run0 = 0, run1 = 0; // the two predictors behind the groups done so far
  bool over = false;
  for (uint32_t g0 = 0; g0 < ngroups; g0 += 32u) {
    const uint32_t g = g0 + (uint32_t)lane;
    const bool have = g < ngroups;
    const uint32_t d = have ? __ldg(desc + g) : 0u;
    const uint32_t p0 = d & P1_POS_MASK, l0 = (d >> 20) & 15u, l1 = (d >> 24) & 15u, hdr = d >> 28;
    const uint32_t b0 = p1_bits_of_len(l0), b1 = p1_bits_of_len(l1);
    const uint32_t pend = p0 + 4u * (b0 + b1);
    // the words that hold the groups of this step
    const uint32_t nhere = min(32u, ngroups - g0);
    const uint32_t wfirst = __shfl_sync(0xFFFFFFFFu, p0, 0) >> 5;
    const uint32_t wlast = (__shfl_sync(0xFFFFFFFFu, pend, (int)nhere - 1) + 31u) >> 5;
    __syncwarp();
    for (uint32_t i = (uint32_t)lane; i <= wlast - wfirst + 1u; i += 32u)
      stage[i] = p1_chunk(base, size, 4u * (wfirst + i));
    __syncwarp();
    uint32_t c[8];
    uint32_t tlast = 0, t1 = 0, t3 = 0, t5 = 0;
    {
      uint32_t rel = p0 - 32u * wfirst;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint32_t n = (k & 1) ? b1 : b0, len = (k & 1) ? l1 : l0;
        uint32_t v = have ? p1_field(stage, rel, n) : 0u;
        if (n != 16u)
          v = v + 1u - (1u << (len - 1u));
        c[k] = v;
        if (k == 1) t1 = rel;
        if (k == 3) t3 = rel;
        if (k == 5) t5 = rel;
        if (k == 7) tlast = rel;
        rel += n;
      }
    }
    const uint32_t off = 32u * wfirst; // (positions of the odd pixels, for the over-read rule)
    t1 += off; t3 += off; t5 += off; tlast += off;
    (void)hdr;
    // per parity: prefix inside the group, then the scan over the groups
    const uint32_t raw0 = (have && b0 == 16u) ? 1u : 0u, raw1 = (have && b1 == 16u) ? 1u : 0u;
    if (!raw0) {
      c[2] += c[0];
      c[4] += c[2];
      c[6] += c[4];
    }
    if (!raw1) {
      c[3] += c[1];
      c[5] += c[3];
      c[7] += c[5];
    }
    uint32_t r0 = raw0, a0 = have ? c[6] : 0u, r1 = raw1, a1 = have ? c[7] : 0u;
    p1_seg_scan(r0, a0, lane);
    p1_seg_scan(r1, a1, lane);
    // what the predictors hold behind lane i: absolute after a restart, else carry + sum
    const uint32_t out0 = r0 ? a0 : run0 + a0, out1 = r1 ? a1 : run1 + a1;
    uint32_t base0 = __shfl_up_sync(0xFFFFFFFFu, out0, 1), base1 = __shfl_up_sync(0xFFFFFFFFu, out1, 1);
    if (lane == 0) {
      base0 = run0;
      base1 = run1;
    }
    run0 = __shfl_sync(0xFFFFFFFFu, out0, 31);
    run1 = __shfl_sync(0xFFFFFFFFu, out1, 31);
    if (have) {
      if (!raw0) {
        c[0] += base0;
        c[2] += base0;
        c[4] += base0;
        c[6] += base0;
      }
      if (!raw1) {
        c[1] += base1;
        c[3] += base1;
        c[5] += base1;
        c[7] += base1;
      }
      uint32_t* o = o32 + 4u * g;
      if (t1 <= tmax)
        o[0] = (c[0] & 0xFFFFu) | (c[1] << 16);
      if (t3 <= tmax)
        o[1] = (c[2] & 0xFFFFu) | (c[3] << 16);
      if (t5 <= tmax)
        o[2] = (c[4] & 0xFFFFu) | (c[5] << 16);
      if (tlast <= tmax)
        o[3] = (c[6] & 0xFFFFu) | (c[7] << 16);
      over = over || tlast > tmax;
    }
  }
  // the last width % 8 pixels: raw 16-bit values (an even number: the width is even)
  const uint32_t ntail = w & 7u;
  if ((uint32_t)lane * 2u < ntail) {
    const uint32_t pt = __ldg(desc + ngroups) + 32u * (uint32_t)lane; // my pair
    const uint32_t a = p1_window(base, size, pt) >> 16, b = p1_window(base, size, pt + 16u) >> 16;
    if (pt + 16u <= tmax)
      o32[4u * ngroups + (uint32_t)lane] = a | (b << 16);
    over = over || pt + 16u > tmax;
  }
  if (__ballot_sync(0xFFFFFFFFu, over) != 0u && lane == 0)
    atomicOr(bad_jobs + st.job, 1u);
}

#ifndef RSB200_EMU
__global__ void __launch_bounds__(P1W_NT)
    p1_walk_kernel(const uint8_t* __restrict__ in, const P1StripDev* __restrict__ strips, uint32_t nstrips,
                   const P1JobDev* __restrict__ jobs, uint32_t gstride, uint32_t* __restrict__ gdesc,
                   uint32_t* __restrict__ rowflag, int first_form) {
  __shared__ P1WalkShared sh;
  // 0 (default) = 7: "lines" (128-byte lines through a per-row ring in shared memory), the form chosen
  // during development; the forms have not been compared on H100
  if (first_form == 1)
    p1_walk_entry<false, 0>(sh, in, strips, nstrips, jobs, gstride, gdesc, rowflag);
  else if (first_form == 2)
    p1_walk_entry<true, 0>(sh, in, strips, nstrips, jobs, gstride, gdesc, rowflag);
  else if (first_form == 3)
    p1_walk_entry<true, 2>(sh, in, strips, nstrips, jobs, gstride, gdesc, rowflag);
  else if (first_form == 4)
    p1_walk_entry<true, 3>(sh, in, strips, nstrips, jobs, gstride, gdesc, rowflag);
  else if (first_form == 5)
    p1_walk_entry<true, 1>(sh, in, strips, nstrips, jobs, gstride, gdesc, rowflag);
  else if (first_form == 6)
    p1_walk_entry<true, 4>(sh, in, strips, nstrips, jobs, gstride, gdesc, rowflag);
  else
    p1_walk_entry<true, 5>(sh, in, strips, nstrips, jobs, gstride, gdesc, rowflag);
}
__global__ void __launch_bounds__(P1D_NT)
    p1_decode_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                     const P1StripDev* __restrict__ strips, uint32_t nstrips,
                     const P1JobDev* __restrict__ jobs, uint32_t gstride, const uint32_t* __restrict__ gdesc,
                     const uint32_t* __restrict__ rowflag, uint32_t* __restrict__ bad_jobs) {
  __shared__ P1DecodeShared sh;
  p1_decode_entry(sh, in, out, strips, nstrips, jobs, gstride, gdesc, rowflag, bad_jobs);
}
#endif

} // namespace rsb200
