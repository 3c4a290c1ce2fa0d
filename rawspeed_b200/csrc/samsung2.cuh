// samsung2.cuh -- Samsung SRW V2 row codec (SamsungV2Decompressor), sm_90a.
//
// Replaces SamsungV2Decompressor::decompress (decompressors/SamsungV2Decompressor.cpp:145-355).  Two
// dependencies are serial in the reference and are broken here:
//  * Row starts are implicit: a row's MSB32 stream starts at the first multiple of 16 bytes (from the
//    start of the data) at or after ceil(bits / 8) of the row before.  Only such positions can start
//    a row, so every one of them is walked speculatively, once per row class, reading block headers
//    only (a difference section is skipped as 4 * the sum of its lengths).  The bit lengths depend on
//    nothing but the four lengths of the last block that was not skipped, the row parity and whether
//    the row is 0 or 1, so a walk from a candidate is exact whatever came before.
//  * Reconstruction is a DAG with clamps: a block with motion 7 starts from the last two pixels of the
//    block to its left (initVal at column 0), the others from one or two rows up (maybe averaged),
//    and every pixel is clamped to the bit depth.  Rows go one after the other in one CTA per frame;
//    inside a row the two left chains (one per parity) are a scan of clamp-add maps
//    x -> min(max(x + a, lo), hi), which are closed under composition.
//
// Stages (one launch each for all frames of a plan):
//   s2_cand_kernel    a thread per (frame, class, 16-byte candidate): the header walk of one row from
//                     there -> the candidate of the next row, or the failure (code, value, block)
//   s2_pair_kernel    the two-row step even -> odd -> next even start, per candidate
//   s2_double_kernel  S2_JUMP rounds of pointer doubling on it (failures absorb)
//   s2_coarse_kernel  a thread per frame: rows 0 and 1, then a checkpoint every S2_CHUNK rows
//   s2_fine_kernel    a thread per checkpoint: every row start of its chunk, and the frame's failure
//   s2_desc_kernel    a thread per true row: the walk again, writing one descriptor per block
//   s2_diff_kernel    a CTA per row: every difference, sign-extended and put in pixel order
//   s2_recon_kernel   a CTA per frame: rows in order through a ring of three rows in shared memory
// No index is taken from the stream without a bound: candidate entries stay within 0..ncand, motions
// that would reach outside the rows fail in the walk (and the ring reads are clamped besides).
#pragma once

#ifndef RSB200_EMU
#include "common.cuh"
#endif
#include "phaseone.cuh" // p1_window: 32 bits of an MSB32 strip from any bit, zero past its end
#include <stdint.h>
#include <string.h>

namespace rsb200 {

constexpr int S2W_NT = 128;  // candidate walk / descriptor walk: threads per CTA
constexpr int S2J_NT = 256;  // pair, doubling, coarse and fine steps
constexpr int S2_JUMP = 5;   // doubling rounds: a jump covers 2^S2_JUMP row pairs
constexpr uint32_t S2_CHUNK = 2u << S2_JUMP; // rows per checkpoint
constexpr int S2X_NT = 256;  // differences: a CTA per row
constexpr int S2R_NT = 512;  // reconstruction: a CTA per frame (one thread per block: nb <= 406)
constexpr int S2_MAXW = 6496;
constexpr uint32_t S2_FAIL = 1u << 31; // candidate entry: S2_FAIL | code << 27 | value << 22 | block
constexpr uint32_t S2F_START_MOTION = 1, S2F_MOTION_BEGIN = 2, S2F_MOTION_END = 3, S2F_UNDERFLOW = 4,
                   S2F_TOO_MANY = 5, S2F_OVERREAD = 6, S2F_SHORT = 7, S2F_BYTESTREAM = 8;
constexpr uint32_t S2_SKIP = 1, S2_MV = 2, S2_QP = 4;

struct S2FrameDev {
  uint64_t in_offset;  // first byte of the data (behind the 16-byte header)
  uint64_t out_offset;
  uint64_t tab_base;   // first candidate entry: classes 0, 1, 2 of (ncand + 1) each, then row 0
  uint64_t desc_base;  // first block descriptor (h * nb)
  uint64_t px_base;    // first difference (h * w)
  uint32_t size;       // data bytes
  uint32_t out_pitch;
  uint32_t w, h, nb, flags, init, bits;
  uint32_t ncand;      // candidates c < ncand start at 16 c <= size; c == ncand lies past the end
  uint32_t jump_base;  // first pair-step entry (ncand + 1)
  uint32_t row_base;   // first row start (sum of the heights before)
  uint32_t cp_base;    // first checkpoint (ceil(h / S2_CHUNK))
};

// Host side: bits [pos, pos + n) of the 16-byte header read as MSB32 (SamsungV2Decompressor.cpp:103-131)
inline uint32_t s2_header_bits(const uint8_t* hd, uint32_t pos, uint32_t n) {
  uint32_t v = 0;
  for (uint32_t b = pos; b < pos + n; ++b) {
    const uint8_t* w = hd + 4 * (b >> 5);
    const uint32_t word = (uint32_t)w[0] | (uint32_t)w[1] << 8 | (uint32_t)w[2] << 16 | (uint32_t)w[3] << 24;
    v = v << 1 | ((word >> (31u - (b & 31u))) & 1u);
  }
  return v;
}

// Host side: a plan's scratch so far (entries of each table)
struct S2Totals {
  uint64_t tab = 0, jump = 0, rows = 0, cps = 0, desc = 0, px = 0;
};

// Host side: one frame's descriptor from a strip whose header the constructor accepted, placed behind
// the frames before it in every scratch table; `starts` (four per-frame searches of nf each: candidate
// entries, pair steps, rows, checkpoints) gets its first indices.
inline void s2_place_frame(S2FrameDev& f, S2Totals& t, uint32_t* starts, uint32_t nf, uint32_t i, uint64_t in_offset,
                           uint32_t in_size, const uint8_t* header, uint32_t bits, uint32_t w, uint32_t h,
                           uint64_t out_offset, uint32_t out_pitch) {
  memset(&f, 0, sizeof f);
  f.in_offset = in_offset + 16;
  f.out_offset = out_offset;
  f.out_pitch = out_pitch;
  f.size = in_size - 16;
  f.w = w;
  f.h = h;
  f.nb = w / 16;
  f.flags = s2_header_bits(header, 84, 4);
  f.init = s2_header_bits(header, 114, 14);
  f.bits = bits;
  f.ncand = f.size / 16 + 1;
  starts[i] = (uint32_t)t.tab;
  starts[nf + i] = (uint32_t)t.jump;
  starts[2 * nf + i] = (uint32_t)t.rows;
  starts[3 * nf + i] = (uint32_t)t.cps;
  f.tab_base = t.tab;
  f.jump_base = (uint32_t)t.jump;
  f.row_base = (uint32_t)t.rows;
  f.cp_base = (uint32_t)t.cps;
  f.desc_base = t.desc;
  f.px_base = t.px;
  t.tab += 3ull * (f.ncand + 1) + 1;
  t.jump += f.ncand + 1;
  t.rows += f.h;
  t.cps += (f.h + S2_CHUNK - 1) / S2_CHUNK;
  t.desc += (uint64_t)f.h * f.nb;
  t.px += (uint64_t)f.h * f.w;
}

// the frame of flattened index x: the last f with starts[f] <= x (starts ascending, starts[0] == 0)
__device__ __forceinline__ uint32_t s2_frame_of(const uint32_t* __restrict__ starts, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1u) {
    const uint32_t mid = (lo + hi) >> 1;
    if (starts[mid] <= x)
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}

__device__ __forceinline__ uint32_t s2_fail(uint32_t code, uint32_t value, uint32_t block) {
  return S2_FAIL | code << 27 | value << 22 | block;
}

// The header walk of one row from candidate c (SamsungV2Decompressor.cpp:152-350 without the
// differences).  cls: 0 an even row >= 2, 1 an odd row >= 3, 2 row 1, 3 row 0.  -> the candidate of
// the next row's start, or a failure entry.  With DESC, desc[k] = (bit of block k's differences from
// the start of the data, lengths | motion << 16 | (scale + 256) << 19) for every block it passes.
// The pump (BitStreamer.h) refills 4 bytes when fewer bits are cached than an operation reads and
// throws when that refill starts more than 8 bytes behind the end: an operation fails iff it ends
// past lim = 32 ((size + 8) / 4 + 1); an operation of 0 bits reads nothing.
template <bool DESC>
__device__ __forceinline__ uint32_t s2_walk(const uint8_t* __restrict__ data, const S2FrameDev& f, uint32_t c,
                                            uint32_t cls, uint2* __restrict__ desc) {
  if (c >= f.ncand) // (the skip to this boundary passed the end)
    return s2_fail(S2F_BYTESTREAM, 0, 0);
  const uint32_t s = 16u * c, size = f.size - s;
  if (size < 4u) // BitStreamer constructor
    return s2_fail(S2F_SHORT, 0, 0);
  const uint8_t* base = data + s;
  const uint32_t lim = 32u * ((size + 8u) / 4u + 1u);
  const bool early = cls >= 2u;
  const uint32_t maxlen = f.bits + 1u;
  uint32_t prev = early ? 0x7777u : 0x4444u; // four lengths, 4 bits each
  uint32_t T = 0, motion = 7;
  int scale = 0;
#define S2_TAKE(n, v)                                                                                        \
  do {                                                                                                       \
    if (T + (n) > lim)                                                                                       \
      return s2_fail(S2F_OVERREAD, 0, k);                                                                    \
    v = p1_window(base, size, T) >> (32u - (n));                                                             \
    T += (n);                                                                                                \
  } while (0)
  for (uint32_t k = 0; k < f.nb; ++k) {
    uint32_t v;
    if (!(f.flags & S2_QP) && (k & 3u) == 0u) {
      S2_TAKE(2u, v);
      if (v < 3u) {
        scale += v == 1u ? -2 : (v == 2u ? 2 : 0);
      } else {
        S2_TAKE(12u, v);
        scale = (int)v;
      }
    }
    S2_TAKE(1u, v);
    if (f.flags & S2_MV) {
      motion = v ? 3u : 7u;
    } else if (!v) {
      S2_TAKE(3u, v);
      motion = v;
    }
    if (early && motion != 7u)
      return s2_fail(S2F_START_MOTION, 0, k);
    if (motion != 7u && (k == 0u || k + 1u == f.nb)) { // (only the first and last blocks reach outside)
      const int off = (int)((0x8644220u >> (4u * motion)) & 15u) - 4; // -4 -2 -2 0 0 2 4
      const bool avg = motion == 2u || motion == 4u;
      const uint32_t par = cls & 1u; // the row's parity (rows 0 and 1 never get here)
      for (uint32_t i = 0; i < 16u; ++i) {
        int rc = (int)(16u * k + i) + off;
        if (!((par + i) & 1u))
          rc += (i & 1u) ? -1 : 1;
        if (rc < 0)
          return s2_fail(S2F_MOTION_BEGIN, motion, k);
        if (rc >= (int)f.w || (avg && rc + 2 >= (int)f.w))
          return s2_fail(S2F_MOTION_END, motion, k);
      }
    }
    bool skip = false;
    if (!(f.flags & S2_SKIP)) {
      S2_TAKE(1u, v);
      skip = v != 0u;
    }
    uint32_t lens = 0, sum = 0;
    if (!skip) {
      uint32_t fl;
      S2_TAKE(8u, fl); // (four 2-bit reads: the first to fail ends past lim iff the 8 bits do)
      for (uint32_t i = 0; i < 4u; ++i) {
        const uint32_t code = (fl >> (6u - 2u * i)) & 3u, p = (prev >> (4u * i)) & 15u;
        uint32_t L;
        if (code == 0u) {
          L = p;
        } else if (code == 1u) {
          L = p + 1u;
        } else if (code == 2u) {
          if (p == 0u)
            return s2_fail(S2F_UNDERFLOW, 0, k);
          L = p - 1u;
        } else {
          S2_TAKE(4u, L);
        }
        if (L > maxlen)
          return s2_fail(S2F_TOO_MANY, L, k);
        lens |= L << (4u * i);
        sum += L;
      }
      prev = lens;
      if (sum && T + 4u * sum > lim)
        return s2_fail(S2F_OVERREAD, 0, k);
    }
    if (DESC)
      desc[k] = make_uint2(8u * s + T, lens | motion << 16 | (uint32_t)(scale + 256) << 19);
    T += 4u * sum;
  }
#undef S2_TAKE
  const uint32_t e = (T + 7u) / 8u; // BitStreamer::getStreamPosition, then ByteStream::skipBytes
  if (e > size)
    return s2_fail(S2F_BYTESTREAM, 0, f.nb);
  return (s + e + 15u) / 16u;
}

// ---- candidate walk: entry x of the flattened tables
__device__ __forceinline__ void s2_cand_entry(const uint8_t* __restrict__ in, const S2FrameDev* __restrict__ fr,
                                              const uint32_t* __restrict__ starts, uint32_t nf, uint32_t total,
                                              uint32_t* __restrict__ tab) {
  const uint32_t x = blockIdx.x * S2W_NT + threadIdx.x;
  if (x >= total)
    return;
  const uint32_t fi = s2_frame_of(starts, nf, x);
  const S2FrameDev f = fr[fi];
  const uint32_t i = x - (uint32_t)f.tab_base, n1 = f.ncand + 1u;
  const uint32_t cls = i / n1, c = cls < 3u ? i - cls * n1 : 0u;
  tab[x] = s2_walk<false>(in + f.in_offset, f, c, cls, nullptr);
}

// ---- the two-row step: even row at c, odd row behind it -> the next even row's candidate
__device__ __forceinline__ void s2_pair_entry(const S2FrameDev* __restrict__ fr, const uint32_t* __restrict__ starts,
                                              uint32_t nf, uint32_t total, const uint32_t* __restrict__ tab,
                                              uint32_t* __restrict__ jump) {
  const uint32_t x = blockIdx.x * S2J_NT + threadIdx.x;
  if (x >= total)
    return;
  const S2FrameDev f = fr[s2_frame_of(starts, nf, x)];
  const uint32_t* t = tab + f.tab_base;
  const uint32_t e = t[x - f.jump_base];
  jump[x] = (e & S2_FAIL) ? S2_FAIL : t[f.ncand + 1u + e];
}

__device__ __forceinline__ void s2_double_entry(const S2FrameDev* __restrict__ fr, const uint32_t* __restrict__ starts,
                                                uint32_t nf, uint32_t total, const uint32_t* __restrict__ src,
                                                uint32_t* __restrict__ dst) {
  const uint32_t x = blockIdx.x * S2J_NT + threadIdx.x;
  if (x >= total)
    return;
  const uint32_t e = src[x];
  uint32_t r = S2_FAIL;
  if (!(e & S2_FAIL)) {
    const S2FrameDev f = fr[s2_frame_of(starts, nf, x)];
    r = src[f.jump_base + e];
  }
  dst[x] = (r & S2_FAIL) ? S2_FAIL : r;
}

// ---- a thread per frame: rows 0 and 1, then checkpoints every S2_CHUNK rows until a jump fails
// fail[f] = (failing row or h, its entry); ncp[f] = checkpoints written
__device__ __forceinline__ void s2_coarse_entry(const S2FrameDev* __restrict__ fr, uint32_t nf,
                                                const uint32_t* __restrict__ tab, const uint32_t* __restrict__ jump,
                                                uint32_t* __restrict__ rowstart, uint32_t* __restrict__ cp,
                                                uint32_t* __restrict__ ncp, uint2* __restrict__ fail) {
  const uint32_t fi = blockIdx.x * S2J_NT + threadIdx.x;
  if (fi >= nf)
    return;
  const S2FrameDev f = fr[fi];
  const uint32_t* t = tab + f.tab_base;
  const uint32_t n1 = f.ncand + 1u;
  uint32_t* rs = rowstart + f.row_base;
  uint2 fl = make_uint2(f.h, 0u);
  uint32_t m = 0;
  rs[0] = 0;
  const uint32_t r0 = t[3u * n1];
  if (r0 & S2_FAIL) {
    fl = make_uint2(0u, r0);
  } else if (f.h > 1u) {
    rs[1] = r0;
    const uint32_t r1 = t[2u * n1 + r0];
    if (r1 & S2_FAIL) {
      fl = make_uint2(1u, r1);
    } else if (f.h > 2u) {
      uint32_t cur = r1, row = 2;
      for (;;) {
        cp[f.cp_base + m++] = cur;
        if (row + S2_CHUNK >= f.h)
          break;
        const uint32_t g = jump[f.jump_base + cur];
        if (g & S2_FAIL)
          break;
        cur = g;
        row += S2_CHUNK;
      }
    }
  }
  ncp[fi] = m;
  fail[fi] = fl;
}

// ---- a thread per checkpoint slot: the row starts of its chunk; the one chunk that fails records it
__device__ __forceinline__ void s2_fine_entry(const S2FrameDev* __restrict__ fr, const uint32_t* __restrict__ starts,
                                              uint32_t nf, uint32_t total, const uint32_t* __restrict__ tab,
                                              const uint32_t* __restrict__ cp, const uint32_t* __restrict__ ncp,
                                              uint32_t* __restrict__ rowstart, uint2* __restrict__ fail) {
  const uint32_t x = blockIdx.x * S2J_NT + threadIdx.x;
  if (x >= total)
    return;
  const uint32_t fi = s2_frame_of(starts, nf, x);
  const S2FrameDev f = fr[fi];
  const uint32_t m = x - f.cp_base;
  if (m >= ncp[fi])
    return;
  const uint32_t* t = tab + f.tab_base;
  const uint32_t n1 = f.ncand + 1u;
  uint32_t cur = cp[x];
  const uint32_t r0 = 2u + m * S2_CHUNK, r1 = min(r0 + S2_CHUNK, f.h);
  for (uint32_t r = r0; r < r1; ++r) {
    rowstart[f.row_base + r] = cur;
    const uint32_t e = t[(r & 1u) * n1 + cur];
    if (e & S2_FAIL) {
      fail[fi] = make_uint2(r, e);
      return;
    }
    cur = e;
  }
}

// ---- a thread per row: descriptors of the rows up to the failing one
__device__ __forceinline__ void s2_desc_entry(const uint8_t* __restrict__ in, const S2FrameDev* __restrict__ fr,
                                              const uint32_t* __restrict__ starts, uint32_t nf, uint32_t total,
                                              const uint32_t* __restrict__ rowstart, const uint2* __restrict__ fail,
                                              uint2* __restrict__ desc) {
  const uint32_t x = blockIdx.x * S2W_NT + threadIdx.x;
  if (x >= total)
    return;
  const uint32_t fi = s2_frame_of(starts, nf, x);
  const S2FrameDev f = fr[fi];
  const uint32_t r = x - f.row_base;
  if (r > fail[fi].x || r >= f.h)
    return;
  const uint32_t cls = r == 0u ? 3u : (r == 1u ? 2u : (r & 1u));
  s2_walk<true>(in + f.in_offset, f, rowstart[x], cls, desc + f.desc_base + (uint64_t)r * f.nb);
}

// blocks of row r that are decoded: all before the failing row, those before the failing block in it
__device__ __forceinline__ uint32_t s2_blocks(const S2FrameDev& f, uint2 fl, uint32_t r) {
  return r < fl.x ? f.nb : (r == fl.x ? min(fl.y & 511u, f.nb) : 0u);
}

// ---- a CTA per row: differences (signExtend of each length's bits), in pixel order, as int16
__device__ __forceinline__ void s2_diff_entry(const uint8_t* __restrict__ in, const S2FrameDev* __restrict__ fr,
                                              const uint32_t* __restrict__ starts, uint32_t nf,
                                              const uint2* __restrict__ fail, const uint2* __restrict__ desc,
                                              int16_t* __restrict__ px) {
  const uint32_t x = blockIdx.x;
  const uint32_t fi = s2_frame_of(starts, nf, x);
  const S2FrameDev f = fr[fi];
  const uint32_t r = x - f.row_base;
  const uint32_t nbl = s2_blocks(f, fail[fi], r);
  const uint2* d = desc + f.desc_base + (uint64_t)r * f.nb;
  int16_t* o = px + f.px_base + (uint64_t)r * f.w;
  const uint8_t* data = in + f.in_offset;
  for (uint32_t idx = threadIdx.x; idx < nbl * 16u; idx += S2X_NT) {
    const uint32_t k = idx >> 4, j = idx & 15u, g = j >> 2;
    const uint2 dd = d[k];
    const uint32_t len = (dd.y >> (4u * g)) & 15u;
    uint32_t off = dd.x + (j & 3u) * len;
    for (uint32_t q = 0; q < g; ++q)
      off += 4u * ((dd.y >> (4u * q)) & 15u);
    int v = 0;
    if (len) {
      const uint32_t b = p1_window(data, f.size, off) >> (32u - len);
      v = (int)(b << (32u - len)) >> (32u - len);
    }
    // stream order 0 2 4 .. 14 1 3 .. 15 (even rows), 1 3 .. 15 0 2 .. 14 (odd rows)
    const uint32_t p = (r & 1u) ? ((j & 7u) << 1) + 1u - (j >> 3) : ((j & 7u) << 1) + (j >> 3);
    o[16u * k + p] = (int16_t)v;
  }
}

// ---- reconstruction: clamp-add maps x -> min(max(x + a, lo), hi); `then` applies f, then g
struct S2Map {
  int a, lo, hi;
};
constexpr int S2_BIG = 1 << 29, S2_ACLAMP = 1 << 20; // (inputs < 2^14: |a| past 2^20 saturates the same)
__device__ __forceinline__ int s2_clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }
__device__ __forceinline__ S2Map s2_then(S2Map f, S2Map g) {
  return S2Map{s2_clampi(f.a + g.a, -S2_ACLAMP, S2_ACLAMP), s2_clampi(f.lo + g.a, g.lo, g.hi),
               s2_clampi(f.hi + g.a, g.lo, g.hi)};
}
__device__ __forceinline__ S2Map s2_shfl_up(S2Map m, int d) {
  return S2Map{(int)__shfl_up_sync(0xFFFFFFFFu, m.a, d), (int)__shfl_up_sync(0xFFFFFFFFu, m.lo, d),
               (int)__shfl_up_sync(0xFFFFFFFFu, m.hi, d)};
}

struct S2Smem {
  uint16_t ring[3][S2_MAXW];
  uint16_t chain[2][S2R_NT + 1]; // value in front of block k, per parity (chain[p][0] = initVal)
  S2Map warp[2][S2R_NT / 32];
};

// baseline of pixel i of an up block (SamsungV2Decompressor.cpp:224-257), from the ring
__device__ __forceinline__ int s2_up_base(const S2Smem& sm, const S2FrameDev& f, uint32_t r, uint32_t col,
                                          uint32_t i, uint32_t motion) {
  const int off = (int)((0x8644220u >> (4u * motion)) & 15u) - 4;
  const bool avg = motion == 2u || motion == 4u;
  uint32_t rr;
  int rc = (int)(col + i) + off;
  if ((r + i) & 1u) {
    rr = r - 2u;
  } else {
    rr = r - 1u;
    rc += (i & 1u) ? -1 : 1;
  }
  const uint16_t* ref = sm.ring[rr % 3u];
  const int w1 = (int)f.w - 1;
  const int a = ref[s2_clampi(rc, 0, w1)];
  return avg ? (a + ref[s2_clampi(rc + 2, 0, w1)] + 1) >> 1 : a;
}

__device__ __forceinline__ int s2_sdiff(const int16_t* __restrict__ o, uint32_t c, int scale) {
  return (int)o[c] * (scale * 2 + 1) + scale;
}

__device__ __forceinline__ void s2_recon_entry(const S2FrameDev* __restrict__ fr, const uint2* __restrict__ fail,
                                               const uint2* __restrict__ desc, const int16_t* __restrict__ px,
                                               uint8_t* __restrict__ out, uint2* __restrict__ results, S2Smem& sm) {
  const uint32_t fi = blockIdx.x, t = threadIdx.x, lane = t & 31u, wp = t >> 5;
  const S2FrameDev f = fr[fi];
  const uint2 fl = fail[fi];
  const int maxv = (1 << f.bits) - 1;
  const uint32_t last = min(fl.x, f.h - 1u);
  for (uint32_t r = 0; r <= last; ++r) {
    const uint32_t nbl = s2_blocks(f, fl, r);
    if (nbl == 0u)
      break;
    const uint2* d = desc + f.desc_base + (uint64_t)r * f.nb;
    const int16_t* o = px + f.px_base + (uint64_t)r * f.w;
    // the maps of the two chains through block t: pixel 14 (even) and 15 (odd)
    S2Map me{0, -S2_BIG, S2_BIG}, mo{0, -S2_BIG, S2_BIG};
    if (t < nbl) {
      const uint32_t y = d[t].y, motion = (y >> 16) & 7u;
      const int scale = (int)(y >> 19) - 256;
      const int se = s2_clampi(s2_sdiff(o, 16u * t + 14u, scale), -S2_ACLAMP, S2_ACLAMP);
      const int so = s2_clampi(s2_sdiff(o, 16u * t + 15u, scale), -S2_ACLAMP, S2_ACLAMP);
      if (motion == 7u) {
        me = S2Map{se, 0, maxv};
        mo = S2Map{so, 0, maxv};
      } else {
        const int ve = s2_clampi(s2_up_base(sm, f, r, 16u * t, 14u, motion) + se, 0, maxv);
        const int vo = s2_clampi(s2_up_base(sm, f, r, 16u * t, 15u, motion) + so, 0, maxv);
        me = S2Map{0, ve, ve};
        mo = S2Map{0, vo, vo};
      }
    }
    for (int dd = 1; dd < 32; dd <<= 1) {
      const S2Map pe = s2_shfl_up(me, dd), po = s2_shfl_up(mo, dd);
      if (lane >= (uint32_t)dd) {
        me = s2_then(pe, me);
        mo = s2_then(po, mo);
      }
    }
    if (lane == 31u) {
      sm.warp[0][wp] = me;
      sm.warp[1][wp] = mo;
    }
    __syncthreads();
    if (wp == 0u) {
      S2Map we = lane < S2R_NT / 32 ? sm.warp[0][lane] : S2Map{0, -S2_BIG, S2_BIG};
      S2Map wo = lane < S2R_NT / 32 ? sm.warp[1][lane] : S2Map{0, -S2_BIG, S2_BIG};
      for (int dd = 1; dd < 32; dd <<= 1) {
        const S2Map pe = s2_shfl_up(we, dd), po = s2_shfl_up(wo, dd);
        if (lane >= (uint32_t)dd) {
          we = s2_then(pe, we);
          wo = s2_then(po, wo);
        }
      }
      if (lane < S2R_NT / 32) {
        sm.warp[0][lane] = we;
        sm.warp[1][lane] = wo;
      }
    }
    __syncthreads();
    if (wp > 0u) {
      me = s2_then(sm.warp[0][wp - 1u], me);
      mo = s2_then(sm.warp[1][wp - 1u], mo);
    }
    if (t < nbl) {
      sm.chain[0][t + 1u] = (uint16_t)s2_clampi((int)f.init + me.a, me.lo, me.hi);
      sm.chain[1][t + 1u] = (uint16_t)s2_clampi((int)f.init + mo.a, mo.lo, mo.hi);
    }
    if (t == 0u) {
      sm.chain[0][0] = (uint16_t)f.init;
      sm.chain[1][0] = (uint16_t)f.init;
    }
    __syncthreads();
    // the pixels, a pair per thread
    uint16_t* ring = sm.ring[r % 3u];
    uint8_t* orow = out + f.out_offset + (uint64_t)r * f.out_pitch;
    for (uint32_t q = t; q < nbl * 8u; q += S2R_NT) {
      const uint32_t k = q >> 3, c = 2u * q, i = c & 15u;
      const uint32_t y = d[k].y, motion = (y >> 16) & 7u;
      const int scale = (int)(y >> 19) - 256;
      int v[2];
      for (uint32_t e = 0; e < 2u; ++e) {
        const int base = motion == 7u ? (int)sm.chain[e][k] : s2_up_base(sm, f, r, 16u * k, i + e, motion);
        v[e] = s2_clampi(base + s2_sdiff(o, c + e, scale), 0, maxv);
        ring[c + e] = (uint16_t)v[e];
      }
      *reinterpret_cast<uint32_t*>(orow + 2u * c) = (uint32_t)v[0] | (uint32_t)v[1] << 16;
    }
    __syncthreads();
  }
  if (t == 0u) {
    if (fl.x >= f.h) {
      results[fi] = make_uint2(0u, 0u);
    } else {
      const uint32_t code = (fl.y >> 27) & 15u;
      results[fi] = make_uint2(code >= S2F_OVERREAD ? 2u : 1u, // RSB200_ERR_IOE / _RDE
                               code << 28 | ((fl.y >> 22) & 31u) << 22 | fl.x << 9 | (fl.y & 511u));
    }
  }
}

#ifndef RSB200_EMU
__global__ void __launch_bounds__(S2W_NT)
    s2_cand_kernel(const uint8_t* __restrict__ in, const S2FrameDev* __restrict__ fr,
                   const uint32_t* __restrict__ starts, uint32_t nf, uint32_t total, uint32_t* __restrict__ tab) {
  s2_cand_entry(in, fr, starts, nf, total, tab);
}

__global__ void __launch_bounds__(S2J_NT)
    s2_pair_kernel(const S2FrameDev* __restrict__ fr, const uint32_t* __restrict__ starts, uint32_t nf,
                   uint32_t total, const uint32_t* __restrict__ tab, uint32_t* __restrict__ jump) {
  s2_pair_entry(fr, starts, nf, total, tab, jump);
}

__global__ void __launch_bounds__(S2J_NT)
    s2_double_kernel(const S2FrameDev* __restrict__ fr, const uint32_t* __restrict__ starts, uint32_t nf,
                     uint32_t total, const uint32_t* __restrict__ src, uint32_t* __restrict__ dst) {
  s2_double_entry(fr, starts, nf, total, src, dst);
}

__global__ void __launch_bounds__(S2J_NT)
    s2_coarse_kernel(const S2FrameDev* __restrict__ fr, uint32_t nf, const uint32_t* __restrict__ tab,
                     const uint32_t* __restrict__ jump, uint32_t* __restrict__ rowstart, uint32_t* __restrict__ cp,
                     uint32_t* __restrict__ ncp, uint2* __restrict__ fail) {
  s2_coarse_entry(fr, nf, tab, jump, rowstart, cp, ncp, fail);
}

__global__ void __launch_bounds__(S2J_NT)
    s2_fine_kernel(const S2FrameDev* __restrict__ fr, const uint32_t* __restrict__ starts, uint32_t nf,
                   uint32_t total, const uint32_t* __restrict__ tab, const uint32_t* __restrict__ cp,
                   const uint32_t* __restrict__ ncp, uint32_t* __restrict__ rowstart, uint2* __restrict__ fail) {
  s2_fine_entry(fr, starts, nf, total, tab, cp, ncp, rowstart, fail);
}

__global__ void __launch_bounds__(S2W_NT)
    s2_desc_kernel(const uint8_t* __restrict__ in, const S2FrameDev* __restrict__ fr,
                   const uint32_t* __restrict__ starts, uint32_t nf, uint32_t total,
                   const uint32_t* __restrict__ rowstart, const uint2* __restrict__ fail, uint2* __restrict__ desc) {
  s2_desc_entry(in, fr, starts, nf, total, rowstart, fail, desc);
}

__global__ void __launch_bounds__(S2X_NT)
    s2_diff_kernel(const uint8_t* __restrict__ in, const S2FrameDev* __restrict__ fr,
                   const uint32_t* __restrict__ starts, uint32_t nf, const uint2* __restrict__ fail,
                   const uint2* __restrict__ desc, int16_t* __restrict__ px) {
  s2_diff_entry(in, fr, starts, nf, fail, desc, px);
}

__global__ void __launch_bounds__(S2R_NT)
    s2_recon_kernel(const S2FrameDev* __restrict__ fr, const uint2* __restrict__ fail,
                    const uint2* __restrict__ desc, const int16_t* __restrict__ px, uint8_t* __restrict__ out,
                    uint2* __restrict__ results) {
  __shared__ S2Smem sm;
  s2_recon_entry(fr, fail, desc, px, out, results, sm);
}
#endif

} // namespace rsb200
