// samsung1.cuh -- Samsung SRW V1 (SamsungV1Decompressor::decompress, decompressors/
// SamsungV1Decompressor.cpp:81-140, paths relative to src/librawspeed of rawspeed), sm_90a.
//
// The reference reads one plain MSB stream (BitStreamerMSB) with a fill(23) before every symbol.  A
// symbol is one of 14 fixed prefix codes (lengths 2..10, intervals assigned in table order, so not
// canonical) followed by `diffLen` bits through extend().  Each row keeps one running value per
// column parity, started from out(row - 2, 0 / 1) (0 on rows 0 and 1); every value must stay in
// 0..4095 (isIntN(value, 12)) or "decoded value out of bounds" is thrown at that pixel.
//
// Entropy stage.  Every code is at most 10 bits, shorter than LUT_BITS, so a DevTable whose LUT is
// filled directly from the 14 (encLen, diffLen) pairs (samsung1_dev_table, maxlen = 0: the F.16
// walk never runs) decodes every window; the multi-CTA range decoder (ljpeg_ranges.cuh, DevScan::kind
// 5, plain MSB pump) writes the differences in stream order.  A zero difference is the code 110100:
// speculative starts inside a run of them are moved to its phase (samsung1_run_phase).  At the end
// of the data the range kernels parse symbols that start up to 8 bytes + 9 bits behind it, reading
// zero bits there.
//
// End of the stream.  Before the code that starts at stream bit T the pump has done
// ceil((T + 23) / 32) refills, and refill number (size + 8) / 4 + 2 throws IOException
// (BitStreamer.h:125-127): the first symbol that fails is the first one that starts at or after
// T* = 32 * floor((size + 8) / 4) + 10.  A stream of fewer than 4 bytes throws before any symbol
// (BitStreamer.h:58-59).  Each code carries exactly one diffLen, the bit length of |difference|, so a
// symbol's length is recovered from its difference and a prefix sum gives every start bit.
//
// Reconstruction (keys (row << 14) | col order the pixels as the stream does):
//   s1_column_kernel  one warp per (frame, row parity, column 0/1): the first two values of every
//                     row, and the first out-of-range one among them
//   s1_row_kernel     one warp per row: the row's values (first out-of-range pixel), its stream
//                     bits and the offset of its last symbol
//   s1_scan_kernel    one CTA per frame: prefix of the row bits, the symbol whose refill fails, the
//                     outcome and the first pixel that is not written
//   s1_store_kernel   one warp per row: the values again, stored up to that pixel
#pragma once

#ifndef RSB200_EMU
#include "common.cuh"
#endif
#include "ljpeg_types.h"
#include <string.h>

namespace rsb200 {

// SamsungV1Decompressor.cpp:88-101: (encLen, diffLen) in the order the code intervals are assigned
constexpr uint8_t S1_TAB[14][2] = {{3, 4}, {3, 7}, {2, 6},  {2, 5},   {4, 3},  {6, 0}, {7, 9},
                                   {8, 10}, {9, 11}, {10, 12}, {10, 13}, {5, 1}, {4, 8}, {4, 2}};

// the code length of each diffLen 0..13 (SSSS of a difference = bit length of its magnitude)
RSB_LJ_HD inline uint32_t s1_enclen(uint32_t ssss) {
  // diffLen:            0  1  2  3  4  5  6  7  8  9 10 11 12  13
  // encLen:             6  5  4  4  3  2  2  3  4  7  8  9 10  10
  // packed 4 bits per entry (entries 0..7 in lo, 8..13 in hi)
  const uint32_t lo = 0x32234456u, hi = 0x00AA9874u;
  return ssss < 8 ? (lo >> (4 * ssss)) & 15u : (hi >> (4 * (ssss - 8))) & 15u;
}

// stream bits of the symbol of difference d (|d| < 2^13 for every decoded symbol; larger values only
// appear in scratch behind the failing symbol, where any positive length will do)
__device__ __forceinline__ uint32_t s1_sym_bits(int d) {
  const uint32_t L = 32u - (uint32_t)__clz((uint32_t)(d < 0 ? -d : d));
  return L > 13 ? 10u + L : s1_enclen(L) + L;
}

// The LUT-only table of the range decoder: entry = codelen | diffLen << 5 | (codelen + diffLen) << 10
inline void samsung1_dev_table(DevTable& t) {
  memset(&t, 0, sizeof t);
  for (int l = 0; l < 18; ++l)
    t.maxcode[l] = -1;
  uint32_t n = 0; // in the reference's 10-bit index space
  for (int k = 0; k < 14; ++k) {
    const uint32_t el = S1_TAB[k][0], dl = S1_TAB[k][1];
    const uint16_t e = (uint16_t)(el | (dl << 5) | ((el + dl) << 10));
    const uint32_t cnt = 1024u >> el;
    for (uint32_t c = 2 * n; c < 2 * (n + cnt); ++c)
      t.lut[c] = e;
    n += cnt;
  }
  t.maxlen = 0;
  t.fix16 = 0;
}

// T*: first stream bit at which a symbol's refill fails (0: the pump's constructor throws)
inline uint32_t samsung1_tstar(uint32_t size) {
  return size < 4 ? 0u : 32u * ((size + 8u) / 4u) + 10u;
}

struct DevS1 {
  uint64_t diff_offset; // first difference of the frame in the plan's diff buffer
  uint64_t out_offset;
  uint32_t w, h;
  uint32_t out_pitch;
  uint32_t tstar;
  uint32_t scan;     // index of the frame's scan / result
  uint32_t row_base; // first row of the frame in the per-row scratch
};

constexpr uint32_t S1_NOKEY = 0xFFFFFFFFu;
constexpr uint32_t S1_OOB = 0x80000000u; // RSB200_PENTAX_OOB

__device__ __forceinline__ uint32_t s1_key(uint32_t row, uint32_t col) { return (row << 14) | col; }
__device__ __forceinline__ bool s1_bad(int v) { return ((uint32_t)v >> 12) != 0; }

__global__ void s1_column_kernel(const DevS1* __restrict__ fr, int nframes,
                                 const uint16_t* __restrict__ diffs, uint16_t* __restrict__ colvals,
                                 uint32_t* __restrict__ oob) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int fi = warp >> 2;
  if (fi >= nframes)
    return;
  const DevS1 f = fr[fi];
  const uint32_t q = (warp >> 1) & 1u, c = warp & 1u; // row parity, column
  const int16_t* d = reinterpret_cast<const int16_t*>(diffs + f.diff_offset) + c;
  uint16_t* cv = colvals + 2ull * f.row_base + c;
  const uint32_t nj = (f.h - q + 1) / 2;
  int run = 0;
  uint32_t first_bad = S1_NOKEY;
  for (uint32_t j0 = 0; j0 < nj; j0 += 32) {
    const uint32_t j = j0 + lane, r = q + 2 * j;
    int v = (j < nj) ? (int)d[(uint64_t)r * f.w] : 0;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
      const int n = __shfl_up_sync(0xFFFFFFFFu, v, k);
      if (lane >= k)
        v += n;
    }
    v += run;
    if (j < nj) {
      cv[2ull * r] = (uint16_t)v;
      if (s1_bad(v))
        first_bad = min(first_bad, s1_key(r, c));
    }
    run = __shfl_sync(0xFFFFFFFFu, v, 31);
  }
  if (first_bad != S1_NOKEY)
    atomicMin(&oob[fi], first_bad);
}

constexpr int S1_NT = 256;
constexpr uint32_t S1_PER = 4; // pairs per lane and step (one 16-byte load of differences)

// One warp's walk of row r: values v[k] / u[k] of the pairs (2p, 2p + 1) of each step are handed to
// `use(p, va, vb, da, db)` in order (da / db: the differences, for the symbol lengths).
template <class F>
__device__ __forceinline__ void s1_row_walk(const DevS1& f, uint32_t r, const uint16_t* diffs,
                                            const uint16_t* colvals, F&& use) {
  const int lane = threadIdx.x & 31;
  const uint32_t npairs = f.w / 2;
  // rows start 64-byte aligned in the scratch (diff_offset % 8 == 0, width % 32 == 0)
  const uint4* d = reinterpret_cast<const uint4*>(diffs + f.diff_offset + (uint64_t)r * f.w);
  const uint32_t cv = *reinterpret_cast<const uint32_t*>(colvals + 2ull * (f.row_base + r));
  int run0 = 0, run1 = 0;
  for (uint32_t p0 = 0; p0 < npairs; p0 += 32 * S1_PER) {
    const uint32_t pb = p0 + lane * S1_PER; // npairs % 16 == 0: a lane's four pairs are all there
    const bool on = pb < npairs;
    uint4 w4 = make_uint4(0, 0, 0, 0);
    if (on)
      w4 = __ldg(d + pb / S1_PER);
    const uint32_t wv[4] = {w4.x, w4.y, w4.z, w4.w};
    int e[S1_PER], g[S1_PER];
    int s0 = 0, s1 = 0;
#pragma unroll
    for (uint32_t k = 0; k < S1_PER; ++k) {
      int a = (int)(int16_t)(wv[k] & 0xFFFFu), b = (int)(int16_t)(wv[k] >> 16);
      if (pb + k == 0) { // the column kernel holds the first two values of the row
        a = (int)(cv & 0xFFFFu);
        b = (int)(cv >> 16);
      }
      s0 += a;
      s1 += b;
      e[k] = s0;
      g[k] = s1;
    }
    int i0 = s0, i1 = s1;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
      const int x = __shfl_up_sync(0xFFFFFFFFu, i0, k);
      const int y = __shfl_up_sync(0xFFFFFFFFu, i1, k);
      if (lane >= k) {
        i0 += x;
        i1 += y;
      }
    }
    const int b0 = run0 + i0 - s0, b1 = run1 + i1 - s1;
    if (on) {
#pragma unroll
      for (uint32_t k = 0; k < S1_PER; ++k)
        use(pb + k, b0 + e[k], b1 + g[k], (int)(int16_t)(wv[k] & 0xFFFFu), (int)(int16_t)(wv[k] >> 16));
    }
    run0 += __shfl_sync(0xFFFFFFFFu, i0, 31);
    run1 += __shfl_sync(0xFFFFFFFFu, i1, 31);
  }
}

// The row kernels take `rb` CTAs of S1_NT / 32 rows per frame, frame after frame along x (no limit on
// the frames of a plan).
constexpr uint32_t S1_ROWS_PER_CTA = S1_NT / 32;

// first out-of-range pixel of the row, its bits and its last symbol's offset
__global__ void __launch_bounds__(S1_NT)
    s1_row_kernel(const DevS1* __restrict__ fr, uint32_t rb, const uint16_t* __restrict__ diffs,
                  const uint16_t* __restrict__ colvals, uint2* __restrict__ rowbits,
                  uint32_t* __restrict__ oob) {
  const uint32_t fi = blockIdx.x / rb;
  const DevS1 f = fr[fi];
  const uint32_t r = ((blockIdx.x % rb) * S1_NT + threadIdx.x) >> 5;
  if (r >= f.h)
    return;
  const int lane = threadIdx.x & 31;
  uint32_t first_bad = S1_NOKEY, bits = 0, lastlen = 0;
  s1_row_walk(f, r, diffs, colvals, [&](uint32_t p, int va, int vb, int da, int db) {
    if (s1_bad(va))
      first_bad = min(first_bad, s1_key(r, 2 * p));
    if (s1_bad(vb))
      first_bad = min(first_bad, s1_key(r, 2 * p + 1));
    lastlen = s1_sym_bits(db);
    bits += s1_sym_bits(da) + lastlen;
  });
#pragma unroll
  for (int k = 16; k; k >>= 1) {
    first_bad = min(first_bad, __shfl_xor_sync(0xFFFFFFFFu, first_bad, k));
    bits += __shfl_xor_sync(0xFFFFFFFFu, bits, k);
  }
  // the row's last pair belongs to the last lane that has pairs: lane (w / 8 - 1) % 32
  lastlen = __shfl_sync(0xFFFFFFFFu, lastlen, ((f.w / 2 / S1_PER) - 1) & 31);
  if (lane == 0) {
    rowbits[f.row_base + r] = make_uint2(bits, bits - lastlen);
    if (first_bad != S1_NOKEY)
      atomicMin(&oob[fi], first_bad);
  }
}

constexpr int S1_SCAN_NT = 1024;

struct S1ScanShared {
  uint32_t w[S1_SCAN_NT / 32];
  uint32_t row, base;
};

// one CTA per frame: the outcome; lim[frame] = key of the first pixel that is not written
__device__ __forceinline__ void s1_scan_body(const DevS1* __restrict__ fr, const uint16_t* __restrict__ diffs,
                                             const uint2* __restrict__ rowbits,
                                             const uint32_t* __restrict__ oob, uint32_t* __restrict__ lim,
                                             DevResult* __restrict__ results, S1ScanShared& sh) {
  uint32_t* const s_w = sh.w;
  uint32_t& s_row = sh.row;
  uint32_t& s_base = sh.base;
  const DevS1 f = fr[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0)
    s_row = S1_NOKEY;
  uint32_t carry = 0;
  for (uint32_t r0 = 0; r0 < f.h; r0 += S1_SCAN_NT) {
    const uint32_t r = r0 + tid;
    const uint2 rb = r < f.h ? rowbits[f.row_base + r] : make_uint2(0, 0);
    uint32_t v = rb.x;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
      const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, v, k);
      if (lane >= k)
        v += x;
    }
    if (lane == 31)
      s_w[wid] = v;
    __syncthreads();
    uint32_t add = 0, tot = 0;
    for (int k = 0; k < S1_SCAN_NT / 32; ++k) {
      add += k < wid ? s_w[k] : 0u;
      tot += s_w[k];
    }
    // (bits of a frame: at most 23 * 5664 * 3714 < 2^32)
    const uint32_t B = carry + add + v - rb.x; // stream bit of the row's first symbol
    if (r < f.h && B + rb.y >= f.tstar) { // the row holds a symbol that starts at or after T*
      atomicMin(&s_row, r);
    }
    carry += tot;
    __syncthreads();
    if (s_row != S1_NOKEY) {
      if (r == s_row)
        s_base = B;
      break;
    }
  }
  __syncthreads();
  uint32_t ioe = S1_NOKEY;
  if (s_row != S1_NOKEY) {
    if (wid == 0) { // the failing symbol inside the row
      const uint32_t r = s_row;
      const int16_t* d = reinterpret_cast<const int16_t*>(diffs + f.diff_offset + (uint64_t)r * f.w);
      uint32_t base = s_base, col = S1_NOKEY;
      for (uint32_t c0 = 0; c0 < f.w && col == S1_NOKEY; c0 += 32) {
        const uint32_t sb = s1_sym_bits(d[c0 + lane]); // (width % 32 == 0)
        uint32_t x = sb;
#pragma unroll
        for (int k = 1; k < 32; k <<= 1) {
          const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, k);
          if (lane >= k)
            x += y;
        }
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, base + x - sb >= f.tstar);
        if (m)
          col = c0 + (uint32_t)__ffs(m) - 1u;
        base += __shfl_sync(0xFFFFFFFFu, x, 31);
      }
      if (lane == 0)
        s_base = s1_key(r, col);
    }
    __syncthreads();
    ioe = s_base;
  }
  if (tid == 0) {
    const uint32_t viol = oob[blockIdx.x];
    DevResult res;
    res.status = 0;
    res.consumed = 0;
    if (ioe != S1_NOKEY && ioe <= viol) { // a failed refill throws before its symbol is read
      res.status = 2u;
      res.consumed = ioe;
    } else if (viol != S1_NOKEY) {
      res.status = 1u;
      res.consumed = S1_OOB | viol;
    }
    lim[blockIdx.x] = min(ioe, viol);
    results[f.scan] = res;
  }
}

#ifndef RSB200_EMU
__global__ void __launch_bounds__(S1_SCAN_NT)
    s1_scan_kernel(const DevS1* __restrict__ fr, const uint16_t* __restrict__ diffs,
                   const uint2* __restrict__ rowbits, const uint32_t* __restrict__ oob,
                   uint32_t* __restrict__ lim, DevResult* __restrict__ results) {
  __shared__ S1ScanShared sh;
  s1_scan_body(fr, diffs, rowbits, oob, lim, results, sh);
}
#endif

// the pixels before lim[frame]
__global__ void __launch_bounds__(S1_NT)
    s1_store_kernel(const DevS1* __restrict__ fr, uint32_t rb, const uint16_t* __restrict__ diffs,
                    const uint16_t* __restrict__ colvals, const uint32_t* __restrict__ lim,
                    uint8_t* __restrict__ out) {
  const uint32_t fi = blockIdx.x / rb;
  const DevS1 f = fr[fi];
  const uint32_t r = ((blockIdx.x % rb) * S1_NT + threadIdx.x) >> 5;
  if (r >= f.h)
    return;
  const uint32_t l = lim[fi];
  if (l <= s1_key(r, 0))
    return;
  uint32_t* o = reinterpret_cast<uint32_t*>(out + f.out_offset + (uint64_t)r * f.out_pitch);
  const bool whole = l > s1_key(r, f.w - 1);
  s1_row_walk(f, r, diffs, colvals, [&](uint32_t p, int va, int vb, int, int) {
    const uint32_t w = ((uint32_t)va & 0xFFFFu) | ((uint32_t)vb << 16);
    if (whole || l > s1_key(r, 2 * p + 1))
      o[p] = w;
    else if (l > s1_key(r, 2 * p))
      reinterpret_cast<uint16_t*>(o)[2 * p] = (uint16_t)w;
  });
}

} // namespace rsb200
