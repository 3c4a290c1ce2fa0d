// kodak.cuh -- Kodak DCR segment codec (KodakDecompressor), sm_90a.
//
// Replaces KodakDecompressor::decompress (decompressors/KodakDecompressor.cpp:67-150).  A row is cut
// into segments of min(256, width - col) pixels; a segment of b pixels is b / 2 bytes of 4-bit lengths
// (low nibble first), two more bytes when b % 8 == 4, then 4-byte refills whenever the bit cache holds
// fewer bits than the next length.  The payload is a string of 16-bit big-endian words read LSB first
// in word order, so pixel i's difference is bits [S_{i-1}, S_i) of it, S_i the sum of the first i + 1
// lengths.  The only serial dependence is where a segment starts, and it breaks cleanly:
//  * A segment's byte length is a closed form of its header: with h = b / 2, e = 2 when b % 8 == 4
//    (else 0) and S the sum of the header's nibbles, len = h + e + 4 ceil(max(0, S - 8 e) / 32).  With
//    a prefix sum of the nibbles over the input, a segment's length from any offset costs O(1).  The
//    segment over-reads iff p + len > size, and then none of its pixels is written (the reference
//    decodes the whole segment before it writes any).
//  * Full segments are 0 (mod 4) bytes long and the tail of t = width % 256 pixels t / 2 + e (mod 4),
//    an even number, so row starts are even offsets, and multiples of 4 when t / 2 + e is.  Every such
//    candidate is walked once, a row's worth of segments, and the chain from offset 0 is resolved by
//    pointer doubling, as for Samsung V2.
//  * The predictors reset for every segment, so a warp decodes a segment on its own: one scan for the
//    bit offsets, one per parity for the values.
// Stages (one launch each for all frames of a plan):
//   kd_tsum_kernel    a CTA per tile of KD_TILE byte pairs: the tile's nibble sum
//   kd_tscan_kernel   a CTA per frame: exclusive scan of its tile sums
//   kd_prefix_kernel  a CTA per tile: q[k] = nibble sum of the bytes before 2 k
//   kd_cand_kernel    a thread per candidate: the next row's candidate, or the failing segment
//   kd_double_kernel  KD_JUMP rounds of pointer doubling on it (failures absorb)
//   kd_coarse_kernel  a thread per frame: a checkpoint every KD_CHUNK rows
//   kd_fine_kernel    a thread per checkpoint: every row start of its chunk, and the failing row
//   kd_check_kernel   a warp per segment: the first out-of-range pixel of the frame (atomicMin)
//   kd_store_kernel   a warp per segment: the pixels before the frame's failure, and its result
// No index is taken from the stream without a bound: a segment's nibble sum is read at offsets checked
// against the size first, and candidate entries stay within 0..ncand - 1.
#pragma once

#ifndef RSB200_EMU
#include "common.cuh"
#endif
#include <stdint.h>
#include <string.h>

namespace rsb200 {

constexpr int KD_NT = 256;            // threads per CTA (every kernel)
constexpr uint32_t KD_TILE = 16u * KD_NT; // byte pairs per prefix tile (16 per thread)
constexpr int KD_JUMP = 5;            // doubling rounds: a jump covers 2^KD_JUMP rows
constexpr uint32_t KD_CHUNK = 1u << KD_JUMP; // rows per checkpoint
constexpr uint32_t KD_FAIL = 1u << 31; // candidate entry: KD_FAIL | the failing segment of the row
constexpr uint32_t KD_MAXW = 4516, KD_MAXH = 3012;
constexpr uint32_t KD_MAX_IN = 1u << 28; // in_size bound: every nibble sum difference fits 32 bits

struct KdFrameDev {
  uint64_t in_offset;
  uint64_t out_offset;
  uint32_t size;      // input bytes
  uint32_t out_pitch;
  uint32_t w, h, bps;
  uint32_t stride;    // bytes between candidates (2 or 4)
  uint32_t nseg;      // segments per row
  uint32_t table;     // first entry of the job's table in the plan's tables, or ~0u for none
  uint32_t tile_base, ntile; // prefix tiles
  uint32_t q_base;    // first prefix entry (size / 2 + 1 of them)
  uint32_t cand_base, ncand; // candidates: offsets stride * c, c < ncand = size / stride + 1
  uint32_t row_base;  // first row start
  uint32_t cp_base;   // first checkpoint (ceil(h / KD_CHUNK))
  uint32_t seg_base;  // first segment (h * nseg)
};

// Host side: a plan's scratch so far (entries of each table)
struct KdTotals {
  uint64_t tiles = 0, q = 0, cand = 0, rows = 0, cps = 0, segs = 0;
};

// Host side: one frame's descriptor, placed behind the frames before it in every scratch table;
// `starts` (four per-frame searches of nf each: tiles, candidates, checkpoints, segments) gets its
// first indices.  table: the first entry of the job's table, or ~0u.
inline void kd_place_frame(KdFrameDev& f, KdTotals& t, uint32_t* starts, uint32_t nf, uint32_t i, uint64_t in_offset,
                           uint32_t in_size, uint32_t w, uint32_t h, uint32_t bps, uint32_t table, uint64_t out_offset,
                           uint32_t out_pitch) {
  memset(&f, 0, sizeof f);
  f.in_offset = in_offset;
  f.out_offset = out_offset;
  f.size = in_size;
  f.out_pitch = out_pitch;
  f.w = w;
  f.h = h;
  f.bps = bps;
  f.table = table;
  f.nseg = (w + 255u) / 256u;
  const uint32_t tail = w % 256u, e = (tail & 7u) == 4u ? 2u : 0u;
  f.stride = ((tail / 2u + e) & 3u) == 0u ? 4u : 2u;
  const uint32_t nq = in_size / 2u + 1u;
  f.ntile = (nq + KD_TILE - 1u) / KD_TILE;
  f.ncand = in_size / f.stride + 1u;
  starts[i] = (uint32_t)t.tiles;
  starts[nf + i] = (uint32_t)t.cand;
  starts[2 * nf + i] = (uint32_t)t.cps;
  starts[3 * nf + i] = (uint32_t)t.segs;
  f.tile_base = (uint32_t)t.tiles;
  f.q_base = (uint32_t)t.q;
  f.cand_base = (uint32_t)t.cand;
  f.row_base = (uint32_t)t.rows;
  f.cp_base = (uint32_t)t.cps;
  f.seg_base = (uint32_t)t.segs;
  t.tiles += f.ntile;
  t.q += nq;
  t.cand += f.ncand;
  t.rows += h;
  t.cps += (h + KD_CHUNK - 1u) / KD_CHUNK;
  t.segs += (uint64_t)h * f.nseg;
}

// the frame of flattened index x: the last f with starts[f] <= x (starts ascending, starts[0] == 0)
__device__ __forceinline__ uint32_t kd_frame_of(const uint32_t* __restrict__ starts, uint32_t n, uint32_t x) {
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

// pixels of segment k of a row
__device__ __forceinline__ uint32_t kd_bsize(const KdFrameDev& f, uint32_t k) { return min(256u, f.w - 256u * k); }

// bytes the segment of b pixels at offset p reads, or 0 when it reads past the end
// (KodakDecompressor.cpp:67-118; the refills are the closed form above).  q: the frame's prefix.
__device__ __forceinline__ uint32_t kd_seg_len(const uint32_t* __restrict__ q, uint32_t size, uint32_t p, uint32_t b) {
  const uint32_t h = b >> 1, e = (b & 7u) == 4u ? 2u : 0u;
  if (h > size - p) // (p <= size)
    return 0u;
  const uint32_t s = q[(p + h) >> 1] - q[p >> 1]; // (p, h even; differences of sums < 2^32 are exact)
  const uint32_t len = h + e + 4u * ((s > 8u * e ? s - 8u * e + 31u : 0u) >> 5);
  return len > size - p ? 0u : len;
}

// ---- nibble-sum prefix: pair k of a frame is bytes 2k and 2k + 1 (0 past the end)
__device__ __forceinline__ uint32_t kd_pair(const uint8_t* __restrict__ data, uint32_t size, uint32_t k) {
  uint32_t s = 0;
  if (2u * k < size) {
    const uint32_t a = __ldg(data + 2u * k);
    s = (a & 15u) + (a >> 4);
  }
  if (2u * k + 1u < size) {
    const uint32_t a = __ldg(data + 2u * k + 1u);
    s += (a & 15u) + (a >> 4);
  }
  return s;
}

// exclusive scan of v over the CTA; *total gets the sum
__device__ __forceinline__ uint32_t kd_cta_scan(uint32_t v, uint32_t* __restrict__ warp_sums, uint32_t* total) {
  const uint32_t lane = threadIdx.x & 31u, wp = threadIdx.x >> 5;
  uint32_t x = v;
  for (uint32_t d = 1; d < 32u; d <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d);
    if (lane >= d)
      x += y;
  }
  if (lane == 31u)
    warp_sums[wp] = x;
  __syncthreads();
  uint32_t before = 0, all = 0;
  for (uint32_t i = 0; i < (uint32_t)KD_NT / 32u; ++i) {
    const uint32_t ws = warp_sums[i];
    before += i < wp ? ws : 0u;
    all += ws;
  }
  __syncthreads();
  *total = all;
  return before + x - v;
}

// the 16 pairs of this thread in tile i of frame f, and their sum
__device__ __forceinline__ uint32_t kd_tile_pairs(const uint8_t* __restrict__ in, const KdFrameDev& f, uint32_t i,
                                                  uint32_t* s) {
  const uint8_t* data = in + f.in_offset;
  const uint32_t k0 = i * KD_TILE + 16u * threadIdx.x;
  uint32_t sum = 0;
#pragma unroll
  for (uint32_t j = 0; j < 16u; ++j) {
    s[j] = kd_pair(data, f.size, k0 + j);
    sum += s[j];
  }
  return sum;
}

__device__ __forceinline__ void kd_tsum_entry(const uint8_t* __restrict__ in, const KdFrameDev* __restrict__ fr,
                                              const uint32_t* __restrict__ starts, uint32_t nf,
                                              uint32_t* __restrict__ tsum, uint32_t* __restrict__ warp_sums) {
  const uint32_t x = blockIdx.x;
  const KdFrameDev f = fr[kd_frame_of(starts, nf, x)];
  uint32_t s[16], total;
  kd_cta_scan(kd_tile_pairs(in, f, x - f.tile_base, s), warp_sums, &total);
  if (threadIdx.x == 0u)
    tsum[x] = total;
}

// a CTA per frame: tsum[tile_base ..) becomes the exclusive scan of itself
__device__ __forceinline__ void kd_tscan_entry(const KdFrameDev* __restrict__ fr, uint32_t* __restrict__ tsum,
                                               uint32_t* __restrict__ warp_sums) {
  const KdFrameDev f = fr[blockIdx.x];
  uint32_t carry = 0;
  for (uint32_t b = 0; b < f.ntile; b += KD_NT) {
    const uint32_t i = b + threadIdx.x;
    const uint32_t v = i < f.ntile ? tsum[f.tile_base + i] : 0u;
    uint32_t total;
    const uint32_t ex = kd_cta_scan(v, warp_sums, &total);
    if (i < f.ntile)
      tsum[f.tile_base + i] = carry + ex;
    carry += total;
  }
}

__device__ __forceinline__ void kd_prefix_entry(const uint8_t* __restrict__ in, const KdFrameDev* __restrict__ fr,
                                                const uint32_t* __restrict__ starts, uint32_t nf,
                                                const uint32_t* __restrict__ tsum, uint32_t* __restrict__ q,
                                                uint32_t* __restrict__ warp_sums) {
  const uint32_t x = blockIdx.x;
  const KdFrameDev f = fr[kd_frame_of(starts, nf, x)];
  const uint32_t i = x - f.tile_base, nq = f.size / 2u + 1u;
  uint32_t s[16], total;
  uint32_t acc = tsum[x] + kd_cta_scan(kd_tile_pairs(in, f, i, s), warp_sums, &total);
  const uint32_t k0 = i * KD_TILE + 16u * threadIdx.x;
#pragma unroll
  for (uint32_t j = 0; j < 16u; ++j) {
    if (k0 + j < nq)
      q[f.q_base + k0 + j] = acc;
    acc += s[j];
  }
}

// ---- the row from candidate c: the next row's candidate, or KD_FAIL | the segment that over-reads
__device__ __forceinline__ uint32_t kd_row(const uint32_t* __restrict__ q, const KdFrameDev& f, uint32_t c) {
  uint32_t p = c * f.stride;
  for (uint32_t k = 0; k < f.nseg; ++k) {
    const uint32_t len = kd_seg_len(q, f.size, p, kd_bsize(f, k));
    if (len == 0u)
      return KD_FAIL | k;
    p += len;
  }
  return p / f.stride; // (p <= size, and a multiple of the stride: see the top of the file)
}

__device__ __forceinline__ void kd_cand_entry(const KdFrameDev* __restrict__ fr, const uint32_t* __restrict__ starts,
                                              uint32_t nf, uint32_t total, const uint32_t* __restrict__ q,
                                              uint32_t* __restrict__ tab) {
  const uint32_t x = blockIdx.x * KD_NT + threadIdx.x;
  if (x >= total)
    return;
  const KdFrameDev f = fr[kd_frame_of(starts, nf, x)];
  tab[x] = kd_row(q + f.q_base, f, x - f.cand_base);
}

__device__ __forceinline__ void kd_double_entry(const KdFrameDev* __restrict__ fr, const uint32_t* __restrict__ starts,
                                                uint32_t nf, uint32_t total, const uint32_t* __restrict__ src,
                                                uint32_t* __restrict__ dst) {
  const uint32_t x = blockIdx.x * KD_NT + threadIdx.x;
  if (x >= total)
    return;
  const uint32_t e = src[x];
  uint32_t r = KD_FAIL;
  if (!(e & KD_FAIL)) {
    const KdFrameDev f = fr[kd_frame_of(starts, nf, x)];
    r = src[f.cand_base + e];
  }
  dst[x] = (r & KD_FAIL) ? KD_FAIL : r;
}

// ---- a thread per frame: a checkpoint every KD_CHUNK rows until a jump fails; ncp[f] = checkpoints
// written.  Also resets the frame's failure: fail[f] = (h, 0), key[f] = ~0u.
__device__ __forceinline__ void kd_coarse_entry(const KdFrameDev* __restrict__ fr, uint32_t nf,
                                                const uint32_t* __restrict__ jump, uint32_t* __restrict__ cp,
                                                uint32_t* __restrict__ ncp, uint2* __restrict__ fail,
                                                uint32_t* __restrict__ key) {
  const uint32_t fi = blockIdx.x * KD_NT + threadIdx.x;
  if (fi >= nf)
    return;
  const KdFrameDev f = fr[fi];
  uint32_t cur = 0, row = 0, m = 0;
  for (;;) {
    cp[f.cp_base + m++] = cur;
    if (row + KD_CHUNK >= f.h)
      break;
    const uint32_t g = jump[f.cand_base + cur];
    if (g & KD_FAIL)
      break;
    cur = g;
    row += KD_CHUNK;
  }
  ncp[fi] = m;
  fail[fi] = make_uint2(f.h, 0u);
  key[fi] = ~0u;
}

// ---- a thread per checkpoint slot: the row starts of its chunk; the one chunk that fails records it
__device__ __forceinline__ void kd_fine_entry(const KdFrameDev* __restrict__ fr, const uint32_t* __restrict__ starts,
                                              uint32_t nf, uint32_t total, const uint32_t* __restrict__ tab,
                                              const uint32_t* __restrict__ cp, const uint32_t* __restrict__ ncp,
                                              uint32_t* __restrict__ rowstart, uint2* __restrict__ fail) {
  const uint32_t x = blockIdx.x * KD_NT + threadIdx.x;
  if (x >= total)
    return;
  const uint32_t fi = kd_frame_of(starts, nf, x);
  const KdFrameDev f = fr[fi];
  const uint32_t m = x - f.cp_base;
  if (m >= ncp[fi])
    return;
  uint32_t cur = cp[x];
  const uint32_t r0 = m * KD_CHUNK, r1 = min(r0 + KD_CHUNK, f.h);
  for (uint32_t r = r0; r < r1; ++r) {
    rowstart[f.row_base + r] = cur;
    const uint32_t e = tab[f.cand_base + cur];
    if (e & KD_FAIL) {
      fail[fi] = make_uint2(r, e & ~KD_FAIL);
      return;
    }
    cur = e;
  }
}

// ---- a warp per segment.  The frame's failure is key = 2 F + (1 for an out-of-range pixel, 0 for a
// segment that over-reads), F = row * w + column of the failing pixel or of the segment's first: the
// earliest in decode order wins (an over-read at F comes before the check of pixel F).
struct KdSeg {
  KdFrameDev f;
  uint32_t fi, r, k, b; // frame, row, segment, its pixels
  uint32_t first;       // row * w + its first column
  bool live;            // decoded by the reference (its row start is known and it does not over-read)
};

__device__ __forceinline__ KdSeg kd_seg_of(const KdFrameDev* __restrict__ fr, const uint32_t* __restrict__ starts,
                                           uint32_t nf, uint32_t gw, const uint2* __restrict__ fail) {
  KdSeg s;
  s.fi = kd_frame_of(starts, nf, gw);
  s.f = fr[s.fi];
  const uint32_t local = gw - s.f.seg_base;
  s.r = local / s.f.nseg;
  s.k = local - s.r * s.f.nseg;
  s.b = kd_bsize(s.f, s.k);
  s.first = s.r * s.f.w + 256u * s.k;
  const uint2 fl = fail[s.fi];
  s.live = s.r < fl.x || (s.r == fl.x && s.k < fl.y);
  return s;
}

// the segment's values (pixels 8 lane .. 8 lane + 7; those past b are 0); -> false when it is not live
__device__ __forceinline__ void kd_decode(const uint8_t* __restrict__ in, const uint32_t* __restrict__ q,
                                          const uint32_t* __restrict__ rowstart, const KdSeg& s, int* v) {
  const KdFrameDev& f = s.f;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t* fq = q + f.q_base;
  uint32_t p = rowstart[f.row_base + s.r] * f.stride;
  for (uint32_t j = 0; j < s.k; ++j) // (full segments in front, none of which over-reads)
    p += kd_seg_len(fq, f.size, p, 256u);
  const uint8_t* data = in + f.in_offset;
  const uint32_t h = s.b >> 1;
  // lengths: header byte 4 lane + m holds pixels 8 lane + 2 m (low nibble) and + 1 (high)
  uint32_t len[8], sum = 0;
#pragma unroll
  for (uint32_t m = 0; m < 4u; ++m) {
    const uint32_t i = 4u * lane + m;
    const uint32_t byte = i < h ? (uint32_t)__ldg(data + p + i) : 0u;
    len[2 * m] = byte & 15u;
    len[2 * m + 1] = byte >> 4;
    sum += len[2 * m] + len[2 * m + 1];
  }
  uint32_t off = sum;
  for (uint32_t d = 1; d < 32u; d <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, off, d);
    if (lane >= d)
      off += y;
  }
  off -= sum;
  // differences: bits [off, off + len) of the BE16 words from p + h, LSB first; sign per extend()
  const uint32_t pb = p + h;
  int pe = 0, po = 0;
#pragma unroll
  for (uint32_t j = 0; j < 8u; ++j) {
    const uint32_t L = len[j];
    int d = 0;
    if (L) {
      const uint32_t at = pb + 2u * (off >> 4);
      uint32_t wv = 0;
#pragma unroll
      for (uint32_t t = 0; t < 4u; ++t) {
        const uint32_t bb = at + t < f.size ? (uint32_t)__ldg(data + at + t) : 0u;
        wv |= bb << (t & 1u ? 8u * (t - 1u) : 8u * (t + 1u)); // bytes hi lo hi lo -> word0 | word1 << 16
      }
      const uint32_t bits = (wv >> (off & 15u)) & ((1u << L) - 1u);
      d = (bits >> (L - 1u)) ? (int)bits : (int)bits - (int)((1u << L) - 1u);
    }
    off += L;
    v[j] = d;
    if (j & 1u)
      po += d;
    else
      pe += d;
  }
  // per-parity prefix over the segment
  int xe = pe, xo = po;
  for (uint32_t dd = 1; dd < 32u; dd <<= 1) {
    const int ye = (int)__shfl_up_sync(0xFFFFFFFFu, (uint32_t)xe, dd);
    const int yo = (int)__shfl_up_sync(0xFFFFFFFFu, (uint32_t)xo, dd);
    if (lane >= dd) {
      xe += ye;
      xo += yo;
    }
  }
  xe -= pe;
  xo -= po;
#pragma unroll
  for (uint32_t j = 0; j < 8u; ++j) {
    if (j & 1u) {
      xo += v[j];
      v[j] = xo;
    } else {
      xe += v[j];
      v[j] = xe;
    }
  }
}

// the first pixel of this warp's segment with a value outside [0, 2^bps), as 2 F + 1; ~0u if none
__device__ __forceinline__ uint32_t kd_first_bad(const KdSeg& s, const int* v) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t j0 = 8u;
#pragma unroll
  for (uint32_t j = 0; j < 8u; ++j)
    if (j0 == 8u && 8u * lane + j < s.b && (uint32_t)v[j] >> s.f.bps)
      j0 = j;
  const uint32_t any = __ballot_sync(0xFFFFFFFFu, j0 < 8u);
  if (!any)
    return ~0u;
  const uint32_t l0 = (uint32_t)__ffs((int)any) - 1u;
  const uint32_t jb = __shfl_sync(0xFFFFFFFFu, j0, (int)l0);
  return 2u * (s.first + 8u * l0 + jb) + 1u;
}

__device__ __forceinline__ void kd_check_entry(const uint8_t* __restrict__ in, const KdFrameDev* __restrict__ fr,
                                               const uint32_t* __restrict__ starts, uint32_t nf, uint32_t total,
                                               const uint32_t* __restrict__ q, const uint32_t* __restrict__ rowstart,
                                               const uint2* __restrict__ fail, uint32_t* __restrict__ key) {
  const uint32_t gw = blockIdx.x * (KD_NT / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  if (gw >= total)
    return;
  const KdSeg s = kd_seg_of(fr, starts, nf, gw, fail);
  if (s.r == 0u && s.k == 0u && lane == 0u) {
    const uint2 fl = fail[s.fi];
    if (fl.x < s.f.h)
      atomicMin(key + s.fi, 2u * (fl.x * s.f.w + 256u * fl.y));
  }
  if (!s.live)
    return;
  int v[8];
  kd_decode(in, q, rowstart, s, v);
  const uint32_t bad = kd_first_bad(s, v);
  if (bad != ~0u && lane == 0u)
    atomicMin(key + s.fi, bad);
}

// consumed = code << 28 | row << 13 | column (RSB200_KODAK_*); values[f] the value an out-of-range
// pixel prints (0 otherwise)
__device__ __forceinline__ void kd_store_entry(const uint8_t* __restrict__ in, const KdFrameDev* __restrict__ fr,
                                               const uint32_t* __restrict__ starts, uint32_t nf, uint32_t total,
                                               const uint32_t* __restrict__ q, const uint32_t* __restrict__ rowstart,
                                               const uint2* __restrict__ fail, const uint32_t* __restrict__ key,
                                               const uint16_t* __restrict__ tables, uint8_t* __restrict__ out,
                                               uint2* __restrict__ results, int32_t* __restrict__ values) {
  const uint32_t gw = blockIdx.x * (KD_NT / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  if (gw >= total)
    return;
  const KdSeg s = kd_seg_of(fr, starts, nf, gw, fail);
  const uint32_t kk = key[s.fi], lim = kk == ~0u ? ~0u : kk >> 1;
  if (s.r == 0u && s.k == 0u && lane == 0u) {
    if (kk == ~0u) {
      results[s.fi] = make_uint2(0u, 0u);
    } else {
      const uint32_t rde = kk & 1u, row = lim / s.f.w, col = lim - row * s.f.w;
      results[s.fi] = make_uint2(rde ? 1u : 2u, // RSB200_ERR_RDE / _IOE
                                 (rde ? 1u : 2u) << 28 | row << 13 | col);
    }
    if (kk == ~0u || !(kk & 1u))
      values[s.fi] = 0;
  }
  if (!s.live || s.first > lim)
    return;
  int v[8];
  kd_decode(in, q, rowstart, s, v);
  const KdFrameDev& f = s.f;
  uint8_t* orow = out + f.out_offset + (uint64_t)s.r * f.out_pitch + 2u * (256u * s.k + 8u * lane);
  const uint32_t px0 = s.first + 8u * lane;
#pragma unroll
  for (uint32_t m = 0; m < 4u; ++m) {
    const uint32_t j = 2u * m;
    if (8u * lane + j >= s.b || px0 + j > lim)
      break;
    if (px0 + j == lim) { // the failing pixel: only its value
      if (kk & 1u)
        values[s.fi] = v[j];
      break;
    }
    uint32_t a = (uint32_t)v[j], c = (uint32_t)v[j + 1];
    if (f.table != ~0u) {
      a = tables[f.table + a];
      if (px0 + j + 1u < lim)
        c = tables[f.table + c];
    }
    if (px0 + j + 1u < lim) {
      *reinterpret_cast<uint32_t*>(orow + 4u * m) = (a & 0xFFFFu) | c << 16;
    } else {
      *reinterpret_cast<uint16_t*>(orow + 4u * m) = (uint16_t)a;
      if (px0 + j + 1u == lim && (kk & 1u))
        values[s.fi] = v[j + 1];
      break;
    }
  }
}

#ifndef RSB200_EMU
__global__ void __launch_bounds__(KD_NT)
    kd_tsum_kernel(const uint8_t* __restrict__ in, const KdFrameDev* __restrict__ fr,
                   const uint32_t* __restrict__ starts, uint32_t nf, uint32_t* __restrict__ tsum) {
  __shared__ uint32_t warp_sums[KD_NT / 32];
  kd_tsum_entry(in, fr, starts, nf, tsum, warp_sums);
}

__global__ void __launch_bounds__(KD_NT) kd_tscan_kernel(const KdFrameDev* __restrict__ fr, uint32_t* __restrict__ tsum) {
  __shared__ uint32_t warp_sums[KD_NT / 32];
  kd_tscan_entry(fr, tsum, warp_sums);
}

__global__ void __launch_bounds__(KD_NT)
    kd_prefix_kernel(const uint8_t* __restrict__ in, const KdFrameDev* __restrict__ fr,
                     const uint32_t* __restrict__ starts, uint32_t nf, const uint32_t* __restrict__ tsum,
                     uint32_t* __restrict__ q) {
  __shared__ uint32_t warp_sums[KD_NT / 32];
  kd_prefix_entry(in, fr, starts, nf, tsum, q, warp_sums);
}

__global__ void __launch_bounds__(KD_NT)
    kd_cand_kernel(const KdFrameDev* __restrict__ fr, const uint32_t* __restrict__ starts, uint32_t nf,
                   uint32_t total, const uint32_t* __restrict__ q, uint32_t* __restrict__ tab) {
  kd_cand_entry(fr, starts, nf, total, q, tab);
}

__global__ void __launch_bounds__(KD_NT)
    kd_double_kernel(const KdFrameDev* __restrict__ fr, const uint32_t* __restrict__ starts, uint32_t nf,
                     uint32_t total, const uint32_t* __restrict__ src, uint32_t* __restrict__ dst) {
  kd_double_entry(fr, starts, nf, total, src, dst);
}

__global__ void __launch_bounds__(KD_NT)
    kd_coarse_kernel(const KdFrameDev* __restrict__ fr, uint32_t nf, const uint32_t* __restrict__ jump,
                     uint32_t* __restrict__ cp, uint32_t* __restrict__ ncp, uint2* __restrict__ fail,
                     uint32_t* __restrict__ key) {
  kd_coarse_entry(fr, nf, jump, cp, ncp, fail, key);
}

__global__ void __launch_bounds__(KD_NT)
    kd_fine_kernel(const KdFrameDev* __restrict__ fr, const uint32_t* __restrict__ starts, uint32_t nf,
                   uint32_t total, const uint32_t* __restrict__ tab, const uint32_t* __restrict__ cp,
                   const uint32_t* __restrict__ ncp, uint32_t* __restrict__ rowstart, uint2* __restrict__ fail) {
  kd_fine_entry(fr, starts, nf, total, tab, cp, ncp, rowstart, fail);
}

__global__ void __launch_bounds__(KD_NT)
    kd_check_kernel(const uint8_t* __restrict__ in, const KdFrameDev* __restrict__ fr,
                    const uint32_t* __restrict__ starts, uint32_t nf, uint32_t total, const uint32_t* __restrict__ q,
                    const uint32_t* __restrict__ rowstart, const uint2* __restrict__ fail, uint32_t* __restrict__ key) {
  kd_check_entry(in, fr, starts, nf, total, q, rowstart, fail, key);
}

__global__ void __launch_bounds__(KD_NT)
    kd_store_kernel(const uint8_t* __restrict__ in, const KdFrameDev* __restrict__ fr,
                    const uint32_t* __restrict__ starts, uint32_t nf, uint32_t total, const uint32_t* __restrict__ q,
                    const uint32_t* __restrict__ rowstart, const uint2* __restrict__ fail,
                    const uint32_t* __restrict__ key, const uint16_t* __restrict__ tables, uint8_t* __restrict__ out,
                    uint2* __restrict__ results, int32_t* __restrict__ values) {
  kd_store_entry(in, fr, starts, nf, total, q, rowstart, fail, key, tables, out, results, values);
}
#endif

} // namespace rsb200
