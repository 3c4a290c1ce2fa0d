// arw1.cuh -- Sony ARW1 (SonyArw1Decompressor::decompress, decompressors/SonyArw1Decompressor.cpp:
// 58-92, paths relative to src/librawspeed of rawspeed), sm_90a.
//
// The reference reads one plain MSB stream (BitStreamerMSB, a 32-bit fill before every symbol) and
// walks the frame column by column from the right, even rows top to bottom, then odd rows, with one
// running predictor `pred += diff` that must stay in 0..4095 (isIntN(pred, 12)).
//
// Entropy stage.  The code (11 -> 1, 10 -> 2, 011 -> 0, 010 -> 3, 00 0^k 1 -> 4 + k, 00 0^13 -> 17,
// then `len` extra bits through extend()) is not canonical, but its bitwise complement is: code
// lengths 2, 2, 3, 3, 3, then one per length 4..15, in canonical order.  Complementing the extra
// bits negates extend(), so the complemented stream is an ordinary plain-MSB prefix-code stream
// whose differences are the negated ARW1 differences.
// arw1_prep_kernel writes that stream (and 16 bytes of 0xFF: the zero bits the reference may read
// behind the buffer) into a scratch buffer, and the multi-CTA range decoder (ljpeg_ranges.cuh, the
// plain MSB pump, one table) decodes it unchanged.  The table maps length 17 (code 1^15, then 17
// extra bits) to two 16-bit codes with SSSS = 16 and the DNG rule (16 more bits): both lengths 16
// and 17 come out as -32768, a sentinel.  Every length >= 13 has |d| >= 4096 and violates the range
// check at once, so no such symbol ever decodes to a pixel; lengths 13..15 fit int16 as they are.
//
// Reconstruction.  Stream index i is column w-1-i/h, k = i % h, row 2k (k < h/2) or 2(k-h/2)+1.
// The differences are cut into runs of 32 entries of one half-column (run ids in stream order):
//   arw1_runsum_kernel  one warp per run: sum, min / max of the in-run prefix, sentinel, the bits
//                       the run's symbols take (recomputed from each difference's length) and the
//                       offset of its last symbol
//   arw1_scan_kernel    one CTA per frame: exact int32 prefix of the runs in stream order (every
//                       prefix up to the first violation is exact; later wrap is harmless) and of
//                       their bit positions; the first run holding a violation and the first run
//                       holding a symbol whose refill fails (plain_overread) decide the outcome
//   arw1_apply_kernel   one CTA per 64x64 tile (rows 64t.., one run of each half-column of 64
//                       columns): warp scans of the runs into shared memory, then 128-byte row
//                       stores of the decoded pixels; the warp of the deciding run resolves the
//                       exact symbol and writes the result
#pragma once

#include "ljpeg.cuh"

namespace rsb200 {

struct DevArw1 {
  uint64_t in_offset;   // first byte of the stream in the input buffer
  uint64_t k_offset;    // first byte of the complemented copy in the scratch buffer
  uint64_t diff_offset; // first difference (stream order) in the plan's diff buffer
  uint64_t run_offset;  // first run of this frame in the run arrays
  uint64_t out_offset;
  uint32_t in_size;
  uint32_t w, h;
  uint32_t out_pitch;
  uint32_t nrh;     // runs per half-column = ceil(h / 64)
  uint32_t tstar;   // first stream bit at which a symbol's refill fails (plain_overread)
  uint32_t scan;    // index of the frame's scan / result
  uint32_t pad;
};

struct Arw1Run {
  int32_t sum;   // sum of the run's differences
  int32_t mn;    // min / max of its inclusive prefix (mn = -2^30 when it holds a sentinel)
  int32_t mx;
  uint32_t bits; // stream bits of its symbols
};

struct Arw1Info {
  uint32_t lim; // first deciding run (0xFFFFFFFF: the frame decodes)
  uint32_t vrun;
  uint32_t erun;
  uint32_t pad;
};

constexpr int ARW1_SENTINEL = -32768;

// stream bits of the symbol of (negated) difference dd: code + extra bits (lengths <= 16)
__device__ __forceinline__ uint32_t arw1_sym_bits(int dd) {
  const uint32_t a = (uint32_t)(dd < 0 ? -dd : dd);
  const uint32_t L = 32u - __clz(a);
  const uint32_t cb = L == 0 ? 3u : (L <= 2 ? 2u : (L == 3 ? 3u : L - 1u));
  return cb + L;
}

// complemented copy of each stream + 16 bytes of 0xFF; grid (words, frames).  The copy is 16-byte
// aligned; each thread writes 4 bytes as one word, read as two aligned words of the input (the
// input base is 16-byte aligned) except at the end of the stream
__global__ void arw1_prep_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ kin,
                                 const DevArw1* __restrict__ fr) {
  const DevArw1 f = fr[blockIdx.y];
  const uint32_t n = f.in_size + 16u;
  const uint32_t sh = 8u * (uint32_t)(f.in_offset & 3u);
  const uint32_t* src = reinterpret_cast<const uint32_t*>(in + (f.in_offset & ~3ull));
  uint32_t* dst = reinterpret_cast<uint32_t*>(kin + f.k_offset);
  for (uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) * 4u; j < n;
       j += gridDim.x * blockDim.x * 4u) {
    uint32_t v;
    if (j + 8u <= f.in_size) {
      v = ~__funnelshift_r(__ldg(src + (j >> 2)), __ldg(src + (j >> 2) + 1), sh);
    } else {
      v = 0;
#pragma unroll
      for (uint32_t b = 0; b < 4; ++b) {
        const uint32_t p = j + b;
        const uint32_t c = p < f.in_size ? (uint8_t)~in[f.in_offset + p] : 0xFFu;
        v |= c << (8 * b);
      }
    }
    dst[j >> 2] = v;
  }
}

struct Arw1Lane {
  int dd;        // negated difference of this lane's symbol (0 for idle lanes)
  int pv;        // inclusive in-run prefix of the differences
  uint32_t sb;   // symbol bits
  uint32_t xb;   // exclusive in-run prefix of the symbol bits
};

__device__ __forceinline__ Arw1Lane arw1_lane(const int16_t* d, uint32_t lane, uint32_t n) {
  Arw1Lane a;
  a.dd = lane < n ? (int)d[lane] : 0;
  a.sb = lane < n ? arw1_sym_bits(a.dd) : 0u;
  int v = -a.dd;
  uint32_t b = a.sb;
#pragma unroll
  for (int k = 1; k < 32; k <<= 1) {
    const int x = __shfl_up_sync(0xFFFFFFFFu, v, k);
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, b, k);
    if ((int)lane >= k) {
      v += x;
      b += y;
    }
  }
  a.pv = v;
  a.xb = b - a.sb;
  return a;
}

// stream base index and length of run r = (ci * 2 + q) * nrh + k
__device__ __forceinline__ void arw1_run_span(const DevArw1& f, uint32_t r, uint32_t& i0,
                                              uint32_t& n) {
  const uint32_t k = r % f.nrh, cq = r / f.nrh, q = cq & 1u, ci = cq >> 1;
  const uint32_t half = f.h / 2u;
  i0 = ci * f.h + q * half + 32u * k;
  n = min(32u, half - 32u * k);
}

constexpr int ARW1_NT = 256;

__global__ void __launch_bounds__(ARW1_NT)
    arw1_runsum_kernel(const DevArw1* __restrict__ fr, const uint16_t* __restrict__ diffs,
                       Arw1Run* __restrict__ runs, uint32_t* __restrict__ lastoff) {
  const DevArw1 f = fr[blockIdx.y];
  const uint32_t r = (blockIdx.x * ARW1_NT + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (r >= f.w * 2u * f.nrh)
    return;
  uint32_t i0, n;
  arw1_run_span(f, r, i0, n);
  const int16_t* d = reinterpret_cast<const int16_t*>(diffs + f.diff_offset + i0);
  const Arw1Lane a = arw1_lane(d, lane, n);
  int mn = lane < n ? a.pv : 0x7FFFFFFF, mx = lane < n ? a.pv : -0x7FFFFFFF - 1;
#pragma unroll
  for (int k = 16; k; k >>= 1) {
    mn = min(mn, __shfl_xor_sync(0xFFFFFFFFu, mn, k));
    mx = max(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, k));
  }
  const bool sent = __any_sync(0xFFFFFFFFu, lane < n && a.dd == ARW1_SENTINEL);
  const int sum = __shfl_sync(0xFFFFFFFFu, a.pv, n - 1);
  const uint32_t last = __shfl_sync(0xFFFFFFFFu, a.xb, n - 1);
  const uint32_t bits = last + __shfl_sync(0xFFFFFFFFu, a.sb, n - 1);
  if (lane == 0) {
    Arw1Run o;
    o.sum = sum;
    o.mn = sent ? -(1 << 30) : mn;
    o.mx = mx;
    o.bits = bits;
    runs[f.run_offset + r] = o;
    lastoff[f.run_offset + r] = last;
  }
}

constexpr int ARW1_SCAN_NT = 1024;
constexpr int ARW1_SCAN_PER = 8; // runs per thread and step

__global__ void __launch_bounds__(ARW1_SCAN_NT)
    arw1_scan_kernel(const DevArw1* __restrict__ fr, const Arw1Run* __restrict__ runs,
                     const uint32_t* __restrict__ lastoff, int2* __restrict__ runpre,
                     Arw1Info* __restrict__ info, DevResult* __restrict__ results) {
  __shared__ uint32_t s_sum[ARW1_SCAN_NT / 32];
  __shared__ uint32_t s_bits[ARW1_SCAN_NT / 32];
  __shared__ uint32_t s_v, s_e;
  const DevArw1 f = fr[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint32_t R = f.w * 2u * f.nrh;
  const Arw1Run* rr = runs + f.run_offset;
  const uint32_t* lo = lastoff + f.run_offset;
  int2* pre = runpre + f.run_offset;
  if (tid == 0)
    s_v = s_e = 0xFFFFFFFFu;
  uint32_t carry = 0, carry_b = 0;
  for (uint32_t base = 0; base < R; base += ARW1_SCAN_NT * ARW1_SCAN_PER) {
    const uint32_t r0 = base + (uint32_t)tid * ARW1_SCAN_PER;
    Arw1Run q[ARW1_SCAN_PER];
    uint32_t s = 0, b = 0;
#pragma unroll
    for (int k = 0; k < ARW1_SCAN_PER; ++k) {
      if (r0 + k < R) {
        q[k] = rr[r0 + k];
      } else {
        q[k].sum = q[k].mn = q[k].mx = 0;
        q[k].bits = 0;
      }
      s += (uint32_t)q[k].sum;
      b += q[k].bits;
    }
    uint32_t is = (uint32_t)s;
    uint32_t ib = b;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
      const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, is, k);
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, ib, k);
      if (lane >= k) {
        is += x;
        ib += y;
      }
    }
    if (lane == 31) {
      s_sum[wid] = is;
      s_bits[wid] = ib;
    }
    __syncthreads();
    uint32_t add = 0, tot = 0, addb = 0, totb = 0;
    for (int k = 0; k < ARW1_SCAN_NT / 32; ++k) {
      if (k < wid) {
        add += s_sum[k];
        addb += s_bits[k];
      }
      tot += s_sum[k];
      totb += s_bits[k];
    }
    // (int32 arithmetic that may wrap behind the first violation: done in uint32)
    uint32_t P = (uint32_t)carry + (uint32_t)add + (uint32_t)is - (uint32_t)s;
    uint32_t B = carry_b + addb + ib - b;
    uint32_t v = 0xFFFFFFFFu, e = 0xFFFFFFFFu;
#pragma unroll
    for (int k = 0; k < ARW1_SCAN_PER; ++k) {
      const uint32_t r = r0 + k;
      if (r < R) {
        pre[r] = make_int2((int)P, (int)B);
        if (v == 0xFFFFFFFFu &&
            ((int)(P + (uint32_t)q[k].mn) < 0 || (int)(P + (uint32_t)q[k].mx) > 4095))
          v = r;
        if (e == 0xFFFFFFFFu && B + __ldg(lo + r) >= f.tstar)
          e = r;
      }
      P += (uint32_t)q[k].sum;
      B += q[k].bits;
    }
    if (v != 0xFFFFFFFFu)
      atomicMin(&s_v, v);
    if (e != 0xFFFFFFFFu)
      atomicMin(&s_e, e);
    carry += tot;
    carry_b += totb;
    __syncthreads();
    if (min(s_v, s_e) != 0xFFFFFFFFu) // runs behind the deciding one are never decoded
      break;
  }
  if (tid == 0) {
    Arw1Info o;
    o.vrun = s_v;
    o.erun = s_e;
    o.lim = min(s_v, s_e);
    o.pad = 0;
    info[blockIdx.x] = o;
    results[f.scan].status = 0;
    results[f.scan].consumed = 0;
  }
}

constexpr int ARW1_TILE = 64;

__global__ void __launch_bounds__(ARW1_NT)
    arw1_apply_kernel(const DevArw1* __restrict__ fr, const uint16_t* __restrict__ diffs,
                      const int2* __restrict__ runpre, const Arw1Info* __restrict__ info,
                      uint8_t* __restrict__ out, DevResult* __restrict__ results) {
  __shared__ uint32_t tile[ARW1_TILE][ARW1_TILE + 1]; // bit 16: pixel decoded
  const DevArw1 f = fr[blockIdx.y];
  const uint32_t ntc = (f.w + ARW1_TILE - 1) / ARW1_TILE;
  if (blockIdx.x >= ntc * f.nrh)
    return;
  const uint32_t tr = blockIdx.x / ntc, tc = blockIdx.x % ntc; // tile row = run index k
  const Arw1Info inf = info[blockIdx.y];
  const int tid = threadIdx.x;
  const uint32_t lane = tid & 31u, wid = tid >> 5;
  for (int i = tid; i < ARW1_TILE * (ARW1_TILE + 1); i += ARW1_NT)
    (&tile[0][0])[i] = 0;
  __syncthreads();
  // 128 runs: (column cc of the tile, half q)
  for (uint32_t p = wid; p < 2u * ARW1_TILE; p += ARW1_NT / 32) {
    const uint32_t q = p & 1u, cc = p >> 1, c = tc * ARW1_TILE + cc;
    if (c >= f.w)
      continue;
    const uint32_t ci = f.w - 1u - c;
    const uint32_t r = (ci * 2u + q) * f.nrh + tr;
    if (r > inf.lim)
      continue;
    uint32_t i0, n;
    arw1_run_span(f, r, i0, n);
    const int16_t* d = reinterpret_cast<const int16_t*>(diffs + f.diff_offset + i0);
    const Arw1Lane a = arw1_lane(d, lane, n);
    const int2 pr = runpre[f.run_offset + r];
    const int pred = (int)((uint32_t)pr.x + (uint32_t)a.pv); // (wraps only behind a violation)
    uint32_t stop = n;
    if (r == inf.lim) {
      const bool viol = r == inf.vrun && lane < n &&
                        (a.dd == ARW1_SENTINEL || pred < 0 || pred > 4095);
      const bool ioe = r == inf.erun && lane < n && (uint32_t)pr.y + a.xb >= f.tstar;
      const uint32_t vm = __ballot_sync(0xFFFFFFFFu, viol), em = __ballot_sync(0xFFFFFFFFu, ioe);
      const uint32_t vl = vm ? (uint32_t)__ffs(vm) - 1u : 32u;
      const uint32_t el = em ? (uint32_t)__ffs(em) - 1u : 32u;
      // a failed refill throws before its symbol is decoded, a violation after its pixel
      stop = min(vl, el);
      if (lane == 0 && stop < 32u) {
        if (el <= vl) {
          results[f.scan].status = 2u;
          results[f.scan].consumed = 0;
        } else {
          const uint32_t row = 2u * (32u * tr + vl) + q;
          results[f.scan].status = 1u;
          results[f.scan].consumed = 0x80000000u | (row << 14) | c; // RSB200_PENTAX_OOB encoding
        }
      }
    }
    if (lane < stop)
      tile[2u * lane + q][cc] = 0x10000u | ((uint32_t)pred & 0xFFFFu);
  }
  __syncthreads();
  const uint32_t cc = tid & (ARW1_TILE - 1), c = tc * ARW1_TILE + cc;
  for (uint32_t rr = tid / ARW1_TILE; rr < ARW1_TILE; rr += ARW1_NT / ARW1_TILE) {
    const uint32_t row = tr * ARW1_TILE + rr;
    const uint32_t v = tile[rr][cc];
    if (row < f.h && c < f.w && (v & 0x10000u))
      *reinterpret_cast<uint16_t*>(out + f.out_offset + (uint64_t)row * f.out_pitch + 2ull * c) =
          (uint16_t)v;
  }
}

} // namespace rsb200
