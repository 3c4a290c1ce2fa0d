// arw2.cuh -- K6: Sony ARW2 block codec (SURVEY 8(f)4), sm_90a.
//
// Replaces the body of SonyArw2Decompressor::decompressRow
// (decompressors/SonyArw2Decompressor.cpp:58-112) and the per-row OpenMP loop
// (:114-133): one byte per pixel; a row is an LSB-first bit stream of 128-bit
// blocks, each block = max(11) min(11) imax(4) imin(4) + 14 x 7-bit deltas for 16
// pixels of the same column parity (the blocks of the even and of the odd pixels
// of 32 columns follow each other).  Every value goes through
// RawImageDataU16::setWithLookUp (common/RawImage.h:335-353).
//
// One thread = 32 columns = two blocks = 32 input bytes -> 64 output bytes (four
// 128-bit stores).  The only serial dependency of the reference, the dither
// state of setWithLookUp (r' = 15700*(r & 65535) + (r >> 16), seeded per row with
// the row's first 24 bits), is a multiply-with-carry generator: for r below
// m = 15700*2^16 - 1 it equals r' = 15700*r mod m, so the state at call n of the
// row is r0 * 15700^n mod m and a thread jumps to its 32 calls with one modular
// multiplication by a constant from a 300-entry table.
#pragma once

#include "common.cuh"

namespace rsb200 {

constexpr int ARW2_NT = 256;
constexpr uint32_t ARW2_M = 15700u * 65536u - 1u; // modulus of the dither generator
constexpr int ARW2_MAX_GROUPS = 300;              // 9600 / 32 columns

struct Arw2JobDev {
  uint64_t in_offset;
  uint64_t out_offset;
  uint32_t out_pitch;
  uint32_t width;
  uint32_t height;
  uint32_t groups_per_row; // width / 32
  uint32_t group_begin;    // first group of this job in the plan
  int32_t table;           // plan table index (-1: no table)
};

__constant__ uint32_t c_arw2_jump[ARW2_MAX_GROUPS]; // 15700^(32 g) mod ARW2_M

// MODE 0: no table, 1: plain table (4096 x u16), 2: dithered table (4096 x {base, delta}).
// SM: the table sits in shared memory (plans with one table), else it is read through L1.
template <int MODE, bool SM>
__device__ __forceinline__ uint32_t arw2_lookup(const uint16_t* __restrict__ tab, uint32_t value,
                                                uint32_t& r) {
  if (MODE == 0)
    return value;
  if (MODE == 1)
    return SM ? (uint32_t)tab[value] : (uint32_t)__ldg(tab + value);
  const uint32_t e = SM ? reinterpret_cast<const uint32_t*>(tab)[value]
                        : __ldg(reinterpret_cast<const uint32_t*>(tab) + value);
  const uint32_t base = e & 0xFFFFu, delta = e >> 16;
  const uint32_t pix = base + ((delta * (r & 2047u) + 1024u) >> 12);
  r = 15700u * (r & 65535u) + (r >> 16);
  return pix & 0xFFFFu;
}

// bits [OFF, OFF+7) of the 128-bit little-endian number w0..w3 (OFF compile-time)
template <int OFF>
__device__ __forceinline__ uint32_t arw2_delta(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
  constexpr int k = OFF >> 5, s = OFF & 31;
  const uint32_t lo = k == 0 ? w0 : (k == 1 ? w1 : (k == 2 ? w2 : w3));
  const uint32_t hi = k == 0 ? w1 : (k == 1 ? w2 : (k == 2 ? w3 : 0u));
  uint32_t v = lo >> s;
  if constexpr (s + 7 > 32)
    v |= hi << (32 - s);
  return v & 127u;
}

// 16 pixels of one block (w0..w3 = the block as a little-endian 128-bit number).  The 14
// deltas sit at fixed bit offsets 30 + 7k; pixel i uses delta i, i-1 or i-2 depending on
// how many of imax / imin lie before it -- two selects instead of a 128-bit shift register.
template <int MODE, bool SM, int I>
__device__ __forceinline__ void arw2_pixels(const uint32_t (&d)[14], int vmax, int vmin,
                                            uint32_t imax, uint32_t imin, uint32_t lo, uint32_t hi,
                                            int sh, const uint16_t* __restrict__ tab, uint32_t& r,
                                            uint32_t (&px)[16]) {
  if constexpr (I < 16) {
    // delta index = I - (lo < I) - (hi < I)
    const uint32_t a = d[I < 14 ? I : 13], b = d[I >= 1 ? (I - 1 < 14 ? I - 1 : 13) : 0],
                   c = d[I >= 2 ? I - 2 : 0];
    const uint32_t dl = ((int)hi < I) ? c : (((int)lo < I) ? b : a);
    int p = min((int)(dl << sh) + vmin, 0x7ff);
    if ((uint32_t)I == imin)
      p = vmin;
    if ((uint32_t)I == imax)
      p = vmax;
    px[I] = arw2_lookup<MODE, SM>(tab, (uint32_t)p << 1, r);
    arw2_pixels<MODE, SM, I + 1>(d, vmax, vmin, imax, imin, lo, hi, sh, tab, r, px);
  }
}

template <int MODE, bool SM>
__device__ __forceinline__ bool arw2_block(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3,
                                           const uint16_t* __restrict__ tab, uint32_t& r,
                                           uint32_t (&px)[16]) {
  const int vmax = (int)(w0 & 0x7FFu), vmin = (int)((w0 >> 11) & 0x7FFu);
  const uint32_t imax = (w0 >> 22) & 15u, imin = (w0 >> 26) & 15u;
  int sh = 0;
  while (sh < 4 && (0x80 << sh) <= (vmax - vmin))
    ++sh;
  uint32_t d[14];
  d[0] = arw2_delta<30>(w0, w1, w2, w3);
  d[1] = arw2_delta<37>(w0, w1, w2, w3);
  d[2] = arw2_delta<44>(w0, w1, w2, w3);
  d[3] = arw2_delta<51>(w0, w1, w2, w3);
  d[4] = arw2_delta<58>(w0, w1, w2, w3);
  d[5] = arw2_delta<65>(w0, w1, w2, w3);
  d[6] = arw2_delta<72>(w0, w1, w2, w3);
  d[7] = arw2_delta<79>(w0, w1, w2, w3);
  d[8] = arw2_delta<86>(w0, w1, w2, w3);
  d[9] = arw2_delta<93>(w0, w1, w2, w3);
  d[10] = arw2_delta<100>(w0, w1, w2, w3);
  d[11] = arw2_delta<107>(w0, w1, w2, w3);
  d[12] = arw2_delta<114>(w0, w1, w2, w3);
  d[13] = arw2_delta<121>(w0, w1, w2, w3);
  arw2_pixels<MODE, SM, 0>(d, vmax, vmin, imax, imin, min(imax, imin), max(imax, imin), sh, tab, r, px);
  return imax != imin;
}

constexpr int ARW2_GPT = 4; // groups (of 32 columns) per thread

template <int MODE, bool SM>
__global__ void __launch_bounds__(ARW2_NT)
    arw2_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                const Arw2JobDev* __restrict__ jobs, int njobs, uint32_t total_groups,
                const uint16_t* __restrict__ tables, uint32_t* __restrict__ bad_jobs) {
  __shared__ __align__(16) uint16_t s_tab[SM ? (MODE == 2 ? 8192 : 4096) : 8];
  if (SM) { // the plan's single table: the 4096 entries a value can reach
    constexpr int n16 = (MODE == 2 ? 8192 : 4096) / 8;
    const uint4* src = reinterpret_cast<const uint4*>(tables);
    uint4* dst = reinterpret_cast<uint4*>(s_tab);
    for (int i = threadIdx.x; i < n16; i += ARW2_NT)
      dst[i] = src[i];
    __syncthreads();
  }
  for (int it = 0; it < ARW2_GPT; ++it) {
    const uint32_t g = (blockIdx.x * ARW2_GPT + it) * ARW2_NT + threadIdx.x;
    if (g >= total_groups)
      return;
    int lo = 0, hi = njobs - 1; // job of this group
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (jobs[mid].group_begin <= g)
        lo = mid;
      else
        hi = mid - 1;
    }
    const Arw2JobDev jb = jobs[lo];
    const uint32_t gl = g - jb.group_begin;
    const uint32_t row = gl / jb.groups_per_row, gx = gl - row * jb.groups_per_row;
    const uint8_t* rowp = in + jb.in_offset + (uint64_t)row * jb.width;
    // 32 input bytes at any alignment: nine aligned words, funnel-shifted
    uint32_t w[8];
    {
      const uint8_t* p = rowp + gx * 32u;
      const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u);
      const uint32_t* pw = reinterpret_cast<const uint32_t*>(p - mis);
      uint32_t a[9];
#pragma unroll
      for (int k = 0; k < 8; ++k)
        a[k] = __ldg(pw + k);
      a[8] = mis ? __ldg(pw + 8) : 0u;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        w[k] = __funnelshift_r(a[k], a[k + 1], 8u * mis);
    }
    const uint16_t* tab = nullptr;
    uint32_t r = 0;
    if (MODE != 0)
      tab = SM ? s_tab : tables + (size_t)jb.table * (MODE == 2 ? 8192u : 4096u);
    if (MODE == 2) {
      // dither state of the row before call 32*gx
      const uint32_t r0 = (uint32_t)rowp[0] | ((uint32_t)rowp[1] << 8) | ((uint32_t)rowp[2] << 16);
      r = (uint32_t)(((uint64_t)r0 * c_arw2_jump[gx]) % ARW2_M);
    }
    uint32_t ev[16], od[16];
    bool ok = arw2_block<MODE, SM>(w[0], w[1], w[2], w[3], tab, r, ev);
    ok = arw2_block<MODE, SM>(w[4], w[5], w[6], w[7], tab, r, od) && ok;
    if (!ok) // "ARW2 invariant failed, same pixel is both min and max"
      atomicOr(bad_jobs + lo, 1u);
    uint8_t* op = out + jb.out_offset + (uint64_t)row * jb.out_pitch + gx * 64u;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint4 o;
      o.x = ev[4 * q + 0] | (od[4 * q + 0] << 16);
      o.y = ev[4 * q + 1] | (od[4 * q + 1] << 16);
      o.z = ev[4 * q + 2] | (od[4 * q + 2] << 16);
      o.w = ev[4 * q + 3] | (od[4 * q + 3] << 16);
      stg_cs_v4(op + 16 * q, o);
    }
  }
}

} // namespace rsb200
