// pana.cuh -- K7: Panasonic RW2 block codecs V4 / V5 / V6 / V7 (SURVEY 8(f)4), sm_90a.
//
// Replaces the bodies of
//   PanasonicV4Decompressor::processBlock / processPixelPacket
//       decompressors/PanasonicV4Decompressor.cpp:171-236 (+ ProxyStream :129-168); the
//       packet arithmetic is in pana4_core.h.  (VER == 4 was developed against a CPU replay,
//       tests/test_pana4_emu.py.)
//   PanasonicV5Decompressor::processBlock / processPixelPacket
//       decompressors/PanasonicV5Decompressor.cpp:188-232 (+ ProxyStream :147-186)
//   PanasonicV6Decompressor::decompressBlock  PanasonicV6Decompressor.cpp:88-221
//   PanasonicV7Decompressor::decompressBlock  PanasonicV7Decompressor.cpp:66-73
// and their OpenMP loops over blocks / rows.  All three cut the image into
// independent 16-byte units read as LSB-first bit streams:
//   V4  packets of 14 pixels (8-bit differences with a per-triplet shift, one 12-bit start
//       value per colour) inside 0x4000-byte blocks whose two sections (split at
//       section_split_offset) are swapped; pixels decoded as 0 can be reported as bad;
//   V5  packets of 10 x 12 or 9 x 14 bits inside 0x4000-byte blocks whose two
//       sections (split at 0x1FF8) are swapped; pixels numbered linearly over
//       the image (width is a multiple of the packet size);
//   V6  blocks of 14 (12 bit) / 11 (14 bit) pixels: 2 full-width pixels, then
//       triplets sharing a 2-bit scale, with an odd/even running reference;
//   V7  blocks of 9 x 14 bits.
// One thread = one unit: 16 input bytes -> 9..14 uint16 (every field offset is a
// compile-time constant).  HBM-bound streaming maps.
#pragma once

#include "common.cuh"
#include "pana4_core.h"

namespace rsb200 {

constexpr int PANA_NT = 256;

struct PanaJobDev {
  uint64_t in_offset;
  uint64_t out_offset;
  uint32_t out_pitch;
  uint32_t width;
  uint32_t height;
  uint32_t unit_begin; // first unit of this job in the group
  uint32_t units;      // units that carry pixels of the image
  uint32_t split;      // V4: section_split_offset
  uint32_t zero_slot;  // V4: 1 + index of the job's bad-pixel list, 0 = zeros are not bad
};

constexpr uint32_t PANA_ZERO_CAP = 1u << 22; // bad-pixel positions kept per job and run

// n bits at compile-time bit offset OFF of the 128-bit little-endian number w[0..3]
template <int OFF, int N>
__device__ __forceinline__ uint32_t pana_field(const uint32_t (&w)[4]) {
  constexpr int k = OFF >> 5, s = OFF & 31;
  uint32_t v = w[k] >> s;
  if constexpr (s + N > 32 && k < 3)
    v |= w[k + 1] << (32 - s);
  return v & ((1u << N) - 1u);
}

template <int BPS, int I, int NPIX>
__device__ __forceinline__ void pana_unpack(const uint32_t (&w)[4], uint32_t (&px)[14]) {
  if constexpr (I < NPIX) {
    px[I] = pana_field<I * BPS, BPS>(w);
    pana_unpack<BPS, I + 1, NPIX>(w, px);
  }
}

// V6 page buffer (PanasonicV6Decompressor.cpp:88-142): entry K of the buffer; the
// buffer is filled from its end, entry 0/1 are the two full-width pixels.
template <int BPS, int K> __device__ __forceinline__ uint32_t pana6_entry(const uint32_t (&w)[4]) {
  constexpr int NBUF = BPS == 14 ? 14 : 18;
  constexpr int SMALL = BPS == 14 ? 10 : 8;
  constexpr int LEAD = BPS == 14 ? 4 : 0;
  if constexpr (K == 0) {
    return pana_field<128 - BPS, BPS>(w);
  } else if constexpr (K == 1) {
    return pana_field<128 - 2 * BPS, BPS>(w);
  } else {
    // entries NBUF-1 down to 2 in stream order; widths: SMALL, except 2 bits where K % 4 == 2
    constexpr int pos = NBUF - 1 - K; // position in stream order
    constexpr int groups = pos / 4, rem = pos % 4; // each group of 4 = 3 SMALL + one 2-bit
    constexpr int off = LEAD + groups * (3 * SMALL + 2) + rem * SMALL;
    constexpr int n = (K % 4 == 2) ? 2 : SMALL;
    return pana_field<off, n>(w);
  }
}

template <int BPS, int PIX, int CUR>
__device__ __forceinline__ void pana6_pixels(const uint32_t (&w)[4], uint32_t (&px)[14],
                                             uint32_t (&oddeven)[2], uint32_t (&nonzero)[2],
                                             uint32_t& pmul, uint32_t& pixel_base) {
  constexpr int NPIX = BPS == 14 ? 11 : 14;
  if constexpr (PIX < NPIX) {
    constexpr uint32_t PixelbaseZero = BPS == 14 ? 0x200u : 0x80u;
    constexpr uint32_t PixelbaseCompare = BPS == 14 ? 0x2000u : 0x800u;
    constexpr uint32_t SpixCompare = BPS == 14 ? 0xffffu : 0x3fffu;
    constexpr uint32_t PixelMask = BPS == 14 ? 0x3fffu : 0xfffu;
    constexpr bool has_base = (PIX % 3 == 2);
    if constexpr (has_base) {
      uint32_t base = pana6_entry<BPS, CUR>(w);
      if (base == 3)
        base = 4;
      pixel_base = PixelbaseZero << base;
      pmul = 1u << base;
    }
    constexpr int E = CUR + (has_base ? 1 : 0);
    uint32_t epixel = pana6_entry<BPS, E>(w);
    constexpr int par = PIX % 2;
    if (oddeven[par]) {
      epixel = (epixel * pmul) & 0xFFFFu;
      if (pixel_base < PixelbaseCompare && nonzero[par] > pixel_base)
        epixel = (epixel + (nonzero[par] - pixel_base)) & 0xFFFFu;
      nonzero[par] = epixel;
    } else {
      oddeven[par] = epixel;
      if (epixel)
        nonzero[par] = epixel;
      else
        epixel = nonzero[par] & 0xFFFFu;
    }
    const uint32_t spix = (uint32_t)((int)epixel - 0xf);
    if (spix <= SpixCompare)
      px[PIX] = spix & SpixCompare;
    else
      px[PIX] = ((uint32_t)((int)(epixel + 0x7ffffff1u) >> 0x1f) & 0xFFFFu) & PixelMask;
    pana6_pixels<BPS, PIX + 1, E + 1>(w, px, oddeven, nonzero, pmul, pixel_base);
  }
}

// VER 4 (BPS 12) / 5 / 6 / 7, BPS 12 / 14.  zero_count / zero_list: V4 bad-pixel lists
// (PANA_ZERO_CAP positions per list), unused otherwise.
template <int VER, int BPS>
__global__ void __launch_bounds__(PANA_NT)
    pana_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                const PanaJobDev* __restrict__ jobs, int njobs, uint32_t total_units,
                uint32_t* __restrict__ zero_count, uint32_t* __restrict__ zero_list) {
  constexpr int NPIX = VER == 4 ? 14 : (VER == 6 ? (BPS == 14 ? 11 : 14) : 128 / BPS);
  const uint32_t u_raw = blockIdx.x * PANA_NT + threadIdx.x;
  const bool live = u_raw < total_units;
  const uint32_t u = live ? u_raw : total_units - 1u; // (idle threads of the last CTA mirror the last unit)
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].unit_begin <= u)
      lo = mid;
    else
      hi = mid - 1;
  }
  const PanaJobDev jb = jobs[lo];
  const uint32_t ul = u - jb.unit_begin;
  const uint8_t* base = in + jb.in_offset;
  uint32_t w[4];
  auto load8 = [&](const uint8_t* p, uint32_t& a, uint32_t& b) {
    // 8 bytes at any alignment: three aligned words, funnel-shifted
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u);
    const uint32_t* pw = reinterpret_cast<const uint32_t*>(p - mis);
    const uint32_t x0 = __ldg(pw), x1 = __ldg(pw + 1), x2 = mis ? __ldg(pw + 2) : 0u;
    a = __funnelshift_r(x0, x1, 8u * mis);
    b = __funnelshift_r(x1, x2, 8u * mis);
  };
  if (VER == 4) {
    // packet ul of the image = packet ul % 1024 of block ul / 1024, through the section swap
    const uint32_t blk = ul >> 10, o = (ul & 1023u) * 16u;
    if ((jb.split & 7u) == 0) { // (the decoder's 0x2008 / 0): an 8-byte half never wraps
      load8(base + pana4_src(blk, o, jb.split), w[0], w[1]);
      load8(base + pana4_src(blk, o + 8u, jb.split), w[2], w[3]);
    } else {
      w[0] = w[1] = w[2] = w[3] = 0u;
#pragma unroll
      for (uint32_t i = 0; i < 16; ++i)
        w[i >> 2] |= (uint32_t)__ldg(base + pana4_src(blk, o + i, jb.split)) << (8u * (i & 3u));
    }
  } else if (VER == 5) {
    // packet ul of the image = packet ul % 1024 of block ul / 1024, read through the
    // section swap: rearranged byte j of a block is original byte (j + 0x1FF8) % 0x4000
    const uint32_t blk = ul >> 10, o = (ul & 1023u) * 16u;
    const uint8_t* bp = base + (uint64_t)blk * 0x4000u;
    load8(bp + ((o + 0x1FF8u) & 0x3FFFu), w[0], w[1]);
    load8(bp + ((o + 8u + 0x1FF8u) & 0x3FFFu), w[2], w[3]);
  } else {
    const uint8_t* p = base + (uint64_t)ul * 16u;
    load8(p, w[0], w[1]);
    load8(p + 8, w[2], w[3]);
  }
  uint32_t px[14];
  if (VER == 4) {
    const uint32_t zeros = pana4_packet(w, px);
    if (live && zeros && jb.zero_slot) {
      // mRaw->mBadPixelPositions (PanasonicV4Decompressor.cpp:206-207, :228-235): (y << 16) | x
      const uint32_t idx0 = ul * 14u;
      const uint32_t row = idx0 / jb.width, col0 = idx0 - row * jb.width;
      for (uint32_t z = zeros; z; z &= z - 1u) {
        const uint32_t i = (uint32_t)__ffs((int)z) - 1u;
        const uint32_t at = atomicAdd(zero_count + (jb.zero_slot - 1u), 1u);
        if (at < PANA_ZERO_CAP)
          zero_list[(uint64_t)(jb.zero_slot - 1u) * PANA_ZERO_CAP + at] = (row << 16) | (col0 + i);
      }
    }
  } else if (VER == 6) {
    uint32_t oddeven[2] = {0, 0}, nonzero[2] = {0, 0}, pmul = 0, pixel_base = 0;
    pana6_pixels<BPS, 0, 0>(w, px, oddeven, nonzero, pmul, pixel_base);
  } else {
    pana_unpack<BPS, 0, NPIX>(w, px);
  }
  // ---- pixels -> image, coalesced: the CTA's units are consecutive pixels of the image
  //      (consecutive units of one job; a job change inside the CTA falls back to direct
  //      stores), so they are staged in shared memory and written out as aligned 32-bit
  //      words, 128 contiguous bytes per warp instruction instead of 32 scattered uint16 ----
  __shared__ uint16_t stage[PANA_NT * 14];
  __shared__ int same_job;
  const uint32_t u0 = blockIdx.x * PANA_NT; // first unit of the CTA
  if (threadIdx.x == 0) {
    const uint32_t ulast = min(u0 + PANA_NT, total_units) - 1u;
    same_job = (jobs[lo].unit_begin <= u0 && ulast - jb.unit_begin < jb.units) ? 1 : 0;
  }
  if (live) {
#pragma unroll
    for (int i = 0; i < NPIX; ++i)
      stage[threadIdx.x * NPIX + i] = (uint16_t)px[i];
  }
  __syncthreads();
  if (!same_job) {
    if (!live)
      return;
    const uint32_t idx = ul * NPIX; // (< 2^32: checked at plan creation) a unit never straddles rows
    const uint32_t row = idx / jb.width, col = idx - row * jb.width;
    uint16_t* o16 = reinterpret_cast<uint16_t*>(out + jb.out_offset + (uint64_t)row * jb.out_pitch) + col;
#pragma unroll
    for (int i = 0; i < NPIX; ++i)
      o16[i] = (uint16_t)px[i];
    return;
  }
  {
    const uint32_t nunits = min((uint32_t)PANA_NT, total_units - u0);
    const uint32_t npx = nunits * NPIX;
    const uint32_t p0 = (u0 - jb.unit_begin) * NPIX; // first pixel of the CTA in the image (< 2^32)
    uint8_t* obase = out + jb.out_offset;
    // pixel k of the CTA -> byte address; rows are out_pitch apart
    uint32_t row = p0 / jb.width;
    uint32_t col = p0 - row * jb.width;
    // walk the CTA's pixels row by row: segment [k0, k1) lies in `row` starting at `col`
    uint32_t k0 = 0;
    while (k0 < npx) {
      const uint32_t k1 = min(npx, k0 + (jb.width - col));
      uint8_t* rowp = obase + (uint64_t)row * jb.out_pitch + 2ull * col;
      const uint32_t n = k1 - k0;
      // leading pixel to reach 4-byte alignment, then pairs, then a trailing pixel
      const uint32_t lead = ((reinterpret_cast<uintptr_t>(rowp) & 2u) && n) ? 1u : 0u;
      if (lead && threadIdx.x == 0)
        *reinterpret_cast<uint16_t*>(rowp) = stage[k0];
      const uint32_t npairs = (n - lead) >> 1;
      uint32_t* o32 = reinterpret_cast<uint32_t*>(rowp + 2u * lead);
      for (uint32_t q = threadIdx.x; q < npairs; q += PANA_NT) {
        const uint32_t a = stage[k0 + lead + 2 * q], b = stage[k0 + lead + 2 * q + 1];
        o32[q] = a | (b << 16);
      }
      if (((n - lead) & 1u) && threadIdx.x == 1)
        reinterpret_cast<uint16_t*>(rowp)[n - 1] = stage[k1 - 1];
      k0 = k1;
      ++row;
      col = 0;
    }
  }
}

} // namespace rsb200
