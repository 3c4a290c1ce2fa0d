// rawforms.cuh -- K1b: the fixed-layout forms of UncompressedDecompressor that are
// not the generic N-bit bit pump (sm_90a).  Reference semantics, paths relative
// to /root/reference/src/librawspeed:
//   decode8BitRaw<uncorrected>            decompressors/UncompressedDecompressor.cpp:270-294
//     (+ RawImageDataU16::setWithLookUp   common/RawImage.h:335-353)
//   decode12BitRawWithControl<e>          decompressors/UncompressedDecompressor.cpp:299-359
//   decode12BitRawUnpackedLeftAligned<e>  decompressors/UncompressedDecompressor.cpp:366-390
//   decodePackedFP<Pump, Binary16/24>     decompressors/UncompressedDecompressor.cpp:171-186
//     (+ extendBinaryFloatingPoint        common/FloatingPoint.h:116-160)
//   32-bit float rows copied as they are  decompressors/UncompressedDecompressor.cpp:214-224
//
// All are pure streaming maps (HBM bound): one thread turns one "item" -- a fixed
// run of input bytes -- into 16 or 20 output bytes.  Input runs start at arbitrary
// byte addresses (row pitches like 1.5*w + (w+2)/10 are not word multiples), so an
// item is fetched as aligned 32-bit words and realigned with funnel shifts; stores
// are 128-bit whenever the destination allows.
#pragma once

#include "common.cuh"
#include "../../include/rawspeed_b200.h"

namespace rsb200 {

struct RawJobDev {
  uint64_t in_offset, out_offset;
  uint32_t out_pitch, in_pitch;
  uint32_t row0, rows, samples, out_col0;
  uint32_t format, table;
  uint32_t ipr;        // items per row
  uint32_t item_begin; // first global item of this job
};

constexpr int RAW_NT = 256;

__host__ __device__ constexpr uint32_t raw_item_samples(int format) {
  switch (format) {
  case RSB200_RAW_12BIT_CONTROL_BE:
  case RSB200_RAW_12BIT_CONTROL_LE:
    return 10;
  case RSB200_RAW_FP16_MSB:
  case RSB200_RAW_FP16_LSB:
  case RSB200_RAW_FP24_MSB:
  case RSB200_RAW_FP24_LSB:
  case RSB200_RAW_F32_COPY:
    return 4;
  default:
    return 8;
  }
}
__host__ __device__ constexpr uint32_t raw_out_sample_bytes(int format) {
  return format >= RSB200_RAW_FP16_MSB ? 4u : 2u;
}
// input bytes of `n` samples that start an item (item-aligned sample index)
__host__ __device__ constexpr uint32_t raw_in_bytes(int format, uint32_t n) {
  switch (format) {
  case RSB200_RAW_8BIT:
  case RSB200_RAW_8BIT_TABLE:
    return n;
  case RSB200_RAW_12BIT_CONTROL_BE:
  case RSB200_RAW_12BIT_CONTROL_LE:
    return n * 3 / 2; // (+ the control byte, never needed)
  case RSB200_RAW_12BIT_LEFT_BE:
  case RSB200_RAW_12BIT_LEFT_LE:
  case RSB200_RAW_FP16_MSB:
  case RSB200_RAW_FP16_LSB:
    return 2 * n;
  case RSB200_RAW_FP24_MSB:
  case RSB200_RAW_FP24_LSB:
    return 3 * n;
  default:
    return 4 * n;
  }
}
// input bytes between the starts of consecutive items of a row
__host__ __device__ constexpr uint32_t raw_item_stride(int format) {
  switch (format) {
  case RSB200_RAW_12BIT_CONTROL_BE:
  case RSB200_RAW_12BIT_CONTROL_LE:
    return 16; // 15 data bytes + 1 control byte
  default:
    return raw_in_bytes(format, raw_item_samples(format));
  }
}

// `nbytes` (<= 16) bytes at in[off..] as little-endian words s[0..3]; bytes at or
// beyond `in_total` read as 0 (never happens for validated jobs; keeps the word
// fetches inside the caller's buffer)
__device__ __forceinline__ void raw_fetch16(const uint8_t* __restrict__ in, uint64_t off,
                                            uint64_t in_total, uint32_t (&s)[4]) {
  const uint64_t a0 = off & ~3ull;
  const uint32_t sh = (uint32_t)(off & 3ull) * 8u;
  uint32_t w[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const uint64_t a = a0 + 4ull * k;
    if (a + 4 <= in_total) {
      w[k] = __ldg(reinterpret_cast<const uint32_t*>(in + a));
    } else {
      w[k] = 0;
      for (int b = 0; b < 4; ++b)
        if (a + b < in_total)
          w[k] |= (uint32_t)in[a + b] << (8 * b);
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k)
    s[k] = __funnelshift_r(w[k], w[k + 1], sh);
}

__device__ __forceinline__ uint32_t raw_byte(const uint32_t (&s)[4], int j) {
  return (s[j >> 2] >> (8 * (j & 3))) & 0xFFu;
}

// extendBinaryFloatingPoint<BinaryN<1+EW+FW>, Binary32> (FloatingPoint.h:116-160)
template <int FW, int EW> __device__ __forceinline__ uint32_t raw_fp_extend(uint32_t n) {
  const uint32_t sign = (n >> (FW + EW)) & 1u;
  const uint32_t e = (n >> FW) & ((1u << EW) - 1u);
  const uint32_t f = n & ((1u << FW) - 1u);
  constexpr int bias = (1 << (EW - 1)) - 1;
  uint32_t we = e - bias + 127;
  uint32_t wf = f << (23 - FW);
  if (e == (1u << EW) - 1u) {
    we = 255; // infinity / NaN: the fraction is kept, widened
  } else if (e == 0) {
    if (f == 0) {
      we = 0;
      wf = 0;
    } else { // subnormal: normalise (one exponent step per shift)
      const uint32_t k = (uint32_t)__clz((int)wf) - 8u;
      we = 1 - bias + 127 - k;
      wf = (wf << k) & 0x7FFFFFu;
    }
  }
  return (sign << 31) | (we << 23) | wf;
}

// out words of one full item; returns the number of 32-bit words produced (4 or 5)
__device__ __forceinline__ int raw_convert(int format, const uint32_t (&s)[4],
                                           const uint16_t* __restrict__ table,
                                           uint32_t (&o)[5]) {
  switch (format) {
  case RSB200_RAW_8BIT:
    o[0] = __byte_perm(s[0], 0, 0x4140);
    o[1] = __byte_perm(s[0], 0, 0x4342);
    o[2] = __byte_perm(s[1], 0, 0x4140);
    o[3] = __byte_perm(s[1], 0, 0x4342);
    return 4;
  case RSB200_RAW_8BIT_TABLE:
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = (uint32_t)__ldg(&table[raw_byte(s, 2 * k)]) |
             ((uint32_t)__ldg(&table[raw_byte(s, 2 * k + 1)]) << 16);
    return 4;
  case RSB200_RAW_12BIT_CONTROL_BE:
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const uint32_t g0 = raw_byte(s, 3 * k), g1 = raw_byte(s, 3 * k + 1),
                     g2 = raw_byte(s, 3 * k + 2);
      o[k] = ((g0 << 4) | (g1 >> 4)) | ((((g1 & 15u) << 8) | g2) << 16);
    }
    return 5;
  case RSB200_RAW_12BIT_CONTROL_LE:
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const uint32_t g0 = raw_byte(s, 3 * k), g1 = raw_byte(s, 3 * k + 1),
                     g2 = raw_byte(s, 3 * k + 2);
      o[k] = (((g1 & 15u) << 8) | g0) | (((g2 << 4) | (g1 >> 4)) << 16);
    }
    return 5;
  case RSB200_RAW_12BIT_LEFT_BE:
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = (__byte_perm(s[k], 0, 0x2301) >> 4) & 0x0FFF0FFFu;
    return 4;
  case RSB200_RAW_12BIT_LEFT_LE:
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = (s[k] >> 4) & 0x0FFF0FFFu;
    return 4;
  case RSB200_RAW_FP16_MSB:
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = raw_fp_extend<10, 5>((raw_byte(s, 2 * k) << 8) | raw_byte(s, 2 * k + 1));
    return 4;
  case RSB200_RAW_FP16_LSB:
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = raw_fp_extend<10, 5>(raw_byte(s, 2 * k) | (raw_byte(s, 2 * k + 1) << 8));
    return 4;
  case RSB200_RAW_FP24_MSB:
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = raw_fp_extend<16, 7>((raw_byte(s, 3 * k) << 16) | (raw_byte(s, 3 * k + 1) << 8) |
                                  raw_byte(s, 3 * k + 2));
    return 4;
  case RSB200_RAW_FP24_LSB:
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = raw_fp_extend<16, 7>(raw_byte(s, 3 * k) | (raw_byte(s, 3 * k + 1) << 8) |
                                  (raw_byte(s, 3 * k + 2) << 16));
    return 4;
  default: // RSB200_RAW_F32_COPY
#pragma unroll
    for (int k = 0; k < 4; ++k)
      o[k] = s[k];
    return 4;
  }
}

// One launch per format present in the plan (FORMAT is a template parameter so the
// conversion is straight-line code).
template <int FORMAT>
__global__ void __launch_bounds__(RAW_NT)
    rawform_kernel(const uint8_t* __restrict__ in, uint64_t in_total, uint8_t* __restrict__ out,
                   const RawJobDev* __restrict__ jobs, int njobs, uint32_t total_items,
                   const uint16_t* __restrict__ tables) {
  const uint32_t item = blockIdx.x * RAW_NT + threadIdx.x;
  if (item >= total_items)
    return;
  // job of this item (jobs are few: binary search over item_begin)
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].item_begin <= item)
      lo = mid;
    else
      hi = mid - 1;
  }
  const RawJobDev j = jobs[lo];
  const uint32_t local = item - j.item_begin;
  const uint32_t r = local / j.ipr, i = local - r * j.ipr;
  constexpr uint32_t K = raw_item_samples(FORMAT);
  constexpr uint32_t OB = raw_out_sample_bytes(FORMAT);
  const uint32_t s0 = i * K;                        // first sample of the item
  const uint32_t n = min(K, j.samples - s0);        // samples in this item
  const uint64_t src = j.in_offset + (uint64_t)r * j.in_pitch + (uint64_t)i * raw_item_stride(FORMAT);
  uint8_t* dst = out + j.out_offset + (uint64_t)(j.row0 + r) * j.out_pitch +
                 (uint64_t)OB * (j.out_col0 + s0);
  uint32_t s[4], o[5];
  raw_fetch16(in, src, in_total, s);
  const uint16_t* table = (FORMAT == RSB200_RAW_8BIT_TABLE) ? tables + (size_t)j.table * 65536u : nullptr;
  const int nw = raw_convert(FORMAT, s, table, o);
  if (n == K) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(dst);
    if (nw == 4 && (a & 15u) == 0) {
      stg_cs_v4(dst, make_uint4(o[0], o[1], o[2], o[3]));
    } else if ((a & 3u) == 0) {
#pragma unroll
      for (int k = 0; k < 5; ++k)
        if (k < nw)
          reinterpret_cast<uint32_t*>(dst)[k] = o[k];
    } else { // 16-bit samples at an odd sample column
#pragma unroll
      for (int k = 0; k < 5; ++k)
        if (k < nw) {
          reinterpret_cast<uint16_t*>(dst)[2 * k] = (uint16_t)o[k];
          reinterpret_cast<uint16_t*>(dst)[2 * k + 1] = (uint16_t)(o[k] >> 16);
        }
    }
  } else { // last, partial item of the row (static indices keep o[] in registers)
#pragma unroll
    for (uint32_t k = 0; k < K; ++k) {
      if (k < n) {
        if (OB == 4)
          reinterpret_cast<uint32_t*>(dst)[k] = o[k < 4 ? k : 0];
        else
          reinterpret_cast<uint16_t*>(dst)[k] = (uint16_t)(o[k >> 1] >> (16 * (k & 1)));
      }
    }
  }
}

} // namespace rsb200
