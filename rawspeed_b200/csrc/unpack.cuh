// unpack.cuh -- K1: packed N-bit -> uint16 (sm_90a).
//
// Replaces the body of UncompressedDecompressor::decodePackedInt<Pump>
// (reference decompressors/UncompressedDecompressor.cpp:188-200) for the four
// fixed bit orders (bitstreams/BitStream{LSB,MSB,MSB16,MSB32}.h:31-43).
//
// Semantics restated (SURVEY appendix A.1): the strip is one continuous bit
// string; row r starts at logical bit 8*r*pitch, sample i of the row covers
// logical bits [8*r*pitch + i*bps, +bps).  MSB-family orders read the bit
// string most-significant-bit first after a byte permutation inside 1/2/4-byte
// chunks anchored at the start of the strip; LSB reads it least-significant-bit
// first.  No state is carried between samples, so the op is embarrassingly
// parallel and purely HBM-bound: bps/8 bytes in, 2 bytes out per sample.
//
// Mapping: one CTA = one (job,row,chunk).  The chunk's packed bytes are staged
// into shared memory with ONE 1-D bulk async copy (TMA unit, cp.async.bulk ->
// SASS UBLKCP) completing on an mbarrier; every thread then extracts groups of
// 8 samples (= bps bytes, always byte aligned) with funnel shifts and emits one
// coalesced 128-bit store per group.
#pragma once

#include "common.cuh"

namespace rsb200 {

struct UnpackJobDev {
  uint64_t in_offset;
  uint64_t in_size;
  uint64_t out_offset;
  int32_t out_pitch, row0, rows, samples, out_col0, in_pitch, bps, order;
  int32_t nchunks;      // chunks per row
  int32_t chunk_groups; // groups of 8 samples per chunk
  uint32_t block_begin; // first CTA of this job
  uint32_t vec_ok;      // output rows are 16-byte aligned -> 128-bit stores
};

constexpr int UNPACK_THREADS = 256;
constexpr int UNPACK_MAX_CHUNK_GROUPS = 1024; // 8192 samples, <= 16 KiB of input
constexpr int UNPACK_SMEM_BYTES = UNPACK_MAX_CHUNK_GROUPS * 16 + 64;

// byte_perm selector turning a little-endian loaded word of the strip into the
// big-endian value of the 4 logical bytes of the MSB-first bit string.
__host__ __device__ inline uint32_t unpack_perm_selector(int order) {
  // MSB: bytes as they come -> bswap; MSB16: swap inside pairs then bswap;
  // MSB32: swap inside quads then bswap == identity.
  return order == 1 ? 0x0123u : order == 2 ? 0x1032u : 0x3210u;
}

template <int BPS, bool LSBO>
__device__ __forceinline__ void unpack_extract8(const uint32_t (&X)[5],
                                                uint32_t (&v)[8], int bps_rt) {
  // X holds the group's bits starting at bit 0 of X[0] (MSB-first for the MSB
  // family, LSB-first for LSB order).
  if constexpr (BPS != 0) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      constexpr int dummy = 0;
      (void)dummy;
      const int bit = j * BPS;
      const int w = bit >> 5, sh = bit & 31;
      if constexpr (LSBO) {
        uint32_t t = __funnelshift_r(X[w], X[w + 1], sh);
        v[j] = BPS == 32 ? t : (t & ((1u << BPS) - 1u));
      } else {
        uint32_t t = __funnelshift_l(X[w + 1], X[w], sh);
        v[j] = t >> (32 - BPS);
      }
    }
  } else {
    // generic bit depth (1..16): dynamic word index, kept out of the hot
    // instantiations
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int bit = j * bps_rt;
      const int w = bit >> 5, sh = bit & 31;
      uint32_t a = w == 0 ? X[0] : w == 1 ? X[1] : w == 2 ? X[2] : X[3];
      uint32_t b = w == 0 ? X[1] : w == 1 ? X[2] : w == 2 ? X[3] : X[4];
      if constexpr (LSBO) {
        v[j] = __funnelshift_r(a, b, sh) & ((1u << bps_rt) - 1u);
      } else {
        v[j] = __funnelshift_l(b, a, sh) >> (32 - bps_rt);
      }
    }
  }
}

template <int BPS, bool LSBO>
__global__ void __launch_bounds__(UNPACK_THREADS)
    unpack_kernel(const uint8_t* __restrict__ in, uint64_t in_total,
                  uint8_t* __restrict__ out, const UnpackJobDev* __restrict__ jobs,
                  int njobs) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;

  // ---- locate job (binary search over block_begin) ----
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].block_begin <= blockIdx.x)
      lo = mid;
    else
      hi = mid - 1;
  }
  const UnpackJobDev job = jobs[lo];
  const int bps = BPS ? BPS : job.bps;
  const uint32_t local = blockIdx.x - job.block_begin;
  const int row = local / job.nchunks;
  const int chunk = local - row * job.nchunks;
  const int total_groups = (job.samples + 7) >> 3;
  const int g0 = chunk * job.chunk_groups;
  const int g1 = min(g0 + job.chunk_groups, total_groups);
  if (g0 >= g1)
    return;

  // strip-relative byte range needed by this chunk (word aligned, +1 word)
  const uint64_t row_byte = (uint64_t)row * (uint64_t)job.in_pitch;
  const uint64_t a0 = (row_byte + (uint64_t)g0 * bps) & ~3ull;
  const uint64_t a1 = ((row_byte + (uint64_t)g1 * bps + 3) & ~3ull) + 4;
  // global window, 16-byte aligned, clamped to the (16-byte padded) buffer
  const uint64_t glo = (job.in_offset + a0) & ~15ull;
  uint64_t ghi = (job.in_offset + a1 + 15) & ~15ull;
  const uint64_t gmax = (in_total + 15) & ~15ull;
  if (ghi > gmax)
    ghi = gmax;
  const uint32_t nbytes = ghi > glo ? (uint32_t)(ghi - glo) : 0u;

  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar, nbytes);
    if (nbytes)
      bulk_g2s(smem, in + glo, nbytes, &bar);
  }
  mbar_wait(&bar, 0);

  const uint32_t* sw = reinterpret_cast<const uint32_t*>(smem);
  const uint32_t sel = unpack_perm_selector(job.order);
  uint8_t* orow = out + job.out_offset +
                  (uint64_t)(job.row0 + row) * (uint64_t)job.out_pitch +
                  2ull * (uint64_t)job.out_col0;

  for (int g = g0 + threadIdx.x; g < g1; g += UNPACK_THREADS) {
    const uint64_t A = row_byte + (uint64_t)g * bps; // strip-relative byte
    const uint64_t k0 = A >> 2;                     // strip-relative word
    // byte address in smem of strip-relative word k0
    const uint32_t s0 = (uint32_t)(job.in_offset + (k0 << 2) - glo);
    const uint32_t wi = s0 >> 2, sk = (s0 & 3) * 8;
    uint32_t L[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      // words past the staged window are never needed for valid samples
      const uint32_t idx = wi + i;
      L[i] = (idx * 4 < nbytes) ? sw[idx] : 0u;
    }
    uint32_t W[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      uint32_t w = __funnelshift_r(L[i], L[i + 1], sk); // LE strip word k0+i
      // bytes at/after the end of the strip read as zero (BitStreamer.h:100-131)
      const uint64_t byte0 = (k0 + i) << 2;
      if (byte0 + 4 > job.in_size) {
        const int valid = byte0 < job.in_size ? (int)(job.in_size - byte0) : 0;
        w = valid ? (w & (0xFFFFFFFFu >> (32 - 8 * valid))) : 0u;
      }
      W[i] = LSBO ? w : __byte_perm(w, 0, sel);
    }
    // align the group to bit 0
    const int gs = (int)(A & 3) * 8;
    uint32_t X[5];
#pragma unroll
    for (int i = 0; i < 4; ++i)
      X[i] = LSBO ? __funnelshift_r(W[i], W[i + 1], gs)
                  : __funnelshift_l(W[i + 1], W[i], gs);
    X[4] = LSBO ? (W[4] >> gs) : (W[4] << gs);
    uint32_t v[8];
    unpack_extract8<BPS, LSBO>(X, v, bps);

    const int s_first = g * 8;
    if (s_first + 8 <= job.samples && job.vec_ok) {
      uint4 o;
      o.x = v[0] | (v[1] << 16);
      o.y = v[2] | (v[3] << 16);
      o.z = v[4] | (v[5] << 16);
      o.w = v[6] | (v[7] << 16);
      stg_cs_v4(orow + 16ull * g, o);
    } else {
      uint16_t* o16 = reinterpret_cast<uint16_t*>(orow) + s_first;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (s_first + j < job.samples)
          o16[j] = (uint16_t)v[j];
    }
  }
}

// ------------------------------------------------------------------
// Fast path: even bit depths, 4-byte aligned strips/pitches, wide rows.
// Work item = 16 samples = 2*BPS bytes (a whole number of 32-bit words), so all
// bit offsets are compile-time constants.  The items of a job are numbered
// row-major across rows ("flattened"), a CTA takes UNPACK_IPB consecutive items
// -- usually spanning a few rows -- and stages each row segment with its own
// 1-D bulk async copy (TMA) onto one mbarrier.
// ------------------------------------------------------------------
constexpr int UNPACK_IPB = 512;    // items per CTA (2 per thread)
constexpr int UNPACK_MAXSEG = 12;  // row segments per CTA (rows >= 64 items wide)
constexpr int UNPACK_FAST_SMEM = UNPACK_IPB * 32 + UNPACK_MAXSEG * 48;

struct UnpackFastJobDev {
  uint64_t in_offset;
  uint64_t out_offset;
  int32_t out_pitch, row0, rows, samples, out_col0, in_pitch, order;
  uint32_t ipr;         // items per row
  uint32_t total_items; // rows * ipr
  uint32_t block_begin;
  uint32_t vec_ok;
  uint32_t row_bytes;
};

template <int BPS, bool LSBO>
__device__ __forceinline__ void unpack_item16(const uint32_t* __restrict__ sw,
                                              uint32_t sel, uint32_t (&o)[8]) {
  constexpr int NW = BPS / 2; // words per item
  uint32_t Wd[NW + 1];
#pragma unroll
  for (int i = 0; i < NW; ++i)
    Wd[i] = LSBO ? sw[i] : __byte_perm(sw[i], 0, sel);
  Wd[NW] = 0;
  uint32_t v[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    constexpr uint32_t mask = BPS == 32 ? 0xFFFFFFFFu : ((1u << BPS) - 1u);
    const int bit = j * BPS;
    const int w = bit >> 5, sh = bit & 31;
    if (LSBO) {
      if (sh + BPS <= 32)
        v[j] = (Wd[w] >> sh) & mask;
      else
        v[j] = __funnelshift_r(Wd[w], Wd[w + 1], sh) & mask;
    } else {
      if (sh + BPS <= 32)
        v[j] = (Wd[w] >> (32 - sh - BPS)) & mask;
      else
        v[j] = __funnelshift_l(Wd[w + 1], Wd[w], sh) >> (32 - BPS);
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k)
    o[k] = v[2 * k] | (v[2 * k + 1] << 16);
}

template <int BPS, bool LSBO>
__global__ void __launch_bounds__(UNPACK_THREADS)
    unpack_fast_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out,
                       const UnpackFastJobDev* __restrict__ jobs, int njobs,
                       uint32_t block_base) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ int32_t seg_delta[UNPACK_MAXSEG + 1]; // smem offset - row-relative byte

  const uint32_t bid = blockIdx.x + block_base; // sub-launches of a plan start mid-grid
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].block_begin <= bid)
      lo = mid;
    else
      hi = mid - 1;
  }
  const UnpackFastJobDev& job = jobs[lo];
  constexpr uint32_t IB = 2 * BPS; // bytes per item
  const uint32_t ipr = job.ipr;
  const uint32_t I0 = (bid - job.block_begin) * UNPACK_IPB;
  const uint32_t I1 = min(I0 + UNPACK_IPB, job.total_items);
  const uint32_t r0 = I0 / ipr;

  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
    const uint32_t r1 = (I1 - 1) / ipr;
    // pass 1: sizes
    uint32_t total = 0;
    for (uint32_t r = r0; r <= r1; ++r) {
      const uint32_t ia = max(I0, r * ipr) - r * ipr;
      const uint32_t ib = min(I1, (r + 1) * ipr) - r * ipr;
      const uint64_t g0 = job.in_offset + (uint64_t)r * job.in_pitch + (uint64_t)ia * IB;
      const uint64_t g1 = job.in_offset + (uint64_t)r * job.in_pitch +
                          min((uint64_t)ib * IB, (uint64_t)job.row_bytes);
      const uint64_t a0 = g0 & ~15ull, a1 = (g1 + 15) & ~15ull;
      total += (uint32_t)(a1 - a0);
    }
    mbar_expect_tx(&bar, total);
    uint32_t soff = 0;
    for (uint32_t r = r0; r <= r1; ++r) {
      const uint32_t ia = max(I0, r * ipr) - r * ipr;
      const uint32_t ib = min(I1, (r + 1) * ipr) - r * ipr;
      const uint64_t rowg = job.in_offset + (uint64_t)r * job.in_pitch;
      const uint64_t g0 = rowg + (uint64_t)ia * IB;
      const uint64_t g1 = rowg + min((uint64_t)ib * IB, (uint64_t)job.row_bytes);
      const uint64_t a0 = g0 & ~15ull, a1 = (g1 + 15) & ~15ull;
      bulk_g2s(smem + soff, in + a0, (uint32_t)(a1 - a0), &bar);
      // smem address of row-relative byte x of row r: soff + (rowg + x - a0)
      seg_delta[r - r0] = (int32_t)soff + (int32_t)(int64_t)(rowg - a0);
      soff += (uint32_t)(a1 - a0);
    }
  }
  __syncthreads();
  mbar_wait(&bar, 0);

  const uint32_t sel = unpack_perm_selector(job.order);
  const uint64_t obase = job.out_offset + 2ull * (uint64_t)job.out_col0;
#pragma unroll
  for (int it = 0; it < UNPACK_IPB / UNPACK_THREADS; ++it) {
    const uint32_t I = I0 + it * UNPACK_THREADS + threadIdx.x;
    if (I >= I1)
      break;
    const uint32_t r = I / ipr;
    const uint32_t i = I - r * ipr;
    const uint32_t saddr = (uint32_t)(seg_delta[r - r0] + (int32_t)(i * IB));
    uint32_t o[8];
    unpack_item16<BPS, LSBO>(reinterpret_cast<const uint32_t*>(smem + saddr), sel, o);
    uint8_t* dst = out + obase + (uint64_t)(job.row0 + (int)r) * (uint64_t)job.out_pitch +
                   32ull * i;
    const uint32_t s_first = i * 16;
    if (job.vec_ok && s_first + 16 <= (uint32_t)job.samples) {
      stg_cs_v4(dst, make_uint4(o[0], o[1], o[2], o[3]));
      stg_cs_v4(dst + 16, make_uint4(o[4], o[5], o[6], o[7]));
    } else {
      uint16_t* d16 = reinterpret_cast<uint16_t*>(dst);
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (s_first + j < (uint32_t)job.samples)
          d16[j] = (uint16_t)(o[j >> 1] >> ((j & 1) * 16));
    }
  }
}

} // namespace rsb200
