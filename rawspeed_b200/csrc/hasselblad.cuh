// hasselblad.cuh -- K2H: HasselbladDecompressor on the device (sm_90a).
//
// Reference: decompressors/HasselbladDecompressor.cpp:72-100 (decompress), :60-70 (getBits),
// HasselbladLJpegDecoder.cpp:50-69; bit source BitStreamerMSB32 (bitstreams/BitStreamMSB32.h:
// 32-bit little-endian chunks consumed MSB first; BitStreamer.h:100-132 replenisher, :216-229 fill).
//
// One frame is ONE Huffman stream without restart points (up to 100 MP):
//     per pair of pixels:  [len1 code][len2 code][len1 bits of diff1][len2 bits of diff2]
//     p1 += diff1, p2 += diff2 (both start at initPred in every row), out(row, 2k) = p1, out(row, 2k+1) = p2
// The reference decodes it on one CPU thread.  Here the stream is cut into segments of 4096 bits and
// every segment gets a thread (the stream is read through L1; a thread walks its 512 bytes sequentially):
//   H1  parse   thread i parses pairs (lengths only) from start[i] until it passes the end of its
//               segment: exit[i] = bit where the first pair of the next segment starts, count[i] =
//               pairs that start in [start[i], exit[i]).  start[0] = 0 is exact; start[i > 0] begins
//               as a guess (the segment boundary) -- Huffman streams self-synchronise, so after a few
//               pairs the guessed parse usually runs on true pair boundaries.
//   H1b link    start[i] <- exit[i-1] wherever they differ; a flag says whether anything changed.
//               Rounds of (parse, link) reach the fixed point start[i] == exit[i-1] for all i, and by
//               induction from segment 0 the fixed point IS the sequential parse.  Eight rounds are
//               launched unconditionally (a CTA whose starts did not change returns at once); if the
//               last link still changed something, one thread walks the rest sequentially (exact,
//               never observed).
//   H2  scan    exclusive prefix sum of count[] = index of the first pair of every segment.
//   H3  decode  thread i decodes its pairs from the verified start and writes the two DIFFERENCES
//               (mod 2^16) to the pixels' places; bad codes and the reference's over-read rule are
//               ordered by (pair, operation) with atomicMin so that the first failure in stream order
//               decides the status; the thread that holds the last pair writes `consumed`.
//   H4  rows    one warp per image row: in-place prefix sums of the two interleaved components
//               (packed 16-bit adds), both starting at initPred.
// Everything streams: ~1 B/px read per round + 2 B/px written, read and written again by H4.
#pragma once

#ifdef RSB200_EMU
#include "ljpeg_types.h"
#else
#include "common.cuh"
#include "ljpeg_types.h"
#endif

namespace rsb200 {

constexpr int H_NT = 128;                 // threads = segments per CTA
// bits per segment.  A guessed parse locks onto the true pair boundaries with probability ~1 / (bits
// per pair) per pair: ~16 pairs for camera data (16 bits per pair), ~50 pairs for 16-bit noise (48
// bits per pair, 2400 bits).  A segment that does not lock costs its successors one more round;
// CPU replay, 2048 x 256 px: camera-like data settles in 2 rounds at any size, 16-bit noise needs 2 / 3 /
// 5 / 7 rounds at 16384 / 8192 / 4096 / 2048 bits.  Shorter segments = more threads (a 50 MB stream
// has only 24 k segments of 16384 bits: 0.1 waves, each thread walking 2 KiB): 4096 bits, 8 rounds.
#ifndef RSB200_H_SEG_BITS
#define RSB200_H_SEG_BITS 4096
#endif
constexpr uint32_t H_SEG_BITS = RSB200_H_SEG_BITS;
constexpr int H_ROUNDS = 8;               // (parse, link) rounds launched unconditionally
constexpr uint32_t H_NOKEY = 0xFFFFFFFFu; // no failure recorded

struct DevHassJob {
  uint64_t in_offset;  // first byte of the stream in the input buffer (multiple of 4)
  uint32_t in_size;    // bytes
  uint32_t w, h;       // pixels (w even)
  uint32_t out_pitch;  // bytes
  uint64_t out_offset; // first byte of the image in the output buffer
  uint32_t init_pred;
  uint32_t table;      // index of the plan's table
  uint32_t seg_begin;  // first segment of this job in the plan's arrays
  uint32_t nseg;       // segments (covers the stream plus what the pump may read behind it)
  uint32_t cta_begin;  // first CTA of this job (H_NT segments per CTA)
  uint32_t pad;
};

struct DevHassCta {
  uint32_t job;  // index into the job array
  uint32_t seg0; // first segment of this CTA inside its job
};

// per-job failure keys and result
struct DevHassState {
  uint32_t key_ioe; // 4 * pair + operation of the first refill behind the buffer's slack (atomicMin)
  uint32_t key_bad; // 4 * pair + operation of the first code that is not in the table
  uint32_t consumed;
  uint32_t pad;
};

struct HassShared {
  uint32_t scan[H_NT];
  DevTable tab;
};

// little-endian word k of the stream (bytes at or behind `size` read as zero, like the pump's
// partial loads, BitStreamer.h:121-131 / adt/VariableLengthLoad.h)
__device__ __forceinline__ uint32_t h_stream_word(const uint8_t* __restrict__ s, uint32_t size, uint32_t k) {
  const uint64_t b = 4ull * k;
  if (b + 4 <= size)
    return __ldg(reinterpret_cast<const uint32_t*>(s) + k);
  uint32_t v = 0;
  for (uint32_t i = 0; i < 4; ++i)
    if (b + i < size)
      v |= (uint32_t)__ldg(s + b + i) << (8 * i);
  return v;
}

// the stream of one job; 32 bits from stream bit p
struct HassStream {
  const uint8_t* s;
  uint32_t size;
};
__device__ __forceinline__ uint32_t h_win(const HassStream& st, uint32_t p) {
  const uint32_t w = p >> 5;
  return __funnelshift_l(h_stream_word(st.s, st.size, w + 1u), h_stream_word(st.s, st.size, w), p);
}

struct HassPair {
  uint32_t cl1, s1, cl2, s2; // code lengths and difference lengths; cl = 0: the code is not in the table
};

// the two length codes of the pair at bit p
__device__ __forceinline__ HassPair h_pair(const DevTable* tab, const HassStream& st, uint32_t p) {
  HassPair r;
  const SymLen a = decode_sym(tab, h_win(st, p));
  r.cl1 = (uint32_t)a.codelen;
  r.s1 = (uint32_t)a.ssss;
  const SymLen b = decode_sym(tab, h_win(st, p + (r.cl1 ? r.cl1 : 1u)));
  r.cl2 = (uint32_t)b.codelen;
  r.s2 = (uint32_t)b.ssss;
  return r;
}
// bits of a pair; a code that is not in the table counts one bit (any rule does, as long as parse
// and decode agree: the real stream fails there anyway, a guessed parse just moves on)
__device__ __forceinline__ uint32_t h_pair_bits(const HassPair& r) {
  return (r.cl1 ? r.cl1 + r.s1 : 1u) + (r.cl2 ? r.cl2 + r.s2 : 1u);
}

// ---- H1 ----
__device__ __forceinline__ void
hass_parse_entry(HassShared& sh, const uint8_t* __restrict__ in, const DevHassJob* __restrict__ jobs,
                 const DevTable* __restrict__ tables, const DevHassCta* __restrict__ ctas,
                 const uint32_t* __restrict__ start, uint32_t* __restrict__ parsed,
                 uint32_t* __restrict__ exitp, uint32_t* __restrict__ count) {
  const DevHassCta c = ctas[blockIdx.x];
  const DevHassJob& j = jobs[c.job];
  const uint32_t seg = c.seg0 + threadIdx.x;
  const uint32_t g = j.seg_begin + seg;
  const bool mine = seg < j.nseg;
  const uint32_t st = mine ? start[g] : 0u;
  const bool todo = mine && parsed[g] != st;
  if (!__syncthreads_or(todo ? 1 : 0))
    return; // nothing moved in this CTA since its last parse
  {
    const uint4* src = reinterpret_cast<const uint4*>(tables + j.table);
    uint4* dst = reinterpret_cast<uint4*>(&sh.tab);
    for (int i = threadIdx.x; i < (int)(sizeof(DevTable) / 16); i += H_NT)
      dst[i] = src[i];
  }
  __syncthreads();
  if (!todo)
    return;
  const HassStream hs{in + j.in_offset, j.in_size};
  const uint32_t end = (seg + 1u) * H_SEG_BITS; // my boundary
  uint32_t p = st, n = 0;
  while (p < end) {
    p += h_pair_bits(h_pair(&sh.tab, hs, p));
    ++n;
  }
  exitp[g] = p;
  count[g] = n;
  parsed[g] = st;
}

// ---- H1b ----
__device__ __forceinline__ void hass_link_entry(const DevHassJob* __restrict__ jobs, int njobs,
                                                uint32_t nseg_total, const uint32_t* __restrict__ seg_job,
                                                uint32_t* __restrict__ start,
                                                const uint32_t* __restrict__ exitp,
                                                uint32_t* __restrict__ changed) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nseg_total)
    return;
  const DevHassJob& j = jobs[seg_job[g]];
  if (g == j.seg_begin)
    return;
  const uint32_t e = exitp[g - 1];
  if (start[g] != e) {
    start[g] = e;
    *changed = 1u;
  }
}

// ---- fallback: the chain did not settle in H_ROUNDS rounds; one thread per job walks it ----
__device__ __noinline__ void hass_serial_entry(const uint8_t* __restrict__ in,
                                               const DevHassJob* __restrict__ jobs,
                                               const DevTable* __restrict__ tables,
                                               uint32_t* __restrict__ start, uint32_t* __restrict__ parsed,
                                               uint32_t* __restrict__ exitp, uint32_t* __restrict__ count,
                                               const uint32_t* __restrict__ changed) {
  if (*changed == 0u)
    return;
  const DevHassJob& j = jobs[blockIdx.x];
  if (threadIdx.x != 0)
    return;
  const DevTable* t = tables + j.table;
  const HassStream hs{in + j.in_offset, j.in_size};
  for (uint32_t seg = 0; seg < j.nseg; ++seg) {
    const uint32_t g = j.seg_begin + seg;
    if (seg > 0)
      start[g] = exitp[g - 1];
    if (parsed[g] == start[g])
      continue;
    const uint32_t end = (seg + 1u) * H_SEG_BITS;
    uint32_t p = start[g], n = 0;
    while (p < end) {
      p += h_pair_bits(h_pair(t, hs, p));
      ++n;
    }
    exitp[g] = p;
    count[g] = n;
    parsed[g] = start[g];
  }
}

// ---- H2 (two small kernels): sums per CTA of H_NT segments, then their exclusive scan per job ----
__device__ __forceinline__ void hass_ctasum_entry(HassShared& sh, const DevHassJob* __restrict__ jobs,
                                                  const DevHassCta* __restrict__ ctas,
                                                  const uint32_t* __restrict__ count,
                                                  uint32_t* __restrict__ cta_sum) {
  const DevHassCta c = ctas[blockIdx.x];
  const DevHassJob& j = jobs[c.job];
  const uint32_t seg = c.seg0 + threadIdx.x;
  sh.scan[threadIdx.x] = seg < j.nseg ? count[j.seg_begin + seg] : 0u;
  __syncthreads();
  for (int d = H_NT / 2; d > 0; d >>= 1) {
    if ((int)threadIdx.x < d)
      sh.scan[threadIdx.x] += sh.scan[threadIdx.x + d];
    __syncthreads();
  }
  if (threadIdx.x == 0)
    cta_sum[blockIdx.x] = sh.scan[0];
}
// one thread per job: exclusive scan of its CTA sums (a 100 MP frame has < 4000 CTAs)
__device__ __forceinline__ void hass_ctascan_entry(const DevHassJob* __restrict__ jobs, int njobs,
                                                   const uint32_t* __restrict__ cta_sum,
                                                   uint32_t* __restrict__ cta_base) {
  const int jb = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (jb >= njobs)
    return;
  const DevHassJob& j = jobs[jb];
  const uint32_t nc = (j.nseg + H_NT - 1) / H_NT;
  uint32_t acc = 0;
  for (uint32_t c = 0; c < nc; ++c) {
    cta_base[j.cta_begin + c] = acc;
    acc += cta_sum[j.cta_begin + c];
  }
}

// refills the reference has done after a Huffman decode that starts at stream bit T
// (BitStreamer::fill(32) before every code: the cache holds 32..63 bits afterwards)
__device__ __forceinline__ uint32_t h_refills_at_code(uint32_t T) { return (T >> 5) + 1u + ((T & 31u) ? 1u : 0u); }

// ---- H3 ----
__device__ __forceinline__ void
hass_decode_entry(HassShared& sh, const uint8_t* __restrict__ in, const DevHassJob* __restrict__ jobs,
                  const DevTable* __restrict__ tables, const DevHassCta* __restrict__ ctas,
                  const uint32_t* __restrict__ start, const uint32_t* __restrict__ exitp,
                  const uint32_t* __restrict__ count, const uint32_t* __restrict__ cta_base,
                  uint8_t* __restrict__ out, DevHassState* __restrict__ states) {
  const DevHassCta c = ctas[blockIdx.x];
  const DevHassJob& j = jobs[c.job];
  const uint32_t seg = c.seg0 + threadIdx.x;
  const uint32_t g = j.seg_begin + seg;
  const bool mine = seg < j.nseg;
  {
    const uint4* src = reinterpret_cast<const uint4*>(tables + j.table);
    uint4* dst = reinterpret_cast<uint4*>(&sh.tab);
    for (int i = threadIdx.x; i < (int)(sizeof(DevTable) / 16); i += H_NT)
      dst[i] = src[i];
  }
  // exclusive scan of the CTA's counts (Hillis-Steele over H_NT values)
  const uint32_t myc = mine ? count[g] : 0u;
  sh.scan[threadIdx.x] = myc;
  __syncthreads();
  for (int d = 1; d < H_NT; d <<= 1) {
    const uint32_t v = (int)threadIdx.x >= d ? sh.scan[threadIdx.x - d] : 0u;
    __syncthreads();
    sh.scan[threadIdx.x] += v;
    __syncthreads();
  }
  if (!mine)
    return;
  const uint32_t ppr = j.w >> 1; // pairs per row
  const uint64_t npairs = (uint64_t)ppr * j.h;
  uint64_t k = (uint64_t)cta_base[blockIdx.x] + sh.scan[threadIdx.x] - myc; // my first pair
  if (k >= npairs)
    return;
  const HassStream hs{in + j.in_offset, j.in_size};
  const uint32_t end = exitp[g];
  uint32_t p = start[g];
  uint32_t row = (uint32_t)(k / ppr), col = (uint32_t)(k - (uint64_t)row * ppr);
  uint8_t* orow = out + j.out_offset + (uint64_t)row * j.out_pitch;
  // the reference throws at the first refill whose position is more than 8 bytes behind the buffer
  // (BitStreamer.h:120-127, 4-byte chunks): the refill that makes the count reach rlim
  const uint32_t rlim = (j.in_size + 8u) / 4u + 2u;
  DevHassState* stt = states + c.job;
  while (p < end && k < npairs) {
    const HassPair r = h_pair(&sh.tab, hs, p);
    const uint32_t T1 = p;
    const uint32_t c1 = r.cl1 ? r.cl1 : 1u, c2 = r.cl2 ? r.cl2 : 1u;
    const uint32_t T2 = T1 + c1, T3 = T2 + c2, T4 = T3 + (r.cl1 ? r.s1 : 0u);
    const uint32_t Tend = T4 + (r.cl2 ? r.s2 : 0u);
    if (!r.cl1 || !r.cl2)
      atomicMin(&stt->key_bad, (uint32_t)(4u * k) + (r.cl1 ? 1u : 0u));
    if (((Tend + 63u) >> 5) + 2u >= rlim) { // near the end of the buffer: operation by operation
      uint32_t R = h_refills_at_code(T1), op = 4;
      if (R >= rlim) {
        op = 0;
      } else if (r.cl1) {
        R = h_refills_at_code(T2);
        if (R >= rlim) {
          op = 1;
        } else if (r.cl2) {
          if (r.s1 && ((T3 + r.s1 + 31u) >> 5) > R)
            R = (T3 + r.s1 + 31u) >> 5;
          if (R >= rlim) {
            op = 2;
          } else {
            if (r.s2 && ((T4 + r.s2 + 31u) >> 5) > R)
              R = (T4 + r.s2 + 31u) >> 5;
            if (R >= rlim)
              op = 3;
          }
        }
      }
      if (op < 4)
        atomicMin(&stt->key_ioe, (uint32_t)(4u * k) + op);
    }
    // differences (mod 2^16): extend(); the value 65535 (16 one-bits) means -32768
    uint32_t d1 = 0, d2 = 0;
    if (r.cl1 && r.s1) {
      const uint32_t v = h_win(hs, T3) >> (32u - r.s1);
      d1 = (v >> (r.s1 - 1u)) ? v : v - ((1u << r.s1) - 1u);
      if (d1 == 65535u)
        d1 = 0x8000u;
    }
    if (r.cl2 && r.s2) {
      const uint32_t v = h_win(hs, T4) >> (32u - r.s2);
      d2 = (v >> (r.s2 - 1u)) ? v : v - ((1u << r.s2) - 1u);
      if (d2 == 65535u)
        d2 = 0x8000u;
    }
    *reinterpret_cast<uint32_t*>(orow + 4ull * col) = (d1 & 0xFFFFu) | (d2 << 16);
    if (k + 1 == npairs)
      stt->consumed = (Tend + 7u) >> 3; // BitStreamer::getStreamPosition(): pos - fillLevel / 8
    p = Tend;
    ++k;
    if (++col == ppr) {
      col = 0;
      orow += j.out_pitch;
    }
  }
}

// ---- H4: one warp per row ----
__device__ __forceinline__ void hass_rows_entry(const DevHassJob* __restrict__ jobs, int njobs,
                                                const uint32_t* __restrict__ row_job_begin,
                                                uint8_t* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t wrow = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; // global row index over all jobs
  // find the job (few jobs: linear)
  int jb = 0;
  while (jb + 1 < njobs && wrow >= row_job_begin[jb + 1])
    ++jb;
  if (wrow >= row_job_begin[njobs])
    return;
  const DevHassJob& j = jobs[jb];
  const uint32_t row = wrow - row_job_begin[jb];
  uint32_t* o = reinterpret_cast<uint32_t*>(out + j.out_offset + (uint64_t)row * j.out_pitch);
  const uint32_t ppr = j.w >> 1;
  uint32_t carry = (j.init_pred & 0xFFFFu) * 0x00010001u;
  for (uint32_t k0 = 0; k0 < ppr; k0 += 32) {
    const uint32_t k = k0 + lane;
    uint32_t v = k < ppr ? o[k] : 0u;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, v, d);
      if (lane >= (uint32_t)d)
        v = __vadd2(v, t);
    }
    v = __vadd2(v, carry);
    if (k < ppr)
      o[k] = v;
    carry = __shfl_sync(0xFFFFFFFFu, v, 31);
  }
}

#ifndef RSB200_EMU
__global__ void __launch_bounds__(H_NT)
    hass_parse_kernel(const uint8_t* __restrict__ in, const DevHassJob* __restrict__ jobs,
                      const DevTable* __restrict__ tables, const DevHassCta* __restrict__ ctas,
                      const uint32_t* __restrict__ start, uint32_t* __restrict__ parsed,
                      uint32_t* __restrict__ exitp, uint32_t* __restrict__ count) {
  extern __shared__ __align__(16) uint8_t h_smem_raw[];
  hass_parse_entry(*reinterpret_cast<HassShared*>(h_smem_raw), in, jobs, tables, ctas, start, parsed, exitp,
                   count);
}
__global__ void hass_link_kernel(const DevHassJob* __restrict__ jobs, int njobs, uint32_t nseg_total,
                                 const uint32_t* __restrict__ seg_job, uint32_t* __restrict__ start,
                                 const uint32_t* __restrict__ exitp, uint32_t* __restrict__ changed) {
  hass_link_entry(jobs, njobs, nseg_total, seg_job, start, exitp, changed);
}
__global__ void hass_serial_kernel(const uint8_t* __restrict__ in, const DevHassJob* __restrict__ jobs,
                                   const DevTable* __restrict__ tables, uint32_t* __restrict__ start,
                                   uint32_t* __restrict__ parsed, uint32_t* __restrict__ exitp,
                                   uint32_t* __restrict__ count, const uint32_t* __restrict__ changed) {
  hass_serial_entry(in, jobs, tables, start, parsed, exitp, count, changed);
}
__global__ void __launch_bounds__(H_NT)
    hass_ctasum_kernel(const DevHassJob* __restrict__ jobs, const DevHassCta* __restrict__ ctas,
                       const uint32_t* __restrict__ count, uint32_t* __restrict__ cta_sum) {
  extern __shared__ __align__(16) uint8_t h_smem_raw[];
  hass_ctasum_entry(*reinterpret_cast<HassShared*>(h_smem_raw), jobs, ctas, count, cta_sum);
}
__global__ void hass_ctascan_kernel(const DevHassJob* __restrict__ jobs, int njobs,
                                    const uint32_t* __restrict__ cta_sum, uint32_t* __restrict__ cta_base) {
  hass_ctascan_entry(jobs, njobs, cta_sum, cta_base);
}
__global__ void __launch_bounds__(H_NT)
    hass_decode_kernel(const uint8_t* __restrict__ in, const DevHassJob* __restrict__ jobs,
                       const DevTable* __restrict__ tables, const DevHassCta* __restrict__ ctas,
                       const uint32_t* __restrict__ start, const uint32_t* __restrict__ exitp,
                       const uint32_t* __restrict__ count, const uint32_t* __restrict__ cta_base,
                       uint8_t* __restrict__ out, DevHassState* __restrict__ states) {
  extern __shared__ __align__(16) uint8_t h_smem_raw[];
  hass_decode_entry(*reinterpret_cast<HassShared*>(h_smem_raw), in, jobs, tables, ctas, start, exitp, count,
                    cta_base, out, states);
}
__global__ void hass_rows_kernel(const DevHassJob* __restrict__ jobs, int njobs,
                                 const uint32_t* __restrict__ row_job_begin, uint8_t* __restrict__ out) {
  hass_rows_entry(jobs, njobs, row_job_begin, out);
}
// start[i] = segment boundary (a guess for i > 0), parsed = none, states cleared
__global__ void hass_init_kernel(const DevHassJob* __restrict__ jobs, int njobs, uint32_t nseg_total,
                                 const uint32_t* __restrict__ seg_job, uint32_t* __restrict__ start,
                                 uint32_t* __restrict__ parsed, DevHassState* __restrict__ states,
                                 uint32_t* __restrict__ changed) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < (uint32_t)njobs) {
    states[g].key_ioe = H_NOKEY;
    states[g].key_bad = H_NOKEY;
    states[g].consumed = 0;
  }
  if (g <= (uint32_t)H_ROUNDS)
    changed[g] = 0;
  if (g >= nseg_total)
    return;
  const DevHassJob& j = jobs[seg_job[g]];
  start[g] = (g - j.seg_begin) * H_SEG_BITS;
  parsed[g] = 0xFFFFFFFFu;
}
#endif

} // namespace rsb200
