// ljpeg_tile.cuh -- K2G `k2_tile_kernel<R>`: lossless-JPEG tile decode (entropy decode +
// predictor 1), one CTA per entropy-coded segment (DNG tile / restart interval), sm_90a.
// Round-2 successor of k2_fused_kernel (ljpeg_fused.cuh) for the common shape of a DNG tile:
// 1, 2 or 4 components in one MCU row, ONE Huffman table for all of them, rows that are whole
// 8-sample units written with aligned 128-bit stores.  Everything else stays on k2_fused_kernel.
//
// Reference bodies replaced (paths relative to /root/reference/src/librawspeed):
//   BitStreamerJPEG::fillCache              bitstreams/BitStreamerJPEG.h:106-189
//   BitStreamer::fill / getInput            bitstreams/BitStreamer.h:97-131, 216-229
//   PrefixCodeLUTDecoder::decode            codes/PrefixCodeLUTDecoder.h:172-216
//   AbstractPrefixCodeDecoder::processSymbol/extend  codes/AbstractPrefixCodeDecoder.h:43-76
//   LJpegDecompressor::decodeN/decodeRowN   decompressors/LJpegDecompressor.cpp:184-339
//
// What changed against k2_fused_kernel, and why (it spends several warp-instructions per pixel,
// decodes every symbol several times and meets 8-way bank conflicts on the clean buffer):
//   * subsequences are LONG (~50 bytes for R = 1, ~100 for R = 2; an odd number of 32-bit words,
//     so the 32 lanes of a warp read 32 different banks) and every thread except the first starts
//     its length-only parse `preroll` bits BEFORE its subsequence: by the time it crosses into its
//     own range it has almost always synchronised with the true parse, so the fixed-point
//     iteration ("adopt your predecessor's exit") confirms instead of re-decoding;
//   * unstuffing works on 64-byte pieces held in registers: pieces without a stuffing byte (4 of
//     5) are written as whole funnel-shifted words; the others are collected in a list and
//     handled byte by byte afterwards by as many threads as there are such pieces, so the common
//     path carries no per-byte work and no divergent branch;
//   * the predictor stage never re-writes the sample buffer: per-thread totals of an odd number
//     of 8-sample units (bank-conflict-free 128-bit loads) -> one scan -> every unit is summed,
//     offset by its row constant and stored straight from the differences;
//   * a whole number of 8-sample units is finished per batch, so there is no scalar edge path;
//   * the end of the stream follows the reference exactly: bits behind the last data byte / the
//     end marker read as zero, and the segment only fails where BitStreamer::getInput would have
//     thrown (position more than 16 bytes past the buffer at a refill), see tl_replay().
//
// The kernel body compiles for two targets: nvcc (sm_90a) and, with RSB200_EMU defined by
// tests/emu/cuda_emu.h, g++ -- the CPU replay the test-suite runs where there is no GPU.
#pragma once

#ifdef RSB200_EMU
#include "ljpeg_types.h"
#else
#include "ljpeg.cuh"
#endif
#include <stddef.h>

namespace rsb200 {

#ifndef RSB200_TILE_NT
#define RSB200_TILE_NT 256
#endif
constexpr int TL_NT = RSB200_TILE_NT; // threads per CTA
constexpr int TL_PIECE = 64;   // raw bytes per unstuff piece
constexpr int TL_LA = 16;      // clean bytes deferred to the next chunk (see tl_replay)
constexpr int TL_ZEXT = 24;    // zero bytes behind the data the reference can still supply (192 bits)
constexpr int TL_RBMAX = 128;  // row starts per predictor batch
constexpr uint32_t TL_NOPOS = 0xFFFFFFFFu;

template <int R> struct TileGeom {
#ifndef RSB200_TILE_NPIECE1
#define RSB200_TILE_NPIECE1 208
#endif
#ifndef RSB200_TILE_DCAP1
#define RSB200_TILE_DCAP1 15360
#endif
  // R = 1: 55 KB of shared memory -> four CTAs per SM (an H100 SM has 228 KB, 227 KB of it for
  // one block); R = 2: 105 KB -> two
  // CTAs per SM with subsequences twice as long
  static constexpr int NPIECE = R == 1 ? RSB200_TILE_NPIECE1 : 448; // pieces per chunk (at most)
  static constexpr int RAWMAX = NPIECE * TL_PIECE;   // raw bytes per chunk (at most)
  static constexpr int UBBYTES = RAWMAX + 128;       // carried tail + chunk + zero extension + slack
  static constexpr int DCAP = R == 1 ? RSB200_TILE_DCAP1 : 32000; // samples per predictor batch (at most)
  static constexpr int UPT = ((DCAP / 8 + TL_NT - 1) / TL_NT) | 1; // units per thread (odd), at most
  static constexpr int MIN_RS = 8 * UPT;             // a thread's units hold at most one row start
};

struct TileCarry {
  uint32_t pos;       // bit position (relative to ub[0]) of the next symbol
  uint32_t sym;       // symbols decoded so far
  uint32_t tail_len;  // clean bytes carried at the front of ub
  uint32_t tail_raw;  // raw offset (from the aligned base) of the source of ub byte 0
  uint32_t ubytes;    // clean bytes that precede ub[0] in the segment
  uint32_t prev_ff;   // last raw byte of the previous chunk was FF (inside the segment)
  uint32_t ended;     // marker seen or end of buffer reached
  uint32_t leftover;  // differences (< 8) carried to the next batch / chunk
  uint32_t left[4];   // ... their values (the raw staging of the next chunk overwrites dbuf)
  uint32_t proc;      // samples already written (multiple of 8)
  uint32_t pc01, pc23;   // running per-component sums carried (4 x 16 bit)
  uint32_t col01, col23; // value of the first MCU of the previous row
  uint32_t rb01, rb23;   // additive constant of the row in progress
};

// where the last needed symbol of the segment was met (written by one thread of the final pass)
struct TileLast {
  uint32_t seen;
  uint32_t p_last; // bit position (in ub of that chunk) of the last needed symbol
};

template <int R> struct alignas(128) TileShared {
  using G = TileGeom<R>;
  DevScan sc;
  TileCarry cy;
  TileLast last;
  alignas(8) uint64_t bar;
  uint32_t mpos;
  uint32_t bad_code;
  uint32_t nlist;
  uint32_t tail_raw_next; // B: raw offset of the source of the next chunk's ub byte 0
  uint32_t prev_ff_next;  // B: the chunk's last raw byte is an FF inside the segment
  uint32_t coop_n[3];     // B: byte counts of the edge pieces / the piece the marker cuts
  uint32_t rstat;   // result of tl_replay: 0 fine, 2 the reference would have thrown
  uint32_t rcons;   // ... and its getStreamPosition()
  uint32_t exitpos[TL_NT];         // C/D: exit positions of the subsequences
  uint32_t list[G::NPIECE];        // B: irregular pieces
  uint32_t anchor[G::NPIECE + 1];  // clean byte index (in ub) where each raw piece starts
  uint32_t warp_tmp[4][TL_NT / 32];
  uint32_t rowbase[TL_RBMAX + 1][2];
  alignas(16) uint32_t ub[G::UBBYTES / 4];    // clean big-endian words
  alignas(16) uint16_t dbuf[G::DCAP + 16];    // differences; A/B: raw staging (RAWMAX + 16 bytes)
  alignas(16) uint8_t len8[1 << LUT_BITS];    // bits consumed by the symbol at the top of an 11-bit window (0: slow path)
  DevTable tab;
};

template <int R> __host__ __device__ inline size_t tile_smem_bytes() { return sizeof(TileShared<R>); }

// ---- byte flags: 0x80 in every byte of w that is 0xFF / 0x00 (exact, 3 instructions each) ----
__device__ __forceinline__ uint32_t tl_ff_flags(uint32_t w) {
  return ((w & 0x7F7F7F7Fu) + 0x01010101u) & w & 0x80808080u;
}
__device__ __forceinline__ uint32_t tl_zero_flags(uint32_t w) {
  return ~(((w & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | w) & 0x80808080u;
}

__device__ __forceinline__ uint32_t tl_block_scan(uint32_t v, uint32_t* tmp, uint32_t* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, v, d);
    if (lane >= d)
      v += n;
  }
  if (lane == 31)
    tmp[wid] = v;
  __syncthreads();
  uint32_t add = 0, tot = 0;
#pragma unroll
  for (int i = 0; i < TL_NT / 32; ++i) {
    const uint32_t x = tmp[i];
    add += (i < wid) ? x : 0u;
    tot += x;
  }
  *total = tot;
  return v + add;
}

// inclusive block scan of two packed 2x16-bit values (mod 2^16 per half)
__device__ __forceinline__ void tl_block_scan_v2(uint32_t& a, uint32_t& b, uint32_t* tmpa,
                                                 uint32_t* tmpb, uint32_t& tota, uint32_t& totb) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, a, d);
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, b, d);
    if (lane >= d) {
      a = __vadd2(a, x);
      b = __vadd2(b, y);
    }
  }
  if (lane == 31) {
    tmpa[wid] = a;
    tmpb[wid] = b;
  }
  __syncthreads();
  uint32_t adda = 0, addb = 0;
  tota = totb = 0;
#pragma unroll
  for (int i = 0; i < TL_NT / 32; ++i) {
    const uint32_t x = tmpa[i], y = tmpb[i];
    if (i < wid) {
      adda = __vadd2(adda, x);
      addb = __vadd2(addb, y);
    }
    tota = __vadd2(tota, x);
    totb = __vadd2(totb, y);
  }
  a = __vadd2(a, adda);
  b = __vadd2(b, addb);
}

// per-CTA view of the segment's bytes
struct TileStream {
  const uint8_t* gbase; // 16-byte aligned base of the segment window
  uint32_t limit;       // valid raw bytes from gbase
  uint32_t skew;        // offset of the first entropy-coded byte from gbase
  uint64_t readable;    // bytes that may be touched by the bulk copies
  uint32_t chunk_raw;   // raw bytes per chunk (npieces * 64)
  uint32_t npieces;     // pieces per chunk
};

__device__ __forceinline__ uint32_t tl_raw_byte(const TileStream& st, uint32_t p) {
  return p < st.limit ? (uint32_t)st.gbase[p] : 0u;
}

template <int R>
__device__ __forceinline__ void tl_issue_chunk(TileShared<R>& sh, const TileStream& st, uint32_t chunk) {
  const uint64_t g0 = (uint64_t)chunk * st.chunk_raw;
  uint32_t n = 0;
  if (g0 < st.readable)
    n = (uint32_t)min((uint64_t)(st.chunk_raw + 16u), st.readable - g0);
  mbar_expect_tx(&sh.bar, n);
  if (n)
    bulk_g2s(sh.dbuf, st.gbase + g0, n, &sh.bar);
}

struct TileChunk {
  uint32_t len;        // clean bytes in ub (carried tail + this chunk)
  uint32_t Lc;         // clean bytes decodable in this chunk (zero extension included when final)
  uint32_t end_all;    // Lc * 8
  uint32_t mpos;       // chunk-relative raw offset of the end marker (or TL_NOPOS)
  uint32_t total_emit; // clean bytes produced by this chunk
  bool final_chunk;
};

// Is raw byte r (offset from gbase) a data byte?  (BitStreamerJPEG.h:131-158: FF00 -> FF, the
// 00 is dropped; bytes outside the segment and at/after the end marker are not data.)
__device__ __forceinline__ bool tl_keep(const TileStream& st, uint32_t r, uint32_t limit_eff) {
  if (r < st.skew || r >= limit_eff)
    return false;
  if (st.gbase[r] != 0u)
    return true;
  return !(r > st.skew && st.gbase[r - 1] == 0xFFu);
}
// Is raw byte r the second byte of a marker (FF at r-1 inside the segment, non-zero here)?
__device__ __forceinline__ bool tl_marker2(const TileStream& st, uint32_t r) {
  return r > st.skew && r < st.limit && st.gbase[r] != 0u && st.gbase[r - 1] == 0xFFu;
}

// Optional per-phase cycle accounting (profiling builds only: -DRSB200_PHASE_TIMING).
#if defined(RSB200_PHASE_TIMING) && !defined(RSB200_EMU)
__device__ unsigned long long g_tile_phase_cycles[16];
#define TL_TICK(i)                                                                 \
  do {                                                                             \
    if (threadIdx.x == 0) {                                                        \
      const long long t_now = clock64();                                           \
      atomicAdd(&g_tile_phase_cycles[i], (unsigned long long)(t_now - t_phase));   \
      t_phase = t_now;                                                             \
    }                                                                              \
  } while (0)
#define TL_TICK_INIT long long t_phase = clock64()
#define TL_TICK_ARG , long long& t_phase
#define TL_TICK_PASS , t_phase
#else
#define TL_TICK(i) do { } while (0)
#define TL_TICK_INIT do { } while (0)
#define TL_TICK_ARG
#define TL_TICK_PASS
#endif

// ================= B: unstuff one raw chunk (staged in sh.dbuf) into sh.ub =================
// Byte q of the chunk (raw offset cbase + q from gbase), read from the staging buffer; the byte in
// front of the chunk is only known as "was it FF" (carry).
template <int R>
__device__ __forceinline__ uint32_t tl_stage_byte(uint32_t sb_raw, uint32_t q) {
  return lds_u8<0>(sb_raw + q);
}

// One warp looks at one 64-byte piece, two bytes per lane: which bytes are data (w.r.t. the end
// `lim`, a raw offset from gbase), and where does a marker start (first FF followed by a non-zero
// byte inside the segment; the chunk's last piece also answers for the look-ahead byte).
// Returns the two keep flags of this lane; *mk = chunk-relative offset of the first marker whose
// second byte lies in [p0, p0 + 64 (+1)) or TL_NOPOS.
template <int R>
__device__ __forceinline__ uint32_t tl_piece_flags(const TileStream& st, uint32_t sb_raw,
                                                   uint32_t cbase, uint32_t pi, uint32_t prev_ff,
                                                   uint32_t lim, uint32_t* mk) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t q0 = pi * TL_PIECE + 2u * lane;
  const uint32_t pm = q0 > 0 ? tl_stage_byte<R>(sb_raw, q0 - 1) : (prev_ff ? 0xFFu : 0u);
  const uint32_t c0 = tl_stage_byte<R>(sb_raw, q0), c1 = tl_stage_byte<R>(sb_raw, q0 + 1);
  const uint32_t r0 = cbase + q0, r1 = r0 + 1;
  // pairing needs the FF inside the segment: r - 1 >= skew
  const bool k0 = r0 >= st.skew && r0 < lim && !(c0 == 0u && pm == 0xFFu && r0 > st.skew);
  const bool k1 = r1 >= st.skew && r1 < lim && !(c1 == 0u && c0 == 0xFFu && r1 > st.skew);
  bool m0 = r0 > st.skew && r0 < st.limit && c0 != 0u && pm == 0xFFu; // marker at q0 - 1
  bool m1 = r1 > st.skew && r1 < st.limit && c1 != 0u && c0 == 0xFFu; // marker at q0
  uint32_t first = TL_NOPOS;
  const uint32_t b0 = __ballot_sync(0xFFFFFFFFu, m0), b1 = __ballot_sync(0xFFFFFFFFu, m1);
  if (b0 | b1) {
    const uint32_t l0 = b0 ? (uint32_t)__ffs(b0) - 1u : 64u, l1 = b1 ? (uint32_t)__ffs(b1) - 1u : 64u;
    // marker offsets: from m0 of lane l -> piece byte 2l - 1; from m1 of lane l -> 2l
    const uint32_t o0 = b0 ? 2u * l0 : 0xFFFFu, o1 = b1 ? 2u * l1 + 1u : 0xFFFFu; // (+1 biased)
    first = pi * TL_PIECE + min(o0, o1) - 1u; // chunk relative (wraps to -1 only for q = 0: see caller)
  } else if (pi + 1 == st.npieces) {
    // look-ahead byte behind the chunk
    const uint32_t qa = st.npieces * TL_PIECE, ra = cbase + qa;
    if (ra > st.skew && ra < st.limit && tl_stage_byte<R>(sb_raw, qa) != 0u &&
        tl_stage_byte<R>(sb_raw, qa - 1) == 0xFFu)
      first = qa - 1u;
  }
  *mk = first;
  return (k0 ? 1u : 0u) | (k1 ? 2u : 0u);
}

// keep flags only (pass 2b)
template <int R>
__device__ __forceinline__ uint32_t tl_piece_keep(const TileStream& st, uint32_t sb_raw,
                                                  uint32_t cbase, uint32_t pi, uint32_t prev_ff,
                                                  uint32_t lim, uint32_t* c01) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t q0 = pi * TL_PIECE + 2u * lane;
  const uint32_t pm = q0 > 0 ? tl_stage_byte<R>(sb_raw, q0 - 1) : (prev_ff ? 0xFFu : 0u);
  const uint32_t c0 = tl_stage_byte<R>(sb_raw, q0), c1 = tl_stage_byte<R>(sb_raw, q0 + 1);
  const uint32_t r0 = cbase + q0, r1 = r0 + 1;
  const bool k0 = r0 >= st.skew && r0 < lim && !(c0 == 0u && pm == 0xFFu && r0 > st.skew);
  const bool k1 = r1 >= st.skew && r1 < lim && !(c1 == 0u && c0 == 0xFFu && r1 > st.skew);
  *c01 = c0 | (c1 << 8);
  return (k0 ? 1u : 0u) | (k1 ? 2u : 0u);
}

template <int R>
__device__ __forceinline__ TileChunk tl_unstuff(TileShared<R>& sh, const TileStream& st,
                                                const TileCarry& cy, uint32_t chunk TL_TICK_ARG) {
  using G = TileGeom<R>;
  const int tid = threadIdx.x;
  const uint32_t lane = (uint32_t)tid & 31u, wid = (uint32_t)tid >> 5;
  const uint32_t sb_raw = smem_u32(sh.dbuf);
  const uint32_t sb_ub = smem_u32(sh.ub);
  const uint32_t cbase = chunk * st.chunk_raw; // raw offset (from gbase) of the chunk
  TileChunk co;
  if (tid == 0) {
    sh.mpos = TL_NOPOS;
    sh.nlist = 0;
    sh.tail_raw_next = TL_NOPOS;
  }
  // pieces that are not fully inside the segment (its first and its last one): at most two per
  // chunk, known from the geometry alone
  const bool has_edge = chunk == 0 || cbase + st.chunk_raw + 1u > st.limit;
  // ---- pass 1: classify my pieces; regular = 64 data bytes, nothing dropped ----
  uint32_t w[R][16];
  uint32_t n_emit[R];
  bool regular[R], active[R], edge[R];
  uint32_t mk_mine = TL_NOPOS; // chunk-relative offset of the first marker my pieces see
#pragma unroll
  for (int rr = 0; rr < R; ++rr) {
    const uint32_t pi = (uint32_t)rr * TL_NT + (uint32_t)tid;
    const uint32_t p0 = pi * TL_PIECE, r0 = cbase + p0;
    active[rr] = pi < st.npieces && r0 < st.limit;
    regular[rr] = false;
    n_emit[rr] = 0;
    // fully inside the segment, previous byte included (its FF would pair with my first byte)
    const bool inside = active[rr] && r0 > st.skew && r0 + TL_PIECE <= st.limit;
    edge[rr] = active[rr] && !inside;
    if (inside) {
      const uint32_t pa = sb_raw + p0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint4 v = lds_v4<0>(pa + 16 * q);
        w[rr][4 * q + 0] = v.x;
        w[rr][4 * q + 1] = v.y;
        w[rr][4 * q + 2] = v.z;
        w[rr][4 * q + 3] = v.w;
      }
      uint32_t ffp; // FF flags of the word before mine
      if (pi == 0)
        ffp = cy.prev_ff ? 0x80000000u : 0u; // (chunk > 0 here: piece 0 of chunk 0 is never `inside`)
      else
        ffp = tl_ff_flags(lds_u32<0>(pa - 4));
      uint32_t zs_cnt = 0, mk_local = TL_NOPOS; // mk_local: piece-relative index of a marker's SECOND byte
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const uint32_t ffk = tl_ff_flags(w[rr][k]);
        const uint32_t pf = __funnelshift_l(ffp, ffk, 8); // bytes of word k whose predecessor is FF
        if (pf) {
          const uint32_t zf = tl_zero_flags(w[rr][k]);
          zs_cnt += (uint32_t)__popc(pf & zf);
          const uint32_t m2 = pf & ~zf; // second byte of a marker
          if (m2 && mk_local == TL_NOPOS)
            mk_local = 4u * k + (((uint32_t)__ffs(m2) - 1u) >> 3);
        }
        ffp = ffk;
      }
      // the chunk's last piece also answers for the byte behind the chunk
      if (mk_local == TL_NOPOS && pi + 1 == st.npieces && (w[rr][15] >> 24) == 0xFFu &&
          r0 + TL_PIECE < st.limit && tl_stage_byte<R>(sb_raw, p0 + TL_PIECE) != 0u)
        mk_local = TL_PIECE;
      n_emit[rr] = TL_PIECE - zs_cnt;
      regular[rr] = zs_cnt == 0 && mk_local == TL_NOPOS;
      if (mk_local != TL_NOPOS && p0 + mk_local > 0) // the marker's FF sits one byte earlier
        mk_mine = min(mk_mine, p0 + mk_local - 1u);
    }
  }
  TL_TICK(9);
  const int any_mk = __syncthreads_or(mk_mine != TL_NOPOS || has_edge);
  uint32_t mpos = TL_NOPOS;
  if (any_mk) {
    // (a) markers: flagged pieces of pass 1 and, cooperatively, the edge pieces
    if (mk_mine != TL_NOPOS)
      atomicMin(&sh.mpos, mk_mine);
    const uint32_t e1 = min((st.limit - 1u - cbase) / TL_PIECE, st.npieces - 1u); // holds the last byte
    auto is_edge_piece = [&](uint32_t pi) {
      const uint32_t r0 = cbase + pi * TL_PIECE;
      return pi < st.npieces && r0 < st.limit && !(r0 > st.skew && r0 + TL_PIECE <= st.limit);
    };
    if (has_edge && wid < 2) {
      const uint32_t pi = wid == 0 ? 0u : e1;
      if (is_edge_piece(pi) && !(wid == 1 && e1 == 0u)) {
        uint32_t mk;
        tl_piece_flags<R>(st, sb_raw, cbase, pi, cy.prev_ff, st.limit, &mk);
        if (lane == 0 && mk != TL_NOPOS)
          atomicMin(&sh.mpos, mk);
      }
    }
    __syncthreads();
    mpos = sh.mpos; // chunk relative
    // (b) byte counts of the edge pieces and of the piece the marker cuts, w.r.t. the real end
    const uint32_t lim = mpos == TL_NOPOS ? st.limit : min(st.limit, cbase + mpos);
    const uint32_t pm = mpos == TL_NOPOS ? TL_NOPOS : mpos / TL_PIECE;
    if (has_edge || mpos != TL_NOPOS) {
      if (wid < 3) {
        const uint32_t pi = wid == 0 ? 0u : (wid == 1 ? e1 : pm);
        const bool wanted = wid == 2 ? (pm != TL_NOPOS && pm < st.npieces)
                                     : (has_edge && is_edge_piece(pi) && !(wid == 1 && e1 == 0u));
        if (wanted) {
          uint32_t mk;
          const uint32_t kf = tl_piece_flags<R>(st, sb_raw, cbase, pi, cy.prev_ff, lim, &mk);
          const uint32_t n = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, kf & 1u)) +
                             (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, kf & 2u));
          if (lane == 0)
            sh.coop_n[wid] = n;
        }
      }
      __syncthreads();
#pragma unroll
      for (int rr = 0; rr < R; ++rr) {
        const uint32_t pi = (uint32_t)rr * TL_NT + (uint32_t)tid;
        const uint32_t p0 = pi * TL_PIECE;
        if (!active[rr])
          continue;
        if (mpos != TL_NOPOS && p0 >= mpos) { // at / behind the marker: no data
          n_emit[rr] = 0;
          regular[rr] = false;
          active[rr] = false;
        } else if (pi == pm) {
          n_emit[rr] = sh.coop_n[2];
          regular[rr] = false;
        } else if (edge[rr]) {
          n_emit[rr] = sh.coop_n[pi == 0 ? 0 : 1];
          regular[rr] = false;
        }
      }
    }
  }
  const uint32_t limit_eff = mpos == TL_NOPOS ? st.limit : min(st.limit, cbase + mpos);
  TL_TICK(10);
  // ---- positions; the list of the pieces that need byte-wise treatment ----
#pragma unroll
  for (int rr = 0; rr < R; ++rr)
    if (active[rr] && !regular[rr] && n_emit[rr])
      sh.list[atomicAdd(&sh.nlist, 1u)] = (uint32_t)rr * TL_NT + (uint32_t)tid;
  uint32_t dst0[R];
  uint32_t run = cy.tail_len;
#pragma unroll
  for (int rr = 0; rr < R; ++rr) {
    uint32_t tot;
    const uint32_t incl = tl_block_scan(n_emit[rr], sh.warp_tmp[rr & 1], &tot);
    dst0[rr] = run + incl - n_emit[rr];
    run += tot;
    const uint32_t pi = (uint32_t)rr * TL_NT + (uint32_t)tid;
    if (pi <= (uint32_t)G::NPIECE)
      sh.anchor[pi] = dst0[rr];
  }
  const uint32_t total_emit = run - cy.tail_len;
  const uint32_t len = run;
  const bool final_chunk = (mpos != TL_NOPOS) || (cbase + st.chunk_raw >= st.limit);
  co.len = len;
  co.Lc = final_chunk ? len + TL_ZEXT : (len > (uint32_t)TL_LA ? len - TL_LA : 0u);
  const uint32_t Lc = co.Lc;
  TL_TICK(11);
  // ---- pass 2a: regular pieces, whole words (byte i of the clean stream lives at ub8[i ^ 3]) ----
#pragma unroll
  for (int rr = 0; rr < R; ++rr) {
    if (!regular[rr])
      continue;
    const uint32_t d0 = dst0[rr];
    // the source of clean byte Lc becomes the source of ub byte 0 of the next chunk
    if (!final_chunk && Lc - d0 < (uint32_t)TL_PIECE)
      sh.tail_raw_next = cbase + ((uint32_t)rr * TL_NT + (uint32_t)tid) * TL_PIECE + (Lc - d0);
    const uint32_t head = (4u - (d0 & 3u)) & 3u; // bytes up to the next word boundary
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if ((uint32_t)k < head)
        sts_u8<0>(sb_ub + ((d0 + k) ^ 3u), (w[rr][0] >> (8 * k)) & 0xFFu);
    const uint32_t sh8 = head * 8;
    const uint32_t wa = sb_ub + ((d0 + head) & ~3u);
#pragma unroll
    for (int k = 0; k < 15; ++k) {
      const uint32_t le = __funnelshift_r(w[rr][k], w[rr][k + 1], sh8);
      sts_u32<0>(wa + 4 * k, __byte_perm(le, 0, 0x0123));
    }
    if (head == 0) {
      sts_u32<60>(wa, __byte_perm(w[rr][15], 0, 0x0123));
    } else {
#pragma unroll
      for (int k = 1; k < 4; ++k)
        if ((uint32_t)k >= head)
          sts_u8<0>(sb_ub + ((d0 + 60 + k) ^ 3u), (w[rr][15] >> (8 * k)) & 0xFFu);
    }
  }
  // zero padding behind the data (look-ahead loads; zero extension at the end of the segment)
  if (tid < 64) {
    const uint32_t i = len + tid;
    if (i < (uint32_t)G::UBBYTES)
      sts_u8<0>(sb_ub + (i ^ 3u), 0u);
  }
  if (tid == 64) { // was the last raw byte of this chunk an FF inside the segment?
    const uint32_t lastr = cbase + st.chunk_raw - 1u;
    sh.prev_ff_next = (lastr >= st.skew && lastr < st.limit &&
                       tl_stage_byte<R>(sb_raw, st.chunk_raw - 1u) == 0xFFu) ? 1u : 0u;
  }
  TL_TICK(12);
  __syncthreads(); // list + anchors complete
  // ---- pass 2b: the other pieces, one warp per piece, two bytes per lane, from the staging ----
  {
    const uint32_t nl = sh.nlist;
    const uint32_t lt = (1u << lane) - 1u;
    for (uint32_t j = wid; j < nl; j += TL_NT / 32) {
      const uint32_t pi = sh.list[j];
      uint32_t c01;
      const uint32_t kf = tl_piece_keep<R>(st, sb_raw, cbase, pi, cy.prev_ff, limit_eff, &c01);
      const uint32_t b0 = __ballot_sync(0xFFFFFFFFu, kf & 1u), b1 = __ballot_sync(0xFFFFFFFFu, kf & 2u);
      uint32_t d = sh.anchor[pi] + (uint32_t)__popc(b0 & lt) + (uint32_t)__popc(b1 & lt);
      const uint32_t q0 = pi * TL_PIECE + 2u * lane;
      if (kf & 1u) {
        if (!final_chunk && d == Lc)
          sh.tail_raw_next = cbase + q0;
        sts_u8<0>(sb_ub + (d ^ 3u), c01 & 0xFFu);
        ++d;
      }
      if (kf & 2u) {
        if (!final_chunk && d == Lc)
          sh.tail_raw_next = cbase + q0 + 1u;
        sts_u8<0>(sb_ub + (d ^ 3u), c01 >> 8);
      }
    }
  }
  TL_TICK(13);
  co.end_all = co.Lc * 8;
  co.mpos = mpos;
  co.total_emit = total_emit;
  co.final_chunk = final_chunk;
  __syncthreads();
  TL_TICK(14);
  return co;
}

// ---- hot-loop view of shared memory: `sb` = smem_base_opaque(&sh), accesses are reg + constant ----
template <int R> struct TileOff {
  using S = TileShared<R>;
  static constexpr int UB = (int)offsetof(S, ub);
  static constexpr int DBUF = (int)offsetof(S, dbuf);
  static constexpr int LUT = (int)(offsetof(S, tab) + offsetof(DevTable, lut));
  static constexpr int LEN8 = (int)offsetof(S, len8);
};
constexpr uint32_t TL_LUT_TOPMASK = ~((1u << (32 - LUT_BITS)) - 1u);

template <int R> struct TileBits {
  uint32_t p;        // bit position in ub
  uint32_t cur, nxt; // words p/32 and p/32+1
  uint32_t wa;       // shared address (relative to sb + UB) of word p/32+2
  __device__ __forceinline__ void open(uint32_t sb, uint32_t start) {
    p = start;
    wa = sb + ((start >> 3) & ~3u);
    cur = lds_u32<TileOff<R>::UB>(wa);
    nxt = lds_u32<TileOff<R>::UB + 4>(wa);
  }
  __device__ __forceinline__ uint32_t peek() const { return __funnelshift_l(nxt, cur, p); }
  __device__ __forceinline__ void skip(uint32_t n) { // n <= 32: at most one word boundary
    const uint32_t pn = p + n;
    if ((pn ^ p) & 32u) {
      cur = nxt;
      nxt = lds_u32<TileOff<R>::UB + 8>(wa);
      wa += 4;
    }
    p = pn;
  }
};

// keeps a loop-invariant value in its register (ptxas otherwise re-derives it from
// threadIdx.x inside the hot loops when registers are short)
__device__ __forceinline__ uint32_t tl_opaque(uint32_t v) {
#ifndef RSB200_EMU
  asm volatile("mov.u32 %0, %0;" : "+r"(v));
#endif
  return v;
}

template <int R> __device__ __forceinline__ uint32_t tl_lut(uint32_t sb, uint32_t x) {
  return lds_u16<TileOff<R>::LUT>(mad_hi(x & TL_LUT_TOPMASK, 1u << (LUT_BITS + 1), sb));
}

// slow path of a symbol: code longer than the LUT depth, SSSS = 16, or corrupt
__device__ __noinline__ uint32_t tl_long_symbol(const DevTable* t, uint32_t x) {
  return (uint32_t)decode_sym(t, x).total;
}

// lengths-only parse from `start` up to (not including) the first symbol that starts at or
// behind end_bit; returns the position reached and counts the symbols
template <int R> __device__ __forceinline__ uint32_t tl_len8(uint32_t sb, uint32_t x) {
  return lds_u8<TileOff<R>::LEN8>(mad_hi(x, 1u << LUT_BITS, sb)); // sb + (x >> 21)
}

template <int R>
__device__ __forceinline__ uint32_t tl_scan(const TileShared<R>& sh, uint32_t sb, uint32_t start,
                                            uint32_t end_bit, uint32_t& count) {
  uint32_t cnt = 0;
  if (start >= end_bit) {
    count = 0;
    return start;
  }
  end_bit = tl_opaque(end_bit);
  TileBits<R> b;
  b.open(sb, start);
  do {
    const uint32_t x = b.peek();
    uint32_t len = tl_len8<R>(sb, x);
    if (len == 0)
      len = tl_long_symbol(&sh.tab, x);
    ++cnt;
    b.skip(len);
  } while (b.p < end_bit);
  count = cnt;
  return b.p;
}

// One difference (PrefixCodeLUTDecoder.h:172-216 + AbstractPrefixCodeDecoder.h:43-76), mod 2^16
// in the low half; tl = bits consumed.
template <int R>
__device__ __forceinline__ uint32_t tl_decode_diff(TileShared<R>& sh, uint32_t sb, uint32_t x,
                                                   uint32_t& tl) {
  const uint32_t e = tl_lut<R>(sb, x);
  tl = e >> 10;
  if (e == 0) {
    const SymLen s = decode_sym(&sh.tab, x);
    tl = (uint32_t)s.total;
    if (s.codelen == 0)
      sh.bad_code = 1u; // "bad Huffman code"
    return (uint32_t)sym_diff(s, x);
  }
  // extend(), branch free: tt = bits after the code; f = all ones iff their first bit is 0
  // (negative range); (f:tt) << ssss leaves v with ones above it in that case, and
  // v - (2^ssss - 1) == (v | ~mask) + 1.  Funnel shifts wrap at 32: fields of e are used unmasked.
  const uint32_t tt = __funnelshift_l(0u, x, e);
  const uint32_t f = (uint32_t)((int32_t)~tt >> 31);
  return __funnelshift_l(tt, f, e >> 5) - f;
}

struct TileSync {
  uint32_t my_start;
  uint32_t count;
  uint32_t nsub;
  uint32_t subbits;
};

// ================= C: self-synchronising parse of the chunk in sh.ub =================
template <int R>
__device__ __forceinline__ TileSync tl_sync(TileShared<R>& sh, uint32_t sb, const TileCarry& cy,
                                            const TileChunk& co, uint32_t preroll) {
  const int tid = threadIdx.x;
  // subsequence size: an odd number of words, at least 9 (288 bits)
  uint32_t sw = ((co.end_all + 31u) / 32u + TL_NT - 1) / TL_NT;
  sw = max(sw, 9u) | 1u;
  const uint32_t subbits = sw * 32u;
  const uint32_t nsub = (co.end_all + subbits - 1) / subbits;
  const uint32_t sub_lo = (uint32_t)tid * subbits;
  const uint32_t sub_hi = min(sub_lo + subbits, co.end_all);
  const bool active = (uint32_t)tid < nsub;
  uint32_t my_start = 0xFFFFFFF0u, cnt = 0, ex = 0xFFFFFFF0u;
  if (active) {
    if (tid == 0) {
      my_start = cy.pos;
    } else {
      // pre-roll: parse from `preroll` bits before my range; the first symbol that starts inside
      // my range is my guess
      const uint32_t from = sub_lo > preroll ? sub_lo - preroll : 0u;
      uint32_t dummy;
      my_start = from < sub_lo ? tl_scan<R>(sh, sb, from, sub_lo, dummy) : sub_lo;
    }
    ex = tl_scan<R>(sh, sb, my_start, sub_hi, cnt);
  }
  sh.exitpos[tid] = ex;
  __syncthreads();
  // Fixed-point iteration: adopt the predecessor's exit until nothing changes.  Thread 0 starts
  // at the true position, so the fixed point is the sequential parse (induction over threads).
  for (int round = 0; round < TL_NT + 2; ++round) {
    const uint32_t new_start = (tid == 0) ? cy.pos : sh.exitpos[tid - 1];
    const bool changed = active && new_start != my_start;
    const int any = __syncthreads_or(changed ? 1 : 0);
    if (!any)
      break;
    if (changed) {
      my_start = new_start;
      ex = tl_scan<R>(sh, sb, my_start, sub_hi, cnt);
    }
    sh.exitpos[tid] = ex;
    __syncthreads();
  }
  TileSync so;
  so.my_start = my_start;
  so.count = active ? cnt : 0u;
  so.nsub = nsub;
  so.subbits = subbits;
  return so;
}

// fast (row, column) of a global sample index
__device__ __forceinline__ void tl_row_col(uint32_t g, uint32_t RS, uint32_t inv, uint32_t& r,
                                           uint32_t& s) {
  r = __umulhi(g, inv);
  int32_t d = (int32_t)(g - r * RS);
  if (d < 0) {
    --r;
    d += (int32_t)RS;
  }
  if ((uint32_t)d >= RS) {
    ++r;
    d -= (int32_t)RS;
  }
  s = (uint32_t)d;
}

// Raw offset (from the segment start) of the data byte with clean index `need_ub` in the CURRENT
// chunk's ub (it must exist: need_ub <= clean bytes in ub): anchors give the clean index at
// which every 64-byte raw piece starts, the rest is a walk of at most 64 + TL_LA bytes.
template <int R>
__device__ __noinline__ uint32_t tl_raw_of_clean(const TileShared<R>& sh, const TileStream& st,
                                                 const TileCarry& cy, uint32_t chunk,
                                                 uint32_t need_ub) {
  uint32_t rawp, cleanp;
  if (need_ub < cy.tail_len || sh.anchor[0] > need_ub) {
    rawp = cy.tail_raw;
    cleanp = 0;
  } else {
    int a = 0, b = (int)st.npieces - 1;
    while (a < b) {
      const int m = (a + b + 1) >> 1;
      if (sh.anchor[m] <= need_ub)
        a = m;
      else
        b = m - 1;
    }
    rawp = chunk * st.chunk_raw + (uint32_t)a * TL_PIECE;
    cleanp = sh.anchor[a];
    if (rawp < st.skew)
      rawp = st.skew;
    // a stuffing byte may sit exactly at rawp (its FF ended the previous piece)
    if (rawp > st.skew && tl_raw_byte(st, rawp - 1) == 0xFFu && tl_raw_byte(st, rawp) == 0u)
      rawp += 1;
  }
  while (cleanp < need_ub) {
    const uint32_t c0 = tl_raw_byte(st, rawp);
    rawp += (c0 == 0xFFu) ? 2u : 1u; // data FF + its stuffing byte
    ++cleanp;
  }
  return rawp - st.skew;
}

// ================= end of the segment: the reference's pump, replayed =================
// The reference refills its 64-bit cache 4 data bytes at a time, before a symbol whenever fewer
// than 32 bits are left (BitStreamer::fill(32), BitStreamer.h:216-229; one fill per symbol,
// PrefixCodeLUTDecoder.h:172-216), so before the symbol at clean bit offset T it has done
// Rf(T) = T/32 + 1 (+1 if T%32) refills, holds 32*Rf - T bits and its input position is the raw
// offset behind 4*Rf data bytes -- as long as no refill met the end marker.  The refill that does
// stops the input: the cache is topped up with zero bits to 64 and the position jumps to
// size + (4 - i) (BitStreamerJPEG.h:155-183); later refills read zeros and advance by 4, and
// BitStreamer::getInput throws once the position is more than 16 bytes past the buffer
// (BitStreamer.h:120-127).  Without a marker the bytes past the buffer are zero DATA bytes and
// the same check applies.  getStreamPosition() = position of the marker, else the position.
//
// Thread 0 replays that over the last symbols of the segment: from an exact symbol start `from`
// (bit position in ub) at which the cadence formula still holds, up to the symbol at p_last.
template <int R>
__device__ __noinline__ void tl_replay(TileShared<R>& sh, const TileStream& st, uint32_t sb,
                                       const TileCarry& cy, uint32_t chunk, uint32_t from,
                                       uint32_t p_last) {
  const uint32_t size = st.limit - st.skew;
  uint32_t fill, rp;
  const uint64_t T0 = 8ull * cy.ubytes + from;
  if (T0 == 0) {
    fill = 0;
    rp = 0;
  } else {
    const uint64_t Rf = (T0 >> 5) + 1 + ((T0 & 31u) ? 1u : 0u);
    fill = (uint32_t)(32ull * Rf - T0);
    rp = tl_raw_of_clean<R>(sh, st, cy, chunk, (uint32_t)(4ull * Rf - cy.ubytes));
  }
  uint32_t end_pos = TL_NOPOS; // endOfStreamPos
  bool threw = false;
  TileBits<R> b;
  b.open(sb, from);
  for (;;) {
    if (fill < 32) {
      // BitStreamer::getInput: more than 16 bytes past the buffer -> IOException
      if (rp > size + 16u) {
        threw = true;
        break;
      }
      if (end_pos != TL_NOPOS) {
        rp += 4;
        fill += 32;
      } else {
        uint32_t q = rp;
        bool hit = false;
        for (int i = 0; i < 4; ++i) {
          const uint32_t c0 = q < size ? (uint32_t)st.gbase[st.skew + q] : 0u;
          if (c0 != 0xFFu) {
            q += 1;
            continue;
          }
          const uint32_t c1 = q + 1 < size ? (uint32_t)st.gbase[st.skew + q + 1] : 0u;
          if (c1 == 0u) {
            q += 2;
            continue;
          }
          end_pos = q;
          fill = 64;
          rp = size + (uint32_t)(4 - i);
          hit = true;
          break;
        }
        if (!hit) {
          rp = q;
          fill += 32;
        }
      }
    }
    const uint32_t at = b.p;
    const uint32_t x = b.peek();
    uint32_t len = tl_len8<R>(sb, x);
    if (len == 0)
      len = tl_long_symbol(&sh.tab, x);
    b.skip(len);
    fill -= len;
    if (at >= p_last)
      break;
  }
  // (LJpegDecompressor.cpp:334: skipBytes(getStreamPosition()) throws behind the buffer)
  if (end_pos == TL_NOPOS && rp > size)
    threw = true;
  sh.rstat = threw ? 2u : 0u;
  sh.rcons = end_pos != TL_NOPOS ? end_pos : rp;
}

// ================= the kernel body =================
template <int R, int GG>
__device__ __forceinline__ void tl_store_units(TileShared<R>& sh, uint32_t sb, const DevScan& sc,
                                               uint8_t* __restrict__ out, uint32_t S0, uint32_t n,
                                               uint32_t upt, uint32_t base01, uint32_t base23,
                                               uint32_t r_first, uint32_t rb01, uint32_t rb23);

template <int R>
__device__ __forceinline__ void tile_body(TileShared<R>& sh, const uint8_t* __restrict__ in,
                                          uint64_t in_total, uint8_t* __restrict__ out,
                                          DevResult* __restrict__ res, uint32_t npieces,
                                          uint32_t preroll) {
  using G = TileGeom<R>;
  const int tid = threadIdx.x;
  const DevScan& sc = sh.sc;
  const uint64_t abase = sc.in_offset & ~15ull;
  TileStream st;
  st.skew = (uint32_t)(sc.in_offset - abase);
  st.gbase = in + abase;
  st.limit = st.skew + sc.in_size;
  st.readable = ((in_total + 15) & ~15ull) - abase;
  st.npieces = npieces;
  st.chunk_raw = npieces * TL_PIECE;
  const uint32_t GRP = sc.group;
  const uint32_t RS = sc.row_samples;
  const uint32_t sb = smem_base_opaque(&sh);
  uint32_t my_status = 0;
  if (tid == 0)
    tl_issue_chunk<R>(sh, st, 0);
  bool pending = true;
  uint32_t pending_par = 0;
  bool replayed = false;
  TL_TICK_INIT;

  for (uint32_t chunk = 0;; ++chunk) {
    const TileCarry cy = sh.cy;
    if (cy.sym >= sc.n_samples)
      break;
    if (cy.ended) {
      my_status |= 2u; // the zero extension was parsed too and symbols are still missing
      break;
    }
    mbar_wait(&sh.bar, chunk & 1);
    pending = false;
    TL_TICK(0);

    // ================= B: unstuff =================
    const TileChunk co = tl_unstuff<R>(sh, st, cy, chunk TL_TICK_PASS);
    const uint32_t len = co.len, Lc = co.Lc;
    TL_TICK(1);

    // ================= C: self-synchronising parse =================
    const TileSync so = tl_sync<R>(sh, sb, cy, co, preroll);
    const uint32_t my_start = so.my_start;
    TL_TICK(2);

    // ================= D: symbol indices =================
    uint32_t total_syms;
    const uint32_t sincl = tl_block_scan(so.count, sh.warp_tmp[2], &total_syms);
    const uint32_t rel0 = sincl - so.count;                  // chunk-relative index of my first symbol
    const uint32_t chunk_syms = min(total_syms, sc.n_samples - cy.sym);
    const uint32_t exit_all = so.nsub ? sh.exitpos[so.nsub - 1] : cy.pos;
    const uint32_t klast = sc.n_samples - 1 - cy.sym;        // chunk-relative index of the last needed one

    // batches over the chunk's symbols (one batch unless the data is below ~1 byte per sample)
    uint32_t done = 0;
    for (;;) {
      const TileCarry cb = sh.cy; // leftover / proc / prefix state (updated per batch)
      uint32_t cap = min((uint32_t)G::DCAP, (uint32_t)(TL_RBMAX - 1) * RS) & ~7u;
      const uint32_t room = cap - cb.leftover;
      const uint32_t take = min(room, chunk_syms - done);
      // the carried differences first
      if ((uint32_t)tid < cb.leftover)
        sh.dbuf[tid] = (uint16_t)(cb.left[tid >> 1] >> (16 * (tid & 1)));
      // ---- decode + store the differences of symbols [done, done+take) ----
      if (so.count) {
        const uint32_t lo = max(rel0, done), hi = min(rel0 + so.count, done + take);
        if (lo < hi) {
          TileBits<R> b;
          b.open(sb, my_start);
          for (uint32_t k = rel0; k < lo; ++k) { // symbols of earlier batches: lengths only
            const uint32_t x = b.peek();
            uint32_t tl = tl_len8<R>(sb, x);
            if (tl == 0)
              tl = tl_long_symbol(&sh.tab, x);
            b.skip(tl);
          }
          uint32_t dst = sb + 2u * (cb.leftover + (lo - done));
          const uint32_t dst_end = dst + 2u * (hi - lo);
          // the segment's last symbol (its position feeds `consumed`) splits the walk in two
          uint32_t stop = (klast >= lo && klast < hi) ? dst + 2u * (klast - lo) : dst_end;
          uint32_t plast = TL_NOPOS;
          for (;;) {
            while (dst != stop) {
              const uint32_t x = b.peek();
              uint32_t tl;
              const uint32_t diff = tl_decode_diff<R>(sh, sb, x, tl);
              sts_u16<TileOff<R>::DBUF>(dst, diff);
              dst += 2;
              b.skip(tl);
            }
            if (stop == dst_end)
              break;
            plast = b.p;
            stop = dst_end;
          }
          if (plast != TL_NOPOS) {
            sh.last.seen = 1u;
            sh.last.p_last = plast;
          }
        }
      }
      __syncthreads();
      TL_TICK(3);

      // ---- `consumed` / status of the segment, once its last symbol has been met ----
      if (sh.last.seen && !replayed) {
        replayed = true;
        const uint32_t p_last = sh.last.p_last;
        // Far behind the data (only streams that end early get there) the cadence of the
        // reference's pump decides between "zero bits" and IOException: replay it.  Otherwise no
        // refill can have been refused and the closed form gives the position.
        const bool far = co.final_chunk && p_last > 8u * len + 64u;
        if (tid == 0) {
          if (!far) {
            const uint64_t T = 8ull * cy.ubytes + p_last;
            const uint64_t Rf = (T >> 5) + 1 + ((T & 31u) ? 1u : 0u);
            const uint64_t need_abs = 4ull * Rf; // data bytes the pump has taken
            const uint64_t have_abs = (uint64_t)cy.ubytes + len;
            uint32_t cons;
            if (!co.final_chunk || need_abs <= have_abs) {
              cons = tl_raw_of_clean<R>(sh, st, cy, chunk, (uint32_t)(need_abs - cy.ubytes));
            } else if (co.mpos != TL_NOPOS) {
              cons = chunk * st.chunk_raw + co.mpos - st.skew; // it met the marker
            } else {
              // zero data bytes behind the buffer: one position each (a final FF pairs with
              // the first of them)
              const uint32_t at_end = tl_raw_of_clean<R>(sh, st, cy, chunk, len);
              cons = at_end + (uint32_t)(need_abs - have_abs);
            }
            // LJpegDecompressor::decodeN skips `consumed` bytes of its ByteStream afterwards
            // (LJpegDecompressor.cpp:334): a position behind the buffer -- only possible when the
            // pump never met a marker -- is an IOException there
            const bool met_marker = co.final_chunk && need_abs > have_abs && co.mpos != TL_NOPOS;
            sh.rstat = (!met_marker && cons > st.limit - st.skew) ? 2u : 0u;
            sh.rcons = cons;
          } else {
            // an exact symbol start at or before the last 64 data bits, where the cadence holds
            const uint32_t tm_lo = len >= 8u ? 8u * len - 64u : 0u;
            uint32_t from = cy.pos;
            uint32_t s = min(tm_lo / so.subbits, so.nsub ? so.nsub - 1 : 0u);
            while (s > 0 && sh.exitpos[s - 1] > tm_lo)
              --s;
            if (s > 0)
              from = sh.exitpos[s - 1];
            tl_replay<R>(sh, st, sb, cy, chunk, from, p_last);
          }
        }
        __syncthreads();
        my_status |= sh.rstat;
        if (tid == 0)
          res->consumed = sh.rcons;
      }

      TL_TICK(4);
      // ================= E: predictor on whole 8-sample units =================
      const uint32_t have = cb.leftover + take;
      const bool last_batch = (done + take == chunk_syms);
      const bool seg_done = last_batch && (cy.sym + chunk_syms >= sc.n_samples);
      const uint32_t n = seg_done ? have : (have & ~7u); // samples to finish now
      const uint32_t S0 = cb.proc;                         // global index of dbuf[0], multiple of 8
      const uint32_t nun = (n + 7) >> 3;
      const uint32_t upt = ((nun + TL_NT - 1) / TL_NT) | 1u; // odd: conflict-free 128-bit loads
      const uint32_t u0 = (uint32_t)tid * upt, u1 = min(u0 + upt, nun);
      // rows starting inside this batch: first sample index ri = r*RS - S0 in [0, n)
      const uint32_t r_first = (S0 + RS - 1) / RS;
      const uint32_t r_end = n ? (S0 + n - 1) / RS + 1 : r_first;
      const uint32_t nrs = r_end > r_first ? r_end - r_first : 0;
      // E1: value of the first MCU of the previous row, for every row start of the batch
      //     (only the differences are needed); one warp, 32 rows at a time
      if (tid < 32) {
        uint32_t col01 = cb.col01, col23 = cb.col23;
        for (uint32_t rbq = 0; rbq < nrs; rbq += 32) {
          const uint32_t j = rbq + tid;
          uint32_t df01 = 0, df23 = 0;
          if (j < nrs) {
            const uint32_t ri = (r_first + j) * RS - S0;
            uint32_t fv[4] = {0, 0, 0, 0};
            for (uint32_t cc = 0; cc < GRP; ++cc)
              fv[cc] = sh.dbuf[ri + cc];
            df01 = fv[0] | (fv[1] << 16);
            df23 = fv[2] | (fv[3] << 16);
          }
          uint32_t i01 = df01, i23 = df23;
#pragma unroll
          for (int dd = 1; dd < 32; dd <<= 1) {
            const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, i01, dd);
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, i23, dd);
            if (tid >= dd) {
              i01 = __vadd2(i01, x);
              i23 = __vadd2(i23, y);
            }
          }
          if (j < nrs) { // value of the first MCU of the previous row
            sh.rowbase[j][0] = __vadd2(col01, __vsub2(i01, df01));
            sh.rowbase[j][1] = __vadd2(col23, __vsub2(i23, df23));
          }
          col01 = __vadd2(col01, __shfl_sync(0xFFFFFFFFu, i01, 31));
          col23 = __vadd2(col23, __shfl_sync(0xFFFFFFFFu, i23, 31));
        }
        if (tid == 0) {
          sh.cy.col01 = col01;
          sh.cy.col23 = col23;
        }
      }
      // E2: my units' totals, and the partial sum in front of the (one) row start among them
      uint32_t s01 = 0, s23 = 0, part01 = 0, part23 = 0, rowj = TL_NOPOS;
      {
        uint32_t rr, ss;
        tl_row_col(S0 + 8u * u0, RS, sc.rs_inv, rr, ss);
        for (uint32_t u = u0; u < u1; ++u) {
          if (ss == 0) { // unit u starts row rr
            rowj = rr - r_first;
            part01 = s01;
            part23 = s23;
          }
          const uint4 q = lds_v4<TileOff<R>::DBUF>(sb + 16u * u);
          if (GRP == 2) {
            s01 = __vadd2(s01, __vadd2(__vadd2(q.x, q.y), __vadd2(q.z, q.w)));
          } else if (GRP == 4) {
            s01 = __vadd2(s01, __vadd2(q.x, q.z));
            s23 = __vadd2(s23, __vadd2(q.y, q.w));
          } else {
            const uint32_t t = __vadd2(__vadd2(q.x, q.y), __vadd2(q.z, q.w));
            s01 = (s01 + (t & 0xFFFFu) + (t >> 16)) & 0xFFFFu;
          }
          ss += 8;
          if (ss >= RS) {
            ss = 0;
            ++rr;
          }
        }
      }
      uint32_t a01 = s01, a23 = s23, ta, tb;
      tl_block_scan_v2(a01, a23, sh.warp_tmp[0], sh.warp_tmp[1], ta, tb); // (barrier inside: E1 done)
      const uint32_t base01 = __vadd2(__vsub2(a01, s01), cb.pc01); // running sums in front of my units
      const uint32_t base23 = __vadd2(__vsub2(a23, s23), cb.pc23);
      if (rowj != TL_NOPOS) {
        // additive constant of that row: (first MCU of the previous row) - (running sum in front)
        sh.rowbase[rowj][0] = __vsub2(sh.rowbase[rowj][0], __vadd2(base01, part01));
        sh.rowbase[rowj][1] = __vsub2(sh.rowbase[rowj][1], __vadd2(base23, part23));
      }
      __syncthreads();
      TL_TICK(5);
      // E3: values -> image
      if (GRP == 2)
        tl_store_units<R, 2>(sh, sb, sc, out, S0, n, upt, base01, base23, r_first, cb.rb01, cb.rb23);
      else if (GRP == 4)
        tl_store_units<R, 4>(sh, sb, sc, out, S0, n, upt, base01, base23, r_first, cb.rb01, cb.rb23);
      else
        tl_store_units<R, 1>(sh, sb, sc, out, S0, n, upt, base01, base23, r_first, cb.rb01, cb.rb23);
      TL_TICK(6);
      // E4: carry; the unfinished differences (< 8) travel in the carry (dbuf is the staging of
      //     the next chunk's raw bytes)
      if (tid == 0) {
        TileCarry& c2 = sh.cy;
        c2.pc01 = __vadd2(cb.pc01, ta);
        c2.pc23 = __vadd2(cb.pc23, tb);
        if (nrs) {
          c2.rb01 = sh.rowbase[nrs - 1][0];
          c2.rb23 = sh.rowbase[nrs - 1][1];
        }
        c2.proc = S0 + n;
        c2.leftover = have - n;
      }
      if (tid >= 32 && tid < 36) {
        const uint32_t k = 2u * (uint32_t)(tid - 32);
        const uint32_t lo = (k < have - n) ? sh.dbuf[n + k] : 0u;
        const uint32_t hi = (k + 1 < have - n) ? sh.dbuf[n + k + 1] : 0u;
        sh.cy.left[tid - 32] = lo | (hi << 16);
      }
      __syncthreads();
      done += take;
      if (done >= chunk_syms)
        break;
    }

    TL_TICK(7);
    // ================= carry to the next chunk =================
    {
      // deferred tail: clean bytes [Lc, len) move to the front of ub (nobody reads ub any more)
      const uint32_t tail = co.final_chunk ? 0u : len - Lc;
      uint32_t tailbyte = 0;
      if ((uint32_t)tid < tail)
        tailbyte = reinterpret_cast<uint8_t*>(sh.ub)[(Lc + tid) ^ 3u];
      if (tid == 32) {
        TileCarry& c2 = sh.cy;
        c2.sym = cy.sym + total_syms;
        c2.pos = exit_all - Lc * 8u;
        c2.tail_len = tail;
        c2.ubytes = cy.ubytes + Lc;
        if (!co.final_chunk) {
          // raw offset of the clean byte that becomes ub byte 0 (clean index Lc of this chunk):
          // recorded by the piece that holds it; it lies in the carried tail only when this chunk
          // produced fewer than TL_LA bytes
          c2.tail_raw = sh.tail_raw_next != TL_NOPOS
                            ? sh.tail_raw_next
                            : tl_raw_of_clean<R>(sh, st, cy, chunk, Lc) + st.skew;
          c2.prev_ff = sh.prev_ff_next;
        }
        c2.ended = co.final_chunk ? 1u : 0u;
      }
      __syncthreads();
      if ((uint32_t)tid < tail)
        reinterpret_cast<uint8_t*>(sh.ub)[tid ^ 3u] = (uint8_t)tailbyte;
      // the raw staging of the next chunk lands in dbuf: everything above has left it
      const bool more = !co.final_chunk && sh.cy.sym < sc.n_samples;
      if (more) {
        if (tid == 0) {
          fence_proxy_async();
          tl_issue_chunk<R>(sh, st, chunk + 1);
        }
        pending = true;
        pending_par = (chunk + 1) & 1u;
      }
    }
    TL_TICK(8);
  }
  // never leave a bulk copy in flight into this CTA's shared memory
  if (pending)
    mbar_wait(&sh.bar, pending_par);
  {
    const int over = __syncthreads_or((int)(my_status & 2u));
    const int bad = (int)sh.bad_code; // (after the barrier)
    if (tid == 0) {
      res->status = bad ? 1u : (over ? 2u : 0u);
      if (!sh.last.seen)
        res->consumed = 0;
    }
  }
}

// E3 for one group size: every thread walks its units, running sums in registers
template <int R, int GG>
__device__ __forceinline__ void tl_store_units(TileShared<R>& sh, uint32_t sb, const DevScan& sc,
                                               uint8_t* __restrict__ out, uint32_t S0, uint32_t n,
                                               uint32_t upt, uint32_t base01, uint32_t base23,
                                               uint32_t r_first, uint32_t rb01, uint32_t rb23) {
  const int tid = threadIdx.x;
  const uint32_t nun = (n + 7) >> 3;
  const uint32_t u0 = (uint32_t)tid * upt, u1 = min(u0 + upt, nun);
  if (u0 >= u1)
    return;
  const uint32_t RS = sc.row_samples;
  uint32_t rr, ss;
  tl_row_col(S0 + 8u * u0, RS, sc.rs_inv, rr, ss);
  // additive constant of the row my first unit lies in
  uint32_t k01, k23;
  if (rr >= r_first && !(ss == 0)) {
    k01 = sh.rowbase[rr - r_first][0];
    k23 = sh.rowbase[rr - r_first][1];
  } else {
    k01 = rb01; // row in progress from the previous batch (replaced below if a row starts here)
    k23 = rb23;
  }
  uint32_t r01 = __vadd2(base01, k01), r23 = __vadd2(base23, k23); // running sum + row constant
  uint8_t* orow = out + sc.out_offset + (uint64_t)(sc.out_y + rr) * sc.out_pitch + 2ull * sc.out_x;
  for (uint32_t u = u0; u < u1; ++u) {
    if (ss == 0) { // a row starts: switch the constant
      const uint32_t n01 = sh.rowbase[rr - r_first][0], n23 = sh.rowbase[rr - r_first][1];
      r01 = __vadd2(r01, __vsub2(n01, k01));
      r23 = __vadd2(r23, __vsub2(n23, k23));
      k01 = n01;
      k23 = n23;
    }
    const uint4 q = lds_v4<TileOff<R>::DBUF>(sb + 16u * u);
    uint4 o;
    if (GG == 2) {
      r01 = __vadd2(r01, q.x); o.x = r01;
      r01 = __vadd2(r01, q.y); o.y = r01;
      r01 = __vadd2(r01, q.z); o.z = r01;
      r01 = __vadd2(r01, q.w); o.w = r01;
    } else if (GG == 4) {
      r01 = __vadd2(r01, q.x); o.x = r01;
      r23 = __vadd2(r23, q.y); o.y = r23;
      r01 = __vadd2(r01, q.z); o.z = r01;
      r23 = __vadd2(r23, q.w); o.w = r23;
    } else {
      uint32_t r = r01 & 0xFFFFu, lo, hi;
      lo = (r + (q.x & 0xFFFFu)) & 0xFFFFu; hi = (lo + (q.x >> 16)) & 0xFFFFu; o.x = lo | (hi << 16); r = hi;
      lo = (r + (q.y & 0xFFFFu)) & 0xFFFFu; hi = (lo + (q.y >> 16)) & 0xFFFFu; o.y = lo | (hi << 16); r = hi;
      lo = (r + (q.z & 0xFFFFu)) & 0xFFFFu; hi = (lo + (q.z >> 16)) & 0xFFFFu; o.z = lo | (hi << 16); r = hi;
      lo = (r + (q.w & 0xFFFFu)) & 0xFFFFu; hi = (lo + (q.w >> 16)) & 0xFFFFu; o.w = lo | (hi << 16); r = hi;
      r01 = r;
    }
    if (ss + 8 <= sc.store_w) {
      stg_cs_v4(orow + 2ull * ss, o);
    } else if (ss < sc.store_w) { // the crop ends inside this unit
      uint16_t* o16 = reinterpret_cast<uint16_t*>(orow) + ss;
      const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (ss + k < sc.store_w)
          o16[k] = (uint16_t)(ow[k >> 1] >> (16 * (k & 1)));
    }
    ss += 8;
    if (ss >= RS) {
      ss = 0;
      ++rr;
      orow += sc.out_pitch;
    }
  }
}

// plan-time parameters of a segment: raw pieces per chunk and the pre-roll of the parse
struct DevTileParam {
  uint32_t npieces;
  uint32_t preroll;
};

// prologue shared by the kernel and its CPU replay: stage the descriptor and the table, reset the carry
template <int R>
__device__ __forceinline__ void tile_entry(TileShared<R>& sh, const uint8_t* __restrict__ in,
                                           uint64_t in_total, const DevScan* __restrict__ scans,
                                           const DevTable* __restrict__ tables,
                                           uint8_t* __restrict__ out,
                                           DevResult* __restrict__ results_all,
                                           const uint32_t* __restrict__ scan_ids,
                                           const DevTileParam* __restrict__ params,
                                           const uint32_t* __restrict__ redo = nullptr) {
  const int tid = threadIdx.x;
  // second opinion for the one-thread-per-segment path: only the segments it flagged (their last
  // symbols read behind the data, where the reference's refill cadence decides) are decoded again
  if (redo && !redo[blockIdx.x])
    return;
  // (bit 31 of an id is a flag of the thread path's list, see k2_stream_kernel)
  const uint32_t scan_idx = scan_ids ? (scan_ids[blockIdx.x] & 0x7FFFFFFFu) : blockIdx.x;
  DevResult* res = results_all + scan_idx;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&scans[scan_idx]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.sc);
    for (int i = tid; i < (int)(sizeof(DevScan) / 4); i += TL_NT)
      dst[i] = src[i];
  }
  __syncthreads();
  {
    const uint4* src = reinterpret_cast<const uint4*>(&tables[sh.sc.table_idx[0]]);
    uint4* dst = reinterpret_cast<uint4*>(&sh.tab);
    for (int i = tid; i < (int)(sizeof(DevTable) / 16); i += TL_NT)
      dst[i] = src[i];
  }
  __syncthreads();
  for (int i = tid; i < (1 << LUT_BITS); i += TL_NT)
    sh.len8[i] = (uint8_t)(sh.tab.lut[i] >> 10);
  if (tid == 0) {
    res->consumed = 0;
    sh.bad_code = 0;
    sh.rstat = 0;
    sh.rcons = 0;
    sh.last.seen = 0;
    sh.last.p_last = 0;
    mbar_init(&sh.bar, 1);
    fence_mbar_init();
    TileCarry c;
    c.pos = 0;
    c.sym = 0;
    c.tail_len = 0;
    c.tail_raw = (uint32_t)(sh.sc.in_offset & 15ull);
    c.ubytes = 0;
    c.prev_ff = 0;
    c.ended = 0;
    c.leftover = 0;
    c.left[0] = c.left[1] = c.left[2] = c.left[3] = 0;
    c.proc = 0;
    c.pc01 = c.pc23 = 0;
    c.col01 = (uint32_t)sh.sc.init_pred[0] | ((uint32_t)sh.sc.init_pred[1] << 16);
    c.col23 = (uint32_t)sh.sc.init_pred[2] | ((uint32_t)sh.sc.init_pred[3] << 16);
    c.rb01 = c.rb23 = 0;
    sh.cy = c;
  }
  __syncthreads();
  const DevTileParam pr = params[blockIdx.x];
  tile_body<R>(sh, in, in_total, out, res, pr.npieces, pr.preroll);
}

#ifndef RSB200_EMU
#ifndef RSB200_TILE_CTAS1
#define RSB200_TILE_CTAS1 4
#endif
template <int R>
__global__ void __launch_bounds__(TL_NT, (R == 1 ? RSB200_TILE_CTAS1 : 2))
    k2_tile_kernel(const uint8_t* __restrict__ in, uint64_t in_total,
                   const DevScan* __restrict__ scans, const DevTable* __restrict__ tables,
                   uint8_t* __restrict__ out, DevResult* __restrict__ results_all,
                   const uint32_t* __restrict__ scan_ids, const DevTileParam* __restrict__ params,
                   const uint32_t* __restrict__ redo) {
  extern __shared__ __align__(128) uint8_t tl_smem_raw[];
  TileShared<R>& sh = *reinterpret_cast<TileShared<R>*>(tl_smem_raw);
  tile_entry<R>(sh, in, in_total, scans, tables, out, results_all, scan_ids, params, redo);
}
#endif


#ifndef RSB200_EMU
// ------------------------------------------------------------------
// K2C2 `k2_clean2_kernel`: the unstuffing pre-pass of the one-thread-per-segment path (K2T,
// ljpeg_thread.cuh) built from this file's stage B: one CTA per segment, 64-byte pieces in
// registers, whole-word writes for the pieces without a stuffing byte.  Same outputs as
// k2_clean_kernel (ljpeg_clean.cuh): clean big-endian words, one anchor per 256 raw bytes, the
// clean length / marker flag -- at ~1/4 of its instructions per byte for DNG-size tiles.
// ------------------------------------------------------------------
__global__ void __launch_bounds__(TL_NT, 4)
    k2_clean2_kernel(const uint8_t* __restrict__ in, uint64_t in_total,
                     const DevScan* __restrict__ scans, const uint32_t* __restrict__ scan_ids,
                     uint32_t nids, const DevTScan* __restrict__ tscans,
                     uint32_t* __restrict__ clean, uint32_t* __restrict__ anchors,
                     DevTInfo* __restrict__ infos) {
  extern __shared__ __align__(128) uint8_t tl_smem_raw[];
  TileShared<1>& sh = *reinterpret_cast<TileShared<1>*>(tl_smem_raw);
  using G = TileGeom<1>;
  const int tid = threadIdx.x;
  const uint32_t id = blockIdx.x;
  if (id >= nids)
    return;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&scans[scan_ids[id]]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.sc);
    for (int i = tid; i < (int)(sizeof(DevScan) / 4); i += TL_NT)
      dst[i] = src[i];
  }
  if (tid == 0) {
    mbar_init(&sh.bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  const DevScan& sc = sh.sc;
  const DevTScan ts = tscans[id];
  const uint64_t abase = sc.in_offset & ~15ull;
  TileStream st;
  st.skew = (uint32_t)(sc.in_offset - abase);
  st.gbase = in + abase;
  st.limit = st.skew + sc.in_size;
  st.readable = ((in_total + 15) & ~15ull) - abase;
  st.npieces = (uint32_t)G::NPIECE & ~3u; // chunk bases are multiples of 256 raw bytes (anchors)
  st.chunk_raw = st.npieces * TL_PIECE;
  uint32_t* cw = clean + ts.clean_off;
  uint32_t* anc = anchors + ts.anchor_off;
  if (tid == 0)
    tl_issue_chunk<1>(sh, st, 0);
  TileCarry cy;
  cy.tail_len = 0;
  cy.prev_ff = 0;
  uint32_t emitted = 0; // clean bytes produced by the chunks so far
  uint32_t wout = 0;    // words written so far (emitted - 4 * wout bytes wait at the front of ub)
  const uint32_t sb_ub = smem_u32(sh.ub);
  TL_TICK_INIT;
  for (uint32_t chunk = 0;; ++chunk) {
    mbar_wait(&sh.bar, chunk & 1);
    const TileChunk co = tl_unstuff<1>(sh, st, cy, chunk TL_TICK_PASS);
    const uint32_t cbase = chunk * st.chunk_raw;
    // the staging is free again: fetch the next chunk while this one is written out
    const bool more = !co.final_chunk;
    if (more && tid == 0) {
      fence_proxy_async();
      tl_issue_chunk<1>(sh, st, chunk + 1);
    }
    // anchors: clean bytes in front of every 256-byte raw offset of this chunk
    for (uint32_t pi = 4u * (uint32_t)tid; pi < st.npieces; pi += 4u * TL_NT) {
      const uint32_t a = (cbase + pi * TL_PIECE) >> T_ANCHOR_SHIFT;
      if (a < ts.n_anchor)
        anc[a] = emitted + sh.anchor[pi] - cy.tail_len;
    }
    const uint32_t len = co.len; // carried bytes + this chunk's
    const uint32_t nw = co.final_chunk ? (len + 3u) / 4u + T_PAD_WORDS : len / 4u;
    if (co.final_chunk) { // zero words behind the data (tl_unstuff zeroed 64 bytes behind len)
      __syncthreads();
    }
    for (uint32_t w = tid; w < nw; w += TL_NT)
      if (wout + w < ts.cap_words)
        cw[wout + w] = lds_u32<0>(sb_ub + 4u * w);
    emitted += co.total_emit;
    if (co.final_chunk) {
      if (tid == 0) {
        infos[id].clean_len = emitted;
        infos[id].marker = co.mpos != TL_NOPOS ? 1u : 0u;
      }
      // the anchors behind the end of the data
      const uint32_t a0 = ((cbase + st.chunk_raw) >> T_ANCHOR_SHIFT);
      for (uint32_t a = a0 + tid; a < ts.n_anchor; a += TL_NT)
        anc[a] = emitted;
      break;
    }
    // the bytes of the last, incomplete word stay at the front of ub
    const uint32_t keep = len & 3u;
    uint32_t kb = 0;
    if ((uint32_t)tid < keep)
      kb = reinterpret_cast<uint8_t*>(sh.ub)[((len & ~3u) + tid) ^ 3u];
    __syncthreads();
    if ((uint32_t)tid < keep)
      reinterpret_cast<uint8_t*>(sh.ub)[tid ^ 3u] = (uint8_t)kb;
    wout += len / 4u;
    cy.tail_len = keep;
    cy.prev_ff = sh.prev_ff_next;
    __syncthreads();
  }
}
#endif

} // namespace rsb200
