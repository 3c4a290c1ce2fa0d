// ljpeg_fused.cuh -- K2F: fused LJPEG tile decode (entropy decode + predictor),
// one CTA per entropy-coded segment, streaming in 8 KiB chunks (sm_90a).
//
// Same semantics as k2_entropy_kernel + k3_* (see ljpeg.cuh for the reference
// citations) but nothing but the compressed bytes is read from HBM and nothing
// but final pixels is written:
//
//   A  each raw chunk is brought into shared memory by ONE bulk async copy (TMA
//      unit, cp.async.bulk / SASS UBLKCP) on an mbarrier; the copy of chunk c+1
//      is issued as soon as chunk c has been unstuffed, so it overlaps C-E;
//   B  the chunk is "unstuffed" cooperatively (FF00 -> FF, stop at the first
//      FFxx marker: BitStreamerJPEG.h:106-183) into a clean big-endian word
//      buffer, so the hot loops carry no stuffing/marker/bounds logic at all;
//   C  self-synchronising parallel Huffman decode over 32-byte subsequences of
//      the clean buffer (branch-free 2-word bit window, funnel shifts);
//   D  prefix sum of symbol counts, second decode pass writes the differences
//      to a shared-memory sample buffer in stream order;
//   E  predictor 1 as a per-component running sum mod 2^16 over the sample
//      buffer + a per-row additive constant that encodes "the first MCU of a
//      row is predicted from the first MCU of the previous row"
//      (LJpegDecompressor.cpp:200-219,326-332); pixels go out with 128-bit
//      stores.
#pragma once

#include "ljpeg.cuh"

namespace rsb200 {

constexpr int F_NT = 256;
constexpr int F_SUB = 32;            // subsequence size (bytes of clean data)
constexpr int F_RAW = F_NT * F_SUB;  // raw bytes consumed per chunk
constexpr int F_WIN = F_RAW + 16;    // staged window (1 look-ahead byte needed)
constexpr int F_LA = 8;              // clean bytes deferred to the next chunk
constexpr int F_DCAP = 8192;         // samples per predictor batch
constexpr int F_RBMAX = 256;         // row starts per batch handled in one go

struct FusedCarry {
  uint32_t pos;        // bit position (relative to ub[0]) of the next symbol
  uint32_t sym;        // symbols decoded so far (global index of the next one)
  uint32_t tail_len;   // clean bytes carried at the front of ub
  uint32_t tail_raw;   // raw offset (from the 16-byte aligned base) of ub byte 0
  uint32_t ubytes;     // clean bytes that precede ub[0] in the segment
  uint32_t prev_ff;    // last raw byte of the previous chunk was FF
  uint32_t ended;      // marker seen or end of buffer reached
  uint32_t leftover;   // samples (< group) waiting at the front of dbuf
  uint32_t proc;       // samples already run through the predictor
  uint32_t status;
  uint32_t pc01, pc23;     // plain per-component prefix carried (4 x 16 bit)
  uint32_t col01, col23;   // value of the first MCU of the previous row
  uint32_t rb01, rb23;     // additive constant of the row in progress
};

struct FusedShared {
  DevScan sc;
  FusedCarry cy;
  alignas(8) uint64_t bar;
  alignas(16) uint32_t raw[F_WIN / 4];
  alignas(16) uint32_t ub[(F_RAW + 64) / 4];
  alignas(16) uint16_t dbuf[F_DCAP + 32];
  uint32_t exitpos[F_NT];
  uint32_t exitph[F_NT];
  uint32_t anchor[F_NT + 1];
  uint32_t warp_tmp[4][F_NT / 32];
  uint32_t rowbase[F_RBMAX + 1][2];
  uint32_t mpos;
  uint32_t last_raw_byte;
  uint32_t bad_code;    // set by the difference decode when a needed code is not in the table
  uint32_t lutaddr[12]; // shared address of the LUT used at each position of a group
  DevTable tab[4]; // only the first `ntab` are staged / allocated
};

__host__ __device__ inline size_t fused_smem_bytes(int ntab) {
  return sizeof(FusedShared) - sizeof(DevTable) * (size_t)(4 - ntab);
}

// 4-bit mask of the bytes of w equal to 0xFF / 0x00
__device__ __forceinline__ uint32_t byte_eq_mask(uint32_t w, uint32_t pat) {
  const uint32_t eq = __vcmpeq4(w, pat);
  return ((eq >> 7) & 1u) | ((eq >> 14) & 2u) | ((eq >> 21) & 4u) | ((eq >> 28) & 8u);
}

__device__ __forceinline__ uint32_t f_block_scan(uint32_t v, uint32_t* tmp, uint32_t* total) {
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
  for (int i = 0; i < F_NT / 32; ++i) {
    const uint32_t x = tmp[i];
    add += (i < wid) ? x : 0u;
    tot += x;
  }
  *total = tot;
  return v + add;
}

// inclusive block scan of two packed 2x16-bit lanes (mod 2^16 per lane)
__device__ __forceinline__ void f_block_scan_v2(uint32_t& a, uint32_t& b, uint32_t* tmpa,
                                                uint32_t* tmpb, uint32_t& tota,
                                                uint32_t& totb) {
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
  for (int i = 0; i < F_NT / 32; ++i) {
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

// Optional per-phase cycle accounting (profiling builds only: -DRSB200_PHASE_TIMING).
#ifdef RSB200_PHASE_TIMING
__device__ unsigned long long g_phase_cycles[16];
#define F_TICK(i)                                                                  \
  do {                                                                             \
    if (threadIdx.x == 0) {                                                        \
      const long long t_now = clock64();                                           \
      atomicAdd(&g_phase_cycles[i], (unsigned long long)(t_now - t_phase));        \
      t_phase = t_now;                                                             \
    }                                                                              \
  } while (0)
#else
#define F_TICK(i) do { } while (0)
#endif

struct FSub {
  uint32_t exitpos;
  uint32_t count;
};

// slow path of a symbol: code longer than the LUT depth, or corrupt
__device__ __noinline__ uint32_t f_long_symbol(const DevTable* t, uint32_t x) {
  return (uint32_t)decode_sym(t, x).total;
}

// ---- hot-loop view of the clean buffer and the LUTs ----
// `sb` = smem_base_opaque(&sh).  Every access is "register + constant":
constexpr int FO_UB = (int)offsetof(FusedShared, ub);
constexpr int FO_DBUF = (int)offsetof(FusedShared, dbuf);
constexpr int FO_LUTADDR = (int)offsetof(FusedShared, lutaddr);
constexpr int FO_LUT0 = (int)(offsetof(FusedShared, tab) + offsetof(DevTable, lut));
constexpr uint32_t F_LUT_TOPMASK = ~((1u << (32 - LUT_BITS)) - 1u); // top LUT_BITS bits of the window

struct FBits {
  uint32_t p;        // bit position in ub
  uint32_t cur, nxt; // words p/32 and p/32+1
  __device__ __forceinline__ void open(uint32_t sb, uint32_t start) {
    p = start;
    const uint32_t wa = sb + ((start >> 3) & ~3u);
    cur = lds_u32<FO_UB>(wa);
    nxt = lds_u32<FO_UB + 4>(wa);
  }
  // the next 32 bits of the stream
  __device__ __forceinline__ uint32_t peek() const { return __funnelshift_l(nxt, cur, p); }
  __device__ __forceinline__ void skip(uint32_t sb, uint32_t n) {
    const uint32_t pn = p + n;
    if ((pn ^ p) & ~31u) { // crossed into the next word (n <= 32)
      cur = nxt;
      nxt = lds_u32<FO_UB + 4>(mad_hi(pn & ~31u, 1u << 29, sb)); // sb + 4*(pn/32)
    }
    p = pn;
  }
};

// LUT entry of the code at the top of window x.  lutbase: MULTI -> absolute
// shared address of the LUT of this position in the group; else unused.
template <bool MULTI>
__device__ __forceinline__ uint32_t f_lut_entry(uint32_t sb, uint32_t lutbase, uint32_t x) {
  // base + 2*(x >> (32-LUT_BITS)), the shift done by IMAD.HI
  if (MULTI)
    return lds_u16<0>(mad_hi(x & F_LUT_TOPMASK, 1u << (LUT_BITS + 1), lutbase));
  return lds_u16<FO_LUT0>(mad_hi(x & F_LUT_TOPMASK, 1u << (LUT_BITS + 1), sb));
}

// One difference: Huffman code + SSSS mantissa bits at the top of window x
// (PrefixCodeLUTDecoder.h:172-216 + AbstractPrefixCodeDecoder.h:43-76).
// Returns the difference mod 2^16 in the low half; tl = bits consumed.
template <bool MULTI>
__device__ __forceinline__ uint32_t f_decode_diff(FusedShared& sh, uint32_t sb,
                                                  uint32_t lutbase, uint32_t phase, uint32_t x,
                                                  uint32_t& tl) {
  const uint32_t e = f_lut_entry<MULTI>(sb, lutbase, x);
  tl = e >> 10;
  if (e == 0) { // code longer than the LUT, SSSS = 16, or corrupt
    const SymLen s = decode_sym(MULTI ? &sh.tab[sh.sc.table_of[phase]] : &sh.tab[0], x);
    tl = s.total;
    if (s.codelen == 0)
      sh.bad_code = 1u; // "bad Huffman code" (kept out of the registers of the hot loop)
    return (uint32_t)sym_diff(s, x);
  }
  // extend(), branch free.  tt = bits after the code; f = all ones iff their
  // first bit is 0 (negative range); (f:tt) << ssss leaves v with ones above it in
  // that case, and v - (2^ssss - 1) == (v | ~mask) + 1.  Funnel shifts wrap at 32,
  // so the code-length / SSSS fields of e are used unmasked.
  const uint32_t tt = __funnelshift_l(0u, x, e);
  const uint32_t f = (uint32_t)((int32_t)~tt >> 31);
  return __funnelshift_l(tt, f, e >> 5) - f;
}

// lengths-only decode of one subsequence of the clean buffer
template <bool MULTI>
__device__ __forceinline__ FSub f_scan_sub(const FusedShared& sh, uint32_t sb, uint32_t start,
                                           uint32_t end_bit, uint32_t phase) {
  FSub r;
  if (start >= end_bit) {
    r.exitpos = start;
    r.count = 0;
    return r;
  }
  FBits b;
  b.open(sb, start);
  uint32_t cnt = 0, lutbase = 0;
  const uint32_t G = sh.sc.group;
  do {
    const uint32_t x = b.peek();
    if (MULTI)
      lutbase = lds_u32<FO_LUTADDR>(sb + 4 * phase);
    uint32_t len = f_lut_entry<MULTI>(sb, lutbase, x) >> 10;
    if (len == 0) // long code, SSSS = 16, or invalid code (rare)
      len = f_long_symbol(MULTI ? &sh.tab[sh.sc.table_of[phase]] : &sh.tab[0], x);
    ++cnt;
    if (MULTI)
      phase = (phase + 1 == G) ? 0 : phase + 1;
    b.skip(sb, len);
  } while (b.p < end_bit);
  r.exitpos = b.p;
  r.count = cnt;
  return r;
}

__device__ __forceinline__ uint32_t f_raw_byte(const uint8_t* gbase, uint32_t limit,
                                               uint32_t p) {
  return p < limit ? (uint32_t)gbase[p] : 0u;
}

// BitStreamerJPEG::getStreamPosition() of the reference after the last symbol
// (refill cadence of BitStreamer.h:216-229, BitStreamerJPEG.h:106-189; see
// DESIGN.md "consumed").  p = bit position of the last symbol in ub.
__device__ __noinline__ uint32_t f_stream_position(const FusedShared& sh, const FusedCarry& cy,
                                                   const uint8_t* gbase, uint32_t limit,
                                                   uint32_t skew, uint32_t chunk, uint32_t p,
                                                   bool* overrun) {
  const uint32_t ub_byte = p >> 3;
  uint32_t rawp, cleanp;
  if (ub_byte < cy.tail_len) {
    rawp = cy.tail_raw;
    cleanp = 0;
  } else {
    int a = 0, b = F_NT - 1;
    while (a < b) {
      const int m = (a + b + 1) >> 1;
      if (sh.anchor[m] <= ub_byte)
        a = m;
      else
        b = m - 1;
    }
    rawp = chunk * F_RAW + a * F_SUB;
    cleanp = sh.anchor[a];
    if (rawp < skew)
      rawp = skew;
    // a stuffing byte may sit exactly at rawp (its FF ended the previous range)
    if (rawp > skew && f_raw_byte(gbase, limit, rawp - 1) == 0xFFu &&
        f_raw_byte(gbase, limit, rawp) == 0u)
      rawp += 1;
  }
  bool marker = false;
  auto step = [&](uint32_t& rp) {
    const uint32_t c0 = f_raw_byte(gbase, limit, rp);
    if (c0 == 0xFFu) {
      if (f_raw_byte(gbase, limit, rp + 1) != 0u) {
        marker = true;
        return;
      }
      rp += 2;
    } else
      rp += 1;
  };
  while (cleanp < ub_byte && !marker) {
    step(rawp);
    ++cleanp;
  }
  const uint64_t U = (uint64_t)cy.ubytes + ub_byte;
  const uint64_t T = 8ull * U + (p & 7u);
  const uint64_t q = T >> 5;
  const uint64_t R = (T & 31u) ? q + 2 : q + 1;
  uint64_t need = 4ull * R - U;
  while (need > 0 && !marker) {
    step(rawp);
    --need;
  }
  *overrun = !marker && rawp > limit + 20u;
  return rawp - skew;
}

// ---------------- E1: plain per-component running sums, in place ----------------
template <int G>
__device__ __forceinline__ void f_prefix_vec(FusedShared& sh, uint32_t doff, uint32_t n,
                                             uint32_t pc01, uint32_t pc23, uint32_t& ta,
                                             uint32_t& tb) {
  // physical range [doff, doff+n) of dbuf; vector v covers physical [8v, 8v+8)
  const int tid = threadIdx.x;
  const uint32_t total_phys = doff + n;
  const uint32_t nvec = (total_phys + 7) >> 3;
  const uint32_t vpt = (nvec + F_NT - 1) / F_NT;
  const uint32_t v0 = tid * vpt, v1 = min(v0 + vpt, nvec);
  uint4* vec = reinterpret_cast<uint4*>(sh.dbuf);
  auto elem_mask = [&](uint32_t v, uint32_t (&m)[4]) {
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const uint32_t e0 = 8 * v + 2 * w, e1 = e0 + 1;
      m[w] = ((e0 >= doff && e0 < total_phys) ? 0x0000FFFFu : 0u) |
             ((e1 >= doff && e1 < total_phys) ? 0xFFFF0000u : 0u);
    }
  };
  uint32_t s01 = 0, s23 = 0;
  for (uint32_t v = v0; v < v1; ++v) {
    uint4 q = vec[v];
    if (v == 0 || v + 1 == nvec) {
      uint32_t m[4];
      elem_mask(v, m);
      q.x &= m[0]; q.y &= m[1]; q.z &= m[2]; q.w &= m[3];
    }
    if (G == 2) {
      s01 = __vadd2(s01, __vadd2(__vadd2(q.x, q.y), __vadd2(q.z, q.w)));
    } else if (G == 4) {
      s01 = __vadd2(s01, __vadd2(q.x, q.z));
      s23 = __vadd2(s23, __vadd2(q.y, q.w));
    } else { // G == 1
      const uint32_t t = __vadd2(__vadd2(q.x, q.y), __vadd2(q.z, q.w));
      s01 = (s01 + (t & 0xFFFFu) + (t >> 16)) & 0xFFFFu;
    }
  }
  uint32_t a = s01, b = s23;
  f_block_scan_v2(a, b, sh.warp_tmp[0], sh.warp_tmp[1], ta, tb);
  uint32_t r01 = __vadd2(__vsub2(a, s01), pc01);
  uint32_t r23 = __vadd2(__vsub2(b, s23), pc23);
  for (uint32_t v = v0; v < v1; ++v) {
    const uint4 orig = vec[v];
    uint4 q = orig;
    uint32_t m[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
    const bool edge = (v == 0 || v + 1 == nvec);
    if (edge) {
      elem_mask(v, m);
      q.x &= m[0]; q.y &= m[1]; q.z &= m[2]; q.w &= m[3];
    }
    uint4 o;
    if (G == 2) {
      r01 = __vadd2(r01, q.x); o.x = r01;
      r01 = __vadd2(r01, q.y); o.y = r01;
      r01 = __vadd2(r01, q.z); o.z = r01;
      r01 = __vadd2(r01, q.w); o.w = r01;
    } else if (G == 4) {
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
    if (edge) {
      o.x = (o.x & m[0]) | (orig.x & ~m[0]);
      o.y = (o.y & m[1]) | (orig.y & ~m[1]);
      o.z = (o.z & m[2]) | (orig.z & ~m[2]);
      o.w = (o.w & m[3]) | (orig.w & ~m[3]);
    }
    vec[v] = o;
  }
}

// generic (any group size) scalar variant
__device__ __forceinline__ void f_prefix_scalar(FusedShared& sh, uint16_t* DB, uint32_t S0,
                                                uint32_t n, uint32_t G, uint32_t pc01,
                                                uint32_t pc23, uint32_t& ta, uint32_t& tb) {
  const int tid = threadIdx.x;
  const uint32_t per = (n + F_NT - 1) / F_NT;
  const uint32_t i0 = tid * per, i1 = min(i0 + per, n);
  uint32_t s01 = 0, s23 = 0;
  uint32_t c = (S0 + i0) % G;
  for (uint32_t i = i0; i < i1; ++i) {
    const uint32_t v = DB[i];
    if (c == 0) s01 = __vadd2(s01, v);
    else if (c == 1) s01 = __vadd2(s01, v << 16);
    else if (c == 2) s23 = __vadd2(s23, v);
    else s23 = __vadd2(s23, v << 16);
    c = (c + 1 == G) ? 0 : c + 1;
  }
  uint32_t a = s01, b = s23;
  f_block_scan_v2(a, b, sh.warp_tmp[0], sh.warp_tmp[1], ta, tb);
  uint32_t r01 = __vadd2(__vsub2(a, s01), pc01);
  uint32_t r23 = __vadd2(__vsub2(b, s23), pc23);
  c = (S0 + i0) % G;
  for (uint32_t i = i0; i < i1; ++i) {
    const uint32_t v = DB[i];
    uint32_t o;
    if (c == 0) { r01 = __vadd2(r01, v); o = r01 & 0xFFFFu; }
    else if (c == 1) { r01 = __vadd2(r01, v << 16); o = r01 >> 16; }
    else if (c == 2) { r23 = __vadd2(r23, v); o = r23 & 0xFFFFu; }
    else { r23 = __vadd2(r23, v << 16); o = r23 >> 16; }
    DB[i] = (uint16_t)o;
    c = (c + 1 == G) ? 0 : c + 1;
  }
}

// fast (row, column) of a global sample index
__device__ __forceinline__ void f_row_col(uint32_t g, uint32_t RS, uint32_t inv, uint32_t& r,
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

// per-CTA description of the byte range being decoded + TMA pipeline state
struct FStream {
  const uint8_t* gbase; // 16-byte aligned base of the segment window
  uint32_t limit;       // valid raw bytes from gbase (this CTA never looks further)
  uint32_t skew;        // offset of the first entropy-coded byte from gbase
  uint64_t readable;    // bytes that may be touched by the bulk copies
  uint32_t chunk_begin; // first chunk this CTA processes
  uint32_t chunk_end;   // one past the last chunk that may be prefetched
  bool plain;           // plain MSB bit source: no FF00 stuffing, no end marker
  bool pending;         // a bulk copy is in flight (uniform)
  uint32_t pending_par; // ... and completes the mbarrier phase of this parity
};

struct FChunk {
  uint32_t len;        // clean bytes in ub (carried tail + this chunk)
  uint32_t Lc;         // clean bytes decodable in this chunk
  uint32_t end_all;    // Lc * 8
  uint32_t mpos;       // chunk-relative raw offset of the end marker (or ~0)
  uint32_t total_emit; // clean bytes produced by this chunk
  bool final_chunk;
};

__device__ __forceinline__ void f_issue_chunk(FusedShared& sh, const FStream& st, uint32_t chunk) {
  // window [chunk*F_RAW, +F_WIN) clamped to the readable (16-byte padded) buffer
  const uint64_t g0 = (uint64_t)chunk * F_RAW;
  uint32_t n = 0;
  if (g0 < st.readable)
    n = (uint32_t)min((uint64_t)F_WIN, st.readable - g0);
  mbar_expect_tx(&sh.bar, n);
  if (n)
    bulk_g2s(sh.raw, st.gbase + g0, n, &sh.bar);
}

// ================= B: unstuff one raw chunk into sh.ub =================
__device__ __forceinline__ FChunk f_unstuff(FusedShared& sh, FStream& st, const FusedCarry& cy,
                                            uint32_t chunk) {
  const int tid = threadIdx.x;
  FChunk co;
    const uint32_t* rw = sh.raw;
    const uint32_t raw0 = chunk * F_RAW + tid * F_SUB; // raw offset of my first byte
    uint32_t w[8];
    uint32_t ffm = 0;
    {
      const uint4 q0 = reinterpret_cast<const uint4*>(rw)[tid * 2];
      const uint4 q1 = reinterpret_cast<const uint4*>(rw)[tid * 2 + 1];
      w[0] = q0.x; w[1] = q0.y; w[2] = q0.z; w[3] = q0.w;
      w[4] = q1.x; w[5] = q1.y; w[6] = q1.z; w[7] = q1.w;
    }
    if (raw0 + 32 > st.limit) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint32_t b = raw0 + 4 * k;
        if (b + 4 > st.limit)
          w[k] = b >= st.limit ? 0u : (w[k] & (0xFFFFFFFFu >> (32 - 8 * (st.limit - b))));
      }
    }
    if (!st.plain) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (__vcmpeq4(w[k], 0xFFFFFFFFu))
          ffm |= byte_eq_mask(w[k], 0xFFFFFFFFu) << (4 * k);
    }
    // bytes that belong to the segment: [st.skew, st.limit)
    uint32_t valid = 0xFFFFFFFFu;
    if (raw0 < st.skew)
      valid = (st.skew - raw0 >= 32) ? 0u : (0xFFFFFFFFu << (st.skew - raw0));
    if (raw0 + 32 > st.limit)
      valid &= (raw0 >= st.limit) ? 0u : (0xFFFFFFFFu >> (32 - (st.limit - raw0)));
    ffm &= valid;
    uint32_t prev_ff;
    if (tid == 0)
      prev_ff = cy.prev_ff;
    else
      prev_ff = ((rw[tid * 8 - 1] >> 24) == 0xFFu) && (raw0 - 1 >= st.skew) && (raw0 - 1 < st.limit);
    if (st.plain)
      prev_ff = 0;
    uint32_t stuff = 0, mk = 0;
    if (ffm | prev_ff) {
      uint32_t zm = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        zm |= byte_eq_mask(w[k], 0u) << (4 * k);
      uint32_t nb = rw[tid * 8 + 8] & 0xFFu; // first byte after my range
      if (raw0 + 32 >= st.limit)
        nb = 0; // past the end bytes read as zero -> FF is followed by "00"
      stuff = zm & ((ffm << 1) | prev_ff) & valid;
      mk = ffm & ~((zm >> 1) | ((nb == 0u ? 1u : 0u) << 31));
    }
    if (tid == 0)
      sh.mpos = 0xFFFFFFFFu;
    if (tid == F_NT - 1)
      sh.last_raw_byte = w[7] >> 24;
    const int any_mk = __syncthreads_or(mk != 0u);
    if (any_mk) {
      if (mk)
        atomicMin(&sh.mpos, (uint32_t)(tid * F_SUB + __ffs(mk) - 1));
      __syncthreads();
    }
    const uint32_t mpos = any_mk ? sh.mpos : 0xFFFFFFFFu; // chunk relative
    uint32_t emit = valid & ~stuff;
    if (mpos != 0xFFFFFFFFu) {
      const uint32_t my0 = tid * F_SUB;
      if (mpos <= my0)
        emit = 0;
      else if (mpos < my0 + 32)
        emit &= (1u << (mpos - my0)) - 1u;
    }
    const uint32_t n_emit = __popc(emit);
    uint32_t total_emit;
    const uint32_t incl = f_block_scan(n_emit, sh.warp_tmp[0], &total_emit);
    // (the scan's barrier also means every thread has read its raw words: the
    //  staging buffer is free -> prefetch the next chunk now, overlapping C-E)
    const bool final_chunk = (mpos != 0xFFFFFFFFu) || ((chunk + 1) * (uint32_t)F_RAW >= st.limit);
    if (!final_chunk && chunk + 1 < st.chunk_end) {
      if (tid == 0)
        f_issue_chunk(sh, st, chunk + 1);
      st.pending = true;
      st.pending_par = (chunk + 1 - st.chunk_begin) & 1u;
    }
    const uint32_t dst0 = cy.tail_len + incl - n_emit; // clean byte index in ub
    sh.anchor[tid] = dst0;
    {
      uint8_t* ub8 = reinterpret_cast<uint8_t*>(sh.ub);
      if (emit == 0xFFFFFFFFu) {
        // fast path: 32 clean bytes; interior as whole big-endian words
        const uint32_t head = (4u - (dst0 & 3u)) & 3u;
#pragma unroll
        for (int k = 0; k < 3; ++k)
          if ((uint32_t)k < head)
            ub8[(dst0 + k) ^ 3u] = (uint8_t)(w[0] >> (8 * k));
        const uint32_t sh8 = head * 8;
        const uint32_t wbase = (dst0 + head) >> 2;
#pragma unroll
        for (int k = 0; k < 7; ++k) {
          const uint32_t le = __funnelshift_r(w[k], w[k + 1], sh8);
          sh.ub[wbase + k] = __byte_perm(le, 0, 0x0123);
        }
        if (head == 0) {
          sh.ub[wbase + 7] = __byte_perm(w[7], 0, 0x0123);
        } else {
#pragma unroll
          for (int k = 1; k < 4; ++k)
            if ((uint32_t)k >= head)
              ub8[(dst0 + 28 + k) ^ 3u] = (uint8_t)(w[7] >> (8 * k));
        }
      } else if (emit) {
        // general path: word by word, bytes of a word that survive go out one by one
        uint32_t d = dst0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t e4 = (emit >> (4 * k)) & 0xFu;
          if (e4 == 0xFu) {
#pragma unroll
            for (int b = 0; b < 4; ++b)
              ub8[(d + b) ^ 3u] = (uint8_t)(w[k] >> (8 * b));
            d += 4;
          } else if (e4) {
#pragma unroll
            for (int b = 0; b < 4; ++b)
              if ((e4 >> b) & 1u) {
                ub8[d ^ 3u] = (uint8_t)(w[k] >> (8 * b));
                ++d;
              }
          }
        }
      }
    }
    co.len = cy.tail_len + total_emit; // clean bytes now in ub
    const uint32_t len = co.len;
    __syncthreads();
    // zero padding behind the data (read by look-ahead loads / after the end)
    if (tid < 16)
      reinterpret_cast<uint8_t*>(sh.ub)[(len + tid) ^ 3u] = 0;
    if (tid >= 32 && tid < 40) {
      const uint32_t wz = ((len + 16) >> 2) + 1 + (tid - 32);
      if (wz < (F_RAW + 64) / 4)
        sh.ub[wz] = 0;
    }
    co.Lc = final_chunk ? len : (len > F_LA ? len - F_LA : 0u); // decodable bytes
    co.end_all = co.Lc * 8;
    co.mpos = mpos;
    co.total_emit = total_emit;
    co.final_chunk = final_chunk;
    __syncthreads();
    return co;

}

struct FSync {
  uint32_t my_start, my_phase;
  FSub d;
};

// ================= C: self-synchronising decode of the chunk in sh.ub =================
// Sony ARW1 (arw1.cuh): a zero difference is the complemented code 100.  A parse that starts on
// the wrong residue inside a run of them reads 001 (length 1) forever and never resynchronises, so
// speculative starts inside such a run are moved to its phase (f_sync's arw1_align): the offset 0..2 at which the 32
// bits of x0:x1 are 100 repeated, else 0.
__device__ __forceinline__ uint32_t arw1_run_phase(uint32_t x0, uint32_t x1) {
  for (uint32_t o = 0; o < 3; ++o)
    if (__funnelshift_l(x1, x0, o) == 0x92492492u)
      return o;
  return 0;
}

template <bool MULTI>
__device__ __forceinline__ FSync f_sync(FusedShared& sh, uint32_t sb, const FusedCarry& cy,
                                        const FChunk& co, uint32_t G, uint32_t arw1_align = 0) {
  const int tid = threadIdx.x;
    const uint32_t sub_lo = tid * F_SUB * 8u;
    // the last thread also takes every symbol that starts behind the F_NT subsequences: a final
    // chunk holds up to F_LA + F_RAW clean bytes (carried tail + chunk), and the range kernels parse
    // a plain segment's final chunk a further 8 bytes into the zero bits
    const uint32_t sub_hi = tid == F_NT - 1 ? co.end_all : min(sub_lo + F_SUB * 8u, co.end_all);
    const bool active = sub_lo < co.end_all;
    uint32_t my_start = (tid == 0) ? cy.pos : sub_lo;
    uint32_t my_phase = (tid == 0) ? (cy.sym % G) : 0u;
    // arw1_align: 1 = the guesses of threads 1.., 2 = thread 0's start too (a range's halo chunk);
    // they stay guesses: the fixed point below is exact
    // (Samsung V1, DevScan::kind 5: the same with samsung1_run_phase, ljpeg_types.h)
    if (arw1_align > (tid == 0 ? 1u : 0u) && active) // (thread 0: cy.pos == sub_lo == 0 then)
      my_start += sh.sc.kind == 5 ? samsung1_run_phase(sh.ub[sub_lo >> 5], sh.ub[(sub_lo >> 5) + 1])
                                  : arw1_run_phase(sh.ub[sub_lo >> 5], sh.ub[(sub_lo >> 5) + 1]);
    const uint32_t start0 = my_start; // thread 0's start (cy.pos unless aligned)
    if (!active)
      my_start = 0xFFFFFFF0u;
    FSub d;
    d.exitpos = my_start;
    d.count = 0;
    if (active)
      d = f_scan_sub<MULTI>(sh, sb, my_start, sub_hi, my_phase);
    sh.exitpos[tid] = d.exitpos;
    if (MULTI)
      sh.exitph[tid] = (my_phase + d.count) % G;
    __syncthreads();
    // Fixed-point iteration: adopt the predecessor's exit state until nothing
    // changes (thread 0 is exact => the fixed point is the sequential parse).
    // With several tables the phase travels with the position hop by hop; once
    // positions are stable the phases come from a prefix sum of the counts.
    for (int round = 0; round < F_NT + 2; ++round) {
      uint32_t new_start = (tid == 0) ? start0 : sh.exitpos[tid - 1];
      uint32_t new_phase = my_phase;
      if (MULTI)
        new_phase = (tid == 0) ? (cy.sym % G) : sh.exitph[tid - 1];
      const bool pos_changed = active && new_start != my_start;
      const int any_pos = __syncthreads_or(pos_changed ? 1 : 0);
      if (MULTI && !any_pos) {
        uint32_t tot;
        const uint32_t inc = f_block_scan(d.count, sh.warp_tmp[1 + (round & 1)], &tot);
        new_phase = (cy.sym + inc - d.count) % G;
      }
      const bool changed = active && (pos_changed || (MULTI && new_phase != my_phase));
      int any = any_pos;
      if (MULTI)
        any = __syncthreads_or(changed ? 1 : 0);
      if (!any)
        break;
      if (changed) {
        my_start = new_start;
        my_phase = new_phase;
        d = f_scan_sub<MULTI>(sh, sb, my_start, sub_hi, my_phase);
      }
      sh.exitpos[tid] = d.exitpos; // (reads of exitpos[tid-1] precede the vote barrier)
      if (MULTI)
        sh.exitph[tid] = (my_phase + d.count) % G;
      __syncthreads();
    }

    FSync so;
    so.my_start = my_start;
    so.my_phase = my_phase;
    so.d = d;
    return so;
}

template <bool MULTI>
__device__ __forceinline__ void
fused_body(FusedShared& sh, const uint8_t* __restrict__ in, uint64_t in_total,
           const DevTable* __restrict__ tables, uint8_t* __restrict__ out,
           DevResult* __restrict__ results) {
  const int tid = threadIdx.x;
  const DevScan& sc = sh.sc;
  const uint64_t abase = sc.in_offset & ~15ull;
  const uint32_t skew = (uint32_t)(sc.in_offset - abase);
  const uint8_t* gbase = in + abase;
  const uint32_t limit = skew + sc.in_size; // valid raw bytes from gbase
  const uint64_t readable = ((in_total + 15) & ~15ull) - abase;
  const uint32_t G = sc.group;
  const uint32_t RS = sc.row_samples;
  const uint32_t sb = smem_base_opaque(&sh); // shared address of sh, for the hot loops
  const uint32_t nchunks_max = (limit + F_RAW - 1) / F_RAW;

  FStream st;
  st.gbase = gbase;
  st.limit = limit;
  st.skew = skew;
  st.readable = readable;
  st.chunk_begin = 0;
  st.chunk_end = nchunks_max;
  st.plain = sc.pump != 0;
  st.pending = true;
  st.pending_par = 0;
  if (tid == 0)
    f_issue_chunk(sh, st, 0);
  uint32_t my_status = 0;
#ifdef RSB200_PHASE_TIMING
  long long t_phase = clock64();
#endif

  for (uint32_t chunk = 0;; ++chunk) {
    const FusedCarry cy = sh.cy;
    if (cy.sym >= sc.n_samples)
      break;
    if (cy.ended) {
      my_status |= 2u; // data exhausted but samples are still missing
      break;
    }
    mbar_wait(&sh.bar, chunk & 1);
    st.pending = false;
    F_TICK(0);

    // ================= B: unstuff =================
    const FChunk co = f_unstuff(sh, st, cy, chunk);
    const uint32_t len = co.len, Lc = co.Lc, end_all = co.end_all, mpos = co.mpos;
    const uint32_t total_emit = co.total_emit;
    const bool final_chunk = co.final_chunk;
    F_TICK(1);

    // ================= C: self-synchronising decode =================
    const FSync so = f_sync<MULTI>(sh, sb, cy, co, G);
    const uint32_t my_start = so.my_start;
    const FSub d = so.d;
    F_TICK(2);

    // ================= D: symbol indices =================
    uint32_t total_syms;
    const uint32_t sincl = f_block_scan(d.count, sh.warp_tmp[3], &total_syms);
    const uint32_t sym0 = cy.sym + sincl - d.count; // global index of my first symbol
    const uint32_t chunk_syms = min(total_syms, sc.n_samples - cy.sym);
    const uint32_t nsub = min((end_all + F_SUB * 8u - 1) / (F_SUB * 8u), (uint32_t)F_NT);
    const uint32_t exit_all = nsub ? sh.exitpos[nsub - 1] : cy.pos;
    const uint32_t rel0 = sym0 - cy.sym;                     // chunk-relative index of my first symbol
    const uint32_t klast = sc.n_samples - 1 - cy.sym;        // chunk-relative index of the last needed one

    // batches over the chunk's symbols (one batch unless the data is < ~1 byte/sample)
    uint32_t done = 0;
    while (true) {
      const FusedCarry cb = sh.cy; // leftover/proc/prefix state (updated per batch)
      // a batch holds at most F_DCAP samples and at most F_RBMAX-1 row starts
      const uint32_t cap = min((uint32_t)F_DCAP, (uint32_t)(F_RBMAX - 1) * RS);
      const uint32_t room = cap - cb.leftover;
      const uint32_t take = min(room, chunk_syms - done);
      // dbuf is indexed so that (physical index) == (global sample index) mod 8:
      // the 128-bit units of steps E1/E3 are then 16-byte aligned in shared memory
      const uint32_t doff = cb.proc & 7u;
      uint16_t* const DB = sh.dbuf + doff;
      if (tid < 8 && (uint32_t)tid < doff)
        sh.dbuf[tid] = 0;
      // ---- decode + store differences of symbols [done, done+take) ----
      if (d.count) {
        const uint32_t lo = max(rel0, done), hi = min(rel0 + d.count, done + take);
        if (lo < hi) {
          FBits b;
          b.open(sb, my_start);
          uint32_t phase = MULTI ? (sym0 % G) : 0u;
          uint32_t lutbase = 0;
          // symbols of earlier batches: lengths only
          for (uint32_t k = rel0; k < lo; ++k) {
            const uint32_t x = b.peek();
            if (MULTI)
              lutbase = lds_u32<FO_LUTADDR>(sb + 4 * phase);
            uint32_t tl = f_lut_entry<MULTI>(sb, lutbase, x) >> 10;
            if (tl == 0)
              tl = f_long_symbol(MULTI ? &sh.tab[sc.table_of[phase]] : &sh.tab[0], x);
            if (MULTI)
              phase = (phase + 1 == G) ? 0 : phase + 1;
            b.skip(sb, tl);
          }
          // dst walks dbuf; the segment's last symbol (its position feeds
          // `consumed`) splits the walk in two so the loop body stays free of it
          uint32_t dst = sb + 2u * (doff + cb.leftover + (lo - done));
          const uint32_t dst_end = dst + 2u * (hi - lo);
          const uint32_t pl_k = klast; // chunk-relative index of the segment's last symbol
          uint32_t stop = (pl_k >= lo && pl_k < hi) ? dst + 2u * (pl_k - lo) : dst_end;
          uint32_t plast = 0xFFFFFFFFu;
          for (;;) {
            while (dst != stop) {
              const uint32_t x = b.peek();
              if (MULTI)
                lutbase = lds_u32<FO_LUTADDR>(sb + 4 * phase);
              uint32_t tl;
              const uint32_t diff = f_decode_diff<MULTI>(sh, sb, lutbase, phase, x, tl);
              sts_u16<FO_DBUF>(dst, diff);
              dst += 2;
              if (MULTI)
                phase = (phase + 1 == G) ? 0 : phase + 1;
              b.skip(sb, tl);
            }
            if (stop == dst_end)
              break;
            plast = b.p;
            stop = dst_end;
          }
          const uint32_t p = b.p;
          if (final_chunk && p > len * 8u)
            my_status |= 2u; // a needed symbol runs past the end of the data
          if (plast != 0xFFFFFFFFu && !st.plain) {
            bool ovr = false;
            results[blockIdx.x].consumed =
                f_stream_position(sh, cy, gbase, limit, skew, chunk, plast, &ovr);
            if (ovr)
              my_status |= 2u;
          }
        }
      }
      __syncthreads();
      F_TICK(3);

      // ================= E: predictor on whole groups =================
      const uint32_t have = cb.leftover + take;
      const bool last_batch = (done + take == chunk_syms);
      const bool seg_done = last_batch && (cy.sym + chunk_syms >= sc.n_samples);
      const uint32_t n = seg_done ? have : (have / G) * G; // samples to finish now
      const uint32_t S0 = cb.proc;                          // global index of DB[0]
      uint32_t ta = 0, tb = 0;
      // E1: per-component plain running sums, written back in place
      if (G == 2)
        f_prefix_vec<2>(sh, doff, n, cb.pc01, cb.pc23, ta, tb);
      else if (G == 4)
        f_prefix_vec<4>(sh, doff, n, cb.pc01, cb.pc23, ta, tb);
      else if (G == 1)
        f_prefix_vec<1>(sh, doff, n, cb.pc01, cb.pc23, ta, tb);
      else
        f_prefix_scalar(sh, DB, S0, n, G, cb.pc01, cb.pc23, ta, tb);
      __syncthreads();
      F_TICK(4);
      // E2: row constants.  Rows starting inside this batch: first sample index
      // ri = r*RS - S0 in [0, n).  One warp scans them 32 at a time.
      const uint32_t r_first = (S0 + RS - 1) / RS;                // first row starting >= S0
      const uint32_t r_end = n ? (S0 + n - 1) / RS + 1 : r_first; // one past the last
      const uint32_t nrs = r_end > r_first ? r_end - r_first : 0;
      if (tid < 32) {
        uint32_t col01 = cb.col01, col23 = cb.col23;
        for (uint32_t rb = 0; rb < nrs; rb += 32) {
          const uint32_t j = rb + tid;
          uint32_t pp01 = 0, pp23 = 0, df01 = 0, df23 = 0;
          if (j < nrs) {
            const uint32_t ri = (r_first + j) * RS - S0;
            uint32_t pv[4], fv[4];
#pragma unroll
            for (uint32_t cc = 0; cc < 4; ++cc) {
              pv[cc] = 0;
              fv[cc] = 0;
              if (cc < G) {
                pv[cc] = (ri >= G) ? DB[ri - G + cc]
                                   : ((cc < 2 ? cb.pc01 : cb.pc23) >> ((cc & 1) * 16)) & 0xFFFFu;
                fv[cc] = DB[ri + cc];
              }
            }
            pp01 = pv[0] | (pv[1] << 16);
            pp23 = pv[2] | (pv[3] << 16);
            df01 = __vsub2(fv[0] | (fv[1] << 16), pp01);
            df23 = __vsub2(fv[2] | (fv[3] << 16), pp23);
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
          // value of the first MCU of the previous row = col + (inclusive - own)
          const uint32_t prev01 = __vadd2(col01, __vsub2(i01, df01));
          const uint32_t prev23 = __vadd2(col23, __vsub2(i23, df23));
          if (j < nrs && j < F_RBMAX) {
            sh.rowbase[j][0] = __vsub2(prev01, pp01);
            sh.rowbase[j][1] = __vsub2(prev23, pp23);
          }
          col01 = __vadd2(col01, __shfl_sync(0xFFFFFFFFu, i01, 31));
          col23 = __vadd2(col23, __shfl_sync(0xFFFFFFFFu, i23, 31));
        }
        if (tid == 0) {
          sh.cy.col01 = col01;
          sh.cy.col23 = col23;
        }
      }
      __syncthreads();
      F_TICK(5);
      // E3: values -> image.  Units of 8 samples, aligned on the global index.
      {
        const uint32_t u_first = S0 >> 3, u_last = (S0 + n + 7) >> 3; // [u_first, u_last)
        const bool vec_ok = sc.mcu_h == 1 && (G == 1 || G == 2 || G == 4) && (RS & 7u) == 0 &&
                            ((sc.out_offset | sc.out_pitch) & 15u) == 0 && (sc.out_x & 7u) == 0;
        const uint32_t inv = sc.rs_inv;
        for (uint32_t u = u_first + tid; u < u_last; u += F_NT) {
          const uint32_t g0 = u << 3; // global sample index of the unit
          uint32_t r, s;
          f_row_col(g0, RS, inv, r, s);
          const bool whole = g0 >= S0 && g0 + 8 <= S0 + n;
          if (whole && vec_ok && s + 8 <= sc.store_w) {
            uint32_t b01, b23;
            if (r >= r_first) {
              b01 = sh.rowbase[r - r_first][0];
              b23 = sh.rowbase[r - r_first][1];
            } else {
              b01 = cb.rb01;
              b23 = cb.rb23;
            }
            const uint4 q = *reinterpret_cast<const uint4*>(&DB[g0 - S0]);
            uint4 o;
            if (G == 2) {
              o.x = __vadd2(q.x, b01); o.y = __vadd2(q.y, b01);
              o.z = __vadd2(q.z, b01); o.w = __vadd2(q.w, b01);
            } else if (G == 4) {
              o.x = __vadd2(q.x, b01); o.y = __vadd2(q.y, b23);
              o.z = __vadd2(q.z, b01); o.w = __vadd2(q.w, b23);
            } else {
              const uint32_t bb = (b01 & 0xFFFFu) * 0x10001u;
              o.x = __vadd2(q.x, bb); o.y = __vadd2(q.y, bb);
              o.z = __vadd2(q.z, bb); o.w = __vadd2(q.w, bb);
            }
            uint8_t* orow = out + sc.out_offset + (uint64_t)(sc.out_y + r) * sc.out_pitch +
                            2ull * (sc.out_x + s);
            stg_cs_v4(orow, o);
          } else if (!(whole && vec_ok && s >= sc.store_w)) {
            for (uint32_t k = 0; k < 8; ++k) {
              const uint32_t gi = g0 + k;
              if (gi < S0 || gi >= S0 + n)
                continue;
              uint32_t rr, ss;
              f_row_col(gi, RS, inv, rr, ss);
              const uint32_t cc = ss % G;
              uint32_t b01, b23;
              if (rr >= r_first) {
                b01 = sh.rowbase[rr - r_first][0];
                b23 = sh.rowbase[rr - r_first][1];
              } else {
                b01 = cb.rb01;
                b23 = cb.rb23;
              }
              const uint32_t base = ((cc < 2 ? b01 : b23) >> ((cc & 1) * 16)) & 0xFFFFu;
              const uint32_t val = (DB[gi - S0] + base) & 0xFFFFu;
              const uint32_t m = ss / G, pidx = ss - m * G;
              const uint32_t ii = pidx / sc.mcu_w, jj = pidx - ii * sc.mcu_w;
              const uint32_t col = m * sc.mcu_w + jj;
              if (col < sc.store_w) {
                uint16_t* o16 = reinterpret_cast<uint16_t*>(
                    out + sc.out_offset +
                    (uint64_t)(sc.out_y + rr * sc.mcu_h + ii) * sc.out_pitch);
                o16[sc.out_x + col] = (uint16_t)val;
              }
            }
          }
        }
      }
      __syncthreads();
      F_TICK(6);
      // E4: carry
      if (tid == 0) {
        FusedCarry& c2 = sh.cy;
        c2.pc01 = __vadd2(cb.pc01, ta);
        c2.pc23 = __vadd2(cb.pc23, tb);
        if (nrs) {
          const uint32_t jl = min(nrs, (uint32_t)F_RBMAX) - 1;
          c2.rb01 = sh.rowbase[jl][0];
          c2.rb23 = sh.rowbase[jl][1];
        }
        c2.proc = S0 + n;
        c2.leftover = have - n;
      }
      // move the unfinished samples (< G of them) to the front
      uint32_t keep = 0;
      if ((uint32_t)tid < have - n)
        keep = DB[n + tid];
      __syncthreads();
      if ((uint32_t)tid < have - n)
        sh.dbuf[((S0 + n) & 7u) + tid] = (uint16_t)keep;
      __syncthreads();
      F_TICK(7);
      done += take;
      if (done >= chunk_syms)
        break;
    }

    // ================= carry to the next chunk =================
    {
      // deferred tail: clean bytes [Lc, len) move to the front of ub
      const uint32_t tail = len - Lc;
      uint32_t tailbyte = 0;
      if ((uint32_t)tid < tail)
        tailbyte = reinterpret_cast<uint8_t*>(sh.ub)[(Lc + tid) ^ 3u];
      __syncthreads();
      if ((uint32_t)tid < tail)
        reinterpret_cast<uint8_t*>(sh.ub)[tid ^ 3u] = (uint8_t)tailbyte;
      if (tid == 0) {
        FusedCarry& c2 = sh.cy;
        c2.sym = cy.sym + total_syms;
        c2.pos = exit_all - Lc * 8u;
        c2.tail_len = tail;
        c2.ubytes = cy.ubytes + Lc;
        // raw offset of the clean byte that becomes ub byte 0: walk back from the
        // end of this chunk's raw range over `tail` clean bytes
        {
          uint32_t rp = min((chunk + 1) * (uint32_t)F_RAW, limit);
          if (mpos != 0xFFFFFFFFu)
            rp = chunk * F_RAW + mpos;
          uint32_t k = tail;
          if (tail > total_emit) {
            // (only when this chunk produced < F_LA bytes) stay anchored on the old tail
            rp = cy.tail_raw;
            k = 0;
            uint32_t adv = Lc;
            while (adv) {
              const uint32_t c0 = f_raw_byte(gbase, limit, rp);
              rp += (c0 == 0xFFu && !st.plain) ? 2 : 1;
              --adv;
            }
          }
          while (k) {
            --rp;
            if (!st.plain && rp > skew && f_raw_byte(gbase, limit, rp) == 0u &&
                f_raw_byte(gbase, limit, rp - 1) == 0xFFu)
              --rp; // stuffing byte: its FF is the clean byte
            --k;
          }
          c2.tail_raw = rp;
        }
        c2.prev_ff = !st.plain && (sh.last_raw_byte == 0xFFu) &&
                     ((chunk + 1) * (uint32_t)F_RAW - 1 < limit) &&
                     ((chunk + 1) * (uint32_t)F_RAW - 1 >= skew);
        c2.ended = final_chunk ? 1u : 0u;
      }
      __syncthreads();
      F_TICK(8);
    }
  }
  // never leave a bulk copy in flight into this CTA's shared memory
  if (st.pending)
    mbar_wait(&sh.bar, st.pending_par);
  {
    int bad = __syncthreads_or((int)(my_status & 1u));
    bad |= (int)sh.bad_code; // (after the barrier)
    const int over = __syncthreads_or((int)(my_status & 2u));
    if (tid == 0)
      results[blockIdx.x].status = bad ? 1u : (over ? 2u : 0u);
  }
}

__global__ void __launch_bounds__(F_NT, 5)
    k2_fused_kernel(const uint8_t* __restrict__ in, uint64_t in_total,
                    const DevScan* __restrict__ scans, const DevTable* __restrict__ tables,
                    uint8_t* __restrict__ out, DevResult* __restrict__ results_all,
                    const uint32_t* __restrict__ scan_ids) {
  extern __shared__ __align__(128) uint8_t f_smem_raw[];
  FusedShared& sh = *reinterpret_cast<FusedShared*>(f_smem_raw);
  const int tid = threadIdx.x;
  const uint32_t scan_idx = scan_ids ? scan_ids[blockIdx.x] : blockIdx.x;
  DevResult* results = results_all + scan_idx - blockIdx.x; // results[blockIdx.x] is ours
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&scans[scan_idx]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.sc);
    for (int i = tid; i < (int)(sizeof(DevScan) / 4); i += F_NT)
      dst[i] = src[i];
  }
  __syncthreads();
  const DevScan& sc = sh.sc;
  for (int s = 0; s < 4; ++s) {
    if (sc.table_idx[s] < 0)
      continue;
    const uint4* src = reinterpret_cast<const uint4*>(&tables[sc.table_idx[s]]);
    uint4* dst = reinterpret_cast<uint4*>(&sh.tab[s]);
    for (int i = tid; i < (int)(sizeof(DevTable) / 16); i += F_NT)
      dst[i] = src[i];
  }
  if (tid < 12)
    sh.lutaddr[tid] = smem_u32(sh.tab[sc.table_of[tid] & 3].lut);
  if (tid == 0) {
    results[blockIdx.x].consumed = 0;
    sh.bad_code = 0;
    mbar_init(&sh.bar, 1);
    fence_mbar_init();
    FusedCarry c;
    c.pos = 0;
    c.sym = 0;
    c.tail_len = 0;
    c.tail_raw = (uint32_t)(sc.in_offset & 15ull);
    c.ubytes = 0;
    c.prev_ff = 0;
    c.ended = 0;
    c.leftover = 0;
    c.proc = 0;
    c.status = 0;
    c.pc01 = c.pc23 = 0;
    c.col01 = (uint32_t)sc.init_pred[0] | ((uint32_t)sc.init_pred[1] << 16);
    c.col23 = (uint32_t)sc.init_pred[2] | ((uint32_t)sc.init_pred[3] << 16);
    c.rb01 = c.rb23 = 0;
    sh.cy = c;
  }
  __syncthreads();
  if (sc.multi_table)
    fused_body<true>(sh, in, in_total, tables, out, results);
  else
    fused_body<false>(sh, in, in_total, tables, out, results);
}

} // namespace rsb200
