// vc5.cuh -- GoPro VC-5 (VC5Decompressor, DNG compression 9) on the device.
//
// A frame is 4 channels x 10 subbands: per channel one low-pass band of fixed-width values and nine
// high-pass bands, each an independent run-length / prefix-code stream (VC5Decompressor.cpp:649-742),
// then three inverse wavelet levels (:137-380) and a Bayer combine through a log table (:875-931).
//
//   vc5_lowpass_kernel   one thread per low-pass coefficient: `prec` bits MSB-first
//   vc5_walk_kernel      high-pass payloads cut into segments of VC5_SEG bits; a symbol is at most
//                        27 bits (26 code + sign), so a segment's true entry lies in its first 27 bits.
//                        One thread per (segment, candidate entry 0..26) walks to the segment's end:
//                        exit offset into the next segment and coefficients produced (saturated
//                        once a marker is met: whatever follows a marker is never stored).
//   vc5_scan_kernel      VC5 rounds of a Hillis-Steele scan of those maps per band (composition of
//                        exit maps, sum of counts): afterwards map[s][0] is the true exit of segment s
//                        and the coefficients before it, from the band's first segment.
//   vc5_store_kernel     one thread per segment: the true symbols from its exact entry with the
//                        coefficient index they start at, the band's failures keyed by bit position
//                        (first in stream order wins, atomicMin), and the non-zero runs into the
//                        int16 band (the run zeroes the coefficient scratch first).
//   vc5_result_kernel    one thread per frame: the first failing band in the reference's order.
//   vc5_recon_kernel     one per wavelet level 3 and 2: both vertical passes and the horizontal pass
//                        fused, one thread per output pair, int16 truncation between passes.
//   vc5_final_kernel     level 1 of all four channels fused with the final combine: log table, Bayer
//                        phase, a 2x2 store per coefficient (two 32-bit stores); skipped by failed frames.
#pragma once
#include "../../include/rawspeed_b200.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <functional>
#include <utility>
#include <vector>

constexpr uint32_t VC5_NT = 256;
constexpr uint32_t VC5_SEG = 1024;   // bits per segment
constexpr uint32_t VC5_CAND = 27;    // candidate entries per segment
constexpr uint32_t VC5_ROOT = 12;    // bits of the first code-table level
constexpr uint32_t VC5_SUB = 7;      // most bits of a deeper level
// high-pass outcomes (RSB200_VC5_*)
constexpr uint32_t VC5_QUANT = 1, VC5_EARLY_END = 2, VC5_OVERRUN = 3, VC5_NO_END = 4, VC5_SHORT = 5,
                   VC5_OVERREAD = 6;

struct Vc5BandDev {
  uint64_t in_offset;
  uint32_t size;      // bytes
  int32_t param;      // quantization (high pass) or precision (low pass)
  uint32_t w, h;      // band dims
  uint32_t seg_first; // first segment (high pass)
  uint32_t nseg;
  uint64_t coef;      // int16 element offset of the band in the plan's coefficient scratch
};

struct Vc5FrameDev {
  uint32_t w, h;           // image
  uint32_t bw[4], bh[4];   // band dims of wavelets 1..3 (index 0: the image's half)
  uint32_t descale;        // bit 3 * ch + (k - 1): wavelet k of channel ch descales by 2
  uint32_t phase;          // 0 RGGB, 2 GBRG
  uint32_t lut;            // offset of its 4096-entry log table
  uint32_t band0;          // its first band (channel * 10 + subband)
  uint64_t rec[4][2];      // int16 offsets of the level-3 and level-2 reconstructions per channel
  uint64_t out_offset;
  uint32_t out_pitch;
  uint32_t pad;
};

// ---------------------------------------------------------------- bits
// 32 bits of a band's payload from bit p, zeros past its end (the pump's zero fill)
__device__ __forceinline__ uint32_t vc5_peek32(const uint8_t* d, uint32_t size, uint64_t p) {
  const uint64_t b = p >> 3;
  uint64_t w = 0;
#pragma unroll
  for (int k = 0; k < 5; ++k)
    w = w << 8 | (b + k < size ? (uint64_t)__ldg(d + b + k) : 0ull);
  return (uint32_t)(w >> (8 - (p & 7)));
}

// 64 bits of a band's payload from byte b, zeros past its end.  A walk keeps one such window and reads
// its symbols from it until fewer than 32 bits are left: 8 loads per 32 bits or more, not 5 per symbol.
__device__ __forceinline__ uint64_t vc5_load64(const uint8_t* d, uint32_t size, uint64_t b) {
  uint64_t w = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k)
    w = w << 8 | (b + k < size ? (uint64_t)__ldg(d + b + k) : 0ull);
  return w;
}

struct Vc5Window {
  uint64_t w, base;  // bits [8 * base, 8 * base + 64)
  __device__ __forceinline__ uint32_t peek(const uint8_t* d, uint32_t size, uint64_t p) {
    uint64_t off = p - 8 * base;
    if (off > 32) {
      base = p >> 3;
      w = vc5_load64(d, size, base);
      off = p & 7;
    }
    return (uint32_t)((w << off) >> 32);
  }
};

// one symbol at the top of `win`: code length + sign, run count, signed decompanded value
struct Vc5Sym {
  uint32_t bits, count;
  int32_t value;
};

__device__ __forceinline__ Vc5Sym vc5_decode(const uint32_t* __restrict__ code, uint32_t win) {
  uint32_t e = __ldg(code + (win >> (32 - VC5_ROOT)));
  uint32_t used = VC5_ROOT;
  while (e >> 31) {
    const uint32_t width = e & 15u;
    const uint32_t idx = (win << used) >> (32 - width);
    e = __ldg(code + ((e >> 4) & 0x7FFFFFFu) + idx);
    used += width;
  }
  Vc5Sym s;
  const uint32_t len = e & 31u;
  s.count = (e >> 5) & 511u;
  int32_t v = (int32_t)((e >> 14) & 1023u);
  s.bits = len;
  if (v != 0) {
    if ((win << len) >> 31)
      v = -v;
    s.bits = len + 1;
  }
  s.value = v;
  return s;
}

// ---------------------------------------------------------------- low pass
__global__ void __launch_bounds__(VC5_NT) vc5_lowpass_kernel(const uint8_t* __restrict__ in,
                                                               const Vc5BandDev* __restrict__ bands,
                                                               int16_t* __restrict__ coef) {
  const Vc5BandDev b = bands[blockIdx.y * 10];  // channel 0..3 of every frame: band (frame, ch, 0)
  const uint32_t i = blockIdx.x * VC5_NT + threadIdx.x;
  if (i >= b.w * b.h)
    return;
  const uint32_t prec = (uint32_t)b.param;
  const uint32_t v = vc5_peek32(in + b.in_offset, b.size, (uint64_t)i * prec) >> (32 - prec);
  coef[b.coef + i] = (int16_t)v;
}

// ---------------------------------------------------------------- segment walks
__global__ void __launch_bounds__(VC5_NT) vc5_walk_kernel(const uint8_t* __restrict__ in,
                                                            const Vc5BandDev* __restrict__ bands,
                                                            const uint32_t* __restrict__ seg_band, uint32_t nsegs,
                                                            const uint32_t* __restrict__ code,
                                                            uint2* __restrict__ map) {
  const uint32_t t = blockIdx.x * VC5_NT + threadIdx.x;
  if (t >= nsegs * VC5_CAND)
    return;
  const uint32_t s = t / VC5_CAND, c = t % VC5_CAND;
  const Vc5BandDev b = bands[__ldg(seg_band + s)];
  const uint8_t* d = in + b.in_offset;
  const uint64_t start = (uint64_t)(s - b.seg_first) * VC5_SEG;
  const uint64_t end = start + VC5_SEG;
  uint64_t p = start + c;
  uint64_t n = 0;
  Vc5Window win{vc5_load64(d, b.size, p >> 3), p >> 3};
  while (p < end) {
    const Vc5Sym y = vc5_decode(code, win.peek(d, b.size, p));
    p += y.bits;
    // a count-0 symbol (a marker) ends the band's pixels: the segments behind it start "past the end"
    n = y.count ? n + y.count : 0xFFFFFFFFull;
  }
  map[t] = make_uint2((uint32_t)(p - end), (uint32_t)min(n, (uint64_t)0xFFFFFFFFu));
}

// one round of the scan: A'[s] = A[s] o A[s - 2^r] within a band
__global__ void __launch_bounds__(VC5_NT) vc5_scan_kernel(const Vc5BandDev* __restrict__ bands,
                                                            const uint32_t* __restrict__ seg_band, uint32_t nsegs,
                                                            uint32_t r, const uint2* __restrict__ src,
                                                            uint2* __restrict__ dst) {
  const uint32_t t = blockIdx.x * VC5_NT + threadIdx.x;
  if (t >= nsegs * VC5_CAND)
    return;
  const uint32_t s = t / VC5_CAND, c = t % VC5_CAND;
  const uint32_t first = bands[__ldg(seg_band + s)].seg_first;
  const uint32_t step = 1u << r;
  uint2 v = src[t];
  if (s - first >= step) {
    const uint2 a = src[(size_t)(s - step) * VC5_CAND + c];
    const uint2 b = src[(size_t)s * VC5_CAND + a.x];
    v = make_uint2(b.x, (uint32_t)min((uint64_t)a.y + b.y, (uint64_t)0xFFFFFFFFu));
  }
  dst[t] = v;
}

// ---------------------------------------------------------------- store
__global__ void __launch_bounds__(VC5_NT) vc5_store_kernel(const uint8_t* __restrict__ in,
                                                             const Vc5BandDev* __restrict__ bands,
                                                             const uint32_t* __restrict__ seg_band, uint32_t nsegs,
                                                             const uint32_t* __restrict__ code,
                                                             const uint2* __restrict__ map,
                                                             unsigned long long* __restrict__ err,
                                                             int16_t* __restrict__ coef) {
  const uint32_t s = blockIdx.x * VC5_NT + threadIdx.x;
  if (s >= nsegs)
    return;
  const uint32_t bi = __ldg(seg_band + s);
  const Vc5BandDev b = bands[bi];
  const uint8_t* d = in + b.in_offset;
  const uint64_t area = (uint64_t)b.w * b.h;
  const uint64_t start = (uint64_t)(s - b.seg_first) * VC5_SEG;
  const uint64_t end = start + VC5_SEG;
  uint64_t p = start, n = 0;
  if (s != b.seg_first) {
    const uint2 e = map[(size_t)(s - 1) * VC5_CAND];
    p += e.x;
    n = e.y;
  }
  if (n > area)
    return;
  int16_t* out = coef + b.coef;
  unsigned long long fail = ~0ull;
  Vc5Window win{vc5_load64(d, b.size, p >> 3), p >> 3};
  const uint64_t limit = 8ull * b.size + 64;  // a symbol starting past it refills past size + 8
  while (p < end) {
    if (p > limit) {
      fail = p << 3 | VC5_OVERREAD;
      break;
    }
    const Vc5Sym y = vc5_decode(code, win.peek(d, b.size, p));
    if (n == area) {  // verifyIsAtEnd: exactly the end marker, sign 0
      if (!(y.value == 1 && y.count == 0))
        fail = p << 3 | VC5_NO_END;
      break;
    }
    const int32_t q = y.value * b.param;
    if (q < -32768 || q > 32767) {
      fail = p << 3 | VC5_QUANT;
      break;
    }
    if (y.count == 0) {
      fail = p << 3 | VC5_EARLY_END;
      break;
    }
    const uint64_t stop = min(n + y.count, area);
    for (uint64_t k = n; q != 0 && k < stop; ++k)  // (the scratch is zeroed before the walks)
      out[k] = (int16_t)q;
    n += y.count;
    if (n > area) {
      fail = p << 3 | VC5_OVERRUN;
      break;
    }
    p += y.bits;
  }
  if (fail != ~0ull)
    atomicMin(err + bi, fail);
}

// ---------------------------------------------------------------- per frame result
__global__ void __launch_bounds__(VC5_NT) vc5_result_kernel(const Vc5FrameDev* __restrict__ frames, uint32_t nf,
                                                              const Vc5BandDev* __restrict__ bands,
                                                              const unsigned long long* __restrict__ err,
                                                              uint2* __restrict__ res) {
  const uint32_t f = blockIdx.x * VC5_NT + threadIdx.x;
  if (f >= nf)
    return;
  // the reference's decode (one worker) meets subbands 3, 2, 1, 6, 5, 4, 9, 8, 7, each for channels 0..3
  const uint64_t order = 0x789456123ull;  // from the lowest nibble up
  uint2 r = make_uint2(0, 0);
  for (int i = 0; i < 36 && r.x == 0; ++i) {
    const uint32_t sb = (uint32_t)(order >> (4 * (i / 4))) & 15u, ch = (uint32_t)i & 3u;
    const uint32_t bi = frames[f].band0 + ch * 10 + sb;
    uint32_t code = 0;
    if (bands[bi].size < 4)
      code = VC5_SHORT;
    else if (err[bi] != ~0ull)
      code = (uint32_t)(err[bi] & 7u);
    if (code)
      r = make_uint2(code == VC5_SHORT || code == VC5_OVERREAD ? 2u : 1u, code << 28 | ch << 4 | sb);
  }
  res[f] = r;
}

// ---------------------------------------------------------------- reconstruction
// First / Middle / Last tap sets, even and odd (VC5Decompressor.cpp:161-179)
__constant__ int VC5_TAPS[3][2][4] = {{{1, 11, -4, 1}, {-1, 5, 4, -1}}, {{1, 1, 8, -1}, {-1, -1, 8, 1}},
                                      {{1, -1, 4, 5}, {-1, 1, -4, 11}}};

__device__ __forceinline__ int vc5_conv(int tap, int parity, int hi, int l0, int l1, int l2, int descale) {
  const int* t = VC5_TAPS[tap][parity];
  const int lows = t[1] * l0 + t[2] * l1 + t[3] * l2;
  int v = t[0] * hi + ((lows + 4) >> 3);
  v *= 1 << descale;
  return v >> 1;
}

// vertical pass at output row r (w x 2h from a w x h high band and a low plane of pitch lp), column c
__device__ __forceinline__ int vc5_vert(const int16_t* hi, const int16_t* lo, uint32_t lp, uint32_t w, uint32_t h,
                                        uint32_t r, uint32_t c) {
  const uint32_t i = r >> 1;
  const int tap = i == 0 ? 0 : (i + 1 < h ? 1 : 2);
  const uint32_t b = i - (uint32_t)tap;
  return (int16_t)vc5_conv(tap, (int)(r & 1), hi[(size_t)i * w + c], lo[(size_t)b * lp + c],
                           lo[(size_t)(b + 1) * lp + c], lo[(size_t)(b + 2) * lp + c], 0);
}

// one output of wavelet k's reconstruction at (r, 2c + parity): before the clamp / truncation
__device__ __forceinline__ int vc5_level(const int16_t* const* hb, const int16_t* lo, uint32_t lp, uint32_t w,
                                         uint32_t h, uint32_t r, uint32_t c, int parity, int descale) {
  const int tap = c == 0 ? 0 : (c + 1 < w ? 1 : 2);
  const uint32_t b = c - (uint32_t)tap;
  const int l0 = vc5_vert(hb[1], lo, lp, w, h, r, b);
  const int l1 = vc5_vert(hb[1], lo, lp, w, h, r, b + 1);
  const int l2 = vc5_vert(hb[1], lo, lp, w, h, r, b + 2);
  const int hv = vc5_vert(hb[2], hb[0], w, w, h, r, c);
  return vc5_conv(tap, parity, hv, l0, l1, l2, descale);
}

// wavelet level 3 (lvl 0) or 2 (lvl 1) of every channel of every frame: grid.y = frame * 4 + channel
__global__ void __launch_bounds__(VC5_NT) vc5_recon_kernel(const Vc5FrameDev* __restrict__ frames,
                                                             const Vc5BandDev* __restrict__ bands, uint32_t lvl,
                                                             int16_t* __restrict__ coef) {
  const Vc5FrameDev& f = frames[blockIdx.y >> 2];
  const uint32_t ch = blockIdx.y & 3u, k = 3 - lvl;
  const uint32_t w = f.bw[k], h = f.bh[k];
  const uint32_t t = blockIdx.x * VC5_NT + threadIdx.x;
  if (t >= w * 2 * h)
    return;
  const uint32_t r = t / w, c = t % w;
  const Vc5BandDev* bd = bands + f.band0 + ch * 10;
  const uint32_t s0 = 1 + 3 * lvl;
  const int16_t* hb[3] = {coef + bd[s0].coef, coef + bd[s0 + 1].coef, coef + bd[s0 + 2].coef};
  const int16_t* lo = lvl == 0 ? coef + bd[0].coef : coef + f.rec[ch][0];
  const uint32_t lp = lvl == 0 ? w : 2 * f.bw[k + 1];
  const int descale = (f.descale >> (3 * ch + k - 1)) & 1u ? 2 : 0;
  int16_t* dst = coef + f.rec[ch][lvl] + (size_t)r * 2 * w + 2 * c;
  dst[0] = (int16_t)vc5_level(hb, lo, lp, w, h, r, c, 0, descale);
  dst[1] = (int16_t)vc5_level(hb, lo, lp, w, h, r, c, 1, descale);
}

// wavelet level 1 of the four channels and the final combine: one thread per 2x2 output quad
__global__ void __launch_bounds__(VC5_NT) vc5_final_kernel(const Vc5FrameDev* __restrict__ frames,
                                                             const Vc5BandDev* __restrict__ bands,
                                                             const int16_t* __restrict__ coef,
                                                             const uint16_t* __restrict__ luts,
                                                             const uint2* __restrict__ res, uint8_t* __restrict__ out) {
  const uint32_t fi = blockIdx.y;
  if (res[fi].x != 0)  // a failed frame leaves its image untouched
    return;
  const Vc5FrameDev& f = frames[fi];
  const uint32_t qw = f.w / 2, t = blockIdx.x * VC5_NT + threadIdx.x;
  if (t >= qw * (f.h / 2))
    return;
  const uint32_t row = t / qw, col = t % qw;
  const uint32_t w = f.bw[1], h = f.bh[1];
  int v[4];
#pragma unroll
  for (uint32_t ch = 0; ch < 4; ++ch) {
    const Vc5BandDev* bd = bands + f.band0 + ch * 10;
    const int16_t* hb[3] = {coef + bd[7].coef, coef + bd[8].coef, coef + bd[9].coef};
    const int descale = (f.descale >> (3 * ch)) & 1u ? 2 : 0;
    const int x = vc5_level(hb, coef + f.rec[ch][1], 2 * f.bw[2], w, h, row, col >> 1, (int)(col & 1), descale);
    v[ch] = (int16_t)min(max(x, 0), 16383);
  }
  const int gs = v[0], rg = v[1] - 2048, bg = v[2] - 2048, gd = v[3] - 2048;
  int p[4] = {gs + 2 * rg, gs + gd, gs - gd, gs + 2 * bg};  // r g1 g2 b
  const uint16_t* lut = luts + f.lut;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    p[k] = __ldg(lut + min(max(p[k], 0), 4095));
  uint32_t top, bot;
  if (f.phase == 2) {  // GBRG: g1 b / r g2
    top = (uint32_t)p[1] | (uint32_t)p[3] << 16;
    bot = (uint32_t)p[0] | (uint32_t)p[2] << 16;
  } else {
    top = (uint32_t)p[0] | (uint32_t)p[1] << 16;
    bot = (uint32_t)p[2] | (uint32_t)p[3] << 16;
  }
  uint8_t* o = out + f.out_offset + (size_t)(2 * row) * f.out_pitch + 4 * (size_t)col;
  *reinterpret_cast<uint32_t*>(o) = top;
  *reinterpret_cast<uint32_t*>(o + f.out_pitch) = bot;
}

// ---------------------------------------------------------------- host: tables and layout
// The decode table of a codebook: a root of 2^VC5_ROOT entries indexed by the next bits, deeper levels
// of at most 2^VC5_SUB; a leaf is len | count << 5 | decompanded value << 14, a link 1 << 31 | offset
// << 4 | width.  False for a codebook that is not a complete prefix code within the ABI's limits.
static inline bool vc5_build_code(const rsb200_vc5_code* codes, int n, std::vector<uint32_t>& tab) {
  if (n <= 0 || n > 4096)
    return false;
  std::vector<std::pair<uint32_t, int>> ws;  // code left-justified in 32 bits, index
  uint64_t kraft = 0;
  for (int i = 0; i < n; ++i) {
    const rsb200_vc5_code& c = codes[i];
    if (c.size < 1 || c.size > 26 || c.count > 511 || c.value > 255 || (c.bits >> c.size) != 0)
      return false;
    kraft += 1ull << (26 - c.size);
    ws.push_back({c.bits << (32 - c.size), i});
  }
  if (kraft != (1ull << 26))
    return false;
  std::sort(ws.begin(), ws.end());
  for (size_t i = 0; i + 1 < ws.size(); ++i)  // no code is a prefix of the next one
    if ((uint64_t)ws[i].first + (1ull << (32 - codes[ws[i].second].size)) > ws[i + 1].first)
      return false;
  auto leaf = [&](int i) {
    const double c0 = codes[i].value;
    const int v = (int)(c0 + (c0 * c0 * c0 * 768) / (255. * 255. * 255.));  // decompand, <= 1023
    return codes[i].size | codes[i].count << 5 | (uint32_t)v << 14;
  };
  // fills the level at `off` (width bits after `used`) from the codes ws[lo, hi) that share its prefix
  std::function<void(size_t, uint32_t, uint32_t, size_t, size_t)> fill = [&](size_t off, uint32_t used,
                                                                           uint32_t width, size_t lo, size_t hi) {
    for (size_t i = lo; i < hi;) {
      const uint32_t w = ws[i].first, len = codes[ws[i].second].size;
      const uint32_t idx = (w << used) >> (32 - width);
      if (len <= used + width) {
        const uint32_t span = 1u << (used + width - len);
        for (uint32_t k = 0; k < span; ++k)
          tab[off + idx + k] = leaf(ws[i].second);
        ++i;
        continue;
      }
      size_t j = i;
      uint32_t maxlen = 0;
      while (j < hi && ((ws[j].first << used) >> (32 - width)) == idx)
        maxlen = std::max(maxlen, codes[ws[j].second].size), ++j;
      const uint32_t sub = std::min<uint32_t>(VC5_SUB, maxlen - used - width);
      const size_t soff = tab.size();
      tab.resize(soff + (1u << sub));
      tab[off + idx] = 1u << 31 | (uint32_t)soff << 4 | sub;
      fill(soff, used + width, sub, i, j);
      i = j;
    }
  };
  tab.assign(1u << VC5_ROOT, 0);
  fill(0, 0, VC5_ROOT, 0, ws.size());
  return tab.size() < (1u << 27);
}

// The plan's layout of its jobs: frames, 40 bands per frame (channel * 10 + subband), the segments of
// the high-pass bands and the coefficient scratch (bands, then the level-3 and level-2 reconstructions
// of each channel).
struct Vc5Layout {
  std::vector<Vc5FrameDev> frames;
  std::vector<Vc5BandDev> bands;
  std::vector<uint32_t> seg_band;
  uint64_t ncoef = 0;
  uint32_t rounds = 0;  // scan rounds: 2^rounds >= the most segments of a band
  uint32_t max_low = 0, max_rec[2] = {0, 0}, max_quads = 0;
};

// -1, or the first job the ABI refuses (`why` says what)
static inline int vc5_layout(const rsb200_vc5_job* jobs, int njobs, const rsb200_vc5_band* bands, int nbands,
                             Vc5Layout& L, const char** why) {
  L.frames.assign((size_t)njobs, Vc5FrameDev{});
  L.bands.assign((size_t)njobs * 40, Vc5BandDev{});
  uint64_t maxseg = 0;
  for (int i = 0; i < njobs; ++i) {
    const rsb200_vc5_job& j = jobs[i];
    bool ok = j.width > 32 && j.height > 32 && j.width <= 65534 && j.height <= 65534 && j.width % 2 == 0 &&
              j.height % 2 == 0 && j.output_bits >= 1 && j.output_bits <= 16 &&
              (j.phase == RSB200_VC5_RGGB || j.phase == RSB200_VC5_GBRG) &&
              (uint64_t)j.first_band + 40 <= (uint64_t)nbands && j.out_offset % 4 == 0 && j.out_pitch % 4 == 0 &&
              j.out_pitch >= 2ull * (uint32_t)j.width && j.reserved == 0;
    Vc5FrameDev& f = L.frames[(size_t)i];
    f.w = (uint32_t)j.width, f.h = (uint32_t)j.height;
    uint32_t ww = f.w, hh = f.h;
    for (int k = 0; k < 4; ++k) {
      ww = (ww + 1) / 2, hh = (hh + 1) / 2;
      f.bw[k] = ww, f.bh[k] = hh;
    }
    for (int ch = 0; ch < 4; ++ch)
      for (int k = 0; k < 3; ++k) {
        ok = ok && j.prescale[ch][k] <= 3;
        if (j.prescale[ch][k] == 2)
          f.descale |= 1u << (3 * ch + k);
      }
    if (!ok) {
      *why = "malformed descriptor";
      return i;
    }
    f.phase = (uint32_t)j.phase;
    f.lut = (uint32_t)(j.output_bits - 1) * 4096u;
    f.band0 = (uint32_t)i * 40;
    f.out_offset = j.out_offset;
    f.out_pitch = j.out_pitch;
    for (int b = 0; b < 40; ++b) {
      const rsb200_vc5_band& src = bands[j.first_band + (uint32_t)b];
      const int sb = b % 10, k = sb == 0 ? 3 : 3 - (sb - 1) / 3;
      Vc5BandDev& d = L.bands[(size_t)i * 40 + (size_t)b];
      d.in_offset = src.in_offset, d.size = src.in_size, d.param = src.param;
      d.w = f.bw[k], d.h = f.bh[k];
      d.coef = L.ncoef;
      const uint64_t area = (uint64_t)d.w * d.h;
      L.ncoef += (area + 7) & ~7ull;
      d.seg_first = (uint32_t)L.seg_band.size();
      if (sb == 0) {
        ok = src.param >= 8 && src.param <= 16 && src.in_size >= 8 * ((area * (uint64_t)src.param + 63) / 64);
      } else {
        ok = src.in_size % 4 == 0 && src.in_size <= (1u << 28) && src.param >= -32768 && src.param <= 32767;
        if (ok && src.in_size >= 4) {  // symbols may start up to bit 8 * size + 64 (the pump's zero fill)
          d.nseg = (uint32_t)((8ull * src.in_size + 65 + VC5_SEG - 1) / VC5_SEG);
          L.seg_band.insert(L.seg_band.end(), d.nseg, (uint32_t)(i * 40 + b));
          maxseg = std::max<uint64_t>(maxseg, d.nseg);
        }
      }
      if (!ok) {
        *why = "malformed band";
        return i;
      }
    }
    for (int ch = 0; ch < 4; ++ch)
      for (int l = 0; l < 2; ++l) {
        f.rec[ch][l] = L.ncoef;
        L.ncoef += (4ull * f.bw[3 - l] * f.bh[3 - l] + 7) & ~7ull;
      }
    if (L.seg_band.size() * VC5_CAND >= (1ull << 31)) {
      *why = "too much input for one plan";
      return i;
    }
    L.max_low = std::max(L.max_low, f.bw[3] * f.bh[3]);
    L.max_rec[0] = std::max(L.max_rec[0], 2 * f.bw[3] * f.bh[3]);
    L.max_rec[1] = std::max(L.max_rec[1], 2 * f.bw[2] * f.bh[2]);
    L.max_quads = std::max(L.max_quads, (f.w / 2) * (f.h / 2));
  }
  while ((1ull << L.rounds) < maxseg)
    ++L.rounds;
  return -1;
}

// VC5Decompressor::initVC5LogTable (VC5Decompressor.cpp:464-488) for output bits 1..16, 4096 entries each
static inline std::vector<uint16_t> vc5_luts() {
  std::vector<uint16_t> luts(16 * 4096);
  for (int bits = 1; bits <= 16; ++bits)
    for (int i = 0; i < 4096; ++i) {
      const double y = 65535 * ((std::pow(113.0, (double)i / 4095.0) - 1) / 112.0);
      luts[(size_t)(bits - 1) * 4096 + (size_t)i] = (uint16_t)((unsigned)y >> (16 - bits));
    }
  return luts;
}
