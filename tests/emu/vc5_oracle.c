/* vc5_oracle.c -- CPU restatement of the GoPro VC-5 decompressor (VC5Decompressor,
 * decompressors/VC5Decompressor.cpp:382-960): the constructor's checks, the tag walk, the band
 * decoders, the three inverse wavelet levels and the final Bayer combine, plus a writer of band
 * streams, for the tests.  The codebook is an argument (n entries of {size, bits, count, value}).
 * Test infrastructure: pinned against the reference's own decompressor by
 * tests/test_oracle_vc5.py. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* band outcomes (RSB200_VC5_* of the C ABI) */
enum { VC_OK = 0, VC_QUANT = 1, VC_EARLY_END = 2, VC_OVERRUN = 3, VC_NO_END = 4, VC_SHORT = 5, VC_OVERREAD = 6 };
/* outcomes of the constructor and the tag walk (message ids of tests/vc5_oracle.py) */
enum {
  VC_DIMS = 16, VC_WIDTH, VC_HEIGHT, VC_CFA, VC_PHASE, VC_WHITE, VC_MAGIC, VC_CHANNELS, VC_IMG_W, VC_IMG_H,
  VC_PRECISION, VC_CHANNEL_NO, VC_FORMAT, VC_SUBBANDS, VC_BPC, VC_PAT_W, VC_PAT_H, VC_SUBBAND_NO, VC_CPS,
  VC_UNKNOWN_TAG, VC_NO_SUBBAND, VC_SEEN, VC_NO_PRECISION, VC_NO_QUANT, VC_BS_BOUNDS, VC_BUF_OVERFLOW,
  VC_TOO_MANY = 64 /* + band outcome: "Too many errors encountered. Giving up. First Error:\n..." */
};

typedef struct {
  int off, size, param; /* payload in the datablock; quantization or low-pass precision */
} Band;

typedef struct {
  int w, h, bits, phase;
  int bw[4], bh[4];     /* band dims of wavelet 1..3 (index 0: the image's half) */
  int prescale[4][4];   /* [channel][wavelet 1..3] */
  Band band[4][10];     /* [channel][subband] */
} Frame;

/* ---------------------------------------------------------------- codebook */
typedef struct {
  int child[1024][2]; /* > 0: node, < 0: -(entry + 1), 0: none */
  int nodes;
  int count[512], value[512]; /* decompanded value */
} Code;

int vc_decompand(int v) {
  double c = v;
  c += (c * c * c * 768) / (255. * 255. * 255.);
  if (c > 32767)
    return 32767;
  if (c < -32768)
    return -32768;
  return (int)c;
}

static int build_code(Code* c, const int32_t* e, int n) {
  memset(c, 0, sizeof(*c));
  c->nodes = 1;
  if (n > 512)
    return -1;
  for (int i = 0; i < n; ++i) {
    int node = 0;
    const int len = e[4 * i];
    for (int k = len - 1; k >= 0; --k) {
      const int b = (e[4 * i + 1] >> k) & 1;
      if (k == 0) {
        c->child[node][b] = -(i + 1);
      } else {
        if (c->child[node][b] == 0) {
          if (c->nodes >= 1024)
            return -1;
          c->child[node][b] = c->nodes++;
        }
        node = c->child[node][b];
      }
    }
    c->count[i] = e[4 * i + 2];
    c->value[i] = vc_decompand(e[4 * i + 3]);
  }
  return 0;
}

/* ---------------------------------------------------------------- band decoders */
static int bit_at(const uint8_t* d, int size, int64_t pos) {
  return pos < 8 * (int64_t)size ? (d[pos >> 3] >> (7 - (pos & 7))) & 1 : 0;
}

/* HighPassBand::decode (VC5Decompressor.cpp:683-742) with the BitStreamerMSB pump: a symbol that
 * starts at bit b refills at byte 4 * ceil(b / 32), which fails past size + 8. */
static int decode_high(const Code* c, const uint8_t* d, int size, int w, int h, int quant, int16_t* out) {
  if (size < 4)
    return VC_SHORT;
  const int64_t area = (int64_t)w * h;
  int64_t n = 0, pos = 0;
  for (;;) {
    if (4 * ((pos + 31) / 32) > (int64_t)size + 8)
      return VC_OVERREAD;
    int node = 0;
    while (node >= 0) {
      node = c->child[node][bit_at(d, size, pos++)];
      if (node == 0)
        return -1; /* not a complete code */
    }
    const int e = -node - 1;
    int v = c->value[e];
    if (v != 0 && bit_at(d, size, pos++))
      v = -v;
    const int count = c->count[e];
    if (n == area) /* verifyIsAtEnd */
      return v == 1 && count == 0 ? VC_OK : VC_NO_END;
    const int q = v * quant;
    if (q < -32768 || q > 32767)
      return VC_QUANT;
    if (count == 0)
      return VC_EARLY_END;
    for (int k = 0; k < count && n + k < area; ++k)
      out[n + k] = (int16_t)q;
    n += count;
    if (n > area)
      return VC_OVERRUN;
  }
}

static void decode_low(const uint8_t* d, int size, int w, int h, int prec, int16_t* out) {
  int64_t pos = 0;
  for (int64_t i = 0; i < (int64_t)w * h; ++i) {
    unsigned v = 0;
    for (int k = 0; k < prec; ++k)
      v = v << 1 | (unsigned)bit_at(d, size, pos++);
    out[i] = (int16_t)v;
  }
}

/* ---------------------------------------------------------------- reconstruction */
static const int TAPS[3][2][4] = {{{1, 11, -4, 1}, {-1, 5, 4, -1}},   /* first */
                                  {{1, 1, 8, -1}, {-1, -1, 8, 1}},    /* middle */
                                  {{1, -1, 4, 5}, {-1, 1, -4, 11}}};  /* last */

static int conv(const int* m, int hi, int l0, int l1, int l2, int descale) {
  int lows = m[1] * l0 + m[2] * l1 + m[3] * l2;
  int t = m[0] * hi + ((lows + 4) >> 3);
  t *= 1 << descale;
  return t >> 1;
}

/* vertical pass (reconstructPass): high w x h, low read at rows 0..h-1 with pitch lp -> w x 2h */
static void vertical(const int16_t* hi, const int16_t* lo, int lp, int w, int h, int16_t* dst) {
  for (int r = 0; r < h; ++r) {
    const int s = r == 0 ? 0 : (r + 1 < h ? 1 : 2);
    const int b = r - s;
    for (int c = 0; c < w; ++c) {
      const int l0 = lo[(b + 0) * lp + c], l1 = lo[(b + 1) * lp + c], l2 = lo[(b + 2) * lp + c];
      dst[(2 * r) * w + c] = (int16_t)conv(TAPS[s][0], hi[r * w + c], l0, l1, l2, 0);
      dst[(2 * r + 1) * w + c] = (int16_t)conv(TAPS[s][1], hi[r * w + c], l0, l1, l2, 0);
    }
  }
}

/* horizontal pass (combineLowHighPass): w x h each -> 2w x h */
static void horizontal(const int16_t* lo, const int16_t* hi, int w, int h, int descale, int clamp, int16_t* dst) {
  for (int r = 0; r < h; ++r)
    for (int c = 0; c < w; ++c) {
      const int s = c == 0 ? 0 : (c + 1 < w ? 1 : 2);
      const int b = c - s;
      const int16_t* L = lo + r * w;
      for (int k = 0; k < 2; ++k) {
        int v = conv(TAPS[s][k], hi[r * w + c], L[b], L[b + 1], L[b + 2], descale);
        if (clamp)
          v = v < 0 ? 0 : (v > 16383 ? 16383 : v);
        dst[r * 2 * w + 2 * c + k] = (int16_t)v;
      }
    }
}

/* ---------------------------------------------------------------- tag walk */
typedef struct {
  const uint8_t* d;
  int size, pos;
} Bs;

static int get16(Bs* b, int* v) {
  if (b->size - b->pos < 2)
    return -1;
  *v = b->d[b->pos] << 8 | b->d[b->pos + 1];
  b->pos += 2;
  return 0;
}

/* The constructor (VC5Decompressor.cpp:382-432) and parseVC5 (:490-618, :744-816).  cfa: the
 * BayerPhase 0..3, or 4 for a CFA that is not 2x2.  args: the values the message prints. */
static int parse(Frame* f, const uint8_t* d, int size, int w, int h, int white, int cfa, int* args) {
  memset(f, 0, sizeof(*f));
  if (w <= 0 || h <= 0)
    return VC_DIMS;
  args[0] = w;
  args[1] = 2;
  if (w % 2)
    return VC_WIDTH;
  args[0] = h;
  if (h % 2)
    return VC_HEIGHT;
  if (cfa < 0 || cfa > 3)
    return VC_CFA;
  if (cfa != 0 && cfa != 2)
    return VC_PHASE;
  args[0] = white;
  if (white <= 0 || white > 65535)
    return VC_WHITE;
  f->w = w, f->h = h, f->phase = cfa;
  for (int wp = white; wp; wp >>= 1)
    f->bits++;
  int ww = w, hh = h;
  for (int k = 0; k < 4; ++k) {
    ww = (ww + 1) / 2, hh = (hh + 1) / 2;
    f->bw[k] = ww, f->bh[k] = hh;
  }
  Bs b = {d, size, 0};
  if (size < 4) /* getU32 / getU16 past the end: Buffer::getSubView */
    return VC_BUF_OVERFLOW;
  b.pos = 4;
  if (!(d[0] == 0x56 && d[1] == 0x43 && d[2] == 0x2d && d[3] == 0x35))
    return VC_MAGIC;
  int chan = 0, subband = -1, prec = -1, quant = -1, has_quant = 0;
  int valid[4][4] = {{0}}; /* [channel][wavelet 0..3] band masks */
  for (;;) {
    int t, val;
    if (get16(&b, &t) || get16(&b, &val))
      return VC_BUF_OVERFLOW;
    int16_t tag = (int16_t)t;
    const int optional = (tag & (int16_t)0x8000) != 0;
    if (optional)
      tag = (int16_t)-tag;
    args[0] = val;
    switch (tag) {
    case 0x000c:
      args[1] = 4;
      if (val != 4)
        return VC_CHANNELS;
      break;
    case 0x0014:
      args[1] = w;
      if (val != w)
        return VC_IMG_W;
      break;
    case 0x0015:
      args[1] = h;
      if (val != h)
        return VC_IMG_H;
      break;
    case 0x0023:
      if (val < 8 || val > 16)
        return VC_PRECISION;
      prec = val;
      break;
    case 0x003e:
      if (val >= 4)
        return VC_CHANNEL_NO;
      chan = val;
      break;
    case 0x0054:
      if (val != 4)
        return VC_FORMAT;
      break;
    case 0x000e:
      args[1] = 10;
      if (val != 10)
        return VC_SUBBANDS;
      break;
    case 0x0066:
      args[1] = 12;
      if (val != 12)
        return VC_BPC;
      break;
    case 0x006a:
      args[1] = 2;
      if (val != 2)
        return VC_PAT_W;
      break;
    case 0x006b:
      args[1] = 2;
      if (val != 2)
        return VC_PAT_H;
      break;
    case 0x0030:
      if (val >= 10)
        return VC_SUBBAND_NO;
      subband = val;
      break;
    case 0x0035:
      quant = (int16_t)val;
      has_quant = 1;
      break;
    case 0x006c:
      args[1] = 1;
      if (val != 1)
        return VC_CPS;
      break;
    case 0x006d: /* applies to the current channel (the FIXME at :568) */
      for (int k = 0; k < 3; ++k)
        f->prescale[chan][1 + k] = (val >> (14 - 2 * k)) & 3;
      break;
    default: {
      int64_t chunk = 0;
      if (tag & 0x2000)
        chunk = (int64_t)(tag & 0xff) << 16 | val;
      else if (tag & 0x4000)
        chunk = val;
      if ((tag & 0x6000) == 0x6000) {
        if ((int64_t)size - b.pos < 4 * chunk)
          return VC_BUF_OVERFLOW;
        const int off = b.pos, len = (int)(4 * chunk);
        b.pos += len;
        if (subband < 0)
          return VC_NO_SUBBAND;
        const int wl = subband == 0 ? 3 : 3 - (subband - 1) / 3; /* wavelet 1..3 */
        const int bi = subband == 0 ? 0 : 1 + (subband - 1) % 3;
        if (valid[chan][wl] & (1 << bi)) {
          args[0] = bi, args[1] = wl - 1, args[2] = chan;
          return VC_SEEN;
        }
        Band* bd = &f->band[chan][subband];
        bd->off = off;
        if (subband == 0) {
          if (prec < 0)
            return VC_NO_PRECISION;
          const int64_t bytes = 8 * (((int64_t)f->bw[3] * f->bh[3] * prec + 63) / 64);
          if (bytes > len)
            return VC_BUF_OVERFLOW;
          bd->size = (int)bytes, bd->param = prec;
          prec = -1;
        } else {
          if (!has_quant)
            return VC_NO_QUANT;
          bd->size = len, bd->param = quant;
          has_quant = 0;
        }
        valid[chan][wl] |= 1 << bi;
        if (valid[chan][wl] == 15)
          valid[chan][wl - 1] |= 1;
        subband = -1;
        break;
      }
      int opt = optional;
      if (tag & 0x2000)
        opt = 1, chunk = 0;
      if (!opt) {
        args[0] = (uint16_t)tag;
        return VC_UNKNOWN_TAG;
      }
      if (chunk) {
        if ((int64_t)size - b.pos < 4 * chunk)
          return VC_BS_BOUNDS;
        b.pos += (int)(4 * chunk);
      }
    }
    }
    if ((valid[0][0] & valid[1][0] & valid[2][0] & valid[3][0]) & 1)
      return VC_OK;
  }
}

int vc_parse(const uint8_t* d, int size, int w, int h, int white, int cfa, int32_t* bands, int32_t* prescale,
             int32_t* bits, int32_t* args) {
  Frame f;
  const int rc = parse(&f, d, size, w, h, white, cfa, args);
  if (rc)
    return rc;
  for (int ch = 0; ch < 4; ++ch) {
    for (int s = 0; s < 10; ++s) {
      bands[3 * (ch * 10 + s)] = f.band[ch][s].off;
      bands[3 * (ch * 10 + s) + 1] = f.band[ch][s].size;
      bands[3 * (ch * 10 + s) + 2] = f.band[ch][s].param;
    }
    for (int k = 0; k < 3; ++k)
      prescale[ch * 3 + k] = f.prescale[ch][1 + k];
  }
  *bits = f.bits;
  return 0;
}

/* Decode one band (code: 264-ish entries) into out (w x h); the band outcome. */
int vc_decode_band(const uint8_t* d, int size, int w, int h, int quant, const int32_t* codes, int ncodes,
                   int16_t* out) {
  static Code c;
  if (build_code(&c, codes, ncodes))
    return -1;
  return decode_high(&c, d, size, w, h, quant, out);
}

/* The order in which the reference's decode (one worker) meets the high-pass bands: subbands 3, 2, 1,
 * 6, 5, 4, 9, 8, 7, each for channels 0..3 (recorded by tools/vc5_ref_golden.py --order).  The first
 * failing band in it is the one the message names. */
static const int ORDER_SUBBANDS[9] = {3, 2, 1, 6, 5, 4, 9, 8, 7};

/* VC5Decompressor(bs, img) + decode(0, 0, w, h).  out: h rows of `pitch` uint16, written only on
 * success.  args: printed values of a constructor / tag-walk message; for VC_TOO_MANY + band outcome,
 * args[0..1] = channel, subband of the band named. */
int vc_decompress(const uint8_t* d, int size, int w, int h, int white, int cfa, const int32_t* codes, int ncodes,
                  uint16_t* out, int pitch, int32_t* args) {
  static Code c;
  Frame f;
  int rc = parse(&f, d, size, w, h, white, cfa, args);
  if (rc)
    return rc;
  if (build_code(&c, codes, ncodes))
    return -1;
  const int W1 = f.bw[1], H1 = f.bh[1];
  int16_t* bands[4][10];
  for (int ch = 0; ch < 4; ++ch)
    for (int s = 0; s < 10; ++s) {
      const int k = s == 0 ? 3 : 3 - (s - 1) / 3;
      bands[ch][s] = calloc((size_t)f.bw[k] * f.bh[k], 2);
    }
  int fail = 0;
  for (int i = 0; i < 36 && !fail; ++i) {
    const int ch = i % 4, s = ORDER_SUBBANDS[i / 4], k = 3 - (s - 1) / 3;
    const Band* b = &f.band[ch][s];
    const int r = decode_high(&c, d + b->off, b->size, f.bw[k], f.bh[k], b->param, bands[ch][s]);
    if (r) {
      fail = VC_TOO_MANY + r;
      args[0] = ch, args[1] = s;
    }
  }
  if (!fail) {
    int16_t* fin[4];
    for (int ch = 0; ch < 4; ++ch) {
      const Band* lb = &f.band[ch][0];
      decode_low(d + lb->off, lb->size, f.bw[3], f.bh[3], lb->param, bands[ch][0]);
      const int16_t* low = bands[ch][0];
      int lp = f.bw[3];
      int16_t* prev = NULL;
      for (int k = 3; k >= 1; --k) {
        const int bw = f.bw[k], bh = f.bh[k], s0 = 1 + 3 * (3 - k);
        int16_t* lv = malloc((size_t)bw * bh * 4);
        int16_t* hv = malloc((size_t)bw * bh * 4);
        int16_t* rec = malloc((size_t)bw * bh * 8);
        vertical(bands[ch][s0 + 1], low, lp, bw, bh, lv);
        vertical(bands[ch][s0 + 2], bands[ch][s0], bw, bw, bh, hv);
        horizontal(lv, hv, bw, 2 * bh, f.prescale[ch][k] == 2 ? 2 : 0, k == 1, rec);
        free(lv);
        free(hv);
        free(prev);
        prev = rec;
        low = rec;
        lp = 2 * bw;
      }
      fin[ch] = prev;
    }
    unsigned lut[4096];
    for (int i = 0; i < 4096; ++i) {
      const double y = 65535 * ((pow(113.0, i / 4095.0) - 1) / 112.0);
      lut[i] = (unsigned)y >> (16 - f.bits);
    }
    const int fp = 2 * W1;
    for (int r = 0; r < h / 2; ++r)
      for (int cc = 0; cc < w / 2; ++cc) {
        const int gs = fin[0][r * fp + cc], rg = fin[1][r * fp + cc] - 2048, bg = fin[2][r * fp + cc] - 2048,
                  gd = fin[3][r * fp + cc] - 2048;
        int p[4] = {gs + 2 * rg, gs + gd, gs - gd, gs + 2 * bg}; /* r g1 g2 b */
        for (int k = 0; k < 4; ++k)
          p[k] = (int)lut[p[k] < 0 ? 0 : (p[k] > 4095 ? 4095 : p[k])];
        int q[4] = {p[0], p[1], p[2], p[3]};
        if (f.phase == 2) /* GBRG: g1 b / r g2 */
          q[0] = p[1], q[1] = p[3], q[2] = p[0], q[3] = p[2];
        out[(2 * r) * pitch + 2 * cc] = (uint16_t)q[0];
        out[(2 * r) * pitch + 2 * cc + 1] = (uint16_t)q[1];
        out[(2 * r + 1) * pitch + 2 * cc] = (uint16_t)q[2];
        out[(2 * r + 1) * pitch + 2 * cc + 1] = (uint16_t)q[3];
      }
    (void)H1;
    for (int ch = 0; ch < 4; ++ch)
      free(fin[ch]);
  }
  for (int ch = 0; ch < 4; ++ch)
    for (int s = 0; s < 10; ++s)
      free(bands[ch][s]);
  return fail;
}

/* ---------------------------------------------------------------- writer */
/* Symbols (entry index, sign bit) of band content whose values are +-decompand(m) * quant: a value
 * takes the count-1 code of its magnitude, a zero run the longest zero-run codes that fit, greedily,
 * and the end marker (count 0, value 1, sign 0) closes the band.  -(i + 1) if value i is not
 * encodable, -(area + 1) if cap is too small. */
int64_t vc_symbols(const int16_t* v, int64_t area, int quant, const int32_t* codes, int ncodes, int32_t* syms,
                   int64_t cap) {
  int one[256], zrun[512], nz = 0, end = -1;
  for (int m = 0; m < 256; ++m)
    one[m] = -1;
  for (int i = 0; i < ncodes; ++i) {
    const int count = codes[4 * i + 2], value = codes[4 * i + 3];
    if (count == 1 && value < 256)
      one[value] = i;
    if (value == 0 && count > 1)
      zrun[nz++] = i;
    if (count == 0 && value == 1)
      end = i;
  }
  int64_t n = 0;
  for (int64_t i = 0; i < area;) {
    if (n + 2 > cap)
      return -(area + 1);
    if (v[i] == 0) {
      int64_t z = 1;
      while (z < 512 && i + z < area && v[i + z] == 0)
        ++z;
      int best = one[0], bc = 1;
      for (int k = 0; k < nz; ++k) {
        const int cnt = codes[4 * zrun[k] + 2];
        if (cnt <= z && cnt > bc)
          best = zrun[k], bc = cnt;
      }
      syms[2 * n] = best, syms[2 * n + 1] = 0, ++n;
      i += bc;
      continue;
    }
    const int a = v[i] < 0 ? -v[i] : v[i];
    int m = 1;
    while (m < 256 && vc_decompand(m) * abs(quant) < a)
      ++m;
    if (m == 256 || vc_decompand(m) * abs(quant) != a || one[m] < 0)
      return -(i + 1);
    syms[2 * n] = one[m], syms[2 * n + 1] = (v[i] < 0) != (quant < 0), ++n;
    ++i;
  }
  if (n + 1 > cap)
    return -(area + 1);
  syms[2 * n] = end, syms[2 * n + 1] = 0;
  return n + 1;
}

/* Bit string of n symbols (entry, sign; the sign bit only where the entry's value is not 0), zero-padded
 * to whole 4-byte words.  Returns the bytes written or -1 when cap is too small. */
int64_t vc_pack(const int32_t* syms, int64_t n, const int32_t* codes, uint8_t* out, int64_t cap) {
  int64_t pos = 0;
  memset(out, 0, (size_t)cap);
  for (int64_t i = 0; i < n; ++i) {
    const int e = syms[2 * i], len = codes[4 * e];
    const uint32_t bits = (uint32_t)codes[4 * e + 1];
    const int sb = codes[4 * e + 3] != 0;
    if ((pos + len + sb + 7) / 8 > cap)
      return -1;
    for (int k = len - 1; k >= 0; --k, ++pos)
      if ((bits >> k) & 1)
        out[pos >> 3] |= (uint8_t)(0x80 >> (pos & 7));
    if (sb) {
      if (syms[2 * i + 1])
        out[pos >> 3] |= (uint8_t)(0x80 >> (pos & 7));
      ++pos;
    }
  }
  const int64_t bytes = (pos + 31) / 32 * 4;
  return bytes <= cap ? bytes : -1;
}
