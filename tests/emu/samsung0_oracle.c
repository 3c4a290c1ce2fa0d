/* samsung0_oracle.c -- CPU restatement of SamsungV0Decompressor and a writer of its row streams,
 * for the tests of the Samsung V0 GPU path (tests/test_oracle_samsung0.py, tests/test_samsung0_emu.py,
 * tests/test_gpu_samsung0.py).
 *
 * Reference (paths relative to src/librawspeed of rawspeed):
 *   SamsungV0Decompressor::SamsungV0Decompressor  decompressors/SamsungV0Decompressor.cpp:44-58
 *   SamsungV0Decompressor::computeStripes         decompressors/SamsungV0Decompressor.cpp:61-90
 *   SamsungV0Decompressor::decompress             decompressors/SamsungV0Decompressor.cpp:92-102
 *   SamsungV0Decompressor::calcAdj                decompressors/SamsungV0Decompressor.cpp:104-108
 *   SamsungV0Decompressor::decompressStrip        decompressors/SamsungV0Decompressor.cpp:110-204
 *   BitStreamerMSB32 (over-read rule)             bitstreams/BitStreamer.h:96-104, 214-228
 *   BitStreamer (at least 4 bytes)                bitstreams/BitStreamer.h:56-59
 *   ByteStream::check / Buffer::getSubView        io/ByteStream.h:62-69, io/Buffer.h:76-90
 */
#include <stdint.h>
#include <string.h>

/* Outcomes: 0 decoded, else the message the reference throws (S0_MSG_*): */
enum {
  S0_OK = 0,
  S0_LEN_NEG = 1,     /* RDE "Bit length less than 0." */
  S0_LEN_BIG = 2,     /* RDE "Bit Length more than 16." */
  S0_UP_FIRST = 3,    /* RDE "Upward prediction for the first two rows. Raw corrupt" */
  S0_UP_LAST = 4,     /* RDE "Upward prediction for the last block of pixels. Raw corrupt" */
  S0_OVERREAD = 5,    /* IOE "Buffer overflow read in BitStreamer" */
  S0_SHORT = 6,       /* IOE "Bit stream size is smaller than MaxProcessBytes" */
  S0_DIMS = 7,        /* RDE "Unexpected image dimensions found" (constructor) */
  S0_OFFSETS = 8,     /* RDE "Line offsets are out of sequence or slice is empty." (constructor) */
  S0_BS_SKIP = 9,     /* IOE "Out of bounds access in ByteStream" (constructor: bsr.skipBytes) */
  S0_BS_STREAM = 10,  /* IOE "Buffer overflow: image file may be truncated" (constructor: peek/getStream) */
};

/* 32 bits of a row stream from bit p: 32-bit little-endian chunks read most significant bit first,
 * zero past the end */
static uint32_t window32(const uint8_t* s, uint32_t size, uint64_t p) {
  uint64_t v = 0;
  const uint64_t c = p >> 5;
  for (int k = 0; k < 2; ++k) {
    uint32_t w = 0;
    for (int b = 0; b < 4; ++b) {
      const uint64_t at = 4 * (c + (uint64_t)k) + (uint64_t)b;
      if (at < size)
        w |= (uint32_t)s[at] << (8 * b);
    }
    v = (v << 32) | w;
  }
  return (uint32_t)(v >> (32 - (p & 31)));
}

/* BitStreamerMSB32: fill(n) at consumed bit T refills once when fewer than n bits are cached; the
 * refill that starts at byte 4k throws when 4k > size + 8.  Refills are never undone, so the
 * operation that throws is the first one that needs ceil((T + n) / 32) >= (size + 8) / 4 + 2
 * refills. */
static int overread(uint64_t T, uint32_t n, uint32_t size) {
  return (T + n + 31) / 32 >= (uint64_t)((size + 8u) / 4u) + 2u;
}

static int sign_extend(uint32_t v, int b) { return (int)(v << (32 - b)) >> (32 - b); }

/* One row (decompressStrip).  Returns 0 or the message; *fail_block gets the block of the failure. */
static int strip(const uint8_t* s, uint32_t size, int row, int w, uint16_t* out, int pitch,
                 int* fail_block) {
  *fail_block = 0;
  if (size < 4)
    return S0_SHORT;
  int len[4];
  for (int i = 0; i < 4; ++i)
    len[i] = row < 2 ? 7 : 4;
  uint64_t T = 0;
  uint16_t* o = out + (int64_t)row * pitch;
  for (int col = 0; col < w; col += 16) {
    *fail_block = col / 16;
    if (overread(T, 32, size))
      return S0_OVERREAD;
    const uint32_t x = window32(s, size, T);
    const int dir = (int)(x >> 31);
    int op[4];
    for (int i = 0; i < 4; ++i)
      op[i] = (int)((x >> (29 - 2 * i)) & 3u);
    T += 9;
    for (int i = 0; i < 4; ++i) {
      if (op[i] == 3) {
        if (overread(T, 4, size))
          return S0_OVERREAD;
        len[i] = (int)(window32(s, size, T) >> 28);
        T += 4;
      } else if (op[i] == 2) {
        len[i]--;
      } else if (op[i] == 1) {
        len[i]++;
      }
      if (len[i] < 0)
        return S0_LEN_NEG;
      if (len[i] > 16)
        return S0_LEN_BIG;
    }
    if (dir) {
      if (row < 2)
        return S0_UP_FIRST;
      if (col + 16 >= w)
        return S0_UP_LAST;
    }
    for (int half = 0; half < 2; ++half) {
      const int pred = dir ? 0 : (col != 0 ? o[col - 2 + half] : 128);
      for (int c = half; c < 16; c += 2) {
        const int b = len[(half << 1) | (c >> 3)];
        int adj = 0;
        if (b) {
          if (overread(T, (uint32_t)b, size))
            return S0_OVERREAD;
          adj = sign_extend(window32(s, size, T) >> (32 - b), b);
          T += (uint64_t)b;
        }
        if (dir)
          o[col + c] = (uint16_t)(adj + o[col + c - (int64_t)(1 + half) * pitch]);
        else if (col + c < w)
          o[col + c] = (uint16_t)(adj + pred);
      }
    }
  }
  return S0_OK;
}

/* SamsungV0Decompressor(image w x h, bso, bsr).decompress().  `out` is the uncropped image, `pitch`
 * elements per row.  Returns 0 or S0_*; *where gets row << 9 | block of a failure in decompress(). */
int s0_decompress(const uint8_t* bso, uint32_t bso_size, const uint8_t* bsr, uint32_t bsr_size,
                  int w, int h, uint16_t* out, int pitch, uint32_t* where) {
  *where = 0;
  if (w <= 0 || h <= 0 || w < 16 || w > 5546 || h > 3714)
    return S0_DIMS;
  if ((uint64_t)h * 4u > bso_size) /* bso.peekStream(height, 4) */
    return S0_BS_STREAM;
  uint32_t off[3715];
  for (int y = 0; y < h; ++y)
    off[y] = (uint32_t)bso[4 * y] | (uint32_t)bso[4 * y + 1] << 8 | (uint32_t)bso[4 * y + 2] << 16 |
             (uint32_t)bso[4 * y + 3] << 24;
  off[h] = bsr_size;
  if (off[0] > bsr_size) /* bsr.skipBytes(offsets[0]) */
    return S0_BS_SKIP;
  uint64_t pos = off[0];
  uint32_t so[3714], ss[3714];
  for (int y = 0; y < h; ++y) {
    if (off[y] >= off[y + 1])
      return S0_OFFSETS;
    const uint32_t size = off[y + 1] - off[y];
    if (pos + size > bsr_size) /* bsr.getStream(size) */
      return S0_BS_STREAM;
    so[y] = (uint32_t)pos;
    ss[y] = size;
    pos += size;
  }
  for (int row = 0; row < h; ++row) {
    int blk = 0;
    const int rc = strip(bsr + so[row], ss[row], row, w, out, pitch, &blk);
    if (rc) {
      *where = ((uint32_t)row << 9) | (uint32_t)blk;
      return rc;
    }
  }
  for (int row = 0; row < h - 1; row += 2)
    for (int col = 0; col < w - 1; col += 2) {
      const uint16_t t = out[(int64_t)row * pitch + col + 1];
      out[(int64_t)row * pitch + col + 1] = out[(int64_t)(row + 1) * pitch + col];
      out[(int64_t)(row + 1) * pitch + col] = t;
    }
  return S0_OK;
}

/* ---------------------------------------------------------------- writer */

/* The length of group g (0..3) of block k after its header, the reference's way (no range check):
 * lens walks from the row's initial value.  Writes the row stream of one row: per block the header
 * (dir, op[0..3], 4 bits for each op 3) and 16 values in stream order, the low `len` bits of each.
 * An out-of-range length (the reference throws there) writes its values with the length clamped to
 * 0..16.  Returns the number of bytes (a multiple of 4), or -1 if `cap` is too small. */
int64_t s0_write_row(int row, int nb, const uint8_t* dir, const uint8_t* op, const uint8_t* setlen,
                     const int32_t* adj, uint8_t* out, int64_t cap) {
  uint64_t acc = 0;
  int nacc = 0;
  int64_t o = 0;
#define PUT(v, k)                                                                                  \
  do {                                                                                             \
    if ((k) > 0) {                                                                                 \
      acc = (acc << (k)) | ((uint64_t)(v) & ((1ull << (k)) - 1ull));                               \
      nacc += (k);                                                                                 \
    }                                                                                              \
    while (nacc >= 32) {                                                                           \
      if (o + 4 > cap)                                                                             \
        return -1;                                                                                 \
      const uint32_t wv = (uint32_t)(acc >> (nacc - 32));                                          \
      out[o++] = (uint8_t)wv;                                                                      \
      out[o++] = (uint8_t)(wv >> 8);                                                               \
      out[o++] = (uint8_t)(wv >> 16);                                                              \
      out[o++] = (uint8_t)(wv >> 24);                                                              \
      nacc -= 32;                                                                                  \
    }                                                                                              \
  } while (0)
  int len[4];
  for (int i = 0; i < 4; ++i)
    len[i] = row < 2 ? 7 : 4;
  for (int k = 0; k < nb; ++k) {
    PUT(dir[k], 1);
    for (int i = 0; i < 4; ++i)
      PUT(op[4 * k + i], 2);
    for (int i = 0; i < 4; ++i) {
      const int q = op[4 * k + i];
      if (q == 3) {
        PUT(setlen[4 * k + i], 4);
        len[i] = setlen[4 * k + i] & 15;
      } else if (q == 2) {
        len[i]--;
      } else if (q == 1) {
        len[i]++;
      }
    }
    for (int j = 0; j < 16; ++j) {
      int b = len[j >> 2];
      b = b < 0 ? 0 : (b > 16 ? 16 : b);
      PUT((uint32_t)adj[16 * k + j], b);
    }
  }
  if (nacc)
    PUT(0, 32 - nacc);
#undef PUT
  return o;
}

static int bits_for(int a) { /* the least b whose signExtend range [-2^(b-1), 2^(b-1)) holds a */
  if (a == 0)
    return 0;
  int b = 1;
  while (b < 16 && !(a >= -(1 << (b - 1)) && a < (1 << (b - 1))))
    ++b;
  return b;
}

/* Fits a stream to the image `val` (h rows of w values, before the red/blue swap) for the given
 * directions dir[row * nb + k]: computes each pixel's adj from the reference's predictors, then
 * per group the shortest length that holds its adjs and the op that reaches it (0 keep, 1/2 step,
 * 3 set, preferring the shortest).  adj is written in stream order (16 per block).  Returns 0, or
 * -1 when a group needs 16 bits from a length below 15 (no single op reaches it). */
int s0_fit(int w, int h, const uint16_t* val, const uint8_t* dir, uint8_t* op, uint8_t* setlen,
           int32_t* adj) {
  const int nb = (w + 15) / 16;
  for (int row = 0; row < h; ++row) {
    int len[4];
    for (int i = 0; i < 4; ++i)
      len[i] = row < 2 ? 7 : 4;
    for (int k = 0; k < nb; ++k) {
      const int64_t bi = (int64_t)row * nb + k;
      const int col = 16 * k;
      int need[4] = {0, 0, 0, 0};
      for (int j = 0; j < 16; ++j) {
        const int c = j < 8 ? 2 * j : 2 * (j - 8) + 1;
        const int half = c & 1;
        int a = 0;
        if (col + c < w) {
          int pred;
          if (dir[bi])
            pred = val[(int64_t)(row - 1 - half) * w + col + c];
          else
            pred = col ? val[(int64_t)row * w + col - 2 + half] : 128;
          a = (int)(int16_t)(uint16_t)(val[(int64_t)row * w + col + c] - pred);
        }
        adj[16 * bi + j] = a;
        const int b = bits_for(a);
        if (b > need[j >> 2])
          need[j >> 2] = b;
      }
      for (int i = 0; i < 4; ++i) {
        const int t = need[i], L = len[i];
        int q, nl;
        if (t <= L && L <= 16 && (L - t) < 3) {
          q = 0;
          nl = L;
        } else if (t == L + 1 && L + 1 <= 16) {
          q = 1;
          nl = L + 1;
        } else if (t <= 15) {
          q = 3;
          nl = t;
        } else if (L >= 15) {
          q = L == 15 ? 1 : 0;
          nl = 16;
        } else {
          return -1;
        }
        op[4 * bi + i] = (uint8_t)q;
        setlen[4 * bi + i] = (uint8_t)(q == 3 ? nl : 0);
        len[i] = nl;
      }
    }
  }
  return 0;
}
