/* kodak_oracle.c -- CPU restatement of the Kodak DCR decompressor (KodakDecompressor,
 * decompressors/KodakDecompressor.cpp:46-150) and a writer of its streams, for the tests.  Test
 * infrastructure: pinned against the reference's own decompressor by tests/test_oracle_kodak.py. */
#include <stdint.h>
#include <string.h>

/* outcomes (KD_VALUE and KD_OVERFLOW are RSB200_KODAK_* of the C ABI) */
enum { KD_OK = 0, KD_VALUE = 1, KD_OVERFLOW = 2, KD_CPP = 3, KD_DIMS = 4, KD_BPS = 5, KD_BYTESTREAM = 6 };

/* ByteStream reads: -1 once past the end */
typedef struct {
  const uint8_t* d;
  uint32_t size, pos;
} Bs;

static int get_byte(Bs* b, int* v) {
  if (b->pos >= b->size)
    return -1;
  *v = b->d[b->pos++];
  return 0;
}

/* decodeSegment (KodakDecompressor.cpp:67-118): -1 when it reads past the end */
static int decode_segment(Bs* in, uint32_t bsize, int16_t* out) {
  uint8_t blen[512];
  uint64_t bitbuf = 0;
  uint32_t bits = 0;
  int v, w;
  for (uint32_t i = 0; i < bsize; i += 2) {
    if (get_byte(in, &v))
      return -1;
    blen[i] = (uint8_t)(v & 15);
    blen[i + 1] = (uint8_t)(v >> 4);
  }
  if ((bsize & 7) == 4) {
    if (get_byte(in, &v) || get_byte(in, &w))
      return -1;
    bitbuf = ((uint64_t)v << 8) + (uint64_t)w;
    bits = 16;
  }
  for (uint32_t i = 0; i < bsize; i++) {
    const uint32_t len = blen[i];
    if (bits < len) {
      for (uint32_t j = 0; j < 32; j += 8) {
        if (get_byte(in, &v))
          return -1;
        bitbuf += (uint64_t)(int64_t)v << (bits + (j ^ 8));
      }
      bits += 32;
    }
    const uint32_t diff = (uint32_t)bitbuf & (0xffffu >> (16 - len));
    bitbuf >>= len;
    bits -= len;
    int x = (int)diff;
    if (len != 0 && (diff & (1u << (len - 1))) == 0)
      x -= (1 << len) - 1;
    out[i] = (int16_t)x;
  }
  return 0;
}

/* The constructor's checks and decompress().  mode: 0 no table (or uncorrectedRawValues), 1 a plain
 * table (65536 entries), 2 a dithered one (TableLookUp's 2 x 65536 {base, delta}).  img: h rows of
 * pitch elements.  row / col: the failing pixel (KD_VALUE) or the first of the failing segment
 * (KD_OVERFLOW); value: the value KD_VALUE prints. */
int kd_decompress(const uint8_t* data, uint32_t size, int w, int h, int bps, int cpp, int mode,
                  const uint16_t* table, uint16_t* img, int pitch, int* row, int* col, int* value) {
  *row = *col = *value = 0;
  if (cpp != 1)
    return KD_CPP;
  if (w <= 0 || h <= 0 || w % 4 != 0 || w > 4516 || h > 3012)
    return KD_DIMS;
  if (bps != 10 && bps != 12)
    return KD_BPS;
  if ((uint64_t)size < (uint64_t)w * (uint64_t)h / 2)
    return KD_BYTESTREAM;
  Bs in = {data, size, 0};
  uint32_t random = 0;
  int16_t buf[256];
  for (int r = 0; r < h; r++) {
    for (int c = 0; c < w;) {
      const int len = w - c < 256 ? w - c : 256;
      if (decode_segment(&in, (uint32_t)len, buf)) {
        *row = r;
        *col = c;
        return KD_OVERFLOW;
      }
      int pred[2] = {0, 0};
      for (int i = 0; i < len; ++i, ++c) {
        pred[i & 1] += buf[i];
        const int v = pred[i & 1];
        if (((uint32_t)v >> bps) != 0) {
          *row = r;
          *col = c;
          *value = v;
          return KD_VALUE;
        }
        uint16_t* dst = img + (size_t)r * pitch + c;
        if (mode == 0) {
          *dst = (uint16_t)v;
        } else if (mode == 1) {
          *dst = table[v];
        } else { /* RawImageDataU16::setWithLookUp, common/RawImage.h:335-353 */
          const uint32_t base = table[2 * v], delta = table[2 * v + 1];
          *dst = (uint16_t)(base + ((delta * (random & 2047) + 1024) >> 12));
          random = 15700 * (random & 65535) + (random >> 16);
        }
      }
    }
  }
  return KD_OK;
}

/* Writer: lens[i] (0..15) and codes[i] (the lens[i] low bits) of every pixel in raster order, cut into
 * the decompressor's segments: the header nibbles (low first), then the codes as a bit string of
 * 16-bit big-endian words, LSB first, 2 bytes when the segment's size is 4 (mod 8) and then 4-byte
 * groups, as many as the reader takes.  Returns the bytes written, or -1 past cap. */
int64_t kd_write(const uint8_t* lens, const uint16_t* codes, int w, int h, uint8_t* out, int64_t cap) {
  int64_t n = 0;
  for (int r = 0; r < h; ++r) {
    for (int c0 = 0; c0 < w; c0 += 256) {
      const int b = w - c0 < 256 ? w - c0 : 256;
      const size_t at = (size_t)r * w + c0;
      if (n + b / 2 > cap)
        return -1;
      uint32_t s = 0;
      for (int i = 0; i < b; i += 2) {
        out[n++] = (uint8_t)((lens[at + i] & 15) | (lens[at + i + 1] & 15) << 4);
        s += (lens[at + i] & 15u) + (lens[at + i + 1] & 15u);
      }
      const uint32_t e = (b & 7) == 4 ? 2 : 0;
      const uint32_t pay = e + 4 * ((s > 8 * e ? s - 8 * e + 31 : 0) / 32);
      if (n + (int64_t)pay > cap)
        return -1;
      memset(out + n, 0, pay);
      uint32_t bit = 0;
      for (int i = 0; i < b; ++i) {
        const uint32_t L = lens[at + i] & 15u, v = codes[at + i] & ((1u << L) - 1u);
        for (uint32_t k = 0; k < L; ++k, ++bit) {
          if ((v >> k) & 1u) {
            const uint32_t word = bit >> 4, wb = bit & 15u;
            out[n + 2 * word + (wb < 8 ? 1 : 0)] |= (uint8_t)(1u << (wb & 7u));
          }
        }
      }
      n += pay;
    }
  }
  return n;
}
