/* samsung1_oracle.c -- restatement of SamsungV1Decompressor (decompressors/SamsungV1Decompressor.cpp:
 * 45-140, paths relative to src/librawspeed of rawspeed) for the tests, and a writer of V1 streams.
 *
 * The pump is BitStreamerMSB as the reference drives it: the constructor throws for fewer than 4 bytes
 * (BitStreamer.h:56-60); fill(23) before every symbol refills 4 bytes (zero bits behind the buffer)
 * when fewer than 23 bits are cached, and the refill that starts more than 8 bytes behind the end
 * throws (BitStreamer.h:125-127).  Plain C99, no GPU. */
#include <stdint.h>
#include <string.h>

enum { S1_OK = 0, S1_OOB, S1_OVERREAD, S1_SHORT, S1_DIMS, S1_BITS };

/* SamsungV1Decompressor.cpp:88-101: (encLen, diffLen), code intervals assigned in this order */
static const uint8_t TAB[14][2] = {{3, 4}, {3, 7}, {2, 6},   {2, 5},   {4, 3}, {6, 0}, {7, 9},
                                   {8, 10}, {9, 11}, {10, 12}, {10, 13}, {5, 1}, {4, 8}, {4, 2}};

typedef struct {
  const uint8_t* data;
  uint32_t size;
  uint32_t pos;  /* bytes consumed by refills */
  uint64_t cache;
  int fill;
} Pump;

/* 0, or -1 when the refill throws */
static int pump_fill(Pump* p, int nbits) {
  if (p->fill >= nbits)
    return 0;
  if ((uint64_t)p->pos + 4 > p->size && (uint64_t)p->pos > (uint64_t)p->size + 8)
    return -1;
  uint32_t v = 0;
  for (int k = 0; k < 4; ++k)
    v = (v << 8) | (p->pos + k < p->size ? p->data[p->pos + k] : 0u);
  p->cache |= (uint64_t)v << (32 - p->fill);
  p->fill += 32;
  p->pos += 4;
  return 0;
}

static uint32_t pump_peek(const Pump* p, int n) { return (uint32_t)(p->cache >> (64 - n)); }
static void pump_skip(Pump* p, int n) {
  p->cache <<= n;
  p->fill -= n;
}

/* decompress() on an image of w x h uint16 pixels, row pitch `pitch` elements (pixels the decode does
 * not reach keep their value).  -> S1_*, *where = row << 14 | col of the failing pixel. */
int s1_decompress(const uint8_t* data, uint32_t size, int w, int h, int bit, uint16_t* img, int pitch,
                  uint32_t* where) {
  *where = 0;
  if (bit != 12)
    return S1_BITS;
  if (w <= 0 || h <= 0 || w % 32 != 0 || h % 2 != 0 || w > 5664 || h > 3714)
    return S1_DIMS;
  uint8_t enc[1024][2];
  {
    uint32_t n = 0;
    for (int i = 0; i < 14; ++i)
      for (int c = 0; c < (1024 >> TAB[i][0]); ++c, ++n) {
        enc[n][0] = TAB[i][0];
        enc[n][1] = TAB[i][1];
      }
  }
  if (size < 4)
    return S1_SHORT;
  Pump p = {data, size, 0, 0, 0};
  for (int row = 0; row < h; ++row) {
    int pred[2] = {0, 0};
    if (row >= 2) {
      pred[0] = img[(size_t)(row - 2) * pitch];
      pred[1] = img[(size_t)(row - 2) * pitch + 1];
    }
    for (int col = 0; col < w; ++col) {
      *where = ((uint32_t)row << 14) | (uint32_t)col;
      if (pump_fill(&p, 23))
        return S1_OVERREAD;
      const uint32_t c = pump_peek(&p, 10);
      pump_skip(&p, enc[c][0]);
      const int len = enc[c][1];
      int32_t diff = 0;
      if (len) {
        const uint32_t v = pump_peek(&p, len);
        pump_skip(&p, len);
        diff = (int32_t)v;
        if ((v & (1u << (len - 1))) == 0)
          diff -= (1 << len) - 1;
      }
      pred[col & 1] += diff;
      const int value = pred[col & 1];
      if (((uint32_t)value >> 12) != 0)
        return S1_OOB;
      img[(size_t)row * pitch + col] = (uint16_t)value;
    }
  }
  return S1_OK;
}

/* The stream of the differences d[0..n) (|d| < 2^13) into out (zero bits up to the next byte).
 * -> bytes written, -1 if cap is too small or a difference has no code. */
int64_t s1_encode(const int32_t* d, int64_t n, uint8_t* out, int64_t cap) {
  uint32_t code[14], clen[14]; /* per diffLen: code, its length */
  {
    uint32_t start = 0;
    for (int i = 0; i < 14; ++i) {
      const uint32_t el = TAB[i][0];
      code[TAB[i][1]] = start >> (10 - el);
      clen[TAB[i][1]] = el;
      start += 1024u >> el;
    }
  }
  memset(out, 0, (size_t)cap);
  uint64_t bitpos = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int32_t v = d[i];
    const uint32_t a = (uint32_t)(v < 0 ? -v : v);
    uint32_t len = 0;
    while ((a >> len) != 0)
      ++len;
    if (len > 13)
      return -1;
    const uint32_t extra = v >= 0 ? (uint32_t)v : (uint32_t)(v + (1 << len) - 1);
    const uint64_t sym = ((uint64_t)code[len] << len) | (len ? extra : 0u);
    const uint32_t nb = clen[len] + len;
    if ((int64_t)((bitpos + nb + 7) / 8) > cap)
      return -1;
    for (uint32_t k = 0; k < nb; ++k) {
      const uint32_t bitv = (uint32_t)(sym >> (nb - 1 - k)) & 1u;
      if (bitv)
        out[(bitpos + k) >> 3] |= (uint8_t)(0x80u >> ((bitpos + k) & 7));
    }
    bitpos += nb;
  }
  return (int64_t)((bitpos + 7) / 8);
}

/* The differences the range decoder leaves in stream order: the first n symbols of data read as the
 * reference reads them (zero bits behind the buffer), and each symbol's start bit. */
void s1_parse(const uint8_t* data, uint32_t size, int64_t n, int16_t* diffs, uint64_t* starts) {
  uint8_t enc[1024][2];
  {
    uint32_t k = 0;
    for (int i = 0; i < 14; ++i)
      for (int c = 0; c < (1024 >> TAB[i][0]); ++c, ++k) {
        enc[k][0] = TAB[i][0];
        enc[k][1] = TAB[i][1];
      }
  }
  uint64_t p = 0;
  for (int64_t i = 0; i < n; ++i) {
    uint32_t win = 0; /* 32 bits from p */
    for (int b = 0; b < 32; ++b) {
      const uint64_t q = p + (uint64_t)b;
      const uint32_t byte = q / 8 < size ? data[q / 8] : 0u;
      win = (win << 1) | ((byte >> (7 - q % 8)) & 1u);
    }
    const uint32_t el = enc[win >> 22][0], dl = enc[win >> 22][1];
    int32_t d = 0;
    if (dl) {
      const uint32_t v = (win << el) >> (32 - dl);
      d = (int32_t)v;
      if ((v & (1u << (dl - 1))) == 0)
        d -= (1 << dl) - 1;
    }
    starts[i] = p;
    diffs[i] = (int16_t)d;
    p += el + dl;
  }
}
