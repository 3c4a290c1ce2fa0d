/* arw1_oracle.c -- CPU restatement of SonyArw1Decompressor and a writer of its streams, for the
 * tests of the ARW1 GPU path (tests/test_oracle_arw1.py, tests/test_gpu_arw1.py).
 *
 * Reference (paths relative to src/librawspeed of rawspeed):
 *   SonyArw1Decompressor::SonyArw1Decompressor  decompressors/SonyArw1Decompressor.cpp:39-50
 *   SonyArw1Decompressor::getDiff               decompressors/SonyArw1Decompressor.cpp:52-57
 *   SonyArw1Decompressor::decompress            decompressors/SonyArw1Decompressor.cpp:58-92
 *   BitStreamerMSB (over-read rule)             bitstreams/BitStreamer.h:100-131
 *   BitStreamerMSB (at least 4 bytes)           bitstreams/BitStreamer.h:56-60
 *   PrefixCodeDecoder<>::extend                 codes/AbstractPrefixCodeDecoder.h:43-76
 */
#include <stdint.h>
#include <string.h>

/* BitStreamerMSB reads zero bits behind the buffer and refills 4 bytes at a time; the refill that
 * starts more than 8 bytes behind the end throws.  decompress() fills to 32 bits before every
 * symbol, so before a symbol that starts at stream bit T the pump has done
 * (T >> 5) + 1 + (T & 31 ? 1 : 0) refills, and refill number (size + 8) / 4 + 2 throws. */
static int overread(uint64_t T, uint32_t size) {
  const uint64_t refills = (T >> 5) + 1u + ((T & 31u) ? 1u : 0u);
  return refills >= (uint64_t)((size + 8u) / 4u) + 2u;
}

static uint32_t bits_at(const uint8_t* in, uint32_t size, uint64_t pos, int n) {
  uint32_t v = 0;
  for (int k = 0; k < n; ++k) {
    const uint64_t p = pos + (uint64_t)k;
    const uint32_t byte = (p >> 3) < size ? in[p >> 3] : 0u;
    v = (v << 1) | ((byte >> (7 - (p & 7))) & 1u);
  }
  return v;
}

static int extend(uint32_t diff, uint32_t len) {
  if ((diff & (1u << (len - 1))) == 0)
    return (int)diff - (int)((1u << len) - 1u);
  return (int)diff;
}

/* Returns 0 (decoded), 1 (RawDecoderException "Error decompressing": *where = row << 14 | col of
 * the pixel), 2 (IOException from the bit pump) or 3 (rejected by the constructor).  `out` is the
 * uncropped image, `pitch` elements per row; only decoded pixels are written.  *consumed_bits gets
 * the bit position behind the last symbol read. */
int arw1_decompress(const uint8_t* in, uint32_t size, int w, int h, uint16_t* out, int pitch,
                    uint32_t* where, uint64_t* consumed_bits) {
  *where = 0;
  if (w <= 0 || h <= 0 || h % 2 != 0 || w > 4600 || h > 3072)
    return 3;
  *consumed_bits = 0;
  if (size < 4) /* BitStreamerMSB's constructor: "Bit stream size is smaller than MaxProcessBytes" */
    return 2;
  uint64_t T = 0;
  int pred = 0;
  int rc = 0;
  for (int col = w - 1; col >= 0 && rc == 0; col--) {
    for (int row = 0; row < h + 1; row += 2) {
      if (overread(T, size)) { /* bits.fill(32) */
        rc = 2;
        break;
      }
      if (row == h)
        row = 1;
      uint32_t len = 4 - bits_at(in, size, T, 2);
      T += 2;
      if (len == 3) {
        if (bits_at(in, size, T, 1))
          len = 0;
        T += 1;
      }
      if (len == 4)
        while (len < 17) {
          const uint32_t b = bits_at(in, size, T, 1);
          T += 1;
          if (b)
            break;
          len++;
        }
      int diff = 0;
      if (len) {
        diff = extend(bits_at(in, size, T, (int)len), len);
        T += len;
      }
      pred += diff;
      if (pred < 0 || pred > 4095) { /* !isIntN(pred, 12) */
        *where = ((uint32_t)row << 14) | (uint32_t)col;
        rc = 1;
        break;
      }
      out[(int64_t)row * pitch + col] = (uint16_t)pred;
    }
  }
  *consumed_bits = T;
  return rc;
}

/* Writer: one symbol per difference, with the shortest length that holds it (|d| < 2^17; the
 * length is 0 for d == 0, else the bit length of |d|).  A length may also be forced per symbol
 * (lens[i] >= 0; the value must then fit it).  Returns the number of bytes (the last one padded
 * with `pad_bit`), or -1 if `cap` is too small. */
int64_t arw1_encode(const int32_t* diffs, const int8_t* lens, int64_t n, uint8_t* out, int64_t cap,
                    int pad_bit) {
  uint64_t acc = 0;
  int nacc = 0;
  int64_t o = 0;
#define PUT(v, k)                                                                                  \
  do {                                                                                             \
    acc = (acc << (k)) | ((uint64_t)(v) & ((1ull << (k)) - 1ull));                                 \
    nacc += (k);                                                                                   \
    while (nacc >= 8) {                                                                            \
      if (o >= cap)                                                                                \
        return -1;                                                                                 \
      out[o++] = (uint8_t)(acc >> (nacc - 8));                                                     \
      nacc -= 8;                                                                                   \
    }                                                                                              \
  } while (0)
  for (int64_t i = 0; i < n; ++i) {
    const int32_t d = diffs[i];
    const uint32_t a = (uint32_t)(d < 0 ? -d : d);
    int len = 0;
    while (len < 32 && (a >> len))
      ++len;
    if (lens && lens[i] >= 0)
      len = lens[i];
    if (len > 17)
      return -2;
    /* code: 11 -> 1, 10 -> 2, 011 -> 0, 010 -> 3, 00 0^(len-4) 1 -> 4..16, 00 0^13 -> 17 */
    if (len == 1)
      PUT(3, 2);
    else if (len == 2)
      PUT(2, 2);
    else if (len == 0)
      PUT(3, 3);
    else if (len == 3)
      PUT(2, 3);
    else if (len < 17)
      PUT(1, len - 1);
    else
      PUT(0, 15);
    if (len) {
      /* extend() inverse: negative values are stored as d + 2^len - 1 */
      const uint32_t v = d < 0 ? (uint32_t)(d + (int32_t)((1u << len) - 1u)) : (uint32_t)d;
      PUT(v, len);
    }
  }
  if (nacc) {
    const int k = 8 - nacc;
    PUT(pad_bit ? (1u << k) - 1u : 0u, k);
  }
#undef PUT
  return o;
}
