/* samsung2_oracle.c -- restatement of SamsungV2Decompressor::decompress (decompressors/
 * SamsungV2Decompressor.cpp:145-355, paths relative to src/librawspeed of rawspeed) for the tests, and a
 * writer of V2 row streams.  The constructor's checks and the 16-byte header are done by the caller
 * (tests/samsung2_oracle.py); `data` here is the stream behind the header.
 *
 * Rows: the data position moves to the next multiple of 16 (ByteStream::skipBytes: "Out of bounds
 * access in ByteStream" past the end), a BitStreamerMSB32 is built over the rest ("Bit stream size is
 * smaller than MaxProcessBytes" under 4 bytes), the blocks are decoded, and the position moves on by
 * the pump's stream position, ceil(bits / 8) (skipBytes again).  The pump refills 4 bytes when fewer
 * bits are cached than an operation needs, zero bits behind the buffer, and the refill that starts
 * more than 8 bytes behind the end throws.  Plain C99, no GPU. */
#include <stdint.h>
#include <string.h>

/* outcomes: the reference's messages thrown from decompress() (== RSB200_S2_* of the C ABI) */
enum {
  S2_OK = 0,
  S2_START_MOTION, /* RDE "At start of image and motion isn't 7. File corrupted?"  */
  S2_MOTION_BEGIN, /* RDE "Bad motion %d at the beginning of the row"              */
  S2_MOTION_END,   /* RDE "Bad motion %d at the end of the row"                    */
  S2_UNDERFLOW,    /* RDE "Difference bits underflow. File corrupted?"             */
  S2_TOO_MANY,     /* RDE "Too many difference bits (%u). File corrupted?"         */
  S2_OVERREAD,     /* IOE "Buffer overflow read in BitStreamer"                    */
  S2_SHORT,        /* IOE "Bit stream size is smaller than MaxProcessBytes"        */
  S2_BYTESTREAM    /* IOE "Out of bounds access in ByteStream"                     */
};
enum { F_SKIP = 1, F_MV = 2, F_QP = 4 };

typedef struct {
  const uint8_t* data;
  uint32_t size;
  uint32_t pos; /* bytes consumed by refills */
  uint64_t cache;
  int fill;
  int err;
} Pump;

static void pump_fill(Pump* p, int n) {
  if (p->fill >= n)
    return;
  if ((uint64_t)p->pos > (uint64_t)p->size + 8) {
    p->err = 1;
    return;
  }
  uint32_t v = 0; /* MSB32: a little-endian 32-bit chunk, most significant bit first */
  for (int k = 3; k >= 0; --k)
    v = (v << 8) | (p->pos + (uint32_t)k < p->size ? p->data[p->pos + (uint32_t)k] : 0u);
  p->cache = (p->cache << 32) | v;
  p->fill += 32;
  p->pos += 4;
}

static uint32_t get(Pump* p, int n) {
  pump_fill(p, n);
  if (p->err)
    return 0;
  p->fill -= n;
  return (uint32_t)(p->cache >> p->fill) & (uint32_t)((1ull << n) - 1);
}

static int clampb(int v, int bits) {
  const int m = (1 << bits) - 1;
  return v < 0 ? 0 : (v > m ? m : v);
}

/* ends (optional): the data position behind each decoded row.
 * `where` = value << 22 | row << 9 | block of the failure (block = width / 16 for the skip behind a
 * row, 0 for the alignment skip and the pump at a row's start). */
#define FAIL(code, val, blk)                                                                         \
  do {                                                                                               \
    *where = (uint32_t)(val) << 22 | (uint32_t)row << 9 | (uint32_t)(blk);                           \
    return (code);                                                                                   \
  } while (0)

int s2_decompress(const uint8_t* data, uint32_t size, int bits, int flags, int init, int w, int h,
                  uint16_t* img, int pitch, uint32_t* where, uint32_t* ends) {
  static const int off[7] = {-4, -2, -2, 0, 0, 2, 4}, avg[7] = {0, 0, 1, 0, 1, 0, 0};
  static const int sv[3] = {0, -2, 2};
  const int nb = w / 16;
  uint32_t dpos = 0;
  *where = 0;
  for (int row = 0; row < h; ++row) {
    if (dpos & 15u) {
      const uint32_t n = 16u - (dpos & 15u);
      if ((uint64_t)dpos + n > size)
        FAIL(S2_BYTESTREAM, 0, 0);
      dpos += n;
    }
    if (size - dpos < 4u)
      FAIL(S2_SHORT, 0, 0);
    Pump p = {data + dpos, size - dpos, 0, 0, 0, 0};
    int motion = 7, scale = 0, mode[3][2];
    for (int c = 0; c < 3; ++c)
      mode[c][0] = mode[c][1] = row < 2 ? 7 : 4;
    uint16_t* out = img + (size_t)row * pitch;
    for (int k = 0; k < nb; ++k) {
      const int col = 16 * k;
      int base[16], len[4] = {0, 0, 0, 0};
#define GET(n) get(&p, (n)); if (p.err) FAIL(S2_OVERREAD, 0, k)
      if (!(flags & F_QP) && col % 64 == 0) {
        const uint32_t i = GET(2);
        if (i < 3) {
          scale += sv[i];
        } else {
          const uint32_t s = GET(12);
          scale = (int)s;
        }
      }
      if (flags & F_MV) {
        const uint32_t b = GET(1);
        motion = b ? 3 : 7;
      } else {
        const uint32_t keep = GET(1);
        if (!keep) {
          const uint32_t m = GET(3);
          motion = (int)m;
        }
      }
      if (row < 2 && motion != 7)
        FAIL(S2_START_MOTION, 0, k);
      if (motion == 7) {
        for (int i = 0; i < 16; ++i)
          base[i] = col == 0 ? init : out[col - 2 + (i & 1)];
      } else {
        for (int i = 0; i < 16; ++i) {
          int rr = row, rc = col + i + off[motion];
          if ((row + i) & 1) {
            rr -= 2;
          } else {
            rr -= 1;
            rc += (i & 1) ? -1 : 1;
          }
          if (rc < 0)
            FAIL(S2_MOTION_BEGIN, motion, k);
          if (rc >= w || (avg[motion] && rc + 2 >= w))
            FAIL(S2_MOTION_END, motion, k);
          const uint16_t* ref = img + (size_t)rr * pitch;
          base[i] = avg[motion] ? (ref[rc] + ref[rc + 2] + 1) >> 1 : ref[rc];
        }
      }
      int skip = 0;
      if (!(flags & F_SKIP)) {
        const uint32_t s = GET(1);
        skip = s != 0;
      }
      if (!skip) {
        uint32_t fl[4];
        for (int i = 0; i < 4; ++i) {
          const uint32_t f = GET(2);
          fl[i] = f;
        }
        for (int i = 0; i < 4; ++i) {
          const int c = (row % 2) ? i >> 1 : ((i >> 1) + 2) % 3; /* 0 green, 1 blue, 2 red */
          if (fl[i] == 0) {
            len[i] = mode[c][0];
          } else if (fl[i] == 1) {
            len[i] = mode[c][0] + 1;
          } else if (fl[i] == 2) {
            if (mode[c][0] == 0)
              FAIL(S2_UNDERFLOW, 0, k);
            len[i] = mode[c][0] - 1;
          } else {
            const uint32_t l = GET(4);
            len[i] = (int)l;
          }
          mode[c][0] = mode[c][1];
          mode[c][1] = len[i];
          if (len[i] > bits + 1)
            FAIL(S2_TOO_MANY, len[i], k);
        }
      }
      int d[16], sh[16];
      for (int i = 0; i < 16; ++i) {
        const int n = len[i >> 2];
        d[i] = 0;
        if (n) {
          const uint32_t v = GET(n);
          d[i] = (int)(int32_t)(v << (32 - n)) >> (32 - n);
        }
      }
#undef GET
      for (int i = 0; i < 16; ++i) {
        const int q = (row % 2) ? ((i % 8) << 1) - (i >> 3) + 1 : ((i % 8) << 1) + (i >> 3);
        sh[q] = d[i];
      }
      for (int i = 0; i < 16; ++i)
        out[col + i] = (uint16_t)clampb(base[i] + sh[i] * (scale * 2 + 1) + scale, bits);
    }
    const uint32_t sp = p.pos - (uint32_t)(p.fill >> 3);
    if ((uint64_t)dpos + sp > size)
      FAIL(S2_BYTESTREAM, 0, nb);
    dpos += sp;
    if (ends)
      ends[row] = dpos;
  }
  return S2_OK;
}

/* ------------------------------------------------------------------ writer */
typedef struct {
  uint8_t* out;
  int64_t cap, n; /* bytes written (whole 32-bit chunks) */
  uint32_t acc;
  int nacc;
  uint64_t bits; /* bits put */
} Writer;

static void put(Writer* wr, uint32_t v, int n) {
  for (int b = n - 1; b >= 0; --b) {
    wr->acc = (wr->acc << 1) | ((v >> b) & 1u);
    wr->bits++;
    if (++wr->nacc == 32) {
      if (wr->n + 4 <= wr->cap)
        for (int k = 0; k < 4; ++k)
          wr->out[wr->n + k] = (uint8_t)(wr->acc >> (8 * k));
      wr->n += 4;
      wr->acc = 0;
      wr->nacc = 0;
    }
  }
}

static uint64_t rng_next(uint64_t* s) {
  *s ^= *s << 13;
  *s ^= *s >> 7;
  *s ^= *s << 17;
  return *s;
}

static int need_bits(int d) {
  int n = 0;
  while (n < 16 && !(d >= -(1 << n >> 1) && d <= ((1 << n) >> 1) - (n ? 1 : 0)))
    ++n;
  return n;
}

static int motion_ok(int motion, int row, int col, int w) {
  static const int off[7] = {-4, -2, -2, 0, 0, 2, 4}, avg[7] = {0, 0, 1, 0, 1, 0, 0};
  if (motion == 7)
    return 1;
  if (row < 2)
    return 0;
  for (int i = 0; i < 16; ++i) {
    int rc = col + i + off[motion];
    if (!((row + i) & 1))
      rc += (i & 1) ? -1 : 1;
    if (rc < 0 || rc >= w || (avg[motion] && rc + 2 >= w))
      return 0;
  }
  return 1;
}

static void baseline(const uint16_t* img, int pitch, int row, int col, int motion, int init, int* base) {
  static const int off[7] = {-4, -2, -2, 0, 0, 2, 4}, avg[7] = {0, 0, 1, 0, 1, 0, 0};
  for (int i = 0; i < 16; ++i) {
    if (motion == 7) {
      base[i] = col == 0 ? init : img[(size_t)row * pitch + col - 2 + (i & 1)];
      continue;
    }
    int rr = row, rc = col + i + off[motion];
    if ((row + i) & 1) {
      rr -= 2;
    } else {
      rr -= 1;
      rc += (i & 1) ? -1 : 1;
    }
    const uint16_t* ref = img + (size_t)rr * pitch;
    base[i] = avg[motion] ? (ref[rc] + ref[rc + 2] + 1) >> 1 : ref[rc];
  }
}

/* Writes the data behind the header for `vals` (h rows of w values < 2^bits, row stride `pitch`).
 * policy: 0 the motion with the fewest difference bits (3 or 7 under MV), 1 always 7, 2 always 3
 * (up), 3 averaging (2 / 4 alternating), 4 a random valid motion; blocks fall back to 7 where the
 * motion is not allowed.  Scale stays 0 (the +0 code).  All-zero blocks are skip blocks unless
 * flags has SKIP.  Each row ends with random bits to the end of its byte, then random bytes up to
 * the next multiple of 16: the decoder must never read them.  Returns the byte count, or -1 if
 * `cap` is too small.  `tmp` holds h * pitch values (the decoded image). */
int64_t s2_encode(const uint16_t* vals, int w, int h, int pitch, int bits, int flags, int init, int policy,
                  uint64_t seed, uint16_t* tmp, uint8_t* out, int64_t cap) {
  Writer wr = {out, cap, 0, 0, 0, 0};
  uint64_t rs = seed * 2654435761ull + 0x9E3779B97F4A7C15ull;
  const int nb = w / 16;
  for (int row = 0; row < h; ++row) {
    int motion = 7, state[4];
    for (int i = 0; i < 4; ++i)
      state[i] = row < 2 ? 7 : 4;
    for (int k = 0; k < nb; ++k) {
      const int col = 16 * k;
      int base[16], want = 7;
      if (!(flags & F_QP) && col % 64 == 0)
        put(&wr, 0, 2);
      if (policy == 0) {
        int best = 1 << 30;
        for (int m = 0; m < 8; ++m) {
          if (m == 7 || (flags & F_MV ? m == 3 : 1)) {
            if (!motion_ok(m, row, col, w))
              continue;
            baseline(tmp, pitch, row, col, m, init, base);
            int cost = 0;
            for (int i = 0; i < 16; ++i)
              cost += need_bits((int)vals[(size_t)row * pitch + col + i] - base[i]);
            if (cost < best) {
              best = cost;
              want = m;
            }
          }
        }
      } else if (policy == 2) {
        want = 3;
      } else if (policy == 3) {
        want = (k & 1) ? 4 : 2;
      } else if (policy == 4) {
        want = (int)(rng_next(&rs) % 8);
      }
      if (flags & F_MV && want != 7)
        want = 3;
      if (!motion_ok(want, row, col, w))
        want = 7;
      if (flags & F_MV) {
        put(&wr, want == 3, 1);
      } else if (want == motion) {
        put(&wr, 1, 1);
      } else {
        put(&wr, 0, 1);
        put(&wr, (uint32_t)want, 3);
      }
      motion = want;
      baseline(tmp, pitch, row, col, motion, init, base);
      int d[16], st[16], zero = 1;
      for (int i = 0; i < 16; ++i) {
        d[i] = (int)vals[(size_t)row * pitch + col + i] - base[i];
        tmp[(size_t)row * pitch + col + i] = vals[(size_t)row * pitch + col + i];
        zero &= d[i] == 0;
      }
      for (int i = 0; i < 16; ++i) {
        const int q = (row % 2) ? ((i % 8) << 1) - (i >> 3) + 1 : ((i % 8) << 1) + (i >> 3);
        st[i] = d[q];
      }
      if (!(flags & F_SKIP)) {
        put(&wr, zero, 1);
        if (zero)
          continue;
      }
      int len[4], fl[4];
      for (int g = 0; g < 4; ++g) {
        int need = 0;
        for (int j = 0; j < 4; ++j) {
          const int n = need_bits(st[4 * g + j]);
          need = n > need ? n : need;
        }
        const int prev = state[g];
        if (prev >= 1 && prev - 1 >= need) {
          fl[g] = 2;
          len[g] = prev - 1;
        } else if (prev >= need) {
          fl[g] = 0;
          len[g] = prev;
        } else if (prev + 1 == need) {
          fl[g] = 1;
          len[g] = need;
        } else {
          fl[g] = 3;
          len[g] = need;
        }
        state[g] = len[g];
      }
      for (int g = 0; g < 4; ++g)
        put(&wr, (uint32_t)fl[g], 2);
      for (int g = 0; g < 4; ++g)
        if (fl[g] == 3)
          put(&wr, (uint32_t)len[g], 4);
      for (int i = 0; i < 16; ++i)
        if (len[i >> 2])
          put(&wr, (uint32_t)st[i] & ((1u << len[i >> 2]) - 1u), len[i >> 2]);
    }
    /* random bits to the end of the byte, random bytes to the next multiple of 16 */
    while (wr.bits % 8)
      put(&wr, (uint32_t)(rng_next(&rs) & 1u), 1);
    while ((wr.bits / 8) % 16)
      put(&wr, (uint32_t)(rng_next(&rs) & 0xFFu), 8);
  }
  if (wr.n > cap)
    return -1;
  return wr.n;
}
