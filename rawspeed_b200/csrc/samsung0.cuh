// samsung0.cuh -- K13: Samsung SRW V0 row codec (SamsungV0Decompressor), sm_90a.
//
// Replaces SamsungV0Decompressor::decompress (decompressors/SamsungV0Decompressor.cpp:92-204).  One
// row = one MSB32 bit stream (BitStreamerMSB32); its block lengths restart at every row, so the parse
// is exact and parallel across rows.  The values are not: a pixel of a block that predicts "left"
// adds its difference to the last same-parity pixel of the previous block of its row (128 at column
// 0), one that predicts "up" to the pixel of its column one row (even columns) or two rows (odd
// columns) above.  Every pixel has one parent, so the image is a forest rooted in the constant 128,
// and all sums are taken mod 2^16.
//
// Stages (one launch each for all frames of a plan):
//   s0_walk_kernel   a thread per row: block headers only (9..25 bits each) -> one descriptor per
//                    block (bit of its first pixel, four lengths, dir, pixels before an over-read),
//                    and the row's first failure; descriptors from the failure on are dead
//   s0_diff_kernel   a warp per row: every difference of the row (2 B/px scratch)
//   s0_node_kernel   block nodes N(r,k,p) = the last parity-p pixel of block k (column 16k+14+p):
//                    a left block's node hangs off N(r,k-1,p) (or the root), an up block's off
//                    N(r-1-p,k,p), the same column one or two rows up
//   s0_jump_kernel   pointer jumping (Wyllie) over the nodes, ceil(log2(h + nb + 1)) rounds fixed on
//                    the host, ping-pong buffers
//   s0_scan_kernel   segmented scans down the columns of 32-row tiles (even columns: one chain of step
//   s0_carry_kernel  1; odd columns: two of step 2), reset at every left block to difference + node;
//   s0_store_kernel  a carry pass over the tiles of each column; the tiles again with their carry,
//                    through shared memory to the image with the red/blue swap (no error) or the
//                    reference's partial-write mask (error)
// No index depends on stream content without a bound: dead descriptors and the root stand in for
// invalid parents, up moves exist only from row 2 and never in the last block.
#pragma once

#ifndef RSB200_EMU
#include "common.cuh"
#endif
#include "phaseone.cuh" // p1_window: 32 bits of an MSB32 strip from any bit, zero past its end
#include <stdint.h>

namespace rsb200 {

constexpr int S0W_NT = 64;   // walk: rows per CTA
constexpr int S0D_NT = 128;  // differences: 4 rows per CTA
constexpr int S0N_NT = 256;  // nodes
constexpr int S0C_NT = 128;  // scan tiles: columns (one thread each)
constexpr int S0C_TH = 32;   // ... rows
constexpr uint32_t S0_ROOT = 0xFFFFFFFFu;
constexpr uint32_t S0_DEAD = 1u << 26; // descriptor .y: lengths (5 bits each) | dir << 20 | pixels << 21 | dead
// failure codes (rowfail = code << 24 | pixels decoded in the failing block << 16 | block)
constexpr uint32_t S0F_LEN_NEG = 1, S0F_LEN_BIG = 2, S0F_UP_FIRST = 3, S0F_UP_LAST = 4, S0F_OVERREAD = 5,
                   S0F_SHORT = 6;

struct S0RowDev {
  uint64_t in_offset;
  uint32_t in_size;
  uint32_t job;
  uint32_t row;
  uint32_t pad;
};
struct S0JobDev {
  uint64_t out_offset;
  uint32_t out_pitch, w, h, nb; // nb = blocks per row
  uint64_t blk_base;            // first block descriptor (h * nb, row major)
  uint64_t px_base;             // first difference (h rows of nb * 16)
  uint64_t carry_base;          // first carry word (rtiles * nb * 16 * 2)
  uint32_t node_base;           // first node (h * nb * 2)
  uint32_t row_base;            // first row record
  uint32_t rtiles;              // row tiles of S0C_TH rows
  uint32_t pad;
};

__device__ __forceinline__ uint32_t s0_len(uint32_t y, uint32_t g) { return (y >> (5u * g)) & 31u; }

// stream index (0..15) of column c (0..15) of a block: 8 even pixels, then 8 odd ones
__device__ __forceinline__ uint32_t s0_sidx(uint32_t c) { return (c & 1u) ? 8u + (c >> 1) : c >> 1; }

// ---- walk: a thread per row (SamsungV0Decompressor.cpp:110-160, the header part of each block)
// BitStreamerMSB32 refills 4 bytes when fewer than n bits are cached and throws when the refill starts
// more than 8 bytes past the strip (BitStreamer.h:96-104): an operation (fill(32) for a header,
// getBits(n) otherwise) fails iff it ends past bit lim = 32 ((size + 8) / 4 + 1).
__device__ __forceinline__ void s0_walk_entry(const uint8_t* __restrict__ in, const S0RowDev* __restrict__ rows,
                                              uint32_t nrows, const S0JobDev* __restrict__ jobs,
                                              uint2* __restrict__ desc, uint32_t* __restrict__ rowfail,
                                              uint32_t* __restrict__ jobfail) {
  const uint32_t s = blockIdx.x * S0W_NT + threadIdx.x;
  if (s >= nrows)
    return;
  const S0RowDev st = rows[s];
  const S0JobDev jb = jobs[st.job];
  const uint8_t* base = in + st.in_offset;
  const uint32_t size = st.in_size, row = st.row;
  uint2* d = desc + jb.blk_base + (uint64_t)row * jb.nb;
  const uint32_t lim = 32u * ((size + 8u) / 4u + 1u);
  int len[4];
  for (int i = 0; i < 4; ++i)
    len[i] = row < 2 ? 7 : 4;
  uint32_t T = 0, k = 0, code = size < 4u ? S0F_SHORT : 0u, m = 0;
  for (; k < jb.nb && !code; ++k) {
    if (T + 32u > lim) {
      code = S0F_OVERREAD;
      break;
    }
    const uint32_t x = p1_window(base, size, T);
    const uint32_t dir = x >> 31;
    T += 9;
    for (int i = 0; i < 4 && !code; ++i) {
      const uint32_t op = (x >> (29 - 2 * i)) & 3u;
      if (op == 3u) {
        if (T + 4u > lim) {
          code = S0F_OVERREAD;
          break;
        }
        len[i] = (int)(p1_window(base, size, T) >> 28);
        T += 4;
      } else {
        len[i] += (op == 1u) - (op == 2u);
      }
      if (len[i] < 0)
        code = S0F_LEN_NEG;
      else if (len[i] > 16)
        code = S0F_LEN_BIG;
    }
    if (code)
      break;
    if (dir && row < 2u) {
      code = S0F_UP_FIRST;
      break;
    }
    if (dir && 16u * k + 16u >= jb.w) {
      code = S0F_UP_LAST;
      break;
    }
    // the pixels decoded before the first over-read (a zero length reads nothing)
    uint32_t e = T;
    m = 16;
    for (uint32_t j = 0; j < 16; ++j) {
      e += (uint32_t)len[j >> 2];
      if (e > lim) {
        m = j;
        break;
      }
    }
    const uint32_t y = (uint32_t)len[0] | (uint32_t)len[1] << 5 | (uint32_t)len[2] << 10 |
                       (uint32_t)len[3] << 15 | dir << 20 | m << 21;
    d[k] = make_uint2(T, y);
    if (m < 16u) {
      code = S0F_OVERREAD;
      break;
    }
    T = e;
  }
  uint32_t fail = 0;
  if (code) {
    const bool partial = code == S0F_OVERREAD && m < 16u; // (descriptor k is live: its first m pixels)
    if (!partial)
      m = 0;
    for (uint32_t q = partial ? k + 1u : k; q < jb.nb; ++q)
      d[q] = make_uint2(0u, S0_DEAD);
    fail = code << 24 | m << 16 | k;
    atomicMin(jobfail + st.job, row);
  }
  rowfail[jb.row_base + row] = fail;
}

// ---- differences: a warp per row, lane = (block of a pair, stream index)
// calcAdj (SamsungV0Decompressor.cpp:104-108): signExtend(getBits(b), b), 0 for b == 0
__device__ __forceinline__ void s0_diff_entry(const uint8_t* __restrict__ in, const S0RowDev* __restrict__ rows,
                                              uint32_t nrows, const S0JobDev* __restrict__ jobs,
                                              const uint2* __restrict__ desc, uint16_t* __restrict__ adj) {
  const uint32_t s = blockIdx.x * (S0D_NT / 32) + threadIdx.x / 32u;
  if (s >= nrows)
    return;
  const uint32_t lane = threadIdx.x & 31u, j = lane & 15u;
  const S0RowDev st = rows[s];
  const S0JobDev jb = jobs[st.job];
  const uint8_t* base = in + st.in_offset;
  const uint2* d = desc + jb.blk_base + (uint64_t)st.row * jb.nb;
  uint16_t* o = adj + jb.px_base + (uint64_t)st.row * jb.nb * 16u;
  const uint32_t col = j < 8u ? 2u * j : 2u * (j - 8u) + 1u;
  for (uint32_t k = lane >> 4; k < jb.nb; k += 2) {
    const uint2 dd = d[k];
    int32_t a = 0;
    if (!(dd.y & S0_DEAD) && j < ((dd.y >> 21) & 31u)) {
      const uint32_t g = j >> 2, b = s0_len(dd.y, g);
      uint32_t off = (j & 3u) * b;
      for (uint32_t q = 0; q < g; ++q)
        off += 4u * s0_len(dd.y, q);
      if (b) {
        const uint32_t v = p1_window(base, st.in_size, dd.x + off) >> (32u - b);
        a = (int32_t)(v << (32u - b)) >> (32u - b);
      }
    }
    o[16u * k + col] = (uint16_t)a;
  }
}

// ---- nodes: (parent, value) with value(node) = value + value(parent), the root being 0
__device__ __forceinline__ void s0_node_entry(const S0JobDev* __restrict__ jobs, const uint2* __restrict__ desc,
                                              const uint16_t* __restrict__ adj, uint2* __restrict__ nodes) {
  const S0JobDev jb = jobs[blockIdx.y];
  const uint32_t n = blockIdx.x * S0N_NT + threadIdx.x;
  if (n >= jb.h * jb.nb * 2u)
    return;
  const uint32_t p = n & 1u, blk = n >> 1, r = blk / jb.nb, k = blk - r * jb.nb;
  const uint32_t y = desc[jb.blk_base + blk].y;
  const uint32_t c = 16u * k + 14u + p;
  const uint32_t a = c < jb.w ? adj[jb.px_base + (uint64_t)r * jb.nb * 16u + c] : 0u;
  uint2 v;
  if (y & S0_DEAD)
    v = make_uint2(S0_ROOT, 0u);
  else if (y & (1u << 20)) // (the walk lets dir through only for r >= 2 and k < nb - 1)
    v = make_uint2(jb.node_base + (((r - 1u - p) * jb.nb + k) << 1) + p, a);
  else if (k)
    v = make_uint2(jb.node_base + ((blk - 1u) << 1) + p, a);
  else
    v = make_uint2(S0_ROOT, (a + 128u) & 0xFFFFu);
  nodes[jb.node_base + n] = v;
}

__device__ __forceinline__ void s0_jump_entry(const uint2* __restrict__ src, uint2* __restrict__ dst,
                                              uint32_t nnodes) {
  const uint32_t i = blockIdx.x * S0N_NT + threadIdx.x;
  if (i >= nnodes)
    return;
  uint2 v = src[i];
  if (v.x != S0_ROOT) {
    const uint2 u = src[v.x];
    v = make_uint2(u.x, (v.y + u.y) & 0xFFFFu);
  }
  dst[i] = v;
}

// One column of a tile, rows r0 .. r1 - 1: s0 / s1 run the chains (odd columns: one per row parity,
// even columns: s0 only), bit ch of rs records a reset (a left or dead block) of chain ch inside the
// tile.  With `tile`, each value also goes to tile[(r - r0) * S0C_NT + threadIdx.x].
__device__ __forceinline__ void s0_tile_column(const S0JobDev& jb, const uint2* __restrict__ desc,
                                               const uint16_t* __restrict__ adj, const uint2* __restrict__ nodes,
                                               uint32_t c, uint32_t r0, uint32_t r1, uint32_t& s0, uint32_t& s1,
                                               uint32_t& rs, uint16_t* tile) {
  const uint32_t k = c >> 4, p = c & 1u, W = jb.nb * 16u;
  for (uint32_t r = r0; r < r1; ++r) {
    const uint32_t ch = p & r;
    const uint32_t y = desc[jb.blk_base + (uint64_t)r * jb.nb + k].y;
    const uint32_t a = adj[jb.px_base + (uint64_t)r * W + c];
    uint32_t v = ch ? s1 : s0;
    if ((y & S0_DEAD) || !(y & (1u << 20))) {
      const uint32_t b = (k == 0u || (y & S0_DEAD)) ? 128u
                                                     : nodes[jb.node_base + ((r * jb.nb + k - 1u) << 1) + p].y;
      v = (a + b) & 0xFFFFu;
      rs |= 1u << ch;
    } else {
      v = (v + a) & 0xFFFFu;
    }
    if (ch)
      s1 = v;
    else
      s0 = v;
    if (tile)
      tile[(r - r0) * S0C_NT + threadIdx.x] = (uint16_t)v;
  }
}

// grid (column tiles, row tiles, jobs): each tile's carry-out per chain: value | reset << 16
__device__ __forceinline__ void s0_scan_entry(const S0JobDev* __restrict__ jobs, const uint2* __restrict__ desc,
                                              const uint16_t* __restrict__ adj, const uint2* __restrict__ nodes,
                                              uint32_t* __restrict__ carry) {
  const S0JobDev jb = jobs[blockIdx.z];
  const uint32_t c = blockIdx.x * S0C_NT + threadIdx.x, t = blockIdx.y;
  if (c >= jb.w || t >= jb.rtiles)
    return;
  uint32_t s0 = 0, s1 = 0, rs = 0;
  const uint32_t r0 = t * S0C_TH, r1 = min(r0 + (uint32_t)S0C_TH, jb.h);
  s0_tile_column(jb, desc, adj, nodes, c, r0, r1, s0, s1, rs, nullptr);
  uint32_t* o = carry + jb.carry_base + ((uint64_t)t * jb.nb * 16u + c) * 2u;
  o[0] = s0 | (rs & 1u) << 16;
  o[1] = s1 | (rs >> 1) << 16;
}

// grid (column-chain groups, jobs): carry-outs -> carry-ins, in place, tile after tile
__device__ __forceinline__ void s0_carry_entry(const S0JobDev* __restrict__ jobs, uint32_t* __restrict__ carry) {
  const S0JobDev jb = jobs[blockIdx.y];
  const uint32_t i = blockIdx.x * S0C_NT + threadIdx.x; // column << 1 | chain
  if ((i >> 1) >= jb.w)
    return;
  uint32_t* o = carry + jb.carry_base + i;
  const uint64_t stride = (uint64_t)jb.nb * 32u;
  uint32_t cur = 0;
  for (uint32_t t = 0; t < jb.rtiles; ++t) {
    const uint32_t x = o[t * stride];
    o[t * stride] = cur;
    cur = (x >> 16) ? (x & 0xFFFFu) : ((cur + x) & 0xFFFFu);
  }
}

// grid (column tiles, row tiles, jobs); tile = S0C_TH x S0C_NT values in shared memory.  No error: the
// image with the swap of decompress() (SamsungV0Decompressor.cpp:96-101).  Error at (row rf, block kf,
// mf pixels of it): what the reference wrote before it threw -- rows above rf, blocks of rf before kf,
// the first mf pixels (stream order) of block kf -- and nothing else.  Block (0, 0) of each job writes
// its result: status, consumed = code << 24 | row << 9 | block.
// (two halves around the CTA barrier: the tile's values, then the rows out)
__device__ __forceinline__ void s0_store_tile(const S0JobDev* __restrict__ jobs, const uint2* __restrict__ desc,
                                              const uint16_t* __restrict__ adj, const uint2* __restrict__ nodes,
                                              const uint32_t* __restrict__ carry, uint16_t* tile) {
  const S0JobDev jb = jobs[blockIdx.z];
  const uint32_t c0 = blockIdx.x * S0C_NT, t = blockIdx.y;
  if (c0 >= jb.w || t >= jb.rtiles)
    return;
  const uint32_t r0 = t * S0C_TH, r1 = min(r0 + (uint32_t)S0C_TH, jb.h);
  const uint32_t c = c0 + threadIdx.x;
  if (c < jb.w) {
    const uint32_t* ci = carry + jb.carry_base + ((uint64_t)t * jb.nb * 16u + c) * 2u;
    uint32_t s0 = ci[0], s1 = ci[1], rs = 0;
    s0_tile_column(jb, desc, adj, nodes, c, r0, r1, s0, s1, rs, tile);
  }
}

__device__ __forceinline__ void s0_store_out(const S0JobDev* __restrict__ jobs, const uint32_t* __restrict__ rowfail,
                                             const uint32_t* __restrict__ jobfail, uint8_t* __restrict__ out,
                                             uint2* __restrict__ results, const uint16_t* tile) {
  const S0JobDev jb = jobs[blockIdx.z];
  const uint32_t c0 = blockIdx.x * S0C_NT, t = blockIdx.y;
  if (c0 >= jb.w || t >= jb.rtiles)
    return;
  const uint32_t r0 = t * S0C_TH, r1 = min(r0 + (uint32_t)S0C_TH, jb.h);
  const uint32_t rf = jobfail[blockIdx.z];
  const uint32_t info = rf != S0_ROOT ? rowfail[jb.row_base + rf] : 0u;
  if (blockIdx.x == 0 && t == 0 && threadIdx.x == 0) {
    const uint32_t code = info >> 24;
    results[blockIdx.z] = rf == S0_ROOT ? make_uint2(0u, 0u)
                                        : make_uint2(code >= S0F_OVERREAD ? 2u : 1u, // RSB200_ERR_IOE / _RDE
                                                     code << 24 | rf << 9 | (info & 0xFFFFu));
  }
  const uint32_t kf = info & 0xFFFFu, mf = (info >> 16) & 0xFFu;
  // a thread per pixel pair (c0 + 2 (tid & 63), +1) of every second row
  const uint32_t pc = c0 + 2u * (threadIdx.x & 63u), lc = 2u * (threadIdx.x & 63u);
  const bool wide = ((jb.out_offset | jb.out_pitch) & 3u) == 0u;
  for (uint32_t r = r0 + (threadIdx.x >> 6); r < r1; r += 2) {
    if (pc >= jb.w)
      break;
    const uint32_t lr = r - r0;
    uint32_t v0, v1;
    bool w0 = true, w1 = pc + 1u < jb.w;
    if (rf == S0_ROOT) {
      // out(row, col + 1) <-> out(row + 1, col) for even row < h - 1 and even col < w - 1
      const bool even = (r & 1u) == 0u;
      v0 = (!even && w1) ? tile[(lr - 1u) * S0C_NT + lc + 1u] : tile[lr * S0C_NT + lc];
      v1 = (even && r + 1u < jb.h) ? tile[(lr + 1u) * S0C_NT + lc] : tile[lr * S0C_NT + lc + 1u];
    } else {
      v0 = tile[lr * S0C_NT + lc];
      v1 = tile[lr * S0C_NT + lc + 1u];
      const uint32_t k = pc >> 4;
      const bool before = r < rf || (r == rf && k < kf);
      const bool in_f = r == rf && k == kf;
      w0 = before || (in_f && s0_sidx(pc & 15u) < mf);
      w1 = w1 && (before || (in_f && s0_sidx((pc + 1u) & 15u) < mf));
    }
    uint8_t* o = out + jb.out_offset + (uint64_t)r * jb.out_pitch + 2ull * pc;
    if (wide && w0 && w1) {
      *reinterpret_cast<uint32_t*>(o) = v0 | v1 << 16;
    } else {
      if (w0)
        *reinterpret_cast<uint16_t*>(o) = (uint16_t)v0;
      if (w1)
        *reinterpret_cast<uint16_t*>(o + 2) = (uint16_t)v1;
    }
  }
}

#ifndef RSB200_EMU
__global__ void __launch_bounds__(S0W_NT)
    s0_walk_kernel(const uint8_t* __restrict__ in, const S0RowDev* __restrict__ rows, uint32_t nrows,
                   const S0JobDev* __restrict__ jobs, uint2* __restrict__ desc, uint32_t* __restrict__ rowfail,
                   uint32_t* __restrict__ jobfail) {
  s0_walk_entry(in, rows, nrows, jobs, desc, rowfail, jobfail);
}

__global__ void __launch_bounds__(S0D_NT)
    s0_diff_kernel(const uint8_t* __restrict__ in, const S0RowDev* __restrict__ rows, uint32_t nrows,
                   const S0JobDev* __restrict__ jobs, const uint2* __restrict__ desc, uint16_t* __restrict__ adj) {
  s0_diff_entry(in, rows, nrows, jobs, desc, adj);
}

__global__ void __launch_bounds__(S0N_NT)
    s0_node_kernel(const S0JobDev* __restrict__ jobs, const uint2* __restrict__ desc,
                   const uint16_t* __restrict__ adj, uint2* __restrict__ nodes) {
  s0_node_entry(jobs, desc, adj, nodes);
}

__global__ void __launch_bounds__(S0N_NT)
    s0_jump_kernel(const uint2* __restrict__ src, uint2* __restrict__ dst, uint32_t nnodes) {
  s0_jump_entry(src, dst, nnodes);
}

__global__ void __launch_bounds__(S0C_NT)
    s0_scan_kernel(const S0JobDev* __restrict__ jobs, const uint2* __restrict__ desc,
                   const uint16_t* __restrict__ adj, const uint2* __restrict__ nodes, uint32_t* __restrict__ carry) {
  s0_scan_entry(jobs, desc, adj, nodes, carry);
}

__global__ void __launch_bounds__(S0C_NT)
    s0_carry_kernel(const S0JobDev* __restrict__ jobs, uint32_t* __restrict__ carry) {
  s0_carry_entry(jobs, carry);
}

// (a budget of 12 CTAs per SM gives ptxas 40 registers; with the default it keeps 32 and spills)
__global__ void __launch_bounds__(S0C_NT, 12)
    s0_store_kernel(const S0JobDev* __restrict__ jobs, const uint2* __restrict__ desc,
                    const uint16_t* __restrict__ adj, const uint2* __restrict__ nodes,
                    const uint32_t* __restrict__ carry, const uint32_t* __restrict__ rowfail,
                    const uint32_t* __restrict__ jobfail, uint8_t* __restrict__ out, uint2* __restrict__ results) {
  __shared__ uint16_t tile[S0C_TH * S0C_NT];
  s0_store_tile(jobs, desc, adj, nodes, carry, tile);
  __syncthreads();
  s0_store_out(jobs, rowfail, jobfail, out, results, tile);
}
#endif

} // namespace rsb200
