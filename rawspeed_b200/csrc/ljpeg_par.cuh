// ljpeg_par.cuh -- K2P: LJPEG tile decode for SMALL launches (one frame ... a few dozen frames):
// one CTA per entropy-coded segment, every thread parses a slice of the segment's CLEAN stream
// (K2C, ljpeg_clean.cuh, has removed the stuffing), sm_90a.
//
// Same results as the other LJPEG kernels (reference: PrefixCodeLUTDecoder.h:172-216,
// AbstractPrefixCodeDecoder.h:43-76, LJpegDecompressor.cpp:184-339).
//
// Why another kernel: the thread path (k2_stream_kernel) needs ~5 ms for a 256x256 tile however
// empty the machine is (65536 dependent symbols per thread), the tile kernel (k2_tile_kernel)
// stages the raw bytes in shared memory, which limits it to four CTAs per SM and short
// subsequences (2.4 parse passes + a cooperative unstuff: ~100 thread-instructions per pixel).
// Here the clean stream stays in global memory / L1 (each thread walks a contiguous slice of a few
// hundred bytes), shared memory holds only the chain state, and a CTA runs the whole pipeline:
//   1. speculative parse: thread i parses symbol lengths from start[i] (a guess: its slice
//      boundary) to the end of its slice -> exit[i], count[i]; start[i+1] <- exit[i]; repeat for the
//      threads whose start moved until nothing moves (Huffman streams self-synchronise within
//      ~16 symbols, a slice holds 200+: two rounds for almost every thread, a third for a few).
//      At the fixed point the parse is the sequential one (induction from slice 0).
//   2. block scan of count[] -> index of every thread's first symbol.
//   3. decode: every thread decodes its symbols again, now with values, and writes the DIFFERENCES
//      in stream order to a scratch buffer (contiguous per thread, 128-bit stores).
//   4. predictor 1: a column scan gives every row its start values (the first MCU of a row is
//      predicted from the first MCU of the row above), then one warp per row turns the row's
//      differences into pixels (coalesced 16 bytes per lane in, 16 bytes per lane out).
// End of stream / `consumed` / error classes exactly as k2_thread_kernel: the thread that decodes
// the last needed symbol maps its bit offset back to a raw position through K2C's anchors; a
// segment whose needed symbols reach behind its data is flagged for the tile kernel's exact
// second opinion.
#pragma once

#include "ljpeg_thread.cuh"

namespace rsb200 {

constexpr int P_NT = 256;          // threads = slices per segment
constexpr uint32_t P_MIN_WORDS = 16; // shortest slice (words of clean data)

struct ParShared {
  DevTable tab;
  uint32_t exitp[P_NT];
  uint32_t count[P_NT];
  uint32_t wtmp[P_NT / 32];
  uint32_t colbase[P_NT][4]; // per row chunk: exclusive column sums of the first MCU (4 components max)
  uint32_t flags;            // bit 0: bad code wholly in the data among the needed symbols; bit 2: one that reaches behind it
};

// bits of the symbol at the top of window x (code + mantissa); 0x80000000 set: not a code
__device__ __forceinline__ uint32_t p_symbol_bits(const DevTable* t, uint32_t x) {
  const uint32_t e = t->lut[x >> (32 - LUT_BITS)];
  if (e)
    return e >> 10;
  const SymLen s = decode_sym(t, x);
  return (uint32_t)s.total | (s.codelen == 0 ? 0x80000000u : 0u);
}

__device__ __forceinline__ uint32_t p_win(const uint32_t* __restrict__ cw, uint32_t p) {
  const uint32_t w = p >> 5;
  return __funnelshift_l(__ldg(cw + w + 1), __ldg(cw + w), p);
}

// inclusive block scan (P_NT threads)
__device__ __forceinline__ uint32_t p_block_scan(uint32_t v, uint32_t* tmp, uint32_t* total) {
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
  for (int i = 0; i < P_NT / 32; ++i) {
    const uint32_t x = tmp[i];
    add += (i < wid) ? x : 0u;
    tot += x;
  }
  *total = tot;
  __syncthreads();
  return v + add;
}

template <int G>
__device__ __forceinline__ void
par_body(ParShared& sh, const DevScan* __restrict__ scp, const DevTScan& ts, const DevTInfo info,
         const bool may_redo, const uint8_t* __restrict__ in, const uint32_t* __restrict__ clean,
         const uint32_t* __restrict__ anchors, uint16_t* __restrict__ diffs, uint8_t* __restrict__ out,
         DevResult* __restrict__ res, uint32_t* __restrict__ redo) {
  const uint32_t tid = threadIdx.x;
  const uint32_t* cw = clean + ts.clean_off;
  const uint32_t data_bits = 8u * info.clean_len;
  const uint32_t nwords = (info.clean_len + 3u) >> 2;
  const uint32_t segw = max(P_MIN_WORDS, (nwords + P_NT - 1) / P_NT);
  const uint32_t nseg = max(1u, (nwords + segw - 1) / segw);
  const uint32_t seg_bits = 32u * segw;
  const bool mine = tid < nseg;
  const uint32_t end = mine ? min((tid + 1u) * seg_bits, data_bits) : 0u;
  const DevTable* tab = &sh.tab;
  const uint32_t lutb = smem_u32(sh.tab.lut);

  // ---- 1. speculative parse to the fixed point ----
  uint32_t start = tid * seg_bits, parsed = 0xFFFFFFFFu;
  for (;;) {
    if (mine && start != parsed) {
      // window: three words in registers, each word of the slice is loaded once per pass (the
      // word two ahead is requested when the position enters a new word: off the symbol chain)
      uint32_t p = start, n = 0;
      const uint32_t* wp = cw + (start >> 5);
      uint32_t cur = __ldg(wp), nxt = __ldg(wp + 1), nn = __ldg(wp + 2);
      wp += 3;
      while (p < end) {
        const uint32_t x = __funnelshift_l(nxt, cur, p);
        uint32_t tl = lds_u16<0>(mad_hi(x & ~((1u << (32 - LUT_BITS)) - 1u), 1u << (LUT_BITS + 1), lutb)) >> 10;
        if (tl == 0u) // code longer than the LUT, SSSS = 16, or no code at all (counts one bit)
          tl = p_symbol_bits(tab, x) & 0xFFu;
        const uint32_t pn = p + tl;
        if ((pn ^ p) & 32u) {
          cur = nxt;
          nxt = nn;
          nn = __ldg(wp);
          ++wp;
        }
        p = pn;
        ++n;
      }
      sh.exitp[tid] = p;
      sh.count[tid] = n;
      parsed = start;
    }
    __syncthreads();
    bool moved = false;
    if (mine && tid > 0) {
      const uint32_t e = sh.exitp[tid - 1];
      if (e != start) {
        start = e;
        moved = true;
      }
    }
    if (!__syncthreads_or(moved ? 1 : 0))
      break;
  }

  // ---- 2. first symbol of every thread ----
  const uint32_t myc = mine ? sh.count[tid] : 0u;
  uint32_t total = 0;
  const uint32_t k0 = p_block_scan(myc, sh.wtmp, &total) - myc;
  const uint32_t n_samples = scp->n_samples;
  const uint32_t row_samples = scp->row_samples;
  uint16_t* dq = diffs + scp->diff_offset; // stream order, diff_offset a multiple of 8

  // ---- 3. decode: differences in stream order ----
  if (mine && k0 < n_samples) {
    uint32_t p = start, k = k0, bad = 0;
    // whole aligned groups of 8 differences [kA, kB) leave with one 128-bit store; the ragged ends
    // (groups shared with a neighbour, or cut by the end of the image) with 16-bit stores
    const uint32_t kend = min(k0 + myc, n_samples);
    const uint32_t kA = min((k0 + 7u) & ~7u, kend), kB = max(kA, kend & ~7u);
    uint32_t a0 = 0, a1 = 0, a2 = 0, a3 = 0, lo = 0; // the group's pairs, oldest in a0
    uint32_t tlast = start, plast = start;
    const uint32_t* wp = cw + (start >> 5);
    uint32_t cur = __ldg(wp), nxt = __ldg(wp + 1), nn = __ldg(wp + 2);
    wp += 3;
    while (p < end && k < n_samples) {
      const uint32_t x = __funnelshift_l(nxt, cur, p);
      const uint32_t e = lds_u16<0>(mad_hi(x & ~((1u << (32 - LUT_BITS)) - 1u), 1u << (LUT_BITS + 1), lutb));
      uint32_t d, tl;
      if (e != 0u) { // (same arithmetic as t_decode_diff)
        const uint32_t tt = __funnelshift_l(0u, x, e);
        const uint32_t f = (uint32_t)((int32_t)~tt >> 31);
        d = (__funnelshift_l(tt, f, e >> 5) - f) & 0xFFFFu;
        tl = e >> 10;
      } else {
        const SymLen s = decode_sym(tab, x);
        bad |= s.codelen == 0 ? (p + 16u <= data_bits ? 1u : 4u) : 0u; // (see t_bad_in_data)
        d = (uint32_t)sym_diff(s, x) & 0xFFFFu;
        tl = (uint32_t)s.total;
      }
      tlast = p;
      const uint32_t pn = p + tl;
      if ((pn ^ p) & 32u) {
        cur = nxt;
        nxt = nn;
        nn = __ldg(wp);
        ++wp;
      }
      p = pn;
      plast = p;
      if (k >= kA && k < kB) {
        if (!(k & 1u)) {
          lo = d;
        } else {
          a0 = a1;
          a1 = a2;
          a2 = a3;
          a3 = lo | (d << 16);
          if ((k & 7u) == 7u)
            *reinterpret_cast<uint4*>(dq + (k - 7u)) = make_uint4(a0, a1, a2, a3);
        }
      } else {
        dq[k] = (uint16_t)d;
      }
      ++k;
    }
    if (bad)
      atomicOr(&sh.flags, bad);
    if (k == n_samples && k > k0) { // I hold the last needed symbol
      sh.exitp[P_NT - 1] = tlast; // (slots of the chain are free now)
      sh.count[P_NT - 1] = plast;
      atomicOr(&sh.flags, 2u);
    }
  }
  __syncthreads();
  const bool complete = (sh.flags & 2u) != 0u; // all needed symbols exist in the stream
  // status / consumed (as k2_thread_kernel)
  if (tid == 0) {
    const bool bad_in = (sh.flags & 1u) != 0u, bad = (sh.flags & 5u) != 0u;
    const uint32_t plast = complete ? sh.count[P_NT - 1] : 0xFFFFFFFFu;
    const bool over = !complete || plast > data_bits;
    // (an unassigned code wholly in the data is the answer; one that reaches behind it is not, see
    //  t_bad_in_data)
    const bool again = over && !bad_in && redo && may_redo;
    if (redo)
      *redo = again ? 1u : 0u;
    uint32_t status = bad_in ? 1u : (over ? (again ? 0u : 2u) : (bad ? 1u : 0u));
    uint32_t consumed = 0;
    if (complete) {
      const uint64_t in_offset = scp->in_offset;
      const uint64_t abase = in_offset & ~15ull;
      const uint32_t skew = (uint32_t)(in_offset - abase);
      consumed = t_stream_position(in + abase, skew + scp->in_size, skew, sh.exitp[P_NT - 1],
                                   anchors + ts.anchor_off, ts.n_anchor, info.clean_len);
      if (status != 1u && !again && consumed > scp->in_size)
        status = 2u; // the reference's skipBytes(consumed) behind the buffer
    }
    res->status = status;
    res->consumed = consumed;
  }
  if (!complete)
    return; // (flagged above; nothing sensible to reconstruct)

  // ---- 4. predictor 1 ----
  const uint32_t rows = scp->rows;
  const uint32_t store_w = scp->store_w;
  const uint32_t out_pitch = scp->out_pitch;
  uint8_t* obase = out + scp->out_offset + (uint64_t)scp->out_y * out_pitch + 2ull * scp->out_x;
  const uint32_t lane = tid & 31u, wid = tid >> 5;
  uint32_t carry_col[G]; // column sums of the rows above the current chunk of P_NT rows
#pragma unroll
  for (int c = 0; c < G; ++c)
    carry_col[c] = scp->init_pred[c];
  for (uint32_t r0 = 0; r0 < rows; r0 += P_NT) {
    // column scan of the first MCU of rows r0 .. r0 + P_NT - 1 (exclusive: the row's start values)
    const uint32_t r = r0 + tid;
#pragma unroll
    for (int c = 0; c < G; ++c) {
      const uint32_t v = r < rows ? (uint32_t)dq[(uint64_t)r * row_samples + c] : 0u;
      uint32_t tot = 0;
      const uint32_t incl = p_block_scan(v, sh.wtmp, &tot);
      sh.colbase[tid][c] = (carry_col[c] + incl - v) & 0xFFFFu;
      carry_col[c] = (carry_col[c] + tot) & 0xFFFFu;
    }
    __syncthreads();
    // rows of this chunk: one warp per row, 8 samples per lane and pass
    for (uint32_t rr = wid; rr < P_NT && r0 + rr < rows; rr += P_NT / 32) {
      const uint16_t* drow = dq + (uint64_t)(r0 + rr) * row_samples;
      uint8_t* orow = obase + (uint64_t)(r0 + rr) * out_pitch;
      uint32_t run[G];
#pragma unroll
      for (int c = 0; c < G; ++c)
        run[c] = sh.colbase[rr][c];
      for (uint32_t s0 = 0; s0 < row_samples; s0 += 256) {
        const uint32_t s = s0 + 8u * lane;
        uint4 q = make_uint4(0, 0, 0, 0);
        if (s < row_samples) // (row_samples is a multiple of 8)
          q = *reinterpret_cast<const uint4*>(drow + s);
        uint32_t v[8] = {q.x & 0xFFFFu, q.x >> 16, q.y & 0xFFFFu, q.y >> 16,
                         q.z & 0xFFFFu, q.z >> 16, q.w & 0xFFFFu, q.w >> 16};
        // local inclusive sums per component (sample j belongs to component j % G: 8 % G == 0)
#pragma unroll
        for (int j = G; j < 8; ++j)
          v[j] += v[j - G];
        uint32_t tot[G], off[G];
#pragma unroll
        for (int c = 0; c < G; ++c) {
          tot[c] = v[8 - G + c];
          uint32_t incl = tot[c];
#pragma unroll
          for (int d = 1; d < 32; d <<= 1) {
            const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, incl, d);
            if (lane >= (uint32_t)d)
              incl += n;
          }
          off[c] = run[c] + incl - tot[c];
          run[c] = (run[c] + __shfl_sync(0xFFFFFFFFu, incl, 31)) & 0xFFFFu;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
          v[j] = (v[j] + off[j % G]) & 0xFFFFu;
        if (s + 8u <= store_w) {
          stg_cs_v4(orow + 2ull * s, make_uint4(v[0] | (v[1] << 16), v[2] | (v[3] << 16),
                                                v[4] | (v[5] << 16), v[6] | (v[7] << 16)));
        } else if (s < store_w) {
          uint16_t* o16 = reinterpret_cast<uint16_t*>(orow) + s;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (s + j < store_w)
              o16[j] = (uint16_t)v[j];
        }
      }
    }
    __syncthreads();
  }
}

// A CTA takes segments blockIdx.x, blockIdx.x + gridDim.x, ...: the plan launches one CTA per segment.
// (A persistent grid of 2..5 CTAs per SM, so that the slices the resident CTAs walk fit the L1
// cache, is the experiment RSB200_PAR_CTAS keeps: the kernel wants more warps in flight, not fewer.)
__global__ void __launch_bounds__(P_NT)
    k2_par_kernel(const uint8_t* __restrict__ in, const DevScan* __restrict__ scans,
                  const DevTable* __restrict__ tables, uint8_t* __restrict__ out,
                  DevResult* __restrict__ results, const uint32_t* __restrict__ scan_ids, uint32_t nids,
                  const DevTScan* __restrict__ tscans, const DevTInfo* __restrict__ infos,
                  const uint32_t* __restrict__ clean, const uint32_t* __restrict__ anchors,
                  uint16_t* __restrict__ diffs, uint32_t* __restrict__ redo) {
  __shared__ ParShared sh;
  int32_t loaded_table = -1;
  for (uint32_t id = blockIdx.x; id < nids; id += gridDim.x) {
    const uint32_t sid = scan_ids[id];
    const uint32_t scan_idx = sid & 0x7FFFFFFFu;
    const DevScan* scp = scans + scan_idx;
    __syncthreads(); // (the previous segment is done with the shared state)
    if (scp->table_idx[0] != loaded_table) {
      const uint4* src = reinterpret_cast<const uint4*>(tables + scp->table_idx[0]);
      uint4* dst = reinterpret_cast<uint4*>(&sh.tab);
      for (int i = threadIdx.x; i < (int)(sizeof(DevTable) / 16); i += P_NT)
        dst[i] = src[i];
      loaded_table = scp->table_idx[0];
    }
    if (threadIdx.x == 0)
      sh.flags = 0;
    __syncthreads();
    const DevTScan ts = tscans[id];
    const DevTInfo info = infos[id];
    const bool may_redo = ts.pad != 0u;
    DevResult* res = results + scan_idx;
    uint32_t* rd = redo ? redo + id : nullptr;
    const uint32_t G = scp->group;
    if (G == 1)
      par_body<1>(sh, scp, ts, info, may_redo, in, clean, anchors, diffs, out, res, rd);
    else if (G == 2)
      par_body<2>(sh, scp, ts, info, may_redo, in, clean, anchors, diffs, out, res, rd);
    else
      par_body<4>(sh, scp, ts, info, may_redo, in, clean, anchors, diffs, out, res, rd);
  }
}

} // namespace rsb200
