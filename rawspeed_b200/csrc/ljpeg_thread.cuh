// ljpeg_thread.cuh -- K2T: LJPEG tile decode for LARGE batches, one THREAD per
// entropy-coded segment (DNG tile / restart interval), sm_90a.
//
// Same results as k2_fused_kernel (see ljpeg.cuh / ljpeg_fused.cuh for the
// reference citations: PrefixCodeLUTDecoder.h:172-216,
// AbstractPrefixCodeDecoder.h:43-76, LJpegDecompressor.cpp:184-339).
//
// Why a second kernel: a batch of frames holds 10^4..10^5 independent segments
// (726 tiles per 45 MP frame).  With that many streams the serial dependency of
// a Huffman stream stops being a problem: every thread simply is a sequential
// decoder and the machine is kept busy by the number of streams -- no
// synchronisation rounds, no second decode pass (~30 instructions per sample
// instead of ~160 issue slots per sample in the block-per-segment kernel).  The
// price is latency (a 256x256 tile is 65536 dependent symbols), which is why the
// plan only takes this path when a launch holds enough segments.
//
// A warp runs 32 different streams, so everything data dependent in the loop
// costs issue slots for all 32 lanes.  The stuffing / marker / end-of-buffer logic
// of the JPEG bit source is therefore done beforehand by K2C (ljpeg_clean.cuh,
// cooperative, one CTA per segment); the decoders read clean big-endian words:
//   * bit window = two registers + position, `peek` is one funnel shift, a word
//     crossing is four predicated instructions (next word prefetched two ahead);
//   * Huffman LUTs of the plan (<= 4 tables) in shared memory;
//   * predictor 1 in registers (mod 2^16), the first MCU of a row predicted from
//     the first MCU of the previous row; 8 samples are packed and written with
//     one 128-bit store (rows of a tile are 16-byte aligned);
//   * `consumed` (the reference's BitStreamerJPEG::getStreamPosition()) is rebuilt
//     from the bit offset of the last symbol through K2C's anchors.
#pragma once

#include "ljpeg_clean.cuh"
#include "ljpeg_lane.cuh"

namespace rsb200 {

struct ThreadShared {
  uint32_t ring[T_RING][T_NT]; // word w of a stream at ring[w % T_RING][thread]
  DevTable tab[T_MAXTAB];
};

__host__ __device__ inline size_t thread_smem_bytes(int ntab) {
  return sizeof(uint32_t) * T_RING * T_NT + sizeof(DevTable) * (size_t)ntab;
}

// BitStreamerJPEG::getStreamPosition() of the reference after the last symbol, whose
// first bit is data bit T of the segment: the reference has done R = T/32 + 1 (+1 if
// T % 32 != 0) refills of 4 data bytes by then (BitStreamer::fill(32) before every
// symbol, BitStreamer.h:216-229; 4 data bytes per refill, BitStreamerJPEG.h:106-183),
// so its position is the raw offset behind 4R data bytes, or the end marker if that
// comes first; past the end of the buffer the bytes read as zero data.
__device__ __noinline__ uint32_t t_stream_position(const uint8_t* gbase, uint32_t limit,
                                                   uint32_t skew, uint32_t T,
                                                   const uint32_t* anc, uint32_t n_anchor,
                                                   uint32_t clean_len) {
  const uint32_t R = (T >> 5) + 1u + ((T & 31u) ? 1u : 0u);
  const uint32_t need = 4u * R;
  // last anchor whose clean count is <= need (the raw position of data byte `need`
  // is at least skew + need); anchors that count the whole data may lie behind the
  // end marker and are not used
  uint32_t a = min((skew + need) >> T_ANCHOR_SHIFT, n_anchor - 1u);
  while (a > 0 && (__ldg(anc + a) > need || __ldg(anc + a) >= clean_len))
    --a;
  while (a + 1 < n_anchor && __ldg(anc + a + 1) <= need && __ldg(anc + a + 1) < clean_len)
    ++a;
  uint32_t rawp = a << T_ANCHOR_SHIFT, c = __ldg(anc + a);
  if (rawp < skew)
    rawp = skew;
  auto byte_at = [&](uint32_t q) { return q < limit ? (uint32_t)__ldg(gbase + q) : 0u; };
  // a stuffing byte may sit exactly at rawp (its FF ended the previous block)
  if (rawp > skew && byte_at(rawp - 1) == 0xFFu && byte_at(rawp) == 0u)
    rawp += 1;
  while (c < need) {
    if (byte_at(rawp) == 0xFFu) {
      if (byte_at(rawp + 1) != 0u)
        break; // marker: the position stays on it
      rawp += 2;
    } else {
      rawp += 1;
    }
    ++c;
  }
  return rawp - skew;
}

// one sample of component c: Huffman code + mantissa at bit position p of the window
#define T_SYM(c, val)                                                           \
  do {                                                                          \
    const uint32_t x_ = __funnelshift_l(nxt, cur, p);                           \
    const uint32_t d_ = t_decode_diff(tabp[c], lutb[c], x_, last_tl, bad);      \
    const uint32_t pn_ = p + last_tl;                                           \
    if ((pn_ ^ p) & 32u) { /* into the next word (a symbol is <= 32 bits) */    \
      cur = nxt;                                                                \
      nxt = nn;                                                                 \
      nn = lds_u32<0>(ringb + (wv & T_RMASK)); /* word wv / T_WSTRIDE */        \
      wv += T_WSTRIDE;                                                          \
    }                                                                           \
    p = pn_;                                                                    \
    pred[c] += d_;                                                              \
    val = pred[c];                                                              \
  } while (0)

template <int G>
__device__ __forceinline__ void
thread_body(ThreadShared& sh, const DevScan* __restrict__ scp, const DevTScan& ts,
            const DevTInfo info, const uint8_t* __restrict__ in,
            const uint32_t* __restrict__ clean, const uint32_t* __restrict__ anchors,
            uint8_t* __restrict__ out, DevResult* __restrict__ res, uint32_t* __restrict__ redo) {
  const uint4* cb = reinterpret_cast<const uint4*>(clean + ts.clean_off); // 16-byte blocks
  const uint32_t bmax = (ts.cap_words >> 2) - 1u;
  const uint32_t ringb = smem_u32(&sh.ring[0][threadIdx.x]);
  // prefill: blocks 0 .. T_AHEAD/16 - 1
  uint32_t nblk = T_AHEAD / 16; // blocks requested so far
#pragma unroll
  for (uint32_t b = 0; b < T_AHEAD / 16; ++b) {
    const uint4 q = __ldg(cb + min(b, bmax));
    sh.ring[4 * b + 0][threadIdx.x] = q.x;
    sh.ring[4 * b + 1][threadIdx.x] = q.y;
    sh.ring[4 * b + 2][threadIdx.x] = q.z;
    sh.ring[4 * b + 3][threadIdx.x] = q.w;
  }
  uint32_t cur = sh.ring[0][threadIdx.x], nxt = sh.ring[1][threadIdx.x],
           nn = sh.ring[2][threadIdx.x];
  uint32_t wv = 3u * T_WSTRIDE, p = 0; // wv: ring byte offset of the next word to fetch (unwrapped)

  uint32_t lutb[G];
  const DevTable* tabp[G];
  uint32_t rowstart[G], pred[G];
#pragma unroll
  for (int c = 0; c < G; ++c) {
    tabp[c] = &sh.tab[scp->table_idx[scp->table_of[c]]];
    lutb[c] = smem_u32(tabp[c]->lut);
    rowstart[c] = scp->init_pred[c];
  }
  const uint32_t rows = scp->rows;
  const uint32_t units = scp->row_samples >> 3; // row_samples is a multiple of 8
  const uint32_t store_w = scp->store_w;
  const uint32_t out_pitch = scp->out_pitch;
  uint8_t* orow = out + scp->out_offset + (uint64_t)scp->out_y * out_pitch + 2ull * scp->out_x;
  uint32_t bad = 0, last_tl = 0;

  for (uint32_t r = 0; r < rows; ++r) {
#pragma unroll
    for (int c = 0; c < G; ++c)
      pred[c] = rowstart[c];
    for (uint32_t u = 0; u < units; ++u) {
      // ---- start of the unit: request up to two more blocks (a unit consumes at
      //      most 32 bytes); they are stored to the ring at the END of this unit, so no
      //      load is in flight across the loop edge (ptxas waits for those at the loop
      //      head) and the decode of the unit hides their latency ----
      uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
      uint32_t pend = 0, qb0 = 0, qb1 = 0;
      {
        const uint32_t pos = p >> 3; // bytes consumed
        if (nblk * 16u - pos < T_AHEAD) {
          qb0 = nblk;
          q0 = __ldg(cb + min(nblk, bmax));
          ++nblk;
          pend = 1u;
          if (nblk * 16u - pos < T_AHEAD) {
            qb1 = nblk;
            q1 = __ldg(cb + min(nblk, bmax));
            ++nblk;
            pend = 3u;
          }
        }
      }
      // 8 samples, straight line (component of sample k = k % G)
      uint32_t v0, v1, v2, v3, v4, v5, v6, v7;
      T_SYM(0 % G, v0);
      T_SYM(1 % G, v1);
      T_SYM(2 % G, v2);
      T_SYM(3 % G, v3);
      T_SYM(4 % G, v4);
      T_SYM(5 % G, v5);
      T_SYM(6 % G, v6);
      T_SYM(7 % G, v7);
      const uint32_t o0 = __byte_perm(v0, v1, 0x5410), o1 = __byte_perm(v2, v3, 0x5410),
                     o2 = __byte_perm(v4, v5, 0x5410), o3 = __byte_perm(v6, v7, 0x5410);
      if (u == 0) { // the first MCU of the row predicts the first MCU of the next row
        rowstart[0] = v0;
        if (G >= 2)
          rowstart[1] = v1;
        if (G == 4) {
          rowstart[2] = v2;
          rowstart[3] = v3;
        }
      }
      // ---- end of the unit: the blocks requested at its start go into the ring ----
      if (pend & 1u) {
        const uint32_t a = ringb + ((qb0 * (4u * T_WSTRIDE)) & T_RMASK);
        sts_u32<0>(a, q0.x);
        sts_u32<(int)T_WSTRIDE>(a, q0.y);
        sts_u32<2 * (int)T_WSTRIDE>(a, q0.z);
        sts_u32<3 * (int)T_WSTRIDE>(a, q0.w);
      }
      if (pend & 2u) {
        const uint32_t a = ringb + ((qb1 * (4u * T_WSTRIDE)) & T_RMASK);
        sts_u32<0>(a, q1.x);
        sts_u32<(int)T_WSTRIDE>(a, q1.y);
        sts_u32<2 * (int)T_WSTRIDE>(a, q1.z);
        sts_u32<3 * (int)T_WSTRIDE>(a, q1.w);
      }
      const uint32_t s = u << 3;
      if (s + 8 <= store_w) {
        stg_cs_v4(orow + 16ull * u, make_uint4(o0, o1, o2, o3));
      } else if (s < store_w) {
        uint16_t* o16 = reinterpret_cast<uint16_t*>(orow) + s;
        const uint32_t ow[4] = {o0, o1, o2, o3};
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (s + k < store_w)
            o16[k] = (uint16_t)(ow[k >> 1] >> (16 * (k & 1)));
      }
    }
    orow += out_pitch;
  }
  // A needed symbol used bits that are not there.  Whether the reference reads them as zero bits
  // or throws depends on the refill cadence of its pump (BitStreamer.h:120-127,
  // BitStreamerJPEG.h:155-183): segments the tile kernel can take are flagged and decoded again
  // by it (exact, tl_replay in ljpeg_tile.cuh); for the others the answer stays IOException
  // (DESIGN.md "known deviations").
  const bool over = p > 8u * info.clean_len;
  const bool again = over && !bad && redo && ts.pad;
  if (redo)
    *redo = again ? 1u : 0u;
  res->status = bad ? 1u : ((over && !again) ? 2u : 0u);
  {
    const uint64_t in_offset = scp->in_offset;
    const uint64_t abase = in_offset & ~15ull;
    const uint32_t skew = (uint32_t)(in_offset - abase);
    res->consumed = t_stream_position(in + abase, skew + scp->in_size, skew, p - last_tl,
                                      anchors + ts.anchor_off, ts.n_anchor, info.clean_len);
  }
}
#undef T_SYM

#ifndef RSB200_T_LB
#define RSB200_T_LB 6
#endif
__global__ void __launch_bounds__(T_NT, RSB200_T_LB)
    k2_thread_kernel(const uint8_t* __restrict__ in, const DevScan* __restrict__ scans,
                     const DevTable* __restrict__ tables, int ntab, uint8_t* __restrict__ out,
                     DevResult* __restrict__ results, const uint32_t* __restrict__ scan_ids,
                     uint32_t nids, const DevTScan* __restrict__ tscans,
                     const DevTInfo* __restrict__ infos, const uint32_t* __restrict__ clean,
                     const uint32_t* __restrict__ anchors, uint32_t* __restrict__ redo) {
  extern __shared__ __align__(16) uint8_t t_smem_raw[];
  ThreadShared& sh = *reinterpret_cast<ThreadShared*>(t_smem_raw);
  const int tid = threadIdx.x;
  {
    const uint4* src = reinterpret_cast<const uint4*>(tables);
    uint4* dst = reinterpret_cast<uint4*>(sh.tab);
    const int n = ntab * (int)(sizeof(DevTable) / 16);
    for (int i = tid; i < n; i += T_NT)
      dst[i] = src[i];
  }
  __syncthreads();
  const uint32_t id = blockIdx.x * T_NT + tid;
  if (id >= nids)
    return;
  const uint32_t scan_idx = scan_ids[id];
  const DevScan* scp = scans + scan_idx;
  DevResult* res = results + scan_idx;
  const DevTScan ts = tscans[id];
  const DevTInfo info = infos[id];
  const uint32_t G = scp->group;
  if (G == 1)
    thread_body<1>(sh, scp, ts, info, in, clean, anchors, out, res, redo ? redo + id : nullptr);
  else if (G == 2)
    thread_body<2>(sh, scp, ts, info, in, clean, anchors, out, res, redo ? redo + id : nullptr);
  else
    thread_body<4>(sh, scp, ts, info, in, clean, anchors, out, res, redo ? redo + id : nullptr);
}

} // namespace rsb200
