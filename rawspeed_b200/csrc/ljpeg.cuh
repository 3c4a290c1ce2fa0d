// ljpeg.cuh -- K2 (JPEG entropy decode) + K3 (predictor-1 reconstruction), sm_90a.
//
// Replaces the bodies of
//   LJpegDecompressor::decodeN/decodeRowN   decompressors/LJpegDecompressor.cpp:184-339
//   Cr2Decompressor::decompressN_X_Y        decompressors/Cr2DecompressorImpl.h:396-468
//   BitStreamerJPEG::fillCache              bitstreams/BitStreamerJPEG.h:106-183
//   PrefixCodeLUTDecoder::decode            codes/PrefixCodeLUTDecoder.h:172-216
//   PrefixCodeLookupDecoder::finishReadingPartialSymbol
//                                           codes/PrefixCodeLookupDecoder.h:133-164
//   AbstractPrefixCodeDecoder::processSymbol/extend
//                                           codes/AbstractPrefixCodeDecoder.h:43-76
//
// The reference decodes a segment strictly serially (variable-length code +
// variable-length mantissa per sample, running predictor).  Here:
//
//  K2  A segment's byte stream is cut into fixed SUBSEQ_BYTES "subsequences".
//      One thread decodes one subsequence.  Its true start (bit position of the
//      first code word that begins inside it) is unknown, so threads start at a
//      guess and the CTA iterates "take your predecessor's exit as your start"
//      until nothing changes (self-synchronising Huffman decoding; the fixed
//      point is *exactly* the sequential parse because thread 0 of the first
//      chunk starts at the true segment start).  A block prefix sum of the
//      per-subsequence symbol counts gives every thread its output index, then
//      a second pass decodes the differences and writes them, in stream order,
//      to a linear uint16 scratch buffer.
//  K3  Sums are taken mod 2^16 exactly like the reference's uint16 stores, which
//      makes predictor 1 an associative scan: column-0 chain down the rows, then
//      one warp-shuffle prefix scan per row; the result is scattered to the
//      RawImage through the tile crop / CR2 slice map.
#pragma once

#include "common.cuh"
#include "ljpeg_types.h"

namespace rsb200 {

constexpr int SUBSEQ_BYTES = 32;
constexpr int K2_THREADS = 256;
constexpr int K2_CHUNK_BYTES = SUBSEQ_BYTES * K2_THREADS;

// ------------------------------------------------------------------
// JPEG bit source over raw (stuffed) bytes.
// Window = last 8 data bytes (hi:lo, newest byte in the low bits); the unread
// bits are the low `nbits` bits.  Refills push 32 data bits at a time, dropping
// the 00 after each FF; the first FF xx (xx != 0) ends the data: from there on
// zero bits are supplied and `fake` counts them (BitStreamerJPEG.h:155-179).
// ------------------------------------------------------------------
struct BitSrc {
  const uint32_t* w; // 4-byte aligned base of the segment window
  uint32_t limit;    // valid bytes from base; bytes beyond read as 0
  uint32_t bytepos;  // next raw byte to load (relative to base)
  uint32_t hi, lo;
  int nbits;
  int fake;        // zero bits pushed after the end marker (multiple of 8)
  uint32_t cur_w0; // cached aligned word containing bytepos
  uint32_t cur_idx;
  bool plain = false; // BitStreamerMSB: no stuffing, no markers

  __device__ __forceinline__ uint32_t load_word(uint32_t idx) const {
    const uint32_t b = idx << 2;
    if (b + 4 <= limit)
      return __ldg(w + idx);
    if (b >= limit)
      return 0u;
    return __ldg(w + idx) & (0xFFFFFFFFu >> (32 - 8 * (limit - b)));
  }
  __device__ __forceinline__ uint32_t byte_at(uint32_t p) const {
    if (p >= limit)
      return 0u;
    return (__ldg(w + (p >> 2)) >> ((p & 3) * 8)) & 0xFFu;
  }

  __device__ __forceinline__ void push32(uint32_t be) {
    hi = lo;
    lo = be;
    nbits += 32;
  }

  __device__ void refill_slow() {
    // byte-wise: gather 4 data bytes, honouring FF00 and the end marker
    uint32_t acc = 0;
    int got = 0;
    while (got < 4) {
      if (fake) {
        acc <<= 8;
        fake += 8;
        ++got;
        continue;
      }
      const uint32_t c0 = byte_at(bytepos);
      if (c0 != 0xFFu) {
        acc = (acc << 8) | c0;
        ++bytepos;
        ++got;
        continue;
      }
      const uint32_t c1 = byte_at(bytepos + 1);
      if (c1 == 0u) {
        // NOTE: past the end of the buffer bytes read as zero, so an FF that is
        // the very last byte is followed by a (virtual) 00 as in the reference.
        acc = (acc << 8) | 0xFFu;
        bytepos += 2;
        ++got;
        continue;
      }
      // end-of-stream marker: position stays on the FF
      acc <<= 8;
      fake += 8;
      ++got;
    }
    push32(acc);
    cur_idx = 0xFFFFFFFFu;
  }

  __device__ __forceinline__ void refill() {
    if (!fake) {
      const uint32_t idx = bytepos >> 2;
      uint32_t w0 = (idx == cur_idx) ? cur_w0 : load_word(idx);
      uint32_t w1 = load_word(idx + 1);
      const uint32_t raw = __funnelshift_r(w0, w1, (bytepos & 3) * 8);
      if (plain || __vcmpeq4(raw, 0xFFFFFFFFu) == 0u) {
        push32(__byte_perm(raw, 0, 0x0123));
        bytepos += 4;
        cur_idx = idx + 1;
        cur_w0 = w1;
        return;
      }
    }
    refill_slow();
  }

  // start reading at raw bit position `pos` (8*byte + bit)
  __device__ __forceinline__ void init(const uint32_t* base, uint32_t lim,
                                       uint32_t pos) {
    w = base;
    limit = lim;
    bytepos = pos >> 3;
    hi = lo = 0;
    nbits = 0;
    fake = 0;
    cur_idx = 0xFFFFFFFFu;
    cur_w0 = 0;
    refill();
    refill();
    nbits -= (int)(pos & 7);
  }

  // next 32 unread bits, MSB aligned (needs nbits >= 32)
  __device__ __forceinline__ uint32_t peek32() const {
    return __funnelshift_rc(lo, hi, nbits - 32);
  }
  __device__ __forceinline__ void skip(int n) {
    nbits -= n;
    if (nbits < 32)
      refill();
  }
  // all real bits consumed and we are reading marker padding
  __device__ __forceinline__ bool exhausted() const { return fake >= nbits && fake > 0; }
  __device__ __forceinline__ int real_bits() const { return nbits - fake; }

  // raw bit position of the next unread bit (only valid while real_bits() > 0)
  __device__ __forceinline__ uint32_t position() const {
    const int real = nbits - fake; // > 0
    const int nbytes = (real + 7) >> 3;
    // the `nbytes` data bytes holding the unread real bits sit just above the
    // fake bytes in the window
    uint64_t win = ((uint64_t)hi << 32) | lo;
    win >>= fake;
    if (nbytes < 8)
      win &= (1ull << (8 * nbytes)) - 1ull;
    const uint32_t l = (uint32_t)win, h = (uint32_t)(win >> 32);
    const int nff = plain ? 0
                          : (__popc(__vcmpeq4(l, 0xFFFFFFFFu)) +
                             __popc(__vcmpeq4(h, 0xFFFFFFFFu))) >> 3;
    const uint32_t b = bytepos - (uint32_t)nbytes - (uint32_t)nff;
    const uint32_t o = (8u - ((uint32_t)real & 7u)) & 7u;
    return 8u * b + o;
  }
};

// End of a plain MSB stream (DevScan::pump = 1: Pentax, Nikon).  BitStreamerMSB reads zero bits
// behind the buffer and refills 4 bytes at a time; the refill that starts more than 8 bytes behind
// the end throws (BitStreamer.h:100-131).  Those decoders refill to 32 bits before every code
// (PrefixCodeDecoder), so before a code that starts at stream bit T the pump has done
// (T >> 5) + 1 + (T & 31 ? 1 : 0) refills, and refill number (size + 8) / 4 + 2 is the one that
// throws.  T only grows: the code of the segment's last sample decides.
__device__ __forceinline__ bool plain_overread(uint64_t T, uint32_t size) {
  const uint64_t refills = (T >> 5) + 1u + ((T & 31u) ? 1u : 0u);
  return refills >= (uint64_t)((size + 8u) / 4u) + 2u;
}

// ------------------------------------------------------------------
// K2: one CTA per segment
// ------------------------------------------------------------------
struct K2Shared {
  DevTable tab[4];
  DevScan sc;
  uint32_t exitpos[K2_THREADS];
  uint32_t exitph[K2_THREADS];
  uint32_t ffmask[K2_THREADS];
  uint32_t scan[K2_THREADS];  // symbol-count prefix
  uint32_t ffscan[K2_THREADS]; // FF-count prefix
  uint32_t warp_tmp[2][K2_THREADS / 32];
  uint32_t carry_pos, carry_sym, carry_ff;
  int flag;
};

// inclusive block scan of one uint32 per thread (K2_THREADS threads)
__device__ __forceinline__ uint32_t block_scan_incl(uint32_t v, uint32_t* warp_tmp,
                                                    uint32_t* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t n = __shfl_up_sync(0xFFFFFFFFu, v, d);
    if (lane >= d)
      v += n;
  }
  if (lane == 31)
    warp_tmp[wid] = v;
  __syncthreads();
  uint32_t add = 0, tot = 0;
#pragma unroll
  for (int i = 0; i < K2_THREADS / 32; ++i) {
    const uint32_t x = warp_tmp[i];
    if (i < wid)
      add += x;
    tot += x;
  }
  *total = tot;
  return v + add;
}

struct SubDecode {
  uint32_t exitpos;
  uint32_t count;
};

// Decode (lengths only) from `start` to the end of the subsequence whose last
// byte is byte `sub_end - 1`; phase = position of the first symbol in its group.
template <bool MULTI>
__device__ __forceinline__ SubDecode
k2_scan_sub(const K2Shared& sh, const DevScan& sc, const uint32_t* base,
            uint32_t limit, uint32_t start, uint32_t sub_begin_byte,
            uint32_t ffmask, uint32_t phase) {
  SubDecode r;
  const uint32_t sub_end_bit = (sub_begin_byte + SUBSEQ_BYTES) * 8u;
  if (start == POS_END || start >= sub_end_bit) {
    r.exitpos = start;
    r.count = 0;
    return r;
  }
  // data bits between `start` and the end of the subsequence: raw bytes minus
  // the stuffing bytes, i.e. minus the FF bytes in [start_byte, end-1)
  const uint32_t sb = (start >> 3) - sub_begin_byte; // 0..31
  uint32_t m = ffmask & (0x7FFFFFFFu) & (0xFFFFFFFFu << sb);
  int left = (int)(sub_end_bit - start) - 8 * __popc(m);
  BitSrc bs;
  bs.plain = sc.pump != 0;
  bs.init(base, limit, start);
  uint32_t cnt = 0;
  const DevTable* t0 = &sh.tab[0];
  while (left > 0) {
    const DevTable* t = MULTI ? &sh.tab[sc.table_of[phase]] : t0;
    const SymLen s = decode_sym(t, bs.peek32());
    ++cnt;
    left -= s.total;
    if (MULTI) {
      ++phase;
      if (phase == sc.group)
        phase = 0;
    }
    bs.skip(s.total);
    if (bs.real_bits() <= 0) {
      r.exitpos = POS_END;
      r.count = cnt;
      return r;
    }
  }
  r.exitpos = bs.position();
  r.count = cnt;
  return r;
}

__global__ void __launch_bounds__(K2_THREADS)
    k2_entropy_kernel(const uint8_t* __restrict__ in, uint64_t in_total,
                      const DevScan* __restrict__ scans,
                      const DevTable* __restrict__ tables,
                      uint16_t* __restrict__ diffs, DevResult* __restrict__ results_all,
                      const uint32_t* __restrict__ scan_ids,
                      const uint32_t* __restrict__ enable) {
  extern __shared__ __align__(16) uint8_t k2_smem_raw[];
  K2Shared& sh = *reinterpret_cast<K2Shared*>(k2_smem_raw);
  const int tid = threadIdx.x;
  // exact single-CTA decoder; in a plan it only runs for segments whose
  // speculative multi-CTA parse failed verification (enable[] != 0)
  if (enable && !enable[blockIdx.x])
    return;
  const uint32_t scan_idx = scan_ids ? scan_ids[blockIdx.x] : blockIdx.x;
  DevResult* results = results_all + scan_idx - blockIdx.x; // so that results[blockIdx.x] is ours
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&scans[scan_idx]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.sc);
    for (int i = tid; i < (int)(sizeof(DevScan) / 4); i += K2_THREADS)
      dst[i] = src[i];
  }
  __syncthreads();
  const DevScan& sc = sh.sc;

  // stage this segment's Huffman tables
  for (int s = 0; s < 4; ++s) {
    if (sc.table_idx[s] < 0)
      continue;
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&tables[sc.table_idx[s]]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.tab[s]);
    for (int i = tid; i < (int)(sizeof(DevTable) / 4); i += K2_THREADS)
      dst[i] = src[i];
  }
  // 16-byte aligned window base; positions are bits relative to it
  const uint64_t abase = sc.in_offset & ~15ull;
  const uint32_t skew = (uint32_t)(sc.in_offset - abase);
  const uint32_t* base = reinterpret_cast<const uint32_t*>(in + abase);
  const uint32_t limit = skew + sc.in_size;
  // bytes behind the data in which a needed symbol may start: the JPEG pump keeps the rule of
  // DESIGN.md "consumed"; for the plain pump plain_overread() decides, so the window only has to
  // hold every symbol it allows (they start at most 8 bytes behind the data)
  const uint32_t slack = sc.pump ? 16u : 8u;
  (void)in_total;
  if (tid == 0) {
    sh.carry_pos = skew * 8u;
    sh.carry_sym = 0;
    sh.carry_ff = 0;
  }
  __syncthreads();

  const bool multi = sc.multi_table != 0;
  uint32_t status = 0;
  uint16_t* dout = diffs + sc.diff_offset;

  for (uint32_t chunk = 0;; ++chunk) {
    const uint32_t carry_pos = sh.carry_pos;
    const uint32_t carry_sym = sh.carry_sym;
    const uint32_t carry_ff = sh.carry_ff;
    if (carry_sym >= sc.n_samples)
      break;
    if (carry_pos == POS_END || (carry_pos >> 3) >= limit + slack) {
      // ran out of data before all samples were decoded
      status |= 2u;
      break;
    }
    const uint32_t sub_byte = chunk * K2_CHUNK_BYTES + tid * SUBSEQ_BYTES;
    const bool active = sub_byte < limit + slack;

    // FF map of my subsequence (bit k = byte k is FF)
    uint32_t ffmask = 0;
    if (active && sc.pump == 0) { // (the plain MSB pump has no stuffing: mask stays 0)
#pragma unroll
      for (int k = 0; k < SUBSEQ_BYTES / 4; ++k) {
        const uint32_t idx = (sub_byte >> 2) + k;
        const uint32_t b = idx << 2;
        uint32_t wv = 0;
        if (b + 4 <= limit)
          wv = __ldg(base + idx);
        else if (b < limit)
          wv = __ldg(base + idx) & (0xFFFFFFFFu >> (32 - 8 * (limit - b)));
        const uint32_t eq = __vcmpeq4(wv, 0xFFFFFFFFu); // 0xFF per matching byte
        // compress the 4 byte flags to 4 bits
        const uint32_t bits = ((eq >> 7) & 1u) | ((eq >> 14) & 2u) |
                              ((eq >> 21) & 4u) | ((eq >> 28) & 8u);
        ffmask |= bits << (4 * k);
      }
      if (chunk == 0 && tid == 0)
        ffmask &= ~((1u << skew) - 1u); // bytes before the segment start
    }

    // ---- self-synchronisation ----
    uint32_t my_start = (tid == 0) ? carry_pos : sub_byte * 8u;
    if (tid != 0 && sub_byte > 0 && active && sc.pump == 0) {
      // a guess must not begin on a stuffing byte
      BitSrc probe;
      probe.w = base;
      probe.limit = limit;
      if (probe.byte_at(sub_byte - 1) == 0xFFu && probe.byte_at(sub_byte) == 0u)
        my_start += 8u;
    }
    if (!active)
      my_start = POS_END;
    uint32_t my_phase = (tid == 0) ? (carry_sym % sc.group) : 0u;
    SubDecode d;
    if (multi)
      d = k2_scan_sub<true>(sh, sc, base, limit, my_start, sub_byte, ffmask, my_phase);
    else
      d = k2_scan_sub<false>(sh, sc, base, limit, my_start, sub_byte, ffmask, 0);
    sh.exitpos[tid] = d.exitpos;
    if (multi)
      sh.exitph[tid] = (my_phase + d.count) % sc.group;
    __syncthreads();
    // Fixed-point iteration.  A thread's state is (start position, start phase);
    // each round it adopts its predecessor's exit state (hop by hop, so a wrong
    // guess heals locally through self-synchronisation).  When no position
    // changed in a round the symbol counts are consistent and the phases are
    // taken from a block prefix sum instead (propagates instantly when the
    // tables of the components differ only slightly).  Termination: thread 0 is
    // exact, so after round r threads 0..r are final; the loop ends when every
    // thread's start equals its predecessor's exit => the sequential parse.
    for (int round = 0; round < K2_THREADS + 2; ++round) {
      uint32_t new_start = (tid == 0) ? carry_pos : sh.exitpos[tid - 1];
      uint32_t new_phase = my_phase;
      if (multi)
        new_phase = (tid == 0) ? (carry_sym % sc.group) : sh.exitph[tid - 1];
      const bool pos_changed = new_start != my_start;
      const int any_pos = __syncthreads_or(pos_changed ? 1 : 0);
      if (multi && !any_pos) {
        uint32_t tot;
        const uint32_t incl = block_scan_incl(d.count, sh.warp_tmp[round & 1], &tot);
        new_phase = (carry_sym + incl - d.count) % sc.group;
      }
      const bool changed = pos_changed || (multi && new_phase != my_phase);
      const int any = __syncthreads_or(changed ? 1 : 0);
      if (!any)
        break;
      if (changed) {
        my_start = new_start;
        my_phase = new_phase;
        if (multi)
          d = k2_scan_sub<true>(sh, sc, base, limit, my_start, sub_byte, ffmask, my_phase);
        else
          d = k2_scan_sub<false>(sh, sc, base, limit, my_start, sub_byte, ffmask, 0);
      }
      sh.exitpos[tid] = d.exitpos;
      if (multi)
        sh.exitph[tid] = (my_phase + d.count) % sc.group;
      __syncthreads();
    }

    // ---- output indices ----
    uint32_t total_syms, total_ff;
    const uint32_t incl = block_scan_incl(d.count, sh.warp_tmp[0], &total_syms);
    const uint32_t sym0 = carry_sym + incl - d.count;
    const uint32_t ffcnt = __popc(ffmask);
    const uint32_t ffincl = block_scan_incl(ffcnt, sh.warp_tmp[1], &total_ff);
    const uint32_t ff_before_sub = carry_ff + ffincl - ffcnt; // FFs before my subsequence

    // ---- decode + write differences ----
    if (d.count != 0 && sym0 < sc.n_samples) {
      BitSrc bs;
      bs.plain = sc.pump != 0;
      bs.init(base, limit, my_start);
      uint32_t phase = sym0 % sc.group;
      uint32_t consumed_bits = 0;
      const uint32_t nsym = min(d.count, sc.n_samples - sym0);
      for (uint32_t k = 0; k < nsym; ++k) {
        const DevTable* t = &sh.tab[sc.table_of[phase]];
        const uint32_t x = bs.peek32();
        const SymLen s = decode_sym(t, x);
        if (s.codelen == 0)
          status |= 1u; // bad Huffman code
        if (s.total > bs.real_bits())
          status |= 2u; // symbol runs past the end marker
        dout[sym0 + k] = (uint16_t)sym_diff(s, x);
        if (sym0 + k + 1 == sc.n_samples && sc.pump != 0) {
          // plain MSB pump: no stream position is reported, only its over-read rule
          if (plain_overread(my_start - 8u * skew + consumed_bits, sc.in_size))
            status |= 2u;
        } else if (sym0 + k + 1 == sc.n_samples) {
          // ---- getStreamPosition() of the reference's pump after this, the
          // last, symbol (BitStreamer.h:216-229 refill cadence; see DESIGN.md)
          const uint32_t sb = my_start >> 3;
          // data bytes from the segment start to my start byte
          uint32_t ff_before = ff_before_sub;
          {
            const uint32_t inb = sb - sub_byte; // bytes of my subsequence before start
            ff_before += __popc(ffmask & ((inb >= 32) ? 0xFFFFFFFFu : ((1u << inb) - 1u)));
            if (sb < sub_byte) {
              // start lies in an earlier subsequence (cannot happen: start >= sub begin)
            }
          }
          const uint32_t U = (sb - skew) - ff_before;
          const uint64_t T = 8ull * U + (my_start & 7u) + consumed_bits;
          const uint64_t q = T >> 5;
          const uint64_t R = (T & 31u) ? q + 2 : q + 1;
          uint64_t need = 4ull * R - U; // data bytes to walk from sb
          uint32_t p = sb;
          uint32_t result;
          bool marker = false;
          while (need > 0) {
            const uint32_t c0 = bs.byte_at(p);
            if (c0 == 0xFFu && sc.pump == 0) {
              const uint32_t c1 = bs.byte_at(p + 1);
              if (c1 != 0u) {
                marker = true;
                break;
              }
              p += 2;
            } else
              p += 1;
            --need;
          }
          result = p - skew;
          (void)marker;
          // over-read guard of the reference (BitStreamer.h:125-127): the R-th
          // refill starts at most 16 bytes past the end
          if (!marker && p > limit + 20u)
            status |= 2u;
          results[blockIdx.x].consumed = result;
        }
        consumed_bits += s.total;
        ++phase;
        if (phase == sc.group)
          phase = 0;
        bs.skip(s.total);
      }
    }
    __syncthreads();
    if (tid == K2_THREADS - 1) {
      sh.carry_pos = sh.exitpos[K2_THREADS - 1];
      sh.carry_sym = carry_sym + total_syms;
      sh.carry_ff = carry_ff + total_ff;
    }
    __syncthreads();
  }
  {
    const int bad = __syncthreads_or((int)(status & 1u));
    const int over = __syncthreads_or((int)(status & 2u));
    if (tid == 0) // RSB200_ERR_RDE = 1 (bad Huffman code), RSB200_ERR_IOE = 2
      results[blockIdx.x].status = bad ? 1u : (over ? 2u : 0u);
  }
}

// ------------------------------------------------------------------
// K3a: column-0 chain.  colval[r][c] = init[c] + sum_{r'<=r} D[r'][first_idx[c]]
// (LJpegDecompressor.cpp:326-332 / Cr2DecompressorImpl.h:437-451), mod 2^16.
// One warp per (segment, component).
// ------------------------------------------------------------------
__global__ void k3_column_kernel(const DevScan* __restrict__ scans,
                                 const uint32_t* __restrict__ scan_ids, int nscans,
                                 const uint16_t* __restrict__ diffs,
                                 uint16_t* __restrict__ colvals) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int si = warp >> 2, c = warp & 3;
  if (si >= nscans)
    return;
  const DevScan& sc = scans[scan_ids ? scan_ids[si] : (uint32_t)si];
  if (c >= sc.ncomp || sc.kind == 2) // (kind 2: pentax.cuh reconstructs)
    return;
  const uint16_t* d = diffs + sc.diff_offset + sc.first_idx[c];
  uint16_t* cv = colvals + sc.col_offset + c;
  uint32_t run = sc.init_pred[c];
  for (uint32_t r0 = 0; r0 < sc.rows; r0 += 32) {
    const uint32_t r = r0 + lane;
    uint32_t v = (r < sc.rows) ? d[(uint64_t)r * sc.row_samples] : 0u;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
      uint32_t n = __shfl_up_sync(0xFFFFFFFFu, v, k);
      if (lane >= k)
        v += n;
    }
    v += run;
    if (r < sc.rows)
      cv[(uint64_t)r * 4] = (uint16_t)v;
    run = __shfl_sync(0xFFFFFFFFu, v, 31) & 0xFFFFu;
  }
}

// ------------------------------------------------------------------
// K3b: per-row prefix scan + scatter to the image.  One warp per frame row.
// ------------------------------------------------------------------
struct K3RowRef {
  uint32_t scan;
  uint32_t row;
};

__device__ __forceinline__ void k3_store(const DevScan& sc,
                                         const DevStrip* __restrict__ strips,
                                         uint8_t* __restrict__ out, uint32_t row,
                                         uint32_t s, uint32_t val) {
  // s = sample index inside the frame row
  if (sc.kind == 0) {
    const uint32_t m = s / sc.group, p = s - m * sc.group;
    const uint32_t i = p / sc.mcu_w, j = p - i * sc.mcu_w;
    const uint32_t col = m * sc.mcu_w + j;
    if (col >= sc.store_w)
      return;
    uint16_t* o = reinterpret_cast<uint16_t*>(
        out + sc.out_offset +
        (uint64_t)(sc.out_y + row * sc.mcu_h + i) * sc.out_pitch);
    o[sc.out_x + col] = (uint16_t)val;
  } else {
    // CR2: global group index -> strip -> (row, col)
    const uint32_t frame_groups = sc.row_samples / sc.group;
    const uint32_t gg = s / sc.group, p = s - gg * sc.group;
    const uint32_t g = row * frame_groups + gg;
    int lo = 0, hi = (int)sc.n_strips - 1;
    const DevStrip* st = strips + sc.strip_begin;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (st[mid].g_begin <= g)
        lo = mid;
      else
        hi = mid - 1;
    }
    const DevStrip s0 = st[lo];
    const uint32_t rel = g - s0.g_begin;
    if (rel >= (uint32_t)s0.w * (uint32_t)s0.h)
      return; // beyond the image (frame larger than image)
    const uint32_t rr = rel / (uint32_t)s0.w, cc = rel - rr * (uint32_t)s0.w;
    uint16_t* o = reinterpret_cast<uint16_t*>(
        out + sc.out_offset + (uint64_t)(s0.y + rr) * sc.out_pitch);
    o[(uint32_t)(s0.x + cc) * sc.group + p] = (uint16_t)val;
  }
}

constexpr int K3_THREADS = 256;

// component pattern of a group
//   PAT_PLAIN: c = p                 (LJPEG MCUs, CR2 <2,1,1>/<4,1,1>)
//   PAT_H2V1 : Y Y Cb Cr             (CR2 sRaw <3,2,1>, Cr2DecompressorImpl.h:250-275)
//   PAT_H2V2 : Y Y Y Y Cb Cr         (CR2 sRaw <3,2,2>)
enum { PAT_PLAIN = 0, PAT_H2V1 = 1, PAT_H2V2 = 2 };

template <int G, int PAT> __device__ __forceinline__ constexpr int k3_comp(int p) {
  return PAT == PAT_PLAIN ? p % G
         : PAT == PAT_H2V1 ? (p % 4 < 2 ? 0 : p % 4 - 1)
                           : (p % 6 < 4 ? 0 : p % 6 - 3);
}

template <int G, int PAT>
__device__ __forceinline__ void
k3_row_body(const DevScan& sc, uint32_t row, const uint16_t* __restrict__ diffs,
            const uint16_t* __restrict__ colvals,
            const DevStrip* __restrict__ strips, uint8_t* __restrict__ out) {
  constexpr int PER = (G == 3 || G == 6) ? 24 : 8; // whole groups per lane
  const int lane = threadIdx.x & 31;
  const uint32_t n = sc.row_samples;
  const uint16_t* d = diffs + sc.diff_offset + (uint64_t)row * n;
  uint32_t run[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    run[c] = 0;
    if (c < sc.ncomp)
      run[c] = row == 0 ? sc.init_pred[c]
                        : colvals[sc.col_offset + (uint64_t)(row - 1) * 4 + c];
  }
  const bool vec_in = (PER == 8) && ((n & 7u) == 0u) && ((sc.diff_offset & 7ull) == 0ull);
  // contiguous destination (LJPEG tile with one-row MCUs)
  const bool linear_out = sc.kind == 0 && sc.mcu_h == 1;
  uint8_t* orow = nullptr;
  if (linear_out)
    orow = out + sc.out_offset + (uint64_t)(sc.out_y + row) * sc.out_pitch +
           2ull * sc.out_x;
  const bool vec_out = linear_out && PER == 8 && ((reinterpret_cast<uintptr_t>(orow) & 15) == 0);

  for (uint32_t s0 = 0; s0 < n; s0 += 32u * PER) {
    const uint32_t sb = s0 + lane * PER;
    uint32_t vals[PER];
    if (vec_in && sb + 8 <= n) {
      const uint4 q = *reinterpret_cast<const uint4*>(d + sb);
      vals[0] = q.x & 0xFFFFu; vals[1] = q.x >> 16;
      vals[2] = q.y & 0xFFFFu; vals[3] = q.y >> 16;
      vals[4] = q.z & 0xFFFFu; vals[5] = q.z >> 16;
      vals[6] = q.w & 0xFFFFu; vals[7] = q.w >> 16;
    } else {
#pragma unroll
      for (int k = 0; k < PER; ++k)
        vals[k] = (sb + k < n) ? d[sb + k] : 0u;
    }
    uint32_t sum[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      constexpr int dummy = 0;
      (void)dummy;
      const int c = k3_comp<G, PAT>(k);
      sum[c] += vals[k];
      vals[k] = sum[c];
    }
    uint32_t p01 = (sum[0] & 0xFFFFu) | (sum[1] << 16);
    uint32_t p23 = (sum[2] & 0xFFFFu) | (sum[3] << 16);
    uint32_t i01 = p01, i23 = p23;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
      const uint32_t a = __shfl_up_sync(0xFFFFFFFFu, i01, k);
      const uint32_t b = __shfl_up_sync(0xFFFFFFFFu, i23, k);
      if (lane >= k) {
        i01 = __vadd2(i01, a);
        i23 = __vadd2(i23, b);
      }
    }
    const uint32_t e01 = __vsub2(i01, p01), e23 = __vsub2(i23, p23);
    uint32_t off[4];
    off[0] = run[0] + (e01 & 0xFFFFu);
    off[1] = run[1] + (e01 >> 16);
    off[2] = run[2] + (e23 & 0xFFFFu);
    off[3] = run[3] + (e23 >> 16);
#pragma unroll
    for (int k = 0; k < PER; ++k)
      vals[k] = (vals[k] + off[k3_comp<G, PAT>(k)]) & 0xFFFFu;

    if (linear_out) {
      if (vec_out && sb + 8 <= sc.store_w) {
        uint4 o;
        o.x = vals[0] | (vals[1] << 16);
        o.y = vals[2] | (vals[3] << 16);
        o.z = vals[4] | (vals[5] << 16);
        o.w = vals[6] | (vals[7] << 16);
        stg_cs_v4(orow + 2ull * sb, o);
      } else {
        uint16_t* o16 = reinterpret_cast<uint16_t*>(orow);
#pragma unroll
        for (int k = 0; k < PER; ++k)
          if (sb + k < n && sb + k < sc.store_w)
            o16[sb + k] = (uint16_t)vals[k];
      }
    } else {
#pragma unroll
      for (int k = 0; k < PER; ++k)
        if (sb + k < n)
          k3_store(sc, strips, out, row, sb + k, vals[k]);
    }
    const uint32_t t01 = __shfl_sync(0xFFFFFFFFu, i01, 31);
    const uint32_t t23 = __shfl_sync(0xFFFFFFFFu, i23, 31);
    run[0] = (run[0] + (t01 & 0xFFFFu)) & 0xFFFFu;
    run[1] = (run[1] + (t01 >> 16)) & 0xFFFFu;
    run[2] = (run[2] + (t23 & 0xFFFFu)) & 0xFFFFu;
    run[3] = (run[3] + (t23 >> 16)) & 0xFFFFu;
  }
}

__global__ void __launch_bounds__(K3_THREADS)
    k3_row_kernel(const DevScan* __restrict__ scans,
                  const K3RowRef* __restrict__ rows, uint32_t nrows,
                  const uint16_t* __restrict__ diffs,
                  const uint16_t* __restrict__ colvals,
                  const DevStrip* __restrict__ strips, uint8_t* __restrict__ out) {
  const uint32_t wrow = (blockIdx.x * K3_THREADS + threadIdx.x) >> 5;
  if (wrow >= nrows)
    return;
  const K3RowRef ref = rows[wrow];
  const DevScan& sc = scans[ref.scan];
  if (sc.kind == 2) // pentax.cuh reconstructs
    return;
  // warp-uniform dispatch on the group layout
  if (sc.pattern == PAT_H2V1)
    k3_row_body<4, PAT_H2V1>(sc, ref.row, diffs, colvals, strips, out);
  else if (sc.pattern == PAT_H2V2)
    k3_row_body<6, PAT_H2V2>(sc, ref.row, diffs, colvals, strips, out);
  else if (sc.group == 1)
    k3_row_body<1, PAT_PLAIN>(sc, ref.row, diffs, colvals, strips, out);
  else if (sc.group == 2)
    k3_row_body<2, PAT_PLAIN>(sc, ref.row, diffs, colvals, strips, out);
  else if (sc.group == 3)
    k3_row_body<3, PAT_PLAIN>(sc, ref.row, diffs, colvals, strips, out);
  else
    k3_row_body<4, PAT_PLAIN>(sc, ref.row, diffs, colvals, strips, out);
}

} // namespace rsb200
