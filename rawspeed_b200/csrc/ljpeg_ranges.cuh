// ljpeg_ranges.cuh -- multi-CTA decode of ONE long entropy-coded segment
// (Canon CR2: a whole frame is a single stream without restart markers,
// Cr2DecompressorImpl.h:419; untiled LJPEG DNG strips), sm_90a.
//
// The reference decodes such a stream on one CPU thread.  Here the raw bytes are
// cut into ranges of R_CHUNKS * 8 KiB; three small kernels turn the serial
// parse into a parallel one WITHOUT giving up exactness:
//
//   P1 count   one CTA per range.  Ranges r > 0 do not know where their first
//              code word starts (nor its component phase), so the CTA starts one
//              chunk early at a guess and lets the parse self-synchronise; it
//              records the entry state it ended up with at its range boundary,
//              the exit state at the next boundary, and how many symbols start
//              inside its range.
//   P2 verify  one CTA per segment: entry[r] must equal exit[r-1] (same bit, and a
//              phase that selects the same Huffman tables).  If every needed
//              seam matches, induction from the exact start of range 0 proves
//              the speculative parse IS the sequential parse; prefix sums then
//              give every range its first symbol index.  If a seam does not
//              match (not seen on camera data; tests/test_gpu_ljpeg_ranges.py
//              forces it) a flag makes the exact single-CTA kernel
//              (k2_entropy_kernel) redo that segment.
//   P3 diffs   one CTA per range: decode from the verified entry state and write
//              the differences in stream order; K3 (ljpeg.cuh) reconstructs and
//              scatters through the CR2 slice map / tile crop.
#pragma once

#include "ljpeg_fused.cuh"

namespace rsb200 {

constexpr int R_CHUNKS = 8; // raw chunks (of F_RAW bytes) owned by one range

struct DevRange {
  uint32_t scan; // index into the plan's scan array
  uint32_t r;    // range index inside that segment
};

struct RangeState {
  uint32_t entry_pos;   // bits past the range boundary where the first owned symbol starts
  uint32_t entry_phase; // position in the group of that symbol (under this CTA's own counting)
  uint32_t exit_pos;    // same, at the boundary to the next range
  uint32_t exit_phase;
  uint32_t count;       // symbols that start inside the range
  uint32_t clean_bytes; // data bytes (stuffing removed) of the range
  uint32_t ended;       // the end marker / end of buffer lies in this range
  uint32_t status;
};

struct RangeFinal {
  uint32_t entry_pos;
  uint32_t sym_base;    // global index of the first owned symbol
  uint32_t needed;      // owned symbols that are part of the image
  uint32_t ubytes_base; // clean bytes that precede the range in the segment
};

struct BigScanInfo {
  uint32_t scan;         // index into the plan's scan array
  uint32_t first_range;  // first entry of this segment in the range arrays
  uint32_t nranges;
  uint32_t pad;
};

// symbols that start before `boundary_bit`, decoding from (start, phase)
template <bool MULTI>
__device__ __noinline__ void f_count_before(const FusedShared& sh, uint32_t start, uint32_t phase,
                                            uint32_t boundary_bit, uint32_t* n_out,
                                            uint32_t* pos_out) {
  const uint32_t G = sh.sc.group;
  uint32_t p = start, n = 0;
  while (p < boundary_bit) {
    const uint32_t wi = p >> 5;
    const uint32_t x = __funnelshift_l(sh.ub[wi + 1], sh.ub[wi], p & 31);
    const DevTable* t = MULTI ? &sh.tab[sh.sc.table_of[phase]] : &sh.tab[0];
    uint32_t len = t->lut[x >> (32 - LUT_BITS)] >> 10;
    if (len == 0)
      len = f_long_symbol(t, x);
    p += len;
    ++n;
    if (MULTI)
      phase = (phase + 1 == G) ? 0 : phase + 1;
  }
  *n_out = n;
  *pos_out = p;
}

__device__ __forceinline__ void r_stage(FusedShared& sh, const DevScan* scans,
                                        const DevTable* tables, uint32_t scan_idx) {
  const int tid = threadIdx.x;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&scans[scan_idx]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.sc);
    for (int i = tid; i < (int)(sizeof(DevScan) / 4); i += F_NT)
      dst[i] = src[i];
  }
  __syncthreads();
  for (int s = 0; s < 4; ++s) {
    if (sh.sc.table_idx[s] < 0)
      continue;
    const uint4* src = reinterpret_cast<const uint4*>(&tables[sh.sc.table_idx[s]]);
    uint4* dst = reinterpret_cast<uint4*>(&sh.tab[s]);
    for (int i = tid; i < (int)(sizeof(DevTable) / 16); i += F_NT)
      dst[i] = src[i];
  }
  if (tid < 12)
    sh.lutaddr[tid] = smem_u32(sh.tab[sh.sc.table_of[tid] & 3].lut);
}

__device__ __forceinline__ void r_stream(const FusedShared& sh, const uint8_t* in,
                                         uint64_t in_total, uint32_t r, uint32_t c_first,
                                         FStream& st, uint32_t& c_own0, uint32_t& c_own1) {
  const DevScan& sc = sh.sc;
  const uint64_t abase = sc.in_offset & ~15ull;
  st.skew = (uint32_t)(sc.in_offset - abase);
  st.gbase = in + abase;
  const uint32_t limit = st.skew + sc.in_size;
  c_own0 = r * R_CHUNKS;
  c_own1 = (r + 1) * R_CHUNKS;
  // the CTA never needs more than 32 bytes past its range (one symbol + window)
  {
    const uint64_t cap = (uint64_t)c_own1 * (uint64_t)F_RAW + 32ull;
    st.limit = cap < (uint64_t)limit ? (uint32_t)cap : limit;
  }
  {
    const uint64_t whole = ((in_total + 15) & ~15ull) - abase;
    const uint64_t mine = (uint64_t)((st.limit + 15u) & ~15u) + 16ull;
    st.readable = whole < mine ? whole : mine;
  }
  st.chunk_begin = c_first;
  st.chunk_end = (st.limit + F_RAW - 1) / F_RAW;
  st.plain = sc.pump != 0;
  st.pending = true;
  st.pending_par = 0;
}

// f_unstuff for the range kernels.  The plain MSB pump reads zero bits behind the data, and the
// reference decodes codes that start there as long as the refill before them is allowed
// (plain_overread): at the end of the segment, symbols that start up to 8 bytes behind the last
// data byte are parsed too (ub holds 16 zero bytes behind the data).  The plain pump only comes
// with one table (Pentax, Nikon): MULTI instantiations are plain f_unstuff.  Samsung V1 refills to
// 23 bits, not 32, before a symbol (samsung1.cuh): its symbols start up to 8 bytes + 9 bits behind.
template <bool MULTI>
__device__ __forceinline__ FChunk r_unstuff(FusedShared& sh, FStream& st, const FusedCarry& cy,
                                            uint32_t chunk) {
  FChunk co = f_unstuff(sh, st, cy, chunk);
  if (!MULTI && st.plain && co.final_chunk && st.limit == st.skew + sh.sc.in_size)
    co.end_all += 8u * 8u + (sh.sc.kind == 5 ? 10u : 1u);
  return co;
}

template <bool MULTI>
__device__ __forceinline__ void range_count_body(FusedShared& sh, const uint8_t* in,
                                                 uint64_t in_total, uint32_t r,
                                                 RangeState* out) {
  const int tid = threadIdx.x;
  const uint32_t G = sh.sc.group;
  const uint32_t sb = smem_base_opaque(&sh);
  FStream st;
  uint32_t c_own0, c_own1;
  const uint32_t c_first = r == 0 ? 0u : r * R_CHUNKS - 1u; // one halo chunk for r > 0
  r_stream(sh, in, in_total, r, c_first, st, c_own0, c_own1);
  if (tid == 0) {
    FusedCarry c;
    c.pos = 0; // r == 0: exact (first clean byte); r > 0: a guess
    c.sym = 0;
    c.tail_len = 0;
    c.tail_raw = max(c_first * (uint32_t)F_RAW, st.skew);
    c.ubytes = 0;
    c.prev_ff = (c_first * (uint32_t)F_RAW > st.skew) &&
                (st.gbase[c_first * (uint32_t)F_RAW - 1] == 0xFFu);
    c.ended = 0;
    c.leftover = c.proc = c.status = 0;
    c.pc01 = c.pc23 = c.col01 = c.col23 = c.rb01 = c.rb23 = 0;
    sh.cy = c;
    f_issue_chunk(sh, st, c_first);
  }
  __syncthreads();
  uint32_t owned = 0, clean = 0;
  uint32_t entry_pos = 0, entry_phase = 0, exit_pos = 0, exit_phase = 0, ended = 0;
  for (uint32_t chunk = c_first; chunk < st.chunk_end; ++chunk) {
    const FusedCarry cy = sh.cy;
    if (cy.ended)
      break;
    mbar_wait(&sh.bar, (chunk - c_first) & 1u);
    st.pending = false;
    const FChunk co = r_unstuff<MULTI>(sh, st, cy, chunk);
    // ARW1 and Samsung V1: every speculative start follows a run of zero differences, including this
    // CTA's guess at the start of its halo chunk
    const uint32_t align =
        (!MULTI && (sh.sc.kind == 4 || sh.sc.kind == 5)) ? ((chunk == c_first && r > 0) ? 2u : 1u) : 0u;
    const FSync so = f_sync<MULTI>(sh, sb, cy, co, G, align);
    uint32_t total_syms;
    (void)f_block_scan(so.d.count, sh.warp_tmp[3], &total_syms);
    const uint32_t nsub = min((co.end_all + F_SUB * 8u - 1) / (F_SUB * 8u), (uint32_t)F_NT);
    const uint32_t exit_all = nsub ? sh.exitpos[nsub - 1] : cy.pos;
    // symbols that start inside the carried tail belong to the previous chunk
    uint32_t n_tail = 0, p_tail = cy.pos;
    const bool boundary = (chunk == c_own0 && r > 0) || chunk == c_own1;
    if (boundary) {
      if (tid == 0) {
        f_count_before<MULTI>(sh, cy.pos, cy.sym % G, 8u * cy.tail_len, &n_tail, &p_tail);
        sh.rowbase[0][0] = n_tail;
        sh.rowbase[0][1] = p_tail;
      }
      __syncthreads();
      n_tail = sh.rowbase[0][0];
      p_tail = sh.rowbase[0][1];
      __syncthreads();
    }
    if (chunk == c_own0) {
      entry_pos = p_tail - 8u * cy.tail_len;
      entry_phase = (cy.sym + n_tail) % G;
      owned += total_syms - n_tail;
      clean += co.total_emit;
    } else if (chunk > c_own0 && chunk < c_own1) {
      owned += total_syms;
      clean += co.total_emit;
    } else if (chunk == c_own1) {
      owned += n_tail;
      exit_pos = p_tail - 8u * cy.tail_len;
      exit_phase = (cy.sym + n_tail) % G;
    }
    if (co.final_chunk && chunk < c_own1)
      ended = 1;
    // carry (same bookkeeping as the tile kernel, minus what only it needs)
    {
      const uint32_t tail = co.len - co.Lc;
      uint32_t tailbyte = 0;
      if ((uint32_t)tid < tail)
        tailbyte = reinterpret_cast<uint8_t*>(sh.ub)[(co.Lc + tid) ^ 3u];
      __syncthreads();
      if ((uint32_t)tid < tail)
        reinterpret_cast<uint8_t*>(sh.ub)[tid ^ 3u] = (uint8_t)tailbyte;
      if (tid == 0) {
        FusedCarry& c2 = sh.cy;
        c2.sym = cy.sym + total_syms;
        c2.pos = exit_all - co.Lc * 8u;
        c2.tail_len = tail;
        c2.ubytes = cy.ubytes + co.Lc;
        c2.prev_ff = (sh.last_raw_byte == 0xFFu) &&
                     ((chunk + 1) * (uint32_t)F_RAW - 1 < st.limit) &&
                     ((chunk + 1) * (uint32_t)F_RAW - 1 >= st.skew);
        c2.ended = co.final_chunk ? 1u : 0u;
      }
      __syncthreads();
    }
  }
  if (st.pending)
    mbar_wait(&sh.bar, st.pending_par);
  if (tid == 0) {
    RangeState s;
    s.entry_pos = entry_pos;
    s.entry_phase = entry_phase;
    s.exit_pos = exit_pos;
    s.exit_phase = exit_phase;
    s.count = owned;
    s.clean_bytes = clean;
    s.ended = ended;
    s.status = 0;
    *out = s;
  }
}

__global__ void __launch_bounds__(F_NT, 5)
    k2_range_count_kernel(const uint8_t* __restrict__ in, uint64_t in_total,
                          const DevScan* __restrict__ scans, const DevTable* __restrict__ tables,
                          const DevRange* __restrict__ ranges, RangeState* __restrict__ states) {
  extern __shared__ __align__(128) uint8_t f_smem_raw[];
  FusedShared& sh = *reinterpret_cast<FusedShared*>(f_smem_raw);
  const DevRange rg = ranges[blockIdx.x];
  r_stage(sh, scans, tables, rg.scan);
  if (threadIdx.x == 0) {
    sh.bad_code = 0;
    mbar_init(&sh.bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (sh.sc.multi_table)
    range_count_body<true>(sh, in, in_total, rg.r, &states[blockIdx.x]);
  else
    range_count_body<false>(sh, in, in_total, rg.r, &states[blockIdx.x]);
}

// ------------------------------------------------------------------ P2
constexpr int V_NT = 256;

__global__ void __launch_bounds__(V_NT)
    k2_range_verify_kernel(const DevScan* __restrict__ scans, const BigScanInfo* __restrict__ big,
                           const RangeState* __restrict__ states, RangeFinal* __restrict__ finals,
                           uint32_t* __restrict__ fallback, DevResult* __restrict__ results) {
  __shared__ uint32_t tmp[2][V_NT / 32];
  __shared__ uint32_t s_first_end, s_bad;
  const BigScanInfo bi = big[blockIdx.x];
  const DevScan& sc = scans[bi.scan];
  const int tid = threadIdx.x;
  const uint32_t N = sc.n_samples, G = sc.group;
  if (tid == 0) {
    s_first_end = 0xFFFFFFFFu;
    s_bad = 0;
  }
  __syncthreads();
  for (uint32_t i = tid; i < bi.nranges; i += V_NT)
    if (states[bi.first_range + i].ended)
      atomicMin(&s_first_end, i);
  __syncthreads();
  const uint32_t last = min(s_first_end, bi.nranges - 1); // ranges beyond hold no data
  uint32_t base = 0, ubase = 0;
  for (uint32_t i0 = 0; i0 < bi.nranges; i0 += V_NT) {
    const uint32_t i = i0 + tid;
    RangeState s{};
    if (i <= last && i < bi.nranges)
      s = states[bi.first_range + i];
    // inclusive scans of count and clean bytes (two plain 32-bit scans)
    uint32_t vc = s.count, vb = s.clean_bytes;
    const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t a = __shfl_up_sync(0xFFFFFFFFu, vc, d);
      const uint32_t b = __shfl_up_sync(0xFFFFFFFFu, vb, d);
      if (lane >= d) {
        vc += a;
        vb += b;
      }
    }
    if (lane == 31) {
      tmp[0][wid] = vc;
      tmp[1][wid] = vb;
    }
    __syncthreads();
    uint32_t addc = 0, addb = 0, totc = 0, totb = 0;
#pragma unroll
    for (int k = 0; k < V_NT / 32; ++k) {
      if (k < wid) {
        addc += tmp[0][k];
        addb += tmp[1][k];
      }
      totc += tmp[0][k];
      totb += tmp[1][k];
    }
    const uint32_t my_base = base + vc + addc - s.count;
    const uint32_t my_ubase = ubase + vb + addb - s.clean_bytes;
    if (i < bi.nranges) {
      RangeFinal f;
      f.sym_base = my_base;
      f.ubytes_base = my_ubase;
      f.needed = (i <= last && my_base < N) ? min(s.count, N - my_base) : 0u;
      f.entry_pos = 0;
      if (i > 0 && i <= last) {
        const RangeState prev = states[bi.first_range + i - 1];
        f.entry_pos = prev.exit_pos;
        if (f.needed) {
          bool ok = prev.exit_pos == s.entry_pos;
          // the phase this CTA assumed must select the same tables as the true one
          for (uint32_t k = 0; ok && k < G; ++k)
            ok = sc.table_of[(s.entry_phase + k) % G] == sc.table_of[(my_base + k) % G];
          if (!ok)
            atomicOr(&s_bad, 1u);
        }
      }
      finals[bi.first_range + i] = f;
    }
    base += totc;
    ubase += totb;
    __syncthreads();
  }
  __syncthreads();
  if (tid == 0) {
    fallback[blockIdx.x] = s_bad;
    // the data (and, for the plain pump, the zero bits the reference may read behind it) ends
    // before the last sample: no range decodes it, so P3 cannot see it.  (With a failed seam the
    // counts are speculative: k2_entropy_kernel redoes the segment and decides its status alone.)
    if (base < N && !s_bad)
      atomicOr(&results[bi.scan].status, 2u);
  }
}

// ------------------------------------------------------------------ P3
template <bool MULTI>
__device__ __forceinline__ void range_diffs_body(FusedShared& sh, const uint8_t* in,
                                                 uint64_t in_total, uint32_t r,
                                                 const RangeFinal fin, uint16_t* __restrict__ dout,
                                                 DevResult* __restrict__ result) {
  const int tid = threadIdx.x;
  const DevScan& sc = sh.sc;
  const uint32_t G = sc.group;
  const uint32_t sb = smem_base_opaque(&sh);
  FStream st;
  uint32_t c_own0, c_own1;
  r_stream(sh, in, in_total, r, r * R_CHUNKS, st, c_own0, c_own1);
  const uint32_t n_end = fin.sym_base + fin.needed;
  if (tid == 0) {
    FusedCarry c;
    c.pos = fin.entry_pos;
    c.sym = fin.sym_base;
    c.tail_len = 0;
    c.tail_raw = max(c_own0 * (uint32_t)F_RAW, st.skew);
    c.ubytes = fin.ubytes_base;
    c.prev_ff = (c_own0 * (uint32_t)F_RAW > st.skew) &&
                (st.gbase[c_own0 * (uint32_t)F_RAW - 1] == 0xFFu);
    c.ended = 0;
    c.leftover = c.proc = c.status = 0;
    c.pc01 = c.pc23 = c.col01 = c.col23 = c.rb01 = c.rb23 = 0;
    sh.cy = c;
    f_issue_chunk(sh, st, c_own0);
  }
  __syncthreads();
  uint32_t my_status = 0;
  for (uint32_t chunk = c_own0;; ++chunk) {
    const FusedCarry cy = sh.cy;
    if (cy.sym >= n_end)
      break;
    if (cy.ended || chunk >= st.chunk_end) {
      my_status |= 2u;
      break;
    }
    mbar_wait(&sh.bar, (chunk - c_own0) & 1u);
    st.pending = false;
    const FChunk co = r_unstuff<MULTI>(sh, st, cy, chunk);
    const FSync so =
        f_sync<MULTI>(sh, sb, cy, co, G, (!MULTI && (sh.sc.kind == 4 || sh.sc.kind == 5)) ? 1u : 0u);
    const FSub d = so.d;
    uint32_t total_syms;
    const uint32_t sincl = f_block_scan(d.count, sh.warp_tmp[3], &total_syms);
    const uint32_t sym0 = cy.sym + sincl - d.count;
    const uint32_t chunk_syms = min(total_syms, n_end - cy.sym);
    const uint32_t nsub = min((co.end_all + F_SUB * 8u - 1) / (F_SUB * 8u), (uint32_t)F_NT);
    const uint32_t exit_all = nsub ? sh.exitpos[nsub - 1] : cy.pos;
    const uint32_t rel0 = sym0 - cy.sym;
    const uint32_t klast = sc.n_samples - 1 - cy.sym; // the segment's very last symbol
    if (d.count && rel0 < chunk_syms) {
      const uint32_t hi = min(rel0 + d.count, chunk_syms);
      FBits b;
      b.open(sb, so.my_start);
      uint32_t phase = MULTI ? (sym0 % G) : 0u;
      uint32_t lutbase = 0;
      uint16_t* dst = dout + sym0;
      uint16_t* const dst_end = dst + (hi - rel0);
      uint16_t* stop = (klast >= rel0 && klast < hi) ? dst + (klast - rel0) : dst_end;
      uint32_t plast = 0xFFFFFFFFu;
      for (;;) {
        while (dst != stop) {
          const uint32_t x = b.peek();
          if (MULTI)
            lutbase = lds_u32<FO_LUTADDR>(sb + 4 * phase);
          uint32_t tl;
          *dst++ = (uint16_t)f_decode_diff<MULTI>(sh, sb, lutbase, phase, x, tl);
          if (MULTI)
            phase = (phase + 1 == G) ? 0 : phase + 1;
          b.skip(sb, tl);
        }
        if (stop == dst_end)
          break;
        plast = b.p;
        stop = dst_end;
      }
      if (!MULTI && st.plain) {
        // stream bit of the last code (plain: clean bytes are raw bytes)
        if (plast != 0xFFFFFFFFu && plain_overread(8ull * cy.ubytes + plast, sc.in_size))
          my_status |= 2u;
      } else if (co.final_chunk && b.p > co.len * 8u) {
        my_status |= 2u;
      }
      if (plast != 0xFFFFFFFFu && !st.plain) {
        // the reference's pump looks at the whole buffer, not just this range
        const uint32_t full_limit = st.skew + sc.in_size;
        bool ovr = false;
        result->consumed =
            f_stream_position(sh, cy, st.gbase, full_limit, st.skew, chunk, plast, &ovr);
        if (ovr)
          my_status |= 2u;
      }
    }
    // carry
    {
      const uint32_t tail = co.len - co.Lc;
      uint32_t tailbyte = 0;
      if ((uint32_t)tid < tail)
        tailbyte = reinterpret_cast<uint8_t*>(sh.ub)[(co.Lc + tid) ^ 3u];
      __syncthreads();
      if ((uint32_t)tid < tail)
        reinterpret_cast<uint8_t*>(sh.ub)[tid ^ 3u] = (uint8_t)tailbyte;
      if (tid == 0) {
        FusedCarry& c2 = sh.cy;
        c2.sym = cy.sym + total_syms;
        c2.pos = exit_all - co.Lc * 8u;
        c2.tail_len = tail;
        c2.ubytes = cy.ubytes + co.Lc;
        uint32_t rp = min((chunk + 1) * (uint32_t)F_RAW, st.limit);
        if (co.mpos != 0xFFFFFFFFu)
          rp = chunk * F_RAW + co.mpos;
        uint32_t k = tail;
        while (k) {
          --rp;
          if (!st.plain && rp > st.skew && f_raw_byte(st.gbase, st.limit, rp) == 0u &&
              f_raw_byte(st.gbase, st.limit, rp - 1) == 0xFFu)
            --rp;
          --k;
        }
        c2.tail_raw = rp;
        c2.prev_ff = (sh.last_raw_byte == 0xFFu) &&
                     ((chunk + 1) * (uint32_t)F_RAW - 1 < st.limit) &&
                     ((chunk + 1) * (uint32_t)F_RAW - 1 >= st.skew);
        c2.ended = co.final_chunk ? 1u : 0u;
      }
      __syncthreads();
    }
  }
  if (st.pending)
    mbar_wait(&sh.bar, st.pending_par);
  {
    int bad = __syncthreads_or((int)(my_status & 1u));
    bad |= (int)sh.bad_code; // (after the barrier)
    const int over = __syncthreads_or((int)(my_status & 2u));
    if (tid == 0 && (bad || over))
      atomicOr(&result->status, bad ? 1u : 2u);
  }
}

__global__ void __launch_bounds__(F_NT, 5)
    k2_range_diffs_kernel(const uint8_t* __restrict__ in, uint64_t in_total,
                          const DevScan* __restrict__ scans, const DevTable* __restrict__ tables,
                          const DevRange* __restrict__ ranges, const RangeFinal* __restrict__ finals,
                          uint16_t* __restrict__ diffs, DevResult* __restrict__ results) {
  extern __shared__ __align__(128) uint8_t f_smem_raw[];
  FusedShared& sh = *reinterpret_cast<FusedShared*>(f_smem_raw);
  const DevRange rg = ranges[blockIdx.x];
  const RangeFinal fin = finals[blockIdx.x];
  if (fin.needed == 0)
    return;
  r_stage(sh, scans, tables, rg.scan);
  if (threadIdx.x == 0) {
    sh.bad_code = 0;
    mbar_init(&sh.bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  uint16_t* dout = diffs + sh.sc.diff_offset;
  DevResult* res = &results[rg.scan];
  if (sh.sc.multi_table)
    range_diffs_body<true>(sh, in, in_total, rg.r, fin, dout, res);
  else
    range_diffs_body<false>(sh, in, in_total, rg.r, fin, dout, res);
}

// results of the multi-CTA path are accumulated with atomicOr: clear them first
__global__ void k2_clear_results_kernel(const BigScanInfo* __restrict__ big, int nbig,
                                        DevResult* __restrict__ results,
                                        uint32_t* __restrict__ oob) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nbig) {
    results[big[i].scan].status = 0;
    results[big[i].scan].consumed = 0;
    if (oob)
      oob[big[i].scan] = 0xFFFFFFFFu; // (pentax.cuh: first out-of-bounds pixel)
  }
}

} // namespace rsb200
