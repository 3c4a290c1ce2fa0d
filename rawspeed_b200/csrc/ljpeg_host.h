// ljpeg_host.h -- host half of the LJPEG plans that the CPU replay of the tile kernel shares with
// rsb200.cu: DHT -> device table, C-ABI scan -> device descriptor, eligibility and plan-time
// parameters of k2_tile_kernel.  Plain C++ (no CUDA runtime calls).
#pragma once

#include "../../include/rawspeed_b200.h"
#include "ljpeg_types.h"

#include <algorithm>
#include <cstring>
#include <tuple>
#include <vector>

namespace rsb200 {

// ------------------------------------------------------------------
// Huffman table -> device table (HuffmanCode.h:66-93 code assignment,
// PrefixCodeLookupDecoder.h:97-113 maxcode/offset, LUT as documented in ljpeg.cuh)
// ------------------------------------------------------------------
inline bool build_dev_table(const rsb200_huff_table& h, DevTable& t) {
  memset(&t, 0, sizeof t);
  unsigned count = 0, maxlen = 0;
  for (unsigned l = 1; l <= 16; ++l) {
    count += h.ncodes_per_len[l - 1];
    if (h.ncodes_per_len[l - 1])
      maxlen = l;
  }
  if (maxlen == 0 || count > 162 || count != h.nvalues)
    return false;
  // Kraft / canonical assignment
  unsigned maxCodes = 2;
  uint32_t code = 0;
  unsigned n = 0;
  for (unsigned l = 0; l < 18; ++l) {
    t.maxcode[l] = -1;
    t.valoff[l] = 0;
  }
  for (unsigned l = 1; l <= maxlen; ++l) {
    const unsigned nc = h.ncodes_per_len[l - 1];
    if (nc > maxCodes)
      return false;
    maxCodes = (maxCodes - nc) * 2;
    if (nc) {
      t.valoff[l] = (int32_t)code - (int32_t)n;
      for (unsigned i = 0; i < nc; ++i, ++n, ++code) {
        const unsigned ssss = h.values[n];
        if (ssss > 16)
          return false;
        // SSSS = 16 stays out of the LUT: the decode loops resolve LUT hits with a
        // branch-free extend() that only covers SSSS <= 15; the rare 16 takes the walk
        if (l <= (unsigned)LUT_BITS && ssss != 16) {
          const unsigned total = l + (ssss == 16 ? (h.fix_dng16 ? 16u : 0u) : ssss);
          const uint16_t e = (uint16_t)(l | (ssss << 5) | (total << 10));
          const uint32_t lo = code << (LUT_BITS - l);
          const uint32_t hi = lo | ((1u << (LUT_BITS - l)) - 1u);
          for (uint32_t c = lo; c <= hi; ++c)
            t.lut[c] = e;
        }
      }
      t.maxcode[l] = (int32_t)code - 1;
    }
    code <<= 1;
  }
  memcpy(t.values, h.values, count);
  t.maxlen = (int32_t)maxlen;
  t.fix16 = h.fix_dng16 ? 1 : 0;
  return true;
}

inline void assign_tables(DevScan& d, const uint8_t* table, int ncomp,
                          const uint8_t* comp_of_pos, int group) {
  // block-local slots: slot of component c
  int slot_of_comp[4] = {0, 0, 0, 0};
  int nslots = 0;
  for (int s = 0; s < 4; ++s)
    d.table_idx[s] = -1;
  for (int c = 0; c < ncomp; ++c) {
    int found = -1;
    for (int s = 0; s < nslots; ++s)
      if (d.table_idx[s] == (int)table[c])
        found = s;
    if (found < 0) {
      found = nslots++;
      d.table_idx[found] = table[c];
    }
    slot_of_comp[c] = found;
  }
  d.multi_table = nslots > 1;
  for (int p = 0; p < group && p < 12; ++p)
    d.table_of[p] = (uint8_t)slot_of_comp[comp_of_pos[p] & 3];
}


// k2_tile_kernel<R> (ljpeg_tile.cuh) takes plain DNG-style tiles: one MCU row of 1, 2 or 4
// components that all use one table, rows of whole 8-sample units that hold at most one row start
// per thread of the predictor stage, 16-byte aligned output rows.
inline bool tile_eligible(const DevScan& d, int min_rs) {
  return d.kind == 0 && d.pump == 0 && !d.multi_table && d.mcu_h == 1 &&
         (d.group == 1 || d.group == 2 || d.group == 4) && (d.row_samples & 7u) == 0 &&
         d.row_samples >= (uint32_t)min_rs && ((d.out_offset | d.out_pitch) & 15u) == 0 &&
         (d.out_x & 7u) == 0 && d.n_samples >= 8;
}

// raw 64-byte pieces per chunk: as many as the staging holds, fewer when the data is so compact
// that a chunk would overflow the sample buffer (then it is decoded in batches anyway, this
// only avoids them); pre-roll of the parse: ~44 symbols, the distance after which a parse that
// started at a wrong bit has almost always locked onto the true one.
inline void tile_params(const DevScan& d, int npiece_max, int dcap, int preroll_override,
                        uint32_t& npieces, uint32_t& preroll) {
  const double bits = d.n_samples ? 8.0 * (double)d.in_size / (double)d.n_samples : 8.0;
  double np = 0.90 * (double)dcap * bits / 8.0 / 64.0;
  np = std::min(np, (double)npiece_max);
  np = std::max(np, 16.0);
  npieces = (uint32_t)np;
  // equal chunks: the same number of chunks, none of them nearly empty
  {
    const uint32_t total = ((uint32_t)(d.in_offset & 15ull) + d.in_size + 63u) / 64u;
    const uint32_t nch = std::max(1u, (total + npieces - 1) / npieces);
    npieces = std::max(16u, (total + nch - 1) / nch);
  }
  const uint32_t sub_bits = std::max(288u, npieces * 512u / 256u);
  uint32_t pre = (uint32_t)std::min(1024.0, std::max(128.0, 44.0 * bits));
  pre = (pre + 31u) & ~31u;
  if (2u * pre > sub_bits) // short subsequences: the pre-roll would cost as much as it saves
    pre = 0;
  if (preroll_override >= 0)
    pre = (uint32_t)preroll_override;
  preroll = pre;
}

// Order of the thread path's segments (one per thread, a warp takes 32 consecutive ones).  The lanes of
// a warp flush k2_stream_kernel's output stage together only where they are at the same row and unit of
// the same kernel body, so a warp should hold segments that agree on everything that steers it: the
// group G (one body per G), row_samples (units per row), rows and store_w (staged groups per row).
// Segments of one such shape form a class; classes run by descending samples per segment, then by
// descending stored width (the short edge tiles last), and a class keeps the input order (in scan order
// a warp of interior tiles is one tile row of a frame: neighbouring input and output).  Returns the
// positions in `ids` in that order.
inline std::vector<uint32_t> thread_shape_order(const DevScan* scans, const std::vector<uint32_t>& ids) {
  std::vector<uint32_t> perm(ids.size());
  for (size_t k = 0; k < ids.size(); ++k)
    perm[k] = (uint32_t)k;
  auto key = [&](uint32_t k) {
    const DevScan& d = scans[ids[k]];
    return std::make_tuple(~((uint64_t)d.rows * d.row_samples), ~d.store_w, d.group, d.row_samples, d.rows);
  };
  std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) { return key(a) < key(b); });
  return perm;
}

// C-ABI scan -> device descriptor (validation included); false = malformed
inline bool ljpeg_scan_to_dev(const rsb200_ljpeg_scan& s, int ntables, DevScan& d) {
  static const uint8_t ident[12] = {0, 1, 2, 3, 0, 0, 0, 0, 0, 0, 0, 0};
  const int group = s.mcu_w * s.mcu_h;
  const bool mcu_ok = (s.mcu_h == 1 && s.mcu_w >= 1 && s.mcu_w <= 4) || (s.mcu_w == 2 && s.mcu_h == 2);
  bool ok = mcu_ok && s.rows > 0 && s.frame_w > 0 && s.store_w > 0 &&
            (uint64_t)s.frame_w * s.mcu_w >= s.store_w &&
            ((uint64_t)s.out_x + (uint64_t)s.store_w) * 2 <= s.out_pitch &&
            (s.out_offset & 1ull) == 0 && (s.out_pitch & 1u) == 0 &&
            (uint64_t)s.rows * s.frame_w * group < (1ull << 32) && s.in_size < (1u << 28) &&
            s.in_offset + (uint64_t)s.in_size >= s.in_offset;
  for (int c = 0; ok && c < group; ++c)
    ok = s.table[c] < ntables;
  if (!ok)
    return false;
  memset(&d, 0, sizeof d);
  d.in_offset = s.in_offset;
  d.in_size = s.in_size;
  d.rows = s.rows;
  d.row_samples = s.frame_w * (uint32_t)group;
  d.n_samples = d.rows * d.row_samples;
  d.rs_inv = d.row_samples <= 1 ? 0xFFFFFFFFu
                                : (uint32_t)(((1ull << 32) + d.row_samples - 1) / d.row_samples);
  d.group = (uint8_t)group;
  d.ncomp = (uint8_t)group;
  d.kind = 0;
  d.pattern = 0; // PAT_PLAIN
  assign_tables(d, s.table, group, ident, group);
  for (int c = 0; c < group; ++c) {
    d.first_idx[c] = (uint8_t)c;
    d.init_pred[c] = s.init_pred[c];
  }
  d.out_offset = s.out_offset;
  d.out_pitch = s.out_pitch;
  d.out_x = s.out_x;
  d.out_y = s.out_y;
  d.store_w = s.store_w;
  d.mcu_w = s.mcu_w;
  d.mcu_h = s.mcu_h;
  return true;
}

} // namespace rsb200
