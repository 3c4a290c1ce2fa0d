// ljpeg_types.h -- descriptors and tables shared by the LJPEG kernels, the host-side plan
// builder and the CPU replay of the tile kernel (tests/emu/): plain C++, usable from nvcc and g++.
// (Split out of ljpeg.cuh in round 2; reference citations are in ljpeg.cuh.)
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define RSB_LJ_HD __host__ __device__
#else
#define RSB_LJ_HD
#endif

namespace rsb200 {

// ------------------------------------------------------------------
// device-side tables / descriptors
// ------------------------------------------------------------------
constexpr int LUT_BITS = 11; // same depth as the reference's LookupDepth
constexpr uint32_t POS_END = 0xFFFFFFFFu;

// LUT entry (uint16): [4:0] code length (0 = not in LUT), [9:5] SSSS,
// [15:10] total bits consumed by code + mantissa.
struct alignas(16) DevTable {
  uint16_t lut[1 << LUT_BITS];
  int32_t maxcode[18];  // per code length 1..16; -1 = no code of this length
  int32_t valoff[18];   // code - valoff[len] = index into values
  uint8_t values[164];
  int32_t maxlen;
  int32_t fix16;
};

struct DevScan {
  uint64_t in_offset;   // first entropy-coded byte (absolute in the input buffer)
  uint32_t in_size;     // bytes available
  uint32_t n_samples;   // symbols to decode = rows * row_samples
  uint32_t rows;        // LJPEG (frame) rows
  uint32_t row_samples; // samples per LJPEG row = frame_w * group
  uint64_t diff_offset; // first element of this scan in the linear scratch buffer
  uint8_t group;        // samples per MCU / CR2 group
  uint8_t ncomp;
  uint8_t multi_table;  // components use different tables -> phase matters
  uint8_t kind;         // 0 = LJPEG tile, 1 = CR2, 2 = Pentax (K3P reconstruction), 3 = Nikon,
                        // 4 = Sony ARW1 (arw1.cuh), 5 = Samsung V1 (samsung1.cuh)
  uint8_t table_of[12]; // slot (0..3) of the block-local table of sample p
  uint8_t pattern;      // component pattern of a group (PAT_*)
  uint8_t pump;         // 0 = JPEG bit source (FF00 stuffing, FFxx ends the data);
                        // 1 = plain MSB (BitStreamerMSB: bytes as they are)
  uint8_t pad0[10];
  int32_t table_idx[4]; // plan table index per slot (-1 unused)
  uint8_t first_idx[4]; // position in the group of the first sample of comp c
  uint16_t init_pred[4];
  // output mapping
  uint64_t out_offset;
  uint32_t out_pitch;
  uint32_t out_x, out_y, store_w;
  uint8_t mcu_w, mcu_h;
  uint16_t n_strips;     // CR2
  uint32_t strip_begin;  // CR2: first entry in the strip table
  uint64_t col_offset;   // first element of this scan in the column-chain scratch
  uint32_t row_begin;    // first global row index of this scan (K3 work list)
  uint32_t rs_inv;       // ceil(2^32 / row_samples) (fast row lookup in the fused kernel)
};

// CR2 vertical output strip (Cr2DecompressorImpl.h:162-205), in groups
struct DevStrip {
  uint32_t g_begin; // first group (stream order) of this strip
  int32_t x, y, w, h;
};

struct DevResult {
  uint32_t status;
  uint32_t consumed;
};

// ------------------------------------------------------------------
// symbol decode helpers (tables live in shared memory)
// ------------------------------------------------------------------
struct SymLen {
  int total;   // bits consumed by code + mantissa
  int codelen; // 0 -> invalid code
  int ssss;
};

RSB_LJ_HD inline SymLen decode_sym(const DevTable*  t,
                                             uint32_t x) {
  SymLen s;
  const uint32_t e = t->lut[x >> (32 - LUT_BITS)];
  s.codelen = e & 31;
  s.ssss = (e >> 5) & 31;
  s.total = e >> 10;
  if (s.codelen == 0) {
    // not in the LUT (code longer than LUT_BITS, SSSS = 16, or corrupt): T.81 F.16 walk
    int len = 1;
    for (; len <= t->maxlen; ++len) {
      const int code = (int)(x >> (32 - len));
      if (code <= t->maxcode[len]) {
        s.ssss = t->values[code - t->valoff[len]];
        s.codelen = len;
        s.total = len + (s.ssss == 16 ? (t->fix16 ? 16 : 0) : s.ssss);
        return s;
      }
    }
    s.codelen = 0; // "bad Huffman code"
    s.ssss = 0;
    s.total = 1;
  }
  return s;
}

// Samsung V1 (samsung1.cuh): a zero difference is the code 110100.  A parse that starts on any of
// the 5 wrong residues inside a run of them falls into a cycle of the residues 2 and 4 mod 6 and
// never resynchronises, so speculative starts inside such a run are moved to its phase (f_sync's
// run alignment): the offset 0..5 at which the 32 bits of x0:x1 are 110100 repeated, else 0.
RSB_LJ_HD inline uint32_t samsung1_run_phase(uint32_t x0, uint32_t x1) {
  for (uint32_t o = 0; o < 6; ++o)
    if (((x0 << o) | (o ? x1 >> (32 - o) : 0u)) == 0xD34D34D3u)
      return o;
  return 0;
}

// AbstractPrefixCodeDecoder::processSymbol + extend
RSB_LJ_HD inline int sym_diff(const SymLen& s, uint32_t x) {
  if (s.ssss == 0)
    return 0;
  if (s.ssss == 16)
    return -32768;
  const uint32_t v = (x << s.codelen) >> (32 - s.ssss);
  return (v >> (s.ssss - 1)) ? (int)v : (int)v - (int)((1u << s.ssss) - 1u);
}

} // namespace rsb200
