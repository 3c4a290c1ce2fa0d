// ljpeg_stream_order_emu.cpp -- CPU replay of k2_stream_kernel's full-launch form (ljpeg_stream.cuh) with its
// output stage, as in ljpeg_stream_stage_emu.cpp, but with the lanes of a warp going through the rows and units
// of their segments in step, as the GPU's do: the whole warp stores each other's runs only where all 32 lanes
// flush at the same row and unit.  The segments run in scan order or in the plan's order (thread_shape_order,
// ljpeg_host.h).  The output buffer is fenced by guard bytes.
#include "cuda_emu.h"

#include <vector>

namespace order_emu {
constexpr int WARPS = 4; // T_NT / 32 (checked below)
int gather = 0;
uint32_t arrived[WARPS];   // lanes waiting at a flush
uint64_t at_of[WARPS][32]; // ... at which one: (G, row, unit), ordered as the lane passes them
bool whole[WARPS];         // the answer to the lanes released last

// "every lane of my warp is here": with `gather`, the lanes of a warp go through the rows and units of
// their segments in step, as the GPU's do.  A lane at a flush waits until every lane of its warp that
// has not exited is at one; the lanes at the earliest flush then meet (a lane further on passed that
// row and unit without flushing there), and the answer is whether they are all 32.
inline bool whole_warp(uint64_t at) {
  if (!gather)
    return false;
  cuemu::Cta* c = cuemu::cta();
  const int w = (int)threadIdx.x >> 5, lane = (int)threadIdx.x & 31;
  at_of[w][lane] = at;
  arrived[w] |= 1u << lane;
  auto all_here = [c, w]() {
    for (int i = 32 * w; i < std::min(32 * w + 32, c->nthreads); ++i)
      if (c->th[(size_t)i].state != 2 && !((arrived[w] >> (i & 31)) & 1u))
        return false;
    return true;
  };
  auto released = [w, lane]() { return !((arrived[w] >> lane) & 1u); };
  for (;;) {
    if (!released() && all_here()) {
      uint64_t first = ~0ull;
      for (int i = 0; i < 32; ++i)
        if ((arrived[w] >> i) & 1u)
          first = std::min(first, at_of[w][i]);
      uint32_t meet = 0;
      for (int i = 0; i < 32; ++i)
        if (((arrived[w] >> i) & 1u) && at_of[w][i] == first)
          meet |= 1u << i;
      whole[w] = meet == 0xFFFFFFFFu;
      arrived[w] &= ~meet;
    }
    if (released())
      return whole[w];
    cuemu::yield_until([released, all_here]() { return released() || all_here(); });
  }
}
} // namespace order_emu

#define RSB200_EMU_WHOLE_WARP_AT(at) order_emu::whole_warp(at)
#include "../../rawspeed_b200/csrc/ljpeg_stream.cuh"
#include "../../rawspeed_b200/csrc/ljpeg_host.h"

using namespace rsb200;
static_assert(T_NT == 32 * order_emu::WARPS, "warps per CTA");

// 64-byte runs the last run stored through the stage: by the whole warp (shared = 1) or by the lane
// whose run it is (shared = 0)
extern "C" unsigned long long order_emu_runs(int shared) { return shared ? g_emu_runs_shared : g_emu_runs_own; }
// whether a launch with `ntab` tables holds the output stage
extern "C" int order_emu_staged(int ntab) { return stream_staged(ntab) ? 1 : 0; }

// The plan's order of the thread path (thread_shape_order) of `nscans` scans: perm[k] = the scan decoded
// by thread k.  Returns -3 on a malformed scan.
extern "C" int order_emu_shape_order(const rsb200_ljpeg_scan* scans, int nscans, int ntables, uint32_t* perm) {
  std::vector<DevScan> ds((size_t)nscans);
  std::vector<uint32_t> ids((size_t)nscans);
  for (int i = 0; i < nscans; ++i) {
    if (!ljpeg_scan_to_dev(scans[i], ntables, ds[(size_t)i]))
      return -3;
    ids[(size_t)i] = (uint32_t)i;
  }
  const std::vector<uint32_t> p = thread_shape_order(ds.data(), ids);
  std::copy(p.begin(), p.end(), perm);
  return 0;
}

// One full launch over `out` (out_bytes, placed at out_base = 0 or 16 modulo 32), the scans in the
// plan's order (shape_order = 1) or in scan order.  gather: see whole_warp.  Returns -4 on a read
// outside the readable input, -6 on a store into the guard bytes around the output.
extern "C" int order_emu_run(const uint8_t* in, uint64_t in_total, const rsb200_huff_table* tables, int ntables,
                             const rsb200_ljpeg_scan* scans, int nscans, uint8_t* out, uint64_t out_bytes,
                             int out_base, int gather, int reverse, int shape_order) {
  if (out_base != 0 && out_base != 16)
    return -5;
  std::vector<DevTable> ht((size_t)ntables);
  for (int i = 0; i < ntables; ++i)
    if (!build_dev_table(tables[i], ht[(size_t)i]))
      return -2;
  std::vector<DevScan> ds((size_t)nscans);
  std::vector<uint32_t> ids((size_t)nscans);
  for (int i = 0; i < nscans; ++i) {
    if (!ljpeg_scan_to_dev(scans[i], ntables, ds[(size_t)i]))
      return -3;
    ids[(size_t)i] = (uint32_t)i;
  }
  if (shape_order)
    ids = thread_shape_order(ds.data(), ids); // (positions of scan indices 0..n-1: the order itself)
  for (uint32_t& i : ids)
    i |= 0x80000000u;
  const uint64_t padded = (in_total + 15) & ~15ull;
  std::vector<uint8_t> buf(padded + 128, 0xA5);
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(buf.data()) + 31) & ~(uintptr_t)31);
  memcpy(base, in, in_total);
  constexpr size_t GUARD = 256;
  std::vector<uint8_t> obuf(out_bytes + 2 * GUARD + 64, 0xEE);
  uint8_t* obase = reinterpret_cast<uint8_t*>(((reinterpret_cast<uintptr_t>(obuf.data()) + GUARD + 31) & ~(uintptr_t)31) +
                                              (uintptr_t)out_base);
  memcpy(obase, out, out_bytes);
  std::vector<DevResult> res((size_t)nscans);
  std::vector<uint32_t> redo((size_t)nscans, 7u);
  g_emu_runs_shared = g_emu_runs_own = 0;
  order_emu::gather = gather;
  cuemu::ldg_lo = base;
  cuemu::ldg_hi = base + padded;
  cuemu::ldg_outside = 0;
  const unsigned nblocks = (unsigned)((nscans + T_NT - 1) / T_NT);
  for (unsigned b = 0; b < nblocks; ++b) {
    memset(order_emu::arrived, 0, sizeof order_emu::arrived);
    cuemu::run_cta(b, nblocks, T_NT, std::max(sizeof(StreamShared), stream_smem_bytes(ntables)), reverse != 0,
                   [&](uint8_t* smem) {
                     StreamShared& sh = *reinterpret_cast<StreamShared*>(smem);
                     stream_entry<true>(sh, base, in_total, ds.data(), ht.data(), ntables, obase, res.data(),
                                        ids.data(), (uint32_t)nscans, redo.data(), false);
                   });
  }
  cuemu::ldg_lo = cuemu::ldg_hi = nullptr;
  order_emu::gather = 0;
  memcpy(out, obase, out_bytes);
  if (cuemu::ldg_outside)
    return -4;
  for (const uint8_t* q = obuf.data(); q < obase; ++q)
    if (*q != 0xEE)
      return -6;
  for (const uint8_t* q = obase + out_bytes; q < obuf.data() + obuf.size(); ++q)
    if (*q != 0xEE)
      return -6;
  for (int i = 0; i < nscans; ++i)
    if (res[(size_t)i].status != 0 || redo[(size_t)i] != 0)
      return -7;
  return 0;
}
