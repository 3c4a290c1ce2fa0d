// ljpeg_stream_stage_emu.cpp -- CPU replay of k2_stream_kernel's full-launch form (ljpeg_stream.cuh) with
// its output stage: the kernel body compiled by g++ against tests/emu/cuda_emu.h, as in
// ljpeg_stream_emu.cpp, with the warp-wide flush of the stage replayed both ways -- every lane alone,
// and the lanes of a warp that are still running meeting at the flush (then the whole warp stores
// each other's runs whenever no lane has exited).  The output buffer is fenced by guard bytes.
#include "cuda_emu.h"

#include <vector>

namespace stage_emu {
constexpr int WARPS = 4; // T_NT / 32 (checked below)
int gather = 0;
uint32_t arrived[WARPS];
uint32_t result[WARPS][2];
uint64_t gen[WARPS];

// "every lane of my warp is here": with `gather`, a lane waits until every lane of its warp that has
// not exited has arrived; the answer is whether that is all 32
inline bool whole_warp() {
  if (!gather)
    return false;
  cuemu::Cta* c = cuemu::cta();
  const int w = (int)threadIdx.x >> 5, lane = (int)threadIdx.x & 31;
  const uint64_t g = gen[w];
  arrived[w] |= 1u << lane;
  auto all_here = [c, w]() {
    for (int i = 32 * w; i < std::min(32 * w + 32, c->nthreads); ++i)
      if (c->th[(size_t)i].state != 2 && !((arrived[w] >> (i & 31)) & 1u))
        return false;
    return true;
  };
  if (!all_here())
    cuemu::yield_until([w, g, all_here]() { return gen[w] != g || all_here(); });
  if (gen[w] == g) {
    result[w][g & 1] = arrived[w];
    arrived[w] = 0;
    ++gen[w];
  }
  return result[w][g & 1] == 0xFFFFFFFFu;
}
} // namespace stage_emu

#define RSB200_EMU_WHOLE_WARP() stage_emu::whole_warp()
#include "../../rawspeed_b200/csrc/ljpeg_stream.cuh"
#include "../../rawspeed_b200/csrc/ljpeg_host.h"

using namespace rsb200;
static_assert(T_NT == 32 * stage_emu::WARPS, "warps per CTA");

// 64-byte runs the last run stored through the stage: by the whole warp (shared = 1) or by the lane
// whose run it is (shared = 0)
extern "C" unsigned long long stage_emu_runs(int shared) { return shared ? g_emu_runs_shared : g_emu_runs_own; }
// shared memory of a launch with `ntab` tables, and whether it holds the output stage
extern "C" unsigned long long stage_emu_smem_bytes(int ntab) { return stream_smem_bytes(ntab); }
extern "C" int stage_emu_staged(int ntab) { return stream_staged(ntab) ? 1 : 0; }

// One full launch over `out` (out_bytes, placed at out_base = 0 or 16 modulo 32).  gather: see
// whole_warp.  Returns -4 on a read outside the readable input, -6 on a store into the guard bytes
// around the output.
extern "C" int stage_emu_run(const uint8_t* in, uint64_t in_total, const rsb200_huff_table* tables, int ntables,
                             const rsb200_ljpeg_scan* scans, int nscans, uint8_t* out, uint64_t out_bytes,
                             int out_base, int gather, int reverse) {
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
    ids[(size_t)i] = (uint32_t)i | 0x80000000u;
  }
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
  stage_emu::gather = gather;
  cuemu::ldg_lo = base;
  cuemu::ldg_hi = base + padded;
  cuemu::ldg_outside = 0;
  const unsigned nblocks = (unsigned)((nscans + T_NT - 1) / T_NT);
  for (unsigned b = 0; b < nblocks; ++b) {
    memset(stage_emu::arrived, 0, sizeof stage_emu::arrived);
    memset(stage_emu::gen, 0, sizeof stage_emu::gen);
    cuemu::run_cta(b, nblocks, T_NT, std::max(sizeof(StreamShared), stream_smem_bytes(ntables)), reverse != 0,
                   [&](uint8_t* smem) {
                     StreamShared& sh = *reinterpret_cast<StreamShared*>(smem);
                     stream_entry<true>(sh, base, in_total, ds.data(), ht.data(), ntables, obase, res.data(),
                                        ids.data(), (uint32_t)nscans, redo.data(), false);
                   });
  }
  cuemu::ldg_lo = cuemu::ldg_hi = nullptr;
  stage_emu::gather = 0;
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
