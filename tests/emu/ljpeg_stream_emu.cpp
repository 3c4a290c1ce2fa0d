// ljpeg_stream_emu.cpp -- CPU replay of k2_stream_kernel (rawspeed_b200/csrc/ljpeg_stream.cuh): the
// kernel body itself, compiled by g++ against tests/emu/cuda_emu.h (one fiber per CUDA thread),
// driven with the descriptors the plan builder (ljpeg_host.h) produces.  Test infrastructure: it
// checks the thread-local unstuffer, the ring bookkeeping and the end-of-stream logic where there
// is no GPU; parity of the real kernel is the GPU tests' job.
#include "cuda_emu.h"

#ifndef RSB200_EMU_WIDE
#define RSB200_EMU_WIDE false
#endif

#include "../../rawspeed_b200/csrc/ljpeg_stream.cuh"
#include "../../rawspeed_b200/csrc/ljpeg_host.h"

#include <vector>

using namespace rsb200;

// whole-sector stores (stg_cs_sector) of the last run
extern "C" unsigned long long stream_emu_sector_stores() { return g_emu_sector_stores; }

// in_base / out_base: where the input and output buffers start modulo 32 (0 or 16; the ABI asks for
// 16-byte alignment only).  any_mode 0: a lane fills when it is low itself; 1: every lane with room
// fills at every unit.  may_redo 0: no segment may be handed to the tile kernel (as the plan does for
// segments it cannot take).  Returns -4 if the kernel read outside the caller's readable input.
extern "C" int stream_emu_run(const uint8_t* in, uint64_t in_total, int in_base, const rsb200_huff_table* tables,
                              int ntables, const rsb200_ljpeg_scan* scans, int nscans, uint8_t* out,
                              uint64_t out_bytes, int out_base, rsb200_scan_result* results, uint32_t* redo_out,
                              int reverse, int any_mode, int may_redo) {
  if ((in_base != 0 && in_base != 16) || (out_base != 0 && out_base != 16))
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
    const DevScan& d = ds[(size_t)i];
    // the plan's thread_eligible(): whole 8-sample units, aligned 128-bit stores
    if (!(d.kind == 0 && d.pump == 0 && d.mcu_h == 1 && (d.group == 1 || d.group == 2 || d.group == 4) &&
          (d.row_samples & 7u) == 0 && ((d.out_offset | d.out_pitch) & 15u) == 0 && (d.out_x & 7u) == 0))
      return -1;
    ids[(size_t)i] = (uint32_t)i | (may_redo ? 0x80000000u : 0u);
  }
  // the product's input contract: base 16-byte aligned, readable up to the next 16-byte boundary
  // (the bytes there are garbage; every __ldg outside that window is counted)
  const uint64_t padded = (in_total + 15) & ~15ull;
  std::vector<uint8_t> buf(padded + 128, 0xA5);
  uint8_t* base = reinterpret_cast<uint8_t*>(((reinterpret_cast<uintptr_t>(buf.data()) + 31) & ~(uintptr_t)31) +
                                             (uintptr_t)in_base);
  memcpy(base, in, in_total);
  std::vector<uint8_t> obuf(out_bytes + 64);
  uint8_t* obase = reinterpret_cast<uint8_t*>(((reinterpret_cast<uintptr_t>(obuf.data()) + 31) & ~(uintptr_t)31) +
                                              (uintptr_t)out_base);
  memcpy(obase, out, out_bytes);
  std::vector<DevResult> res((size_t)nscans);
  std::vector<uint32_t> redo((size_t)nscans, 7u);
  g_emu_any_mode = any_mode;
  g_emu_sector_stores = 0;
  cuemu::ldg_lo = base;
  cuemu::ldg_hi = base + padded;
  cuemu::ldg_outside = 0;
  const unsigned nblocks = (unsigned)((nscans + T_NT - 1) / T_NT);
  for (unsigned b = 0; b < nblocks; ++b)
    cuemu::run_cta(b, nblocks, T_NT, std::max(sizeof(StreamShared), stream_smem_bytes(T_MAXTAB)), reverse != 0, [&](uint8_t* smem) {
      StreamShared& sh = *reinterpret_cast<StreamShared*>(smem);
      stream_entry<RSB200_EMU_WIDE>(sh, base, in_total, ds.data(), ht.data(), ntables, obase, res.data(), ids.data(),
                   (uint32_t)nscans, redo.data(), (any_mode & 1) != 0);
    });
  cuemu::ldg_lo = cuemu::ldg_hi = nullptr;
  memcpy(out, obase, out_bytes);
  if (cuemu::ldg_outside) {
    std::fprintf(stderr, "stream_emu: %llu reads outside the readable input\n", cuemu::ldg_outside);
    return -4;
  }
  for (int i = 0; i < nscans; ++i) {
    results[i].status = res[(size_t)i].status;
    results[i].consumed = res[(size_t)i].consumed;
    if (redo_out)
      redo_out[i] = redo[(size_t)i];
  }
  return 0;
}
