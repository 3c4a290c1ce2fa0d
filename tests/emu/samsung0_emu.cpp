// samsung0_emu.cpp -- CPU replay of K13 (rawspeed_b200/csrc/samsung0.cuh: walk, differences, nodes,
// pointer jumping, column scans, carries, store), compiled by g++ against tests/emu/cuda_emu.h and run
// in the plan's order with the plan's layout: through the fiber scheduler (forward or reverse thread
// order), or thread after thread (`plain`, fast enough for full-size frames; the kernels have no
// synchronisation but the store's one CTA barrier, which then falls between its two halves).  Test
// infrastructure (no GPU needed); parity of the real kernels is the GPU tests' job.
#include "cuda_emu.h"

#include "../../rawspeed_b200/csrc/samsung0.cuh"

#include <functional>
#include <vector>

using namespace rsb200;

namespace {
// One CTA of `nthreads`: `phases` in order with a CTA barrier between them.  mode 0 / 1: fibers in
// forward / reverse order; 2: plain.
void cta(unsigned b, int nthreads, size_t smem_bytes, int mode,
         const std::vector<std::function<void(uint8_t*)>>& phases) {
  if (mode < 2) {
    cuemu::run_cta(b, 0, nthreads, smem_bytes, mode == 1, [&](uint8_t* smem) {
      for (size_t i = 0; i < phases.size(); ++i) {
        if (i)
          __syncthreads();
        phases[i](smem);
      }
    });
    return;
  }
  std::vector<uint8_t> smem(smem_bytes + 16, 0xCD);
  blockIdx.x = b;
  blockDim.x = (unsigned)nthreads;
  for (const auto& ph : phases)
    for (int t = 0; t < nthreads; ++t) {
      threadIdx.x = (unsigned)t;
      ph(smem.data());
    }
}
} // namespace

// jobs: w[i], h[i], out_offset[i], out_pitch[i], first strip first[i]; strips: (offset, size) per row.
// results: (status, consumed) per job.  Returns the number of jump rounds run.
extern "C" int s0_emu_run(const uint8_t* in, uint64_t in_total, int njobs, const uint32_t* w, const uint32_t* h,
                          const uint64_t* out_offset, const uint32_t* out_pitch, const uint32_t* first,
                          const uint64_t* soff, const uint32_t* ssize, uint8_t* out, uint32_t* results,
                          int mode) {
  std::vector<uint8_t> buf((size_t)in_total + 512);
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(buf.data()) + 255) & ~(uintptr_t)255);
  memcpy(base, in, (size_t)in_total);
  std::vector<S0JobDev> jobs((size_t)njobs);
  std::vector<S0RowDev> rows;
  uint64_t blk = 0, px = 0, carry = 0;
  uint32_t node = 0, rowb = 0, maxw = 0, maxtiles = 0, maxnodes = 0, depth = 0;
  for (int i = 0; i < njobs; ++i) {
    S0JobDev& j = jobs[(size_t)i];
    memset(&j, 0, sizeof j);
    j.out_offset = out_offset[i];
    j.out_pitch = out_pitch[i];
    j.w = w[i];
    j.h = h[i];
    j.nb = (w[i] + 15) / 16;
    j.blk_base = blk;
    j.px_base = px;
    j.node_base = node;
    j.row_base = rowb;
    j.rtiles = (h[i] + S0C_TH - 1) / S0C_TH;
    j.carry_base = carry;
    blk += (uint64_t)j.h * j.nb;
    px += (uint64_t)j.h * j.nb * 16;
    node += j.h * j.nb * 2;
    rowb += j.h;
    carry += (uint64_t)j.rtiles * j.nb * 32;
    maxw = std::max(maxw, j.w);
    maxtiles = std::max(maxtiles, j.rtiles);
    maxnodes = std::max(maxnodes, j.h * j.nb * 2);
    depth = std::max(depth, j.h + j.nb + 1);
    for (uint32_t r = 0; r < h[i]; ++r)
      rows.push_back(S0RowDev{soff[first[i] + r], ssize[first[i] + r], (uint32_t)i, r, 0});
  }
  int rounds = 0;
  while ((1u << rounds) < depth)
    ++rounds;
  const uint32_t nrows = (uint32_t)rows.size();
  std::vector<uint2> desc((size_t)blk, make_uint2(0xCDCDCDCDu, 0xCDCDCDCDu));
  std::vector<uint16_t> adj((size_t)px, 0xCDCD);
  std::vector<uint2> na((size_t)node), nb2((size_t)node);
  std::vector<uint32_t> carryv((size_t)carry, 0xCDCDCDCDu), rowfail(nrows, 0xCDCDCDCDu),
      jobfail((size_t)njobs, 0xFFFFFFFFu);
  std::vector<uint2> res((size_t)njobs);
  blockIdx.y = blockIdx.z = 0;
  for (uint32_t b = 0; b < (nrows + S0W_NT - 1) / S0W_NT; ++b)
    cta(b, S0W_NT, 0, mode, {[&](uint8_t*) {
          s0_walk_entry(base, rows.data(), nrows, jobs.data(), desc.data(), rowfail.data(), jobfail.data());
        }});
  for (uint32_t b = 0; b < (nrows + S0D_NT / 32 - 1) / (S0D_NT / 32); ++b)
    cta(b, S0D_NT, 0, mode,
        {[&](uint8_t*) { s0_diff_entry(base, rows.data(), nrows, jobs.data(), desc.data(), adj.data()); }});
  for (int i = 0; i < njobs; ++i) {
    blockIdx.y = (unsigned)i;
    for (uint32_t b = 0; b < (maxnodes + S0N_NT - 1) / S0N_NT; ++b)
      cta(b, S0N_NT, 0, mode, {[&](uint8_t*) { s0_node_entry(jobs.data(), desc.data(), adj.data(), na.data()); }});
  }
  blockIdx.y = 0;
  uint2* src = na.data();
  uint2* dst = nb2.data();
  for (int r = 0; r < rounds; ++r) {
    for (uint32_t b = 0; b < (node + S0N_NT - 1) / S0N_NT; ++b)
      cta(b, S0N_NT, 0, mode, {[&](uint8_t*) { s0_jump_entry(src, dst, node); }});
    std::swap(src, dst);
  }
  const uint32_t ctiles = (maxw + S0C_NT - 1) / S0C_NT;
  for (int i = 0; i < njobs; ++i)
    for (uint32_t t = 0; t < maxtiles; ++t) {
      blockIdx.y = t;
      blockIdx.z = (unsigned)i;
      for (uint32_t b = 0; b < ctiles; ++b)
        cta(b, S0C_NT, 0, mode,
            {[&](uint8_t*) { s0_scan_entry(jobs.data(), desc.data(), adj.data(), src, carryv.data()); }});
    }
  blockIdx.z = 0;
  for (int i = 0; i < njobs; ++i) {
    blockIdx.y = (unsigned)i;
    for (uint32_t b = 0; b < (2 * maxw + S0C_NT - 1) / S0C_NT; ++b)
      cta(b, S0C_NT, 0, mode, {[&](uint8_t*) { s0_carry_entry(jobs.data(), carryv.data()); }});
  }
  for (int i = 0; i < njobs; ++i)
    for (uint32_t t = 0; t < maxtiles; ++t) {
      blockIdx.y = t;
      blockIdx.z = (unsigned)i;
      for (uint32_t b = 0; b < ctiles; ++b)
        cta(b, S0C_NT, sizeof(uint16_t) * S0C_TH * S0C_NT, mode,
            {[&](uint8_t* smem) {
               s0_store_tile(jobs.data(), desc.data(), adj.data(), src, carryv.data(),
                             reinterpret_cast<uint16_t*>(smem));
             },
             [&](uint8_t* smem) {
               s0_store_out(jobs.data(), rowfail.data(), jobfail.data(), out, res.data(),
                            reinterpret_cast<uint16_t*>(smem));
             }});
    }
  blockIdx.y = blockIdx.z = 0;
  for (int i = 0; i < njobs; ++i) {
    results[2 * i] = res[(size_t)i].x;
    results[2 * i + 1] = res[(size_t)i].y;
  }
  return rounds;
}
