// cuda_emu.h -- a small "CUDA thread block on fibers" shim (test infrastructure).
//
// Lets a kernel body written for nvcc be compiled by g++ and executed on the CPU, one CTA at a
// time: every CUDA thread is a ucontext fiber, __syncthreads() / warp collectives / mbarrier
// waits are yield points of a deterministic round-robin scheduler (forward or reverse thread
// order, so order-dependent bugs -- a missing barrier -- show up as a difference between the two
// schedules).  Shared memory is one host buffer per CTA; "shared addresses" (smem_u32) are
// offsets into it.  The 1-D bulk copy (TMA) is a memcpy by the issuing thread that completes the
// mbarrier phase.  Nothing here is product code: it exists so that the arithmetic, indexing and
// barrier structure of a kernel can be checked where there is no GPU; parity of the real kernel
// is established by the GPU tests.
#pragma once

#include <stdint.h>
#include <string.h>
#include <ucontext.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <vector>

#define RSB200_EMU 1
#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __launch_bounds__(...)

struct uint2 {
  uint32_t x, y;
};
struct alignas(16) uint4 {
  uint32_t x, y, z, w;
};
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  return uint4{x, y, z, w};
}

namespace cuemu {

struct Dim {
  unsigned x = 0, y = 0, z = 0;
};

struct Fiber {
  ucontext_t ctx;
  std::vector<uint8_t> stack;
  int state = 0; // 0 runnable, 1 waiting (predicate), 2 done
  std::function<bool()> ready;
};

struct Cta {
  std::vector<Fiber> th;
  ucontext_t sched;
  int nthreads = 0;
  int cur = -1;
  bool reverse = false;
  uint8_t* smem = nullptr;
  size_t smem_bytes = 0;
  // CTA barrier
  int bar_arrived = 0;
  uint64_t bar_gen = 0;
  uint32_t bar_or_acc = 0, bar_or_res[2] = {0, 0};
  // warp collectives
  struct Warp {
    uint32_t val[32];
    uint32_t res[2][32];
    uint32_t present[2];
    int arrived = 0;
    uint32_t arrived_mask = 0;
    uint64_t gen = 0;
  };
  std::vector<Warp> warps;
  int live = 0;
  std::function<void()> body;
};

inline Cta*& cta() {
  static Cta* c = nullptr;
  return c;
}

// The global memory a kernel may read through __ldg: [ldg_lo, ldg_hi), set by a runner (unset: no
// check).  A read outside it is counted and not performed (it returns zero).
inline const uint8_t* ldg_lo = nullptr;
inline const uint8_t* ldg_hi = nullptr;
inline unsigned long long ldg_outside = 0;

} // namespace cuemu

// the CUDA built-ins the kernels read
inline cuemu::Dim threadIdx, blockIdx, blockDim, gridDim;

namespace cuemu {

inline void yield_until(std::function<bool()> pred) {
  Cta* c = cta();
  Fiber& f = c->th[(size_t)c->cur];
  f.state = 1;
  f.ready = std::move(pred);
  swapcontext(&f.ctx, &c->sched);
}

inline void fiber_entry() {
  Cta* c = cta();
  c->body();
  Fiber& f = c->th[(size_t)c->cur];
  f.state = 2;
  --c->live;
  // a thread that has exited no longer takes part in barriers
  swapcontext(&f.ctx, &c->sched);
}

// Run one CTA of `nthreads` threads with `smem_bytes` of shared memory.
inline void run_cta(unsigned block, unsigned nblocks, int nthreads, size_t smem_bytes, bool reverse,
                    const std::function<void(uint8_t* smem)>& kernel) {
  Cta c;
  cta() = &c;
  c.nthreads = nthreads;
  c.reverse = reverse;
  std::vector<uint8_t> smem(smem_bytes + 256, 0xCD); // garbage, like real shared memory
  c.smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem.data()) + 127) & ~(uintptr_t)127);
  c.smem_bytes = smem_bytes;
  c.th.resize((size_t)nthreads);
  c.warps.resize((size_t)(nthreads + 31) / 32);
  c.live = nthreads;
  c.body = [&]() { kernel(c.smem); };
  blockIdx.x = block;
  gridDim.x = nblocks;
  blockDim.x = (unsigned)nthreads;
  for (int i = 0; i < nthreads; ++i) {
    Fiber& f = c.th[(size_t)i];
    f.stack.resize(192 * 1024);
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = f.stack.data();
    f.ctx.uc_stack.ss_size = f.stack.size();
    f.ctx.uc_link = &c.sched;
    makecontext(&f.ctx, (void (*)())fiber_entry, 0);
  }
  long idle_rounds = 0;
  while (c.live > 0) {
    bool progressed = false;
    for (int k = 0; k < nthreads; ++k) {
      const int i = reverse ? nthreads - 1 - k : k;
      Fiber& f = c.th[(size_t)i];
      if (f.state == 2)
        continue;
      if (f.state == 1) {
        if (!f.ready())
          continue;
        f.state = 0;
      }
      c.cur = i;
      threadIdx.x = (unsigned)i;
      progressed = true;
      swapcontext(&c.sched, &f.ctx);
    }
    if (!progressed && ++idle_rounds > 4) {
      std::fprintf(stderr, "cuda_emu: deadlock in block %u (%d threads alive)\n", block, c.live);
      std::abort();
    }
    if (progressed)
      idle_rounds = 0;
  }
  cta() = nullptr;
}

inline uint32_t cta_barrier(uint32_t orv, bool want_or) {
  Cta* c = cta();
  const uint64_t g = c->bar_gen;
  c->bar_or_acc |= orv;
  if (++c->bar_arrived >= c->live) {
    c->bar_or_res[g & 1] = c->bar_or_acc;
    c->bar_or_acc = 0;
    c->bar_arrived = 0;
    ++c->bar_gen;
  } else {
    yield_until([c, g]() { return c->bar_gen != g; });
  }
  (void)want_or;
  return c->bar_or_res[g & 1];
}

// every lane named in `mask` contributes v; returns the 32 contributions (and which lanes were there)
inline const uint32_t* warp_exchange(uint32_t mask, uint32_t v, uint32_t* present) {
  Cta* c = cta();
  const int w = (int)threadIdx.x >> 5, lane = (int)threadIdx.x & 31;
  Cta::Warp& W = c->warps[(size_t)w];
  const uint64_t g = W.gen;
  W.val[lane] = v;
  W.arrived_mask |= 1u << lane;
  // lanes of the last (partial) warp that do not exist never arrive
  uint32_t exist = 0xFFFFFFFFu;
  const int base = w * 32;
  if (base + 32 > c->nthreads)
    exist = (1u << (c->nthreads - base)) - 1u;
  const uint32_t need = mask & exist;
  if ((W.arrived_mask & need) == need) {
    memcpy(W.res[g & 1], W.val, sizeof W.val);
    W.present[g & 1] = W.arrived_mask;
    W.arrived_mask = 0;
    ++W.gen;
  } else {
    yield_until([&W, g]() { return W.gen != g; });
  }
  *present = W.present[g & 1];
  return W.res[g & 1];
}

} // namespace cuemu

// ---------------- synchronisation ----------------
static inline void __syncthreads() { cuemu::cta_barrier(0, false); }
static inline int __syncthreads_or(int p) { return cuemu::cta_barrier(p ? 1u : 0u, true) != 0; }
static inline void __syncwarp(uint32_t mask = 0xFFFFFFFFu) {
  uint32_t pr;
  cuemu::warp_exchange(mask, 0, &pr);
}
static inline uint32_t __shfl_sync(uint32_t mask, uint32_t v, int src) {
  uint32_t pr;
  const uint32_t* r = cuemu::warp_exchange(mask, v, &pr);
  return r[src & 31];
}
static inline uint32_t __shfl_up_sync(uint32_t mask, uint32_t v, unsigned d) {
  uint32_t pr;
  const uint32_t* r = cuemu::warp_exchange(mask, v, &pr);
  const int lane = (int)threadIdx.x & 31;
  return lane >= (int)d ? r[lane - (int)d] : v;
}
static inline uint32_t __shfl_down_sync(uint32_t mask, uint32_t v, unsigned d) {
  uint32_t pr;
  const uint32_t* r = cuemu::warp_exchange(mask, v, &pr);
  const int lane = (int)threadIdx.x & 31;
  return lane + (int)d < 32 ? r[lane + (int)d] : v;
}
static inline uint32_t __ballot_sync(uint32_t mask, int p) {
  uint32_t pr;
  const uint32_t* r = cuemu::warp_exchange(mask, p ? 1u : 0u, &pr);
  uint32_t b = 0;
  for (int i = 0; i < 32; ++i)
    if (((pr >> i) & 1u) && r[i])
      b |= 1u << i;
  return b & mask;
}

// ---------------- integer intrinsics ----------------
static inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t s) {
  s &= 31u;
  return s ? (hi << s) | (lo >> (32 - s)) : hi;
}
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t s) {
  s &= 31u;
  return s ? (lo >> s) | (hi << (32 - s)) : lo;
}
static inline uint32_t __funnelshift_lc(uint32_t lo, uint32_t hi, uint32_t s) {
  if (s >= 32)
    return lo;
  return s ? (hi << s) | (lo >> (32 - s)) : hi;
}
static inline uint32_t __funnelshift_rc(uint32_t lo, uint32_t hi, uint32_t s) {
  if (s >= 32)
    return hi;
  return s ? (lo >> s) | (hi << (32 - s)) : lo;
}
static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t sel) {
  const uint64_t v = ((uint64_t)b << 32) | a;
  uint32_t r = 0;
  for (int i = 0; i < 4; ++i) {
    const uint32_t n = (sel >> (4 * i)) & 0xFu;
    uint32_t byte = (uint32_t)(v >> (8 * (n & 7u))) & 0xFFu;
    if (n & 8u)
      byte = (byte & 0x80u) ? 0xFFu : 0u;
    r |= byte << (8 * i);
  }
  return r;
}
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline int __ffs(uint32_t v) { return __builtin_ffs((int)v); }
static inline int __clz(uint32_t v) { return v ? __builtin_clz(v) : 32; }
static inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
static inline uint32_t __vadd2(uint32_t a, uint32_t b) {
  return ((a + b) & 0xFFFFu) | (((a >> 16) + (b >> 16)) << 16);
}
static inline uint32_t __vsub2(uint32_t a, uint32_t b) {
  return ((a - b) & 0xFFFFu) | (((a >> 16) - (b >> 16)) << 16);
}
static inline uint32_t __vcmpeq4(uint32_t a, uint32_t b) {
  uint32_t r = 0;
  for (int i = 0; i < 4; ++i)
    if (((a >> (8 * i)) & 0xFFu) == ((b >> (8 * i)) & 0xFFu))
      r |= 0xFFu << (8 * i);
  return r;
}
template <typename T> static inline T __ldg(const T* p) {
  const uint8_t* b = reinterpret_cast<const uint8_t*>(p);
  if (cuemu::ldg_lo && (b < cuemu::ldg_lo || b + sizeof(T) > cuemu::ldg_hi)) {
    ++cuemu::ldg_outside;
    return T{};
  }
  return *p;
}
static inline long long clock64() { return 0; }
static inline uint32_t atomicMin(uint32_t* p, uint32_t v) {
  const uint32_t o = *p;
  if (v < o)
    *p = v;
  return o;
}
static inline uint32_t atomicOr(uint32_t* p, uint32_t v) {
  const uint32_t o = *p;
  *p = o | v;
  return o;
}
static inline uint32_t atomicAdd(uint32_t* p, uint32_t v) {
  const uint32_t o = *p;
  *p = o + v;
  return o;
}
static inline uint32_t min(uint32_t a, uint32_t b) { return a < b ? a : b; }
static inline uint32_t max(uint32_t a, uint32_t b) { return a > b ? a : b; }
static inline uint64_t min(uint64_t a, uint64_t b) { return a < b ? a : b; }
static inline uint64_t max(uint64_t a, uint64_t b) { return a > b ? a : b; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }

// ---------------- the helpers of csrc/common.cuh ----------------
namespace rsb200 {

static inline uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  memcpy(&r, p, 16);
  return r;
}
static inline void stg_cs_v4(void* p, const uint4& v) { memcpy(p, &v, 16); }
static inline uint32_t smem_u32(const void* p) {
  return (uint32_t)(reinterpret_cast<const uint8_t*>(p) - cuemu::cta()->smem);
}
static inline uint32_t smem_base_opaque(const void* p) { return smem_u32(p); }
static inline uint8_t* emu_saddr(uint32_t saddr, int off, size_t n) {
  cuemu::Cta* c = cuemu::cta();
  const size_t a = (size_t)saddr + (size_t)off;
  if (a + n > c->smem_bytes) {
    std::fprintf(stderr, "cuda_emu: shared access out of bounds: %zu+%zu > %zu (thread %u)\n", a, n,
                 c->smem_bytes, threadIdx.x);
    std::abort();
  }
  if (a % n) {
    std::fprintf(stderr, "cuda_emu: misaligned shared access: %zu size %zu (thread %u)\n", a, n,
                 threadIdx.x);
    std::abort();
  }
  return c->smem + a;
}
template <int OFF = 0> static inline uint32_t lds_u8(uint32_t saddr) { return *emu_saddr(saddr, OFF, 1); }
template <int OFF = 0> static inline uint32_t lds_u16(uint32_t saddr) {
  uint16_t v;
  memcpy(&v, emu_saddr(saddr, OFF, 2), 2);
  return v;
}
template <int OFF = 0> static inline uint32_t lds_u32(uint32_t saddr) {
  uint32_t v;
  memcpy(&v, emu_saddr(saddr, OFF, 4), 4);
  return v;
}
template <int OFF = 0> static inline uint2 lds_v2(uint32_t saddr) {
  uint2 v;
  memcpy(&v, emu_saddr(saddr, OFF, 8), 8);
  return v;
}
template <int OFF = 0> static inline uint4 lds_v4(uint32_t saddr) {
  uint4 v;
  memcpy(&v, emu_saddr(saddr, OFF, 16), 16);
  return v;
}
template <int OFF = 0> static inline void sts_u8(uint32_t saddr, uint32_t v) {
  *emu_saddr(saddr, OFF, 1) = (uint8_t)v;
}
template <int OFF = 0> static inline void sts_u16(uint32_t saddr, uint32_t v) {
  const uint16_t h = (uint16_t)v;
  memcpy(emu_saddr(saddr, OFF, 2), &h, 2);
}
template <int OFF = 0> static inline void sts_u32(uint32_t saddr, uint32_t v) {
  memcpy(emu_saddr(saddr, OFF, 4), &v, 4);
}
template <int OFF = 0> static inline void sts_v2(uint32_t saddr, const uint2& v) {
  memcpy(emu_saddr(saddr, OFF, 8), &v, 8);
}
template <int OFF = 0> static inline void sts_v4(uint32_t saddr, const uint4& v) {
  memcpy(emu_saddr(saddr, OFF, 16), &v, 16);
}
static inline uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) { return __byte_perm(a, b, sel & 0xFFFFu); }
static inline uint32_t mad_hi(uint32_t a, uint32_t b, uint32_t c) {
  return (uint32_t)(((uint64_t)a * b) >> 32) + c;
}

// mbarrier: word 0 = completed phases, word 1 = outstanding transaction bytes
static inline void mbar_init(uint64_t* bar, uint32_t) { *bar = 0; }
static inline void fence_mbar_init() {}
static inline void fence_proxy_async() {}
static inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  uint32_t* w = reinterpret_cast<uint32_t*>(bar);
  w[1] = bytes;
  if (bytes == 0)
    ++w[0];
}
static inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t* w = reinterpret_cast<uint32_t*>(bar);
  if ((w[0] & 1u) == (parity & 1u))
    cuemu::yield_until([w, parity]() { return (w[0] & 1u) != (parity & 1u); });
}
static inline void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  if ((reinterpret_cast<uintptr_t>(smem_dst) | reinterpret_cast<uintptr_t>(gsrc) | bytes) & 15u) {
    std::fprintf(stderr, "cuda_emu: bulk copy not 16-byte aligned\n");
    std::abort();
  }
  memcpy(smem_dst, gsrc, bytes);
  uint32_t* w = reinterpret_cast<uint32_t*>(bar);
  w[1] -= bytes;
  if (w[1] == 0)
    ++w[0];
}

} // namespace rsb200
