// TEST INFRASTRUCTURE.  CUDA names on top of std::thread, for running kernel SOURCE TEXT on the CPU (see
// hotpath_emul.cpp, text_emul.cpp -DEMUL_PARSE_KERNEL): a CTA is a group of threads with a barrier, a warp 32 of them
// with emulated shuffles / ballots / reductions, a bulk copy is a memcpy that completes an emulated mbarrier phase.
// Validates source logic, not machine code.
#pragma once
#include <algorithm>
#include <atomic>
#include <barrier>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <memory>
#include <string>
#include <thread>
#include <vector>

using std::max;
using std::min;

#define __device__
#define __global__
#define __forceinline__ inline
#define __launch_bounds__(x)
#define __restrict__
#define __align__(x)

struct float4 { float x, y, z, w; };
struct uint4 { uint32_t x, y, z, w; };
static inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }
static inline uint4 make_uint4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { return uint4{a, b, c, d}; }

struct Dim3 { unsigned x; };
struct WarpCtx {
  std::barrier<> bar{32};
  uint32_t slot[32];
};
struct CtaCtx {
  CtaCtx(unsigned threads, size_t smem_bytes) : bar((std::ptrdiff_t)threads), warps(threads / 32), smem_store(smem_bytes + 256) {
    smem = smem_store.data();
    smem += (128 - reinterpret_cast<uintptr_t>(smem) % 128) % 128;
  }
  std::barrier<> bar;
  std::vector<WarpCtx> warps;
  std::vector<unsigned char> smem_store;
  unsigned char* smem = nullptr;
  unsigned long long s_cnt[3] = {0, 0, 0};
  unsigned int s_last = 0, s_next = 0;
};
static thread_local Dim3 threadIdx, blockIdx, blockDim, gridDim;
static thread_local CtaCtx* tl_cta = nullptr;

static inline WarpCtx& warp_ctx() { return tl_cta->warps[threadIdx.x >> 5]; }
static inline uint32_t xchg(uint32_t mine, int from_lane) {   // every lane publishes, then reads one lane's word
  WarpCtx& w = warp_ctx();
  w.slot[threadIdx.x & 31] = mine;
  w.bar.arrive_and_wait();
  const uint32_t r = w.slot[from_lane & 31];
  w.bar.arrive_and_wait();
  return r;
}
static inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline void __syncthreads() { tl_cta->bar.arrive_and_wait(); }
static inline void __syncwarp() { warp_ctx().bar.arrive_and_wait(); }
static inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
static inline void __nanosleep(unsigned) { std::this_thread::yield(); }
static inline int __popc(uint32_t x) { return __builtin_popcount(x); }
static inline float __int_as_float(int x) { return u2f((uint32_t)x); }
static inline uint32_t __shfl_xor_sync(unsigned, uint32_t v, int o) { return xchg(v, (threadIdx.x & 31) ^ o); }
static inline float __shfl_xor_sync(unsigned, float v, int o) { return u2f(xchg(f2u(v), (threadIdx.x & 31) ^ o)); }
static inline uint32_t __shfl_sync(unsigned, uint32_t v, int lane) { return xchg(v, lane); }
static inline uint32_t __ballot_sync(unsigned, bool pred) {
  WarpCtx& w = warp_ctx();
  w.slot[threadIdx.x & 31] = pred ? 1u : 0u;
  w.bar.arrive_and_wait();
  uint32_t r = 0;
  for (int l = 0; l < 32; ++l) r |= w.slot[l] << l;
  w.bar.arrive_and_wait();
  return r;
}
static inline uint32_t __reduce_or_sync(unsigned, uint32_t v) {
  WarpCtx& w = warp_ctx();
  w.slot[threadIdx.x & 31] = v;
  w.bar.arrive_and_wait();
  uint32_t r = 0;
  for (int l = 0; l < 32; ++l) r |= w.slot[l];
  w.bar.arrive_and_wait();
  return r;
}
static inline uint32_t __reduce_max_sync(unsigned, uint32_t v) {
  WarpCtx& w = warp_ctx();
  w.slot[threadIdx.x & 31] = v;
  w.bar.arrive_and_wait();
  uint32_t r = 0;
  for (int l = 0; l < 32; ++l) r = std::max(r, w.slot[l]);
  w.bar.arrive_and_wait();
  return r;
}
static inline uint32_t __vmaxu4(uint32_t a, uint32_t b) {
  uint32_t r = 0;
  for (int k = 0; k < 4; ++k) r |= std::max((a >> (8 * k)) & 0xffu, (b >> (8 * k)) & 0xffu) << (8 * k);
  return r;
}
template <class T> static inline T __ldcg(const T* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned int atomicAdd(unsigned int* p, unsigned int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned int atomicOr(unsigned int* p, unsigned int v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }

// ---- the helpers that are inline PTX in the header -------------------------------------------------------------
static inline unsigned long long gtime() {
  return (unsigned long long)std::chrono::duration_cast<std::chrono::nanoseconds>(
             std::chrono::steady_clock::now().time_since_epoch()).count();
}
static inline void pdl_launch_dependents() {}
static inline void pdl_wait_prior_grids() {}   // the driver joins the reduce grid before it starts the fold grid
static inline void spin_until_gpu(const unsigned long long* p, unsigned long long want) {
  while (__atomic_load_n(p, __ATOMIC_ACQUIRE) < want) std::this_thread::yield();
}
static inline void spin_until_sys(const unsigned long long* p, unsigned long long want, unsigned int*, unsigned) {
  spin_until_gpu(p, want);
}
static inline void st_release_u64(unsigned long long* p, unsigned long long v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
static inline void st_release_sys_u64(unsigned long long* p, unsigned long long v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
static inline void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) { __atomic_store_n(p, v, __ATOMIC_RELAXED); }
static inline unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
static inline float4 ldg_stream(const float4* p) { return *p; }
static inline uint4 ldg_stream_u4(const uint4* p) { return *p; }
// an mbarrier is emulated by the number of completed phases; a bulk copy completes its phase when the bytes are there
static inline void mbar_init(uint64_t* bar, uint32_t) { __atomic_store_n(bar, (uint64_t)0, __ATOMIC_RELEASE); }
static inline void mbar_expect_tx(uint64_t*, uint32_t) {}
static inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  while ((__atomic_load_n(bar, __ATOMIC_ACQUIRE) & 1u) == parity) std::this_thread::yield();
}
static inline void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t) {
  if (bytes % 16u != 0 || reinterpret_cast<uintptr_t>(src) % 16u != 0 || reinterpret_cast<uintptr_t>(dst) % 16u != 0) {
    fprintf(stderr, "bulk copy with unaligned address or size (%u bytes)\n", bytes);   // what the hardware rejects
    abort();
  }
  memcpy(dst, src, bytes);
  __atomic_fetch_add(bar, (uint64_t)1, __ATOMIC_RELEASE);
}
static inline uint64_t l2_evict_first_policy() { return 0; }


// ---- more built-ins (the text parse kernel) ------------------------------------------------------------------
static inline unsigned int __float_as_uint(float f) { return f2u(f); }
static inline float __uint_as_float(unsigned int u) { return u2f(u); }
static inline int __ffs(uint32_t x) { return __builtin_ffs((int)x); }
static inline uint32_t __vcmpeq4(uint32_t a, uint32_t b) {
  uint32_t r = 0;
  for (int k = 0; k < 4; ++k)
    if (((a >> (8 * k)) & 0xffu) == ((b >> (8 * k)) & 0xffu)) r |= 0xffu << (8 * k);
  return r;
}
static inline uint32_t __reduce_add_sync(unsigned, uint32_t v) {
  WarpCtx& w = warp_ctx();
  w.slot[threadIdx.x & 31] = v;
  w.bar.arrive_and_wait();
  uint32_t r = 0;
  for (int l = 0; l < 32; ++l) r += w.slot[l];
  w.bar.arrive_and_wait();
  return r;
}
static inline uint32_t __shfl_up_sync(unsigned, uint32_t v, int d) {
  const int lane = (int)(threadIdx.x & 31);
  return xchg(v, lane >= d ? lane - d : lane);   // lanes below d keep their own value
}
static inline bool __all_sync(unsigned, bool pred) { return __ballot_sync(0xffffffffu, pred) == 0xffffffffu; }
static inline int atomicMax(int* p, int v) {
  int old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (old < v && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_SEQ_CST, __ATOMIC_RELAXED)) {
  }
  return old;
}
static inline unsigned int atomicCAS(unsigned int* p, unsigned int expect, unsigned int v) {
  __atomic_compare_exchange_n(p, &expect, v, false, __ATOMIC_SEQ_CST, __ATOMIC_RELAXED);
  return expect;
}

// ---- launching a grid ------------------------------------------------------------------------------------------
// CTAs resident at once (0 = the whole grid).  A kernel whose CTAs never wait for one another — the reduce kernels,
// the single-GPU fold — may run in waves, as on a device with fewer SMs than CTAs; a wide grid of 1024-thread CTAs
// then does not need thousands of threads at once.
static unsigned g_max_resident_ctas = 0;

template <class Fn>
static void launch(unsigned grid, unsigned threads, size_t smem, Fn&& kernel) {
  const unsigned wave = g_max_resident_ctas ? g_max_resident_ctas : std::max(grid, 1u);
  for (unsigned c0 = 0; c0 < grid; c0 += wave) {
    const unsigned c1 = std::min(grid, c0 + wave);
    std::vector<std::unique_ptr<CtaCtx>> ctas;
    std::vector<std::thread> th;
    for (unsigned c = c0; c < c1; ++c) ctas.push_back(std::make_unique<CtaCtx>(threads, smem));
    for (unsigned c = c0; c < c1; ++c)
      for (unsigned t = 0; t < threads; ++t)
        th.emplace_back([&, c, t] {
          threadIdx.x = t, blockIdx.x = c, blockDim.x = threads, gridDim.x = grid;
          tl_cta = ctas[c - c0].get();
          kernel();
        });
    for (auto& t : th) t.join();
  }
}
