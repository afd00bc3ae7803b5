// simpletuner_b200 — sm_90a device primitives shared by every kernel in csrc/.
//
// Thin inline-PTX wrappers for the Hopper async machinery (mbarrier, TMA, wgmma fences and
// shared-memory matrix descriptors).  Bit layouts follow the PTX ISA "matrix descriptor" table of
// the warpgroup-level MMA.  Nothing here is generic: sm_90a only.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

#ifndef STB_WATCHDOG
#define STB_WATCHDOG 1  // bounded mbarrier spins: a wedged pipeline traps instead of hanging the GPU
#endif

namespace stb {

// ----------------------------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// named barriers among `nthreads` threads (a multiple of 32); id 0 is __syncthreads'
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}

// ----------------------------------------------------------------------------------------------
// clusters
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster: release what this thread wrote (barrier init, remote arrives), acquire
// what the others did
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at the same shared offset as `bar` in cluster CTA `rank`.  Default (.release.cta) semantics:
// the stage it hands back was read by wgmma, complete at the wait_group before it, and .release.cluster would compile to
// a GPU-wide memory barrier that waits for the epilogue's outstanding global stores.
__device__ __forceinline__ void mbar_arrive_remote(uint32_t bar, uint32_t rank) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t"
      "}\n" ::"r"(bar), "r"(rank)
      : "memory");
}

// Diagnostics for a wedged pipeline. `tag` identifies the wait site.
__device__ unsigned int g_stb_wedge[8];

// Inline (no printf): a function call inside the consumer loops would make ptxas serialize every wgmma.
__device__ __forceinline__ void mbar_wedged(uint32_t bar, uint32_t parity, int tag) {
  g_stb_wedge[0] = 0xdeadu;
  g_stb_wedge[1] = blockIdx.x;
  g_stb_wedge[2] = threadIdx.x;
  g_stb_wedge[3] = (unsigned)tag;
  g_stb_wedge[4] = bar;
  g_stb_wedge[5] = parity;
  __threadfence_system();
  __trap();
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int tag = 0) {
#if STB_WATCHDOG
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3ffu) == 0 && (clock64() - t0) > 4000000000ll) mbar_wedged(bar, parity, tag);
  }
#else
  while (!mbar_try_wait(bar, parity)) {
  }
#endif
}

// Ring of STAGES shared-memory stages between one TMA producer warp and the consumer warps, each stage guarded by a
// full barrier (one arrival, plus the TMA transaction bytes) and an empty barrier (one arrival per consumer warp).
// `bars` is the shared address of 2 * STAGES mbarriers: full[0, STAGES), then empty[0, STAGES).  Producer and consumers
// each keep their own copy, whose {stage, phase} cursor walks the ring in the same order.
// Inline only, and it never touches accumulator registers: a call inside a consumer loop makes ptxas serialize every
// wgmma.
template <int STAGES>
struct StageRing {
  uint32_t bars;
  int stage = 0;
  uint32_t phase = 0;

  __device__ __forceinline__ uint32_t full_bar(int s) const { return bars + 8u * s; }
  __device__ __forceinline__ uint32_t empty_bar(int s) const { return bars + 8u * (STAGES + s); }
  // one thread, before the __syncthreads that publishes the barriers
  __device__ __forceinline__ void init(uint32_t consumer_warps) const {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), consumer_warps);
    }
    fence_mbar_init();
  }
  __device__ __forceinline__ void advance() {
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1u;
    }
  }
  // n advances at once: a consumer passing over the stages that another consumer takes
  __device__ __forceinline__ void skip(int n) {
    stage += n;
    const int laps = stage / STAGES;
    stage -= laps * STAGES;
    phase ^= uint32_t(laps) & 1u;
  }
  // producer: until the consumers have released the current stage (the first lap passes at once)
  __device__ __forceinline__ void wait_empty(int tag) const { mbar_wait(empty_bar(stage), phase ^ 1u, tag); }
  // consumers: until the current stage's TMA bytes have landed
  __device__ __forceinline__ void wait_full(int tag) const { mbar_wait(full_bar(stage), phase, tag); }
  // consumers: lane 0 of each warp hands stage s back to the producer
  __device__ __forceinline__ void release(int s) const {
    if (lane_id() == 0) mbar_arrive(empty_bar(s));
  }
  // 2-CTA cluster whose producers each fill stage s in both CTAs: lane 0 of each warp hands s back to both producers
  // (the empty barriers then count the consumer warps of both CTAs)
  __device__ __forceinline__ void release_cluster(int s, uint32_t peer) const {
    if (lane_id() == 0) {
      mbar_arrive(empty_bar(s));
      mbar_arrive_remote(empty_bar(s), peer);
    }
  }
};

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) — tile mode, mbarrier completion
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// the box lands at offset `dst` of every cluster CTA in `cta_mask`, and completes bytes on the mbarrier at offset `bar`
// of each of them
__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1,
                                               uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, "
      "{%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// smem -> global tile store (bulk group completion)
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2,
                                             int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// smem -> global tile reduce-add (fp32), bulk group completion
__device__ __forceinline__ void tma_reduce_add_4d(const CUtensorMap* m, uint32_t src, int c0, int c1,
                                                  int c2, int c3) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], "
      "[%1];"
      ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): fences and group completion; the MMA wrappers themselves are in wgmma.cuh
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wg_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor for wgmma, SWIZZLE_128B layouts.
//   [0,14) addr>>4  [16,30) LBO>>4  [32,46) SBO>>4  [62,64) layout (1 = SW128)
// `tile_saddr` is the 1024-byte-aligned base of a SWIZZLE_128B operand tile and `byte_off` a multiple of 16 that
// selects the K step / atom.  The address field holds bits [4, 18) of the address: in a cluster launch a CTA's shared
// addresses carry its rank above bit 18, which must not carry into the LBO field.
//   K-major tile: rows of 64 bf16 (128 B), 8-row groups 1024 B apart (SBO); K step kk -> +kk*32 B.
__device__ __forceinline__ uint64_t sdesc_k(uint32_t tile_saddr, uint32_t byte_off) {
  const uint32_t lo = ((tile_saddr & 0x3ffffu) >> 4) + (byte_off >> 4) + (1u << 16);
  const uint32_t hi = (1024u >> 4) | (1u << 30);
  return (uint64_t(hi) << 32) | lo;
}
//   MN-major tile made of [K rows x 64 MN-elements] boxes `lbo` bytes apart; 8-k groups 1024 B apart;
//   K step of 16 rows -> +2048 B.
__device__ __forceinline__ uint64_t sdesc_mn(uint32_t tile_saddr, uint32_t byte_off, uint32_t lbo) {
  const uint32_t lo = ((tile_saddr & 0x3ffffu) >> 4) + ((byte_off >> 4) + ((lbo >> 4) << 16));
  const uint32_t hi = (1024u >> 4) | (1u << 30);
  return (uint64_t(hi) << 32) | lo;
}

// per-warpgroup register re-allocation (all 4 warps of the warpgroup must execute it)
template <int N>
__device__ __forceinline__ void reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// ----------------------------------------------------------------------------------------------
// numeric helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// tanh-GELU exactly as torch.nn.GELU(approximate="tanh"):
//   0.5 x (1 + tanh( sqrt(2/pi) (x + 0.044715 x^3) ))
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  return 0.5f * x * (1.f + tanhf(u));
}
__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float x2 = x * x;
  float u = k0 * (x + k1 * x * x2);
  float t = tanhf(u);
  float du = k0 * (1.f + 3.f * k1 * x2);
  return 0.5f * (1.f + t) + 0.5f * x * (1.f - t * t) * du;
}

}  // namespace stb
