// simpletuner_b200 — "TN over rows" wgmma GEMM for weight gradients, sm_90a.
//
//   out[r, n] += alpha * sum_{b,s}  L[b, s, r] * Rm[b, s, n]          (fp32 out, atomics across row splits)
//
// Both operands are contracted over their SLOW dimension (the token rows), i.e. both are MN-major
// for the tensor core: A = Rm^T tile [128 n x 64 rows], B = L^T tile [RN x 64 rows], D^T[n, r] in registers
// (RN = the rank block rounded up to 64; TMA zero-fills the columns past R).
// Used for the LoRA weight gradients (autograd of peft lora.Linear, reference common.py:1094-1117):
//   dA = (dY B)^T X      -> L = dY B [M, r],   Rm = X  [M, K]
//   dB^T = (X A^T)^T dY  -> L = X A^T [M, r],  Rm = dY [M, N]
// HBM-bound (reads Rm once); grid = n-tiles x row-splits so that ~all SMs stream concurrently.
// Roles (384 threads): warpgroup 0 TMA producer, warpgroups 1-2 wgmma + epilogue (64 n each).
#pragma once
#include "common.cuh"
#include "wgrad_full.cuh"

namespace stb {

struct WgradParams {
  int S, B, N, R;
  int rows_per_split;   // multiple of 64
  int splits_per_batch;
  float alpha;
  float* out;           // [R, N] fp32
  float* partial;       // deterministic mode: [gridDim.y][R][N] slabs written with plain stores (summed in slab order by
                        // wgrad_reduce_slabs_kernel); nullptr = fp32 atomics straight into `out`
};

struct WgradMaps {
  CUtensorMap rm;  // 3-D (n, s, b) box (64, 64, 1) SWIZZLE_128B
  CUtensorMap l;   // 3-D (r, s, b) box (64, 64, 1) SWIZZLE_128B
};

template <int RN>
struct WgradCfg {
  static constexpr int A_BYTES = 2 * 8192;                // two [64 rows x 64 n] atoms
  static constexpr int B_BYTES = 8192 * (RN / 64);
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = 6;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

template <int RN>  // rank block rounded up to 64 (64 or 128)
__global__ void __launch_bounds__(384, 1)
wgrad_tn_kernel(const __grid_constant__ WgradMaps maps, const WgradParams p) {
  using Cfg = WgradCfg<RN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int A_BYTES = Cfg::A_BYTES;
  constexpr int STAGE_BYTES = Cfg::STAGE_BYTES;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)
  const int n0 = blockIdx.x * 128;
  const int b = blockIdx.y / p.splits_per_batch;
  const int s_begin = (blockIdx.y % p.splits_per_batch) * p.rows_per_split;
  const int s_end = min(p.S, s_begin + p.rows_per_split);
  const int kblocks = (s_end - s_begin + 63) / 64;
  if (kblocks <= 0) return;  // uniform per CTA

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps.rm);
    tma_prefetch_desc(&maps.l);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (warp == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(empty_bar(stage), phase ^ 1u, 60);
        const uint32_t sa = smem_base + stage * STAGE_BYTES;
        const int s = s_begin + kb * 64;
        if (elect_one()) {
          mbar_arrive_expect_tx(full_bar(stage), STAGE_BYTES);
          tma_load_3d(sa, &maps.rm, full_bar(stage), n0, s, b);
          tma_load_3d(sa + 8192, &maps.rm, full_bar(stage), n0 + 64, s, b);
#pragma unroll
          for (int ra = 0; ra < RN / 64; ++ra) tma_load_3d(sa + A_BYTES + ra * 8192, &maps.l, full_bar(stage), ra * 64, s, b);
        }
        __syncwarp();
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
  } else {
    reg_alloc<232>();
    const int cw = wg - 1, wq = warp & 3;
    float acc[RN / 2];
    int stage = 0;
    uint32_t phase = 0;
    uint32_t accumulate = 0;
    int prev_stage = -1;
    for (int kb = 0; kb < kblocks; ++kb) {
      mbar_wait(full_bar(stage), phase, 61);
      const uint32_t sa = smem_base + stage * STAGE_BYTES;
      // a block never reaches into the next split (rows_per_split % 64 == 0); rows >= S are zero-filled by TMA
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        wgmma_mn_mn<RN>(acc, sdesc_mn(sa + cw * 8192, kk * 2048, 8192), sdesc_mn(sa + A_BYTES, kk * 2048, 8192), accumulate);
        accumulate = 1;
      }
      wg_commit();
      wg_wait<1>();
      wg_fence_regs(acc);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));
      prev_stage = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    // acc[4 i + 2 hh + e] = D^T row n_lo + 8 hh (an n), column 8 i + 2 (lane % 4) + e (an r)
    const int n_lo = n0 + cw * 64 + wq * 16 + (lane >> 2);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int n = n_lo + 8 * hh;
      if (n >= p.N) continue;
#pragma unroll
      for (int i = 0; i < RN / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = 8 * i + 2 * (lane & 3) + e;
          if (r < p.R) {
            const float v = acc[4 * i + 2 * hh + e];
            if (p.partial) p.partial[((long long)blockIdx.y * p.R + r) * p.N + n] = v;
            else atomicAdd(p.out + (long long)r * p.N + n, p.alpha * v);
          }
        }
    }
  }
}

// out[i] += alpha * sum_y partial[y][i], slabs in index order (run-to-run reproducible LoRA gradients)
__global__ void __launch_bounds__(256)
wgrad_reduce_slabs_kernel(const float* __restrict__ partial, float* __restrict__ out, int slabs, long long n, float alpha) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int y = 0; y < slabs; ++y) acc += partial[(long long)y * n + i];
    out[i] += alpha * acc;
  }
}

}  // namespace stb
