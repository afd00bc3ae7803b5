// simpletuner_b200 — full-rank weight gradient GEMM on wgmma, sm_90a (full fine-tune, BASELINE config 3).
//
//   dW[n, k] = alpha * sum_{b,s} dY[b, s, n] * X[b, s, k]   (+ dW_old[n, k])        bf16 out, fp32 accumulation
//
// This is the autograd of every nn.Linear weight the reference trains when `model_type=full`
// (reference trainer.py:7126 `accelerator.backward`; SD3 blocks sd3/transformer.py:145-241).  Both operands are contracted
// over their SLOW dimension (the token rows), so both are MN-major for the tensor core — the layout of wgrad.cuh (the
// rank-r LoRA version), generalised to a persistent, tiled kernel:
//   A = dY^T tile [128 n x 64 tokens]  (two   [64 tokens x 64 n] SWIZZLE_128B boxes, one per consumer warpgroup)
//   B = X^T  tile [BN  k x 64 tokens]  (BN/64 [64 tokens x 64 k] boxes),  D tile [128 x BN] fp32 in registers,
// k-blocks run over (batch, 64-token chunk); rows past the end of a batch slab are zero-filled by TMA, so ragged
// sequences and strided [B, S, N] views (a row range of the joint hidden buffer) need no copies.
// Roles (384 threads): warpgroup 0 TMA producer, warpgroups 1-2 wgmma + epilogue (64 n-rows each).
// Algorithmic work: 2 * M * N * K flops (M = B*S tokens) — the same as the forward GEMM of that layer.
#pragma once
#include "common.cuh"
#include "elementwise.cuh"
#include "gemm.cuh"

namespace stb {

struct WgradFullParams {
  int S, B, N, K;
  float alpha;
  int accumulate;               // 1: out += (bf16 read-modify-write)
  __nv_bfloat16* out;           // [N, K]
  long long out_row_stride;
};

struct WgradFullMaps {
  CUtensorMap dy;  // 3-D (n, s, b) box (64, 64, 1) SWIZZLE_128B
  CUtensorMap x;   // 3-D (k, s, b) box (64, 64, 1) SWIZZLE_128B
};

template <int BN>
struct WgradFullCfg {
  static constexpr int A_BYTES = 2 * 8192;
  static constexpr int B_BYTES = (BN / 64) * 8192;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (200 * 1024) / STAGE_BYTES > 8 ? 8 : (200 * 1024) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

// D (64 x N) += A^T B over 16 token rows, both operands MN-major
template <int N>
__device__ __forceinline__ void wgmma_mn_mn(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (N == 256) wgmma_ss_n256<1, 1>(d, a, b, accumulate);
  else if constexpr (N == 128) wgmma_ss_n128<1, 1>(d, a, b, accumulate);
  else wgmma_ss_n64<1, 1>(d, a, b, accumulate);
}

template <int BN>
__global__ void __launch_bounds__(384, 1)
wgrad_full_kernel(const __grid_constant__ WgradFullMaps maps, const WgradFullParams p) {
  using Cfg = WgradFullCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int A_BYTES = Cfg::A_BYTES, STAGE_BYTES = Cfg::STAGE_BYTES;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)
  const int tiles_n = (p.N + 127) / 128;
  const int tiles_k = (p.K + BN - 1) / BN;
  const int num_tiles = tiles_n * tiles_k;
  const int chunks = (p.S + 63) / 64;       // 64-token chunks per batch slab
  const int kblocks = chunks * p.B;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps.dy);
    tma_prefetch_desc(&maps.x);
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
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        // k-tile fastest: CTAs running side by side share the dY columns (A) of one n-tile through L2
        const int tn = tile / tiles_k, tk = tile - tn * tiles_k;
        const int n0 = tn * 128, k0 = tk * BN;
        for (int kb = 0; kb < kblocks; ++kb) {
          const int b = kb / chunks, s = (kb - b * chunks) * 64;
          mbar_wait(empty_bar(stage), phase ^ 1u, 80);
          const uint32_t sa = smem_base + stage * STAGE_BYTES;
          if (elect_one()) {
            mbar_arrive_expect_tx(full_bar(stage), STAGE_BYTES);
            tma_load_3d(sa, &maps.dy, full_bar(stage), n0, s, b);
            tma_load_3d(sa + 8192, &maps.dy, full_bar(stage), n0 + 64, s, b);
#pragma unroll
            for (int a = 0; a < BN / 64; ++a) tma_load_3d(sa + A_BYTES + a * 8192, &maps.x, full_bar(stage), k0 + a * 64, s, b);
          }
          __syncwarp();
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else {
    reg_alloc<232>();
    const int cw = wg - 1, wq = warp & 3;
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int tn = tile / tiles_k, tk = tile - tn * tiles_k;
      const int k0 = tk * BN;
      uint32_t accumulate = 0;
      int prev_stage = -1;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(full_bar(stage), phase, 82);
        const uint32_t sa = smem_base + stage * STAGE_BYTES;
        // tokens past the end of the slab are zeros (TMA fill), so a ragged last chunk runs all four K steps too
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          wgmma_mn_mn<BN>(acc, sdesc_mn(sa + cw * 8192, kk * 2048, 8192), sdesc_mn(sa + A_BYTES, kk * 2048, 8192), accumulate);
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
      if (lane == 0) mbar_arrive(empty_bar(prev_stage));
      // acc[4 i + 2 hh + e] = dW row n_lo + 8 hh, column k0 + 8 i + 2 (lane % 4) + e
      const int n_lo = tn * 128 + cw * 64 + wq * 16 + (lane >> 2);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int n = n_lo + 8 * hh;
        if (n >= p.N) continue;
        __nv_bfloat16* orow = p.out + (long long)n * p.out_row_stride;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const int k = k0 + 8 * i + 2 * (lane & 3);
          if (k < p.K) {   // K % 8 == 0: the pair is whole
            float f0 = p.alpha * acc[4 * i + 2 * hh], f1 = p.alpha * acc[4 * i + 2 * hh + 1];
            uint32_t* dp = reinterpret_cast<uint32_t*>(orow + k);
            if (p.accumulate) {
              const uint32_t o = *dp;
              f0 += bf16_lo(o);
              f1 += bf16_hi(o);
            }
            *dp = pack_bf16x2(f0, f1);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Per-(batch, column) reductions over the token axis, fp32 atomics into zeroed outputs:
//   sum[b, d] = sum_s dy[b, s, d]            (gradient of an adaLN shift, bias gradients when summed over b on the host)
//   dot[b, d] = sum_s dy[b, s, d] * z[b, s, d]   (gradient of an adaLN scale with z = LayerNorm(x), of a gate with z = the
//                                                 gated linear output)
// Either output may be null.  HBM-bound: reads dy (and z) once.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
colsum2_kernel(const __nv_bfloat16* __restrict__ dy, long long dy_b, long long dy_s, const __nv_bfloat16* __restrict__ z,
               long long z_b, long long z_s, float* __restrict__ sum, float* __restrict__ dot, int B, int S, int D,
               int rows_per_cta) {
  const int vecs = D >> 3;
  const int b = blockIdx.z;
  const int s0 = blockIdx.y * rows_per_cta;
  const int s1 = min(S, s0 + rows_per_cta);
  for (int vi = blockIdx.x * blockDim.x + threadIdx.x; vi < vecs; vi += gridDim.x * blockDim.x) {
    const int c = vi * 8;
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, d[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = s0; s < s1; ++s) {
      float g[8];
      unpack8(*reinterpret_cast<const uint4*>(dy + b * dy_b + s * dy_s + c), g);
      if (dot) {
        float zz[8];
        unpack8(*reinterpret_cast<const uint4*>(z + b * z_b + s * z_s + c), zz);
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] += g[j] * zz[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += g[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (sum) atomicAdd(sum + (long long)b * D + c + j, a[j]);
      if (dot) atomicAdd(dot + (long long)b * D + c + j, d[j]);
    }
  }
}

}  // namespace stb
