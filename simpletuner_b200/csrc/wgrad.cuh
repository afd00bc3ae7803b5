// simpletuner_b200 — weight-gradient GEMM on wgmma, sm_90a: the token rows are the contraction.
//
//   D[n, k] = sum_{b,s} A[b, s, n] * B[b, s, k]          fp32 accumulation, two output kinds:
//
//   WGRAD_OUT_F32_RN   out[k, n] (fp32 [R, N], k = r < R <= 128): LoRA weight gradients (autograd of peft lora.Linear,
//                      reference common.py:1094-1117), A = Rm and B = L, the rank-r operand as one BN-wide box (columns
//                      past R are TMA zeros):
//                        dA = (dY B)^T X      -> L = dY B [M, r],   Rm = X  [M, K]
//                        dB^T = (X A^T)^T dY  -> L = X A^T [M, r],  Rm = dY [M, N]
//                      Each token split writes a slab of `partial` with plain stores (summed in slab order by
//                      wgrad_reduce_slabs_kernel, run-to-run reproducible), or, with `partial` null, adds alpha * D
//                      into `out_f32` with fp32 atomics.  HBM-bound (reads Rm once).
//   WGRAD_OUT_BF16_NK  out[n, k] (bf16 [N, K]) = alpha * D (+ out[n, k]): full-rank weight gradients (full fine-tune,
//                      BASELINE config 3; reference trainer.py:7126 `accelerator.backward`, SD3 blocks
//                      sd3/transformer.py:145-241), A = dY and B = X.  2 * M * N * K flops (M = B*S tokens), the same
//                      as the forward GEMM of that layer.
//
// Both operands are contracted over their SLOW dimension, so both are MN-major for the tensor core:
//   A^T tile [128 n x 64 tokens]  (two   [64 tokens x 64 n] SWIZZLE_128B boxes, one per consumer warpgroup)
//   B^T tile [BN  k x 64 tokens]  (BN/64 [64 tokens x 64 k] boxes),  D tile [128 x BN] fp32 in registers.
// A work unit is (token split y, n-tile, column tile), column tile fastest, so that CTAs running side by side share the
// A columns of one n-tile through L2.  Its k-blocks are a contiguous range of the flattened (batch, 64-token chunk)
// index; tokens past the end of a batch slab are zero-filled by TMA, so ragged sequences and strided [B, S, N] views
// (a row range of the joint hidden buffer) need no copies.
// Roles (384 threads): warpgroup 0 TMA producer, warpgroups 1-2 wgmma + epilogue (64 n each); the grid is persistent
// over the units.
#pragma once
#include "common.cuh"

namespace stb {

enum WgradOut : int { WGRAD_OUT_F32_RN = 0, WGRAD_OUT_BF16_NK = 1 };

struct WgradParams {
  int N, K;             // output rows (columns of A) and columns (of B; the rank R for WGRAD_OUT_F32_RN)
  int chunks;           // 64-token chunks per batch slab
  // token splits: split y covers k-blocks [g0, min(g0 + kb_per_split, (y / splits_per_group + 1) * kb_per_group)),
  // g0 = (y / splits_per_group) * kb_per_group + (y % splits_per_group) * kb_per_split.  Every split is non-empty.
  int splits, splits_per_group, kb_per_group, kb_per_split;
  int col_tiles;        // ceil(K / BN)
  float alpha;
  float* partial;       // WGRAD_OUT_F32_RN: [splits][R][N] slabs, or nullptr = atomics into out_f32
  float* out_f32;       // WGRAD_OUT_F32_RN: [R, N]
  __nv_bfloat16* out;   // WGRAD_OUT_BF16_NK: [N, K], rows out_row_stride apart
  long long out_row_stride;
  int accumulate;       // WGRAD_OUT_BF16_NK, 1: out += (bf16 read-modify-write)
};

struct WgradMaps {
  CUtensorMap a;  // 3-D (n, s, b) box (64, 64, 1) SWIZZLE_128B
  CUtensorMap b;  // 3-D (k, s, b) box (64, 64, 1) SWIZZLE_128B
};

template <int BN, int OUT>
struct WgradCfg {
  static constexpr int A_BYTES = 2 * 8192;
  static constexpr int B_BYTES = (BN / 64) * 8192;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES =
      OUT == WGRAD_OUT_F32_RN ? 6 : ((200 * 1024) / STAGE_BYTES > 8 ? 8 : (200 * 1024) / STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

// D (64 x N) += A^T B over 16 token rows, both operands MN-major
template <int N>
__device__ __forceinline__ void wgmma_mn_mn(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (N == 256) wgmma_ss_n256<1, 1>(d, a, b, accumulate);
  else if constexpr (N == 128) wgmma_ss_n128<1, 1>(d, a, b, accumulate);
  else wgmma_ss_n64<1, 1>(d, a, b, accumulate);
}

struct WgradUnit {
  int y, n0, k0, kb_begin, kb_end;
};

__device__ __forceinline__ WgradUnit wgrad_unit(const WgradParams& p, int unit, int tiles_n, int bn) {
  WgradUnit u;
  const int tk = unit % p.col_tiles, rest = unit / p.col_tiles;
  u.y = rest / tiles_n;
  u.n0 = (rest - u.y * tiles_n) * 128;
  u.k0 = tk * bn;
  const int group = u.y / p.splits_per_group;
  u.kb_begin = group * p.kb_per_group + (u.y - group * p.splits_per_group) * p.kb_per_split;
  u.kb_end = min(u.kb_begin + p.kb_per_split, (group + 1) * p.kb_per_group);
  return u;
}

template <int BN, int OUT>
__global__ void __launch_bounds__(384, 1)
wgrad_kernel(const __grid_constant__ WgradMaps maps, const WgradParams p) {
  using Cfg = WgradCfg<BN, OUT>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int A_BYTES = Cfg::A_BYTES, STAGE_BYTES = Cfg::STAGE_BYTES;
  constexpr bool F32 = OUT == WGRAD_OUT_F32_RN;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  StageRing<STAGES> ring{smem_base + STAGES * STAGE_BYTES};

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)
  const int tiles_n = (p.N + 127) / 128;
  const int units = p.splits * tiles_n * p.col_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps.a);
    tma_prefetch_desc(&maps.b);
    ring.init(8);
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (warp == 0) {
      for (int unit = blockIdx.x; unit < units; unit += gridDim.x) {
        const WgradUnit u = wgrad_unit(p, unit, tiles_n, BN);
        // k-block g = (batch b, tokens 64 c ..), walked without a division per k-block: one in the producer's issue
        // path slows the HBM-bound LoRA gradient by ~4 %
        int b = u.kb_begin / p.chunks, c = u.kb_begin - b * p.chunks;
        for (int g = u.kb_begin; g < u.kb_end; ++g) {
          const int s = c * 64;
          ring.wait_empty(F32 ? 60 : 80);
          const uint32_t sa = smem_base + ring.stage * STAGE_BYTES;
          const uint32_t full = ring.full_bar(ring.stage);
          if (elect_one()) {
            mbar_arrive_expect_tx(full, STAGE_BYTES);
            tma_load_3d(sa, &maps.a, full, u.n0, s, b);
            tma_load_3d(sa + 8192, &maps.a, full, u.n0 + 64, s, b);
#pragma unroll
            for (int i = 0; i < BN / 64; ++i) tma_load_3d(sa + A_BYTES + i * 8192, &maps.b, full, u.k0 + i * 64, s, b);
          }
          __syncwarp();
          ring.advance();
          if (++c == p.chunks) {
            c = 0;
            ++b;
          }
        }
      }
    }
  } else {
    reg_alloc<232>();
    const int cw = wg - 1, wq = warp & 3;
    float acc[BN / 2];
    for (int unit = blockIdx.x; unit < units; unit += gridDim.x) {
      const WgradUnit u = wgrad_unit(p, unit, tiles_n, BN);
      uint32_t accumulate = 0;
      int prev_stage = -1;
      for (int g = u.kb_begin; g < u.kb_end; ++g) {
        ring.wait_full(F32 ? 61 : 82);
        const uint32_t sa = smem_base + ring.stage * STAGE_BYTES;
        // tokens past the end of the slab are zeros (TMA fill), so a ragged last chunk runs all four K steps too
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          wgmma_mn_mn<BN>(acc, sdesc_mn(sa + cw * 8192, kk * 2048, 8192), sdesc_mn(sa + A_BYTES, kk * 2048, 8192), accumulate);
          accumulate = 1;
        }
        wg_commit();
        // keep one k-block in flight; the one before it has retired -> free its slot
        wg_wait<1>();
        wg_fence_regs(acc);
        if (prev_stage >= 0) ring.release(prev_stage);
        prev_stage = ring.stage;
        ring.advance();
      }
      wg_wait<0>();
      wg_fence_regs(acc);
      ring.release(prev_stage);
      // acc[4 i + 2 hh + e] = D row n_lo + 8 hh, column k0 + 8 i + 2 (lane % 4) + e
      const int n_lo = u.n0 + cw * 64 + wq * 16 + (lane >> 2);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int n = n_lo + 8 * hh;
        if (n >= p.N) continue;
        if constexpr (F32) {
#pragma unroll
          for (int i = 0; i < BN / 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int r = u.k0 + 8 * i + 2 * (lane & 3) + e;
              if (r < p.K) {
                const float v = acc[4 * i + 2 * hh + e];
                if (p.partial) p.partial[((long long)u.y * p.K + r) * p.N + n] = v;
                else atomicAdd(p.out_f32 + (long long)r * p.N + n, p.alpha * v);
              }
            }
        } else {
          __nv_bfloat16* orow = p.out + (long long)n * p.out_row_stride;
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) {
            const int k = u.k0 + 8 * i + 2 * (lane & 3);
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
