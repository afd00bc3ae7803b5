// simpletuner_b200 — persistent warp-specialised wgmma GEMM for sm_90a.
//
//   D[b, s, n] = epilogue( sum_seg  A_seg[b, s, :] . W_seg[n, :]  + bias[n] )
//
// Every operand is K-major bf16 ("TN": activations [rows, K], nn.Linear weights [N, K]), fp32
// accumulation in registers.  Up to three K-segments are chained in one mainloop so that
//   * torch.cat([attn, mlp], -1) @ W^T          (reference flux/transformer.py:460-464)
//   * x @ W^T + (x A^T) B^T   (PEFT LoRA linear, reference common.py:1094-1117)
// become extra k-blocks of the same tile instead of extra kernels / extra HBM round trips.
//
// Roles (384 threads, three warpgroups): warpgroup 0 = TMA producer (one warp issues), warpgroups 1 and 2 =
// consumers, each owning 64 rows of the CTA's 128 x BN tile: wgmma m64nBNk16 from shared memory, then the fused
// epilogue straight from the accumulator registers.  The grid is persistent, so the producer already streams the
// k-blocks of the next tile while the consumers run the epilogue of the current one.  CONV = true turns the A
// operand into the shifted NHWC window of a 3x3 convolution (implicit GEMM, VAE encoder).
#pragma once
#include <type_traits>
#include "common.cuh"

namespace stb {

enum GemmEpi : int {
  EPI_STORE = 0,        // D = acc + bias
  EPI_GELU = 1,         // D = gelu_tanh(acc + bias); aux (optional) = acc + bias (pre-activation)
  EPI_GATE_RES = 2,     // D = res + gate[b, n] * (acc + bias); optional nan_to_num; aux (optional) = acc + bias
  EPI_MUL_DGELU = 3,    // D = acc * gelu_tanh'(aux)          (dgrad through the activation)
  EPI_ADD_RES = 4,      // D = acc + bias + res                (gradient accumulation; residual add of the text encoders)
  EPI_MUL = 5,          // D = (acc + bias) * aux              (T5 gated feed-forward: gelu(x wi_0) * (x wi_1))
  EPI_QUICK_GELU = 6,   // D = y * sigmoid(1.702 y), y = bf16(acc + bias)   (CLIP text model activation)
};

struct GemmParams {
  int rows_per_batch;  // S : rows in one batch slab of A / D
  int num_batches;     // B
  int N;
  int nseg;
  int kblocks[3];  // ceil(K_seg / 64)
  int w_kn[3];        // 1: the segment's weight is given as [K, N] row-major (contraction index = row): the B operand is
                      // staged MN-major (64 k-rows x 64 n-columns SWIZZLE_128B boxes) — dgrad reads W itself, no W^T copy
  int epi;
  int nan_to_num;
  __nv_bfloat16* D;
  long long d_batch_stride, d_row_stride;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* gate;
  long long gate_batch_stride;
  const __nv_bfloat16* res;
  long long res_batch_stride, res_row_stride;
  __nv_bfloat16* aux;  // EPI_GELU / EPI_GATE_RES: written (optional); EPI_MUL_DGELU: read
  long long aux_batch_stride, aux_row_stride;
  // CONV mode (3x3 NHWC implicit GEMM): a "batch" is one output image row, a "row" an output pixel x.
  // maps.a[0] is then a 4-D map (c, x, y, img) with box (64, 128, 1, 1) and x element-stride = conv_stride;
  // k-block kb covers tap kb / conv_cblocks (dy = tap / 3, dx = tap % 3) and channels (kb % conv_cblocks) * 64.
  int conv_h_out, conv_stride, conv_pad, conv_cblocks;
};

struct GemmMaps {
  CUtensorMap a[3];  // 3-D (k, s, b), box (64, 128, 1), SWIZZLE_128B
  CUtensorMap w[3];  // 2-D (k, n),   box (64, BN),      SWIZZLE_128B;  w_kn: 2-D (n, k), box (64, 64)
};

template <int BN>
struct GemmCfg {
  static constexpr int BM = 128;
  static constexpr int BK = 64;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int W_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + W_BYTES;
  static constexpr int STAGES = (200 * 1024) / STAGE_BYTES > 8 ? 8 : (200 * 1024) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

__device__ __forceinline__ float gemm_bf16r(float x) { return __bfloat162float(__float2bfloat16(x)); }

__device__ __forceinline__ void gemm_tile_coords(int tile, int tiles_m, int tiles_n, int& tm, int& tn) {
  // grouped rasterisation: bands of 8 m-tiles sweep all n-tiles -> square-ish L2 footprint
  constexpr int GM = 8;
  int per_group = GM * tiles_n;
  int g = tile / per_group;
  int first_m = g * GM;
  int gsize = min(GM, tiles_m - first_m);
  int within = tile - g * per_group;
  tm = first_m + within % gsize;
  tn = within / gsize;
}

__device__ __forceinline__ void ld_bf16x2(const __nv_bfloat16* p, bool two, float& a, float& b) {
  if (two) {
    const uint32_t u = *reinterpret_cast<const uint32_t*>(p);
    a = bf16_lo(u);
    b = bf16_hi(u);
  } else {
    a = __bfloat162float(p[0]);
    b = 0.f;
  }
}
__device__ __forceinline__ void st_bf16x2(__nv_bfloat16* p, bool two, float a, float b) {
  if (two) *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(a, b);
  else p[0] = __float2bfloat16(a);
}

// Fused epilogue of two adjacent columns (n, n+1) of one output row; f = accumulator + bias.
__device__ __forceinline__ void gemm_epi_pair(const GemmParams& p, int b, int s, int n, bool two, float f0, float f1) {
  const long long drow = (long long)b * p.d_batch_stride + (long long)s * p.d_row_stride;
  __nv_bfloat16* xp = p.aux ? p.aux + (long long)b * p.aux_batch_stride + (long long)s * p.aux_row_stride + n : nullptr;
  if (p.epi == EPI_GELU) {
    if (xp) st_bf16x2(xp, two, f0, f1);
    // the activation sees the bf16-rounded pre-activation, as the reference's
    // nn.Linear -> nn.GELU chain does (bf16 tensor between the two modules)
    f0 = gelu_tanh(gemm_bf16r(f0));
    f1 = gelu_tanh(gemm_bf16r(f1));
  } else if (p.epi == EPI_GATE_RES) {
    float g0, g1, r0, r1;
    ld_bf16x2(p.gate + (long long)b * p.gate_batch_stride + n, two, g0, g1);
    ld_bf16x2(p.res + (long long)b * p.res_batch_stride + (long long)s * p.res_row_stride + n, two, r0, r1);
    // full fine-tune: keep the (bf16) linear output — the gate gradient is sum_s dOut * y
    if (xp) st_bf16x2(xp, two, f0, f1);
    // reference order: bias -> (bf16 linear output) -> gate * y -> residual + (...)
    // (flux/transformer.py:464-465, 584-586, 652-653); each step is a bf16 tensor there.
    float o[2] = {r0 + gemm_bf16r(g0 * gemm_bf16r(f0)), r1 + gemm_bf16r(g1 * gemm_bf16r(f1))};
    if (p.nan_to_num) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        float v = gemm_bf16r(o[j]);
        if (v != v) v = 0.f;
        else if (v == INFINITY) v = 65504.f;
        else if (v == -INFINITY) v = -65504.f;
        o[j] = v;
      }
    }
    f0 = o[0];
    f1 = o[1];
  } else if (p.epi == EPI_MUL_DGELU) {
    float x0, x1;
    ld_bf16x2(xp, two, x0, x1);
    f0 *= gelu_tanh_grad(x0);
    f1 *= gelu_tanh_grad(x1);
  } else if (p.epi == EPI_MUL) {
    float x0, x1;
    ld_bf16x2(xp, two, x0, x1);
    f0 = gemm_bf16r(f0) * x0;
    f1 = gemm_bf16r(f1) * x1;
  } else if (p.epi == EPI_QUICK_GELU) {
    const float y0 = gemm_bf16r(f0), y1 = gemm_bf16r(f1);
    f0 = y0 / (1.f + __expf(-1.702f * y0));
    f1 = y1 / (1.f + __expf(-1.702f * y1));
  } else if (p.epi == EPI_ADD_RES) {
    float r0, r1;
    ld_bf16x2(p.res + (long long)b * p.res_batch_stride + (long long)s * p.res_row_stride + n, two, r0, r1);
    f0 += r0;
    f1 += r1;
  }
  st_bf16x2(p.D + drow + n, two, f0, f1);
}

template <int BN, int TB>
__device__ __forceinline__ void gemm_wgmma(float (&acc)[BN / 2], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (BN == 256) wgmma_ss_n256<0, TB>(acc, a, b, accumulate);
  else if constexpr (BN == 128) wgmma_ss_n128<0, TB>(acc, a, b, accumulate);
  else wgmma_ss_n64<0, TB>(acc, a, b, accumulate);
}

template <int BN, bool CONV = false>
__global__ void __launch_bounds__(384, 1)
gemm_bf16_tn_kernel(const __grid_constant__ GemmMaps maps, const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * Cfg::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)

  const int tiles_per_batch = (p.rows_per_batch + Cfg::BM - 1) / Cfg::BM;
  const int tiles_m = tiles_per_batch * p.num_batches;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int num_tiles = tiles_m * tiles_n;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nseg; ++s) {
      tma_prefetch_desc(&maps.a[s]);
      tma_prefetch_desc(&maps.w[s]);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);   // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer (warp 0, one elected lane issues) =====================
    reg_dealloc<40>();
    if (warp == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int tm, tn;
        gemm_tile_coords(tile, tiles_m, tiles_n, tm, tn);
        const int b = tm / tiles_per_batch;
        const int s0 = (tm - b * tiles_per_batch) * Cfg::BM;
        const int n0 = tn * BN;
        for (int seg = 0; seg < p.nseg; ++seg) {
          for (int kb = 0; kb < p.kblocks[seg]; ++kb) {
            mbar_wait(empty_bar(stage), phase ^ 1u, 1);
            const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES;
            if (elect_one()) {
              mbar_arrive_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);
              if constexpr (CONV) {
                // implicit-GEMM 3x3 conv: shifted input window; TMA zero-fills the halo (x / y out of range)
                const int tap = kb / p.conv_cblocks;
                const int c0 = (kb - tap * p.conv_cblocks) * 64;
                const int img = b / p.conv_h_out, yo = b - img * p.conv_h_out;
                const int dy = tap / 3, dx = tap - dy * 3;
                tma_load_4d(sa, &maps.a[0], full_bar(stage), c0, s0 * p.conv_stride + dx - p.conv_pad,
                            yo * p.conv_stride + dy - p.conv_pad, img);
              } else {
                tma_load_3d(sa, &maps.a[seg], full_bar(stage), kb * 64, s0, b);
              }
              if (p.w_kn[seg]) {
#pragma unroll
                for (int g = 0; g < BN / 64; ++g)
                  tma_load_2d(sa + Cfg::A_BYTES + g * 8192, &maps.w[seg], full_bar(stage), n0 + g * 64, kb * 64);
              } else {
                tma_load_2d(sa + Cfg::A_BYTES, &maps.w[seg], full_bar(stage), kb * 64, n0);
              }
            }
            __syncwarp();
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1u;
            }
          }
        }
      }
    }
  } else {
    // ===================== consumers: 64 rows each =====================
    reg_alloc<232>();
    const int cw = wg - 1;               // rows [64 cw, 64 cw + 64) of the tile
    const int wq = warp & 3;             // warp within the warpgroup: rows 16 wq .. 16 wq + 15
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int tm, tn;
      gemm_tile_coords(tile, tiles_m, tiles_n, tm, tn);
      const int b = tm / tiles_per_batch;
      const int s0 = (tm - b * tiles_per_batch) * Cfg::BM + cw * 64;
      const int n0 = tn * BN;
      uint32_t accumulate = 0;
      int prev_stage = -1;
      for (int seg = 0; seg < p.nseg; ++seg) {
        const bool wkn = __shfl_sync(0xffffffffu, p.w_kn[seg], 0) != 0;
        for (int kb = 0; kb < p.kblocks[seg]; ++kb) {
          mbar_wait(full_bar(stage), phase, 3);
          const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES + cw * 8192;
          const uint32_t sw = smem_base + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES;
          // K past the end of the segment is zero-filled by TMA, so the last k-block runs all four K steps too
          wg_fence();
          if (wkn) {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) gemm_wgmma<BN, 1>(acc, sdesc_k(sa, kk * 32), sdesc_mn(sw, kk * 2048, 8192), kk > 0 ? 1u : accumulate);
          } else {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) gemm_wgmma<BN, 0>(acc, sdesc_k(sa, kk * 32), sdesc_k(sw, kk * 32), kk > 0 ? 1u : accumulate);
          }
          accumulate = 1;
          wg_commit();
          // keep one k-block in flight; the one before it has retired -> free its slot
          wg_wait<1>();
          wg_fence_regs(acc);
          if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar(prev_stage));
          prev_stage = stage;
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
      wg_wait<0>();
      wg_fence_regs(acc);
      if (lane == 0) mbar_arrive(empty_bar(prev_stage));

      // ===================== epilogue from registers =====================
      // accumulator layout (m64nBN): acc[4 i + 2 h + j] = row 16 wq + lane / 4 + 8 h, column 8 i + 2 (lane % 4) + j
      const int r_lo = s0 + wq * 16 + (lane >> 2);
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int n = n0 + 8 * i + 2 * (lane & 3);
        if (n < p.N) {
          const bool two = n + 1 < p.N;
          float b0 = 0.f, b1 = 0.f;
          if (p.bias) ld_bf16x2(p.bias + n, two, b0, b1);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int s = r_lo + 8 * h;
            if (s < p.rows_per_batch && b < p.num_batches)
              gemm_epi_pair(p, b, s, n, two, acc[4 * i + 2 * h] + b0, acc[4 * i + 2 * h + 1] + b1);
          }
        }
      }
    }
  }
}

}  // namespace stb
