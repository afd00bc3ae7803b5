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
// consumers in ping-pong: each owns whole BM x BN tiles (the CTA's tiles alternate between them), runs wgmma
// m64nBNk16 from shared memory over BM / 64 row blocks, then the fused epilogue (through a shared-memory buffer and TMA
// at 128 x 128, straight from the accumulator registers otherwise).  While one consumer is in its epilogue the other one's MMAs keep the tensor pipe busy, and the grid is
// persistent, so the producer streams the next tile's k-blocks meanwhile.  The epilogue kind is a template parameter.
// CONV = true turns the A operand into the shifted NHWC window of a 3x3 convolution (implicit GEMM, VAE encoder).
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
  EPI_SILU = 7,         // D = y * sigmoid(y), y = bf16(acc + bias)           (Chroma approximator: nn.Linear -> SiLU)
};

struct GemmParams {
  int rows_per_batch;  // S : rows in one batch slab of A / D
  int num_batches;     // B
  int N;
  int nseg;
  int kblocks[3];  // ceil(K_seg / 64)
  int w_kn[3];        // 1: the segment's weight is given as [K, N] row-major (contraction index = row): the B operand is
                      // staged MN-major (64 k-rows x 64 n-columns SWIZZLE_128B boxes) — dgrad reads W itself, no W^T copy
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
  // maps.a[0] is then a 4-D map (c, x, y, img) with box (64, BM, 1, 1) and x element-stride = conv_stride;
  // k-block kb covers tap kb / conv_cblocks (dy = tap / 3, dx = tap % 3) and channels (kb % conv_cblocks) * 64.
  int conv_h_out, conv_stride, conv_pad, conv_cblocks;
};

struct GemmMaps {
  CUtensorMap a[3];  // 3-D (k, s, b), box (64, BM, 1), SWIZZLE_128B
  CUtensorMap w[3];  // 2-D (k, n),   box (64, BN),      SWIZZLE_128B;  w_kn: 2-D (n, k), box (64, 64)
  // shared-memory epilogue (kGemmSmemEpi): 3-D (n, s, b), box (64, 128, 1), SWIZZLE_128B, over D, the [M, N] operand the
  // epilogue reads (res or aux) and the aux output of EPI_GELU / EPI_GATE_RES
  CUtensorMap d, x, aux;
};

// 128 x 128 tiles of the plain GEMM stage the epilogue through shared memory (a TMA load of the operand, TMA stores of
// the results); the other widths and CONV keep the epilogue from registers.
template <int BN, bool CONV>
constexpr bool kGemmSmemEpi = BN == 128 && !CONV;

// A consumer's tile is BM x BN with 128 fp32 accumulators per thread at BN 128 and 256 (64 at BN 64).  SMEM_EPI: one
// BM x BN bf16 epilogue buffer per consumer warpgroup, paid for with one ring stage (5 instead of 6 at 128 x 128).
template <int BN, bool SMEM_EPI = false>
struct GemmCfg {
  static constexpr int BM = BN == 256 ? 64 : 128;
  static constexpr int BK = 64;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int W_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + W_BYTES;
  static constexpr int EPI_BYTES = SMEM_EPI ? BM * BN * 2 : 0;
  static constexpr int STAGES = SMEM_EPI ? 5 : (200 * 1024) / STAGE_BYTES > 8 ? 8 : (200 * 1024) / STAGE_BYTES;
  static constexpr int SMEM_BYTES =
      STAGES * STAGE_BYTES + 2 * EPI_BYTES + 1024 /*align*/ + 256 /*ring, order and epilogue barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory per block");
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
// the pair as one word; a lone last column reads one element and leaves the high half zero
__device__ __forceinline__ uint32_t ld_pair_word(const __nv_bfloat16* p, bool two) {
  return two ? *reinterpret_cast<const uint32_t*>(p) : uint32_t(__bfloat16_as_ushort(p[0]));
}
__device__ __forceinline__ void st_bf16x2(__nv_bfloat16* p, bool two, float a, float b) {
  if (two) *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(a, b);
  else p[0] = __float2bfloat16(a);
}

// The epilogues that read an [M, N] operand element for element: res (GATE_RES, ADD_RES) or aux (MUL_DGELU, MUL).
// The register epilogue loads those words ahead, a chunk of column groups at a time, so that their latencies overlap.
template <int EPI>
constexpr bool kGemmEpiReadsRows = EPI == EPI_GATE_RES || EPI == EPI_ADD_RES || EPI == EPI_MUL_DGELU || EPI == EPI_MUL;
template <int EPI>
__device__ __forceinline__ const __nv_bfloat16* gemm_epi_row_operand(const GemmParams& p, int b, int s, int n) {
  if constexpr (EPI == EPI_GATE_RES || EPI == EPI_ADD_RES)
    return p.res + (long long)b * p.res_batch_stride + (long long)s * p.res_row_stride + n;
  else
    return p.aux + (long long)b * p.aux_batch_stride + (long long)s * p.aux_row_stride + n;
}

// Fused epilogue arithmetic of two adjacent columns of one output row: f = accumulator + bias in, D out; x = the pair's
// res / aux word for the epilogues that read one, g = the pair's gate (EPI_GATE_RES).  The aux output of EPI_GELU /
// EPI_GATE_RES is f itself, written by the caller.
template <int EPI>
__device__ __forceinline__ void gemm_epi_math(const GemmParams& p, float& f0, float& f1, float g0, float g1, uint32_t x) {
  if constexpr (EPI == EPI_GELU) {
    // the activation sees the bf16-rounded pre-activation, as the reference's
    // nn.Linear -> nn.GELU chain does (bf16 tensor between the two modules)
    f0 = gelu_tanh(gemm_bf16r(f0));
    f1 = gelu_tanh(gemm_bf16r(f1));
  } else if constexpr (EPI == EPI_GATE_RES) {
    const float r0 = bf16_lo(x), r1 = bf16_hi(x);
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
  } else if constexpr (EPI == EPI_MUL_DGELU) {
    f0 *= gelu_tanh_grad(bf16_lo(x));
    f1 *= gelu_tanh_grad(bf16_hi(x));
  } else if constexpr (EPI == EPI_MUL) {
    f0 = gemm_bf16r(f0) * bf16_lo(x);
    f1 = gemm_bf16r(f1) * bf16_hi(x);
  } else if constexpr (EPI == EPI_QUICK_GELU) {
    const float y0 = gemm_bf16r(f0), y1 = gemm_bf16r(f1);
    f0 = y0 / (1.f + __expf(-1.702f * y0));
    f1 = y1 / (1.f + __expf(-1.702f * y1));
  } else if constexpr (EPI == EPI_SILU) {
    const float y0 = gemm_bf16r(f0), y1 = gemm_bf16r(f1);
    f0 = y0 / (1.f + __expf(-y0));
    f1 = y1 / (1.f + __expf(-y1));
  } else if constexpr (EPI == EPI_ADD_RES) {
    f0 += bf16_lo(x);
    f1 += bf16_hi(x);
  }
}

// Register epilogue of one pair (n, n+1) of output row s, stored straight to global memory.
template <int EPI>
__device__ __forceinline__ void gemm_epi_pair(const GemmParams& p, int b, int s, int n, bool two, float f0, float f1,
                                              uint32_t x) {
  const long long drow = (long long)b * p.d_batch_stride + (long long)s * p.d_row_stride;
  __nv_bfloat16* xp = p.aux ? p.aux + (long long)b * p.aux_batch_stride + (long long)s * p.aux_row_stride + n : nullptr;
  float g0 = 0.f, g1 = 0.f;
  if constexpr (EPI == EPI_GATE_RES) ld_bf16x2(p.gate + (long long)b * p.gate_batch_stride + n, two, g0, g1);
  // full fine-tune (GATE_RES): keep the (bf16) linear output — the gate gradient is sum_s dOut * y
  if constexpr (EPI == EPI_GELU || EPI == EPI_GATE_RES)
    if (xp) st_bf16x2(xp, two, f0, f1);
  gemm_epi_math<EPI>(p, f0, f1, g0, g1, x);
  st_bf16x2(p.D + drow + n, two, f0, f1);
}

template <int BN, int TB>
__device__ __forceinline__ void gemm_wgmma(float (&acc)[BN / 2], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (BN == 256) wgmma_ss_n256<0, TB>(acc, a, b, accumulate);
  else if constexpr (BN == 128) wgmma_ss_n128<0, TB>(acc, a, b, accumulate);
  else wgmma_ss_n64<0, TB>(acc, a, b, accumulate);
}

// CLUSTER = 2: the CTAs run as 2-CTA clusters.  A cluster's work unit is a pair tile, m-tiles 2 pm and 2 pm + 1 at the
// same n-tile; CTA rank r computes m-tile 2 pm + r.  The two tiles read the same W tile, so each producer loads rows
// [64 r, 64 r + 64) of it and multicasts them into the same stage of both CTAs: 24 KB instead of 32 KB of L2 reads per
// tile and k-block.  Both CTAs walk the same units, so their rings advance in lockstep, and a producer refills a stage
// only when the consumers of both CTAs have released it (empty barriers of 8 warps, release_cluster).  With an odd
// tiles_m the last pair's second tile lies past the end (its A box is zero-filled and its stores are skipped by the
// row / batch guards); that CTA still loads, multicasts, waits on and releases every stage, or its peer would wedge.
// W maps are then boxes of 64 rows (k-major) or the usual 64 x 64 boxes (w_kn).  CONV supports CLUSTER = 1 only.
template <int BN, int EPI, bool CONV = false, int CLUSTER = 1>
__global__ void __launch_bounds__(384, 1)
gemm_bf16_tn_kernel(const __grid_constant__ GemmMaps maps, const GemmParams p) {
  constexpr bool SMEM_EPI = kGemmSmemEpi<BN, CONV>;
  using Cfg = GemmCfg<BN, SMEM_EPI>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int MI = Cfg::BM / 64;   // m64 row blocks of a tile
  static_assert(CLUSTER == 1 || (CLUSTER == 2 && BN == 128 && !CONV), "2-CTA clusters: 128 x 128 GEMM tiles only");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  // shared memory: the ring's stages, the consumers' epilogue buffers (SMEM_EPI), then the barriers
  const uint32_t epi_smem = smem_base + STAGES * Cfg::STAGE_BYTES;
  StageRing<STAGES> ring{epi_smem + 2 * Cfg::EPI_BYTES};
  // order[c]: consumer c may start its next mainloop (the other consumer has waited on every stage of the tile before)
  const uint32_t order_bars = ring.bars + 16u * STAGES;
  // epi_full[c] (SMEM_EPI, epilogues that read an operand): the res / aux block of consumer c's tile is in its buffer
  const uint32_t epi_full_bars = order_bars + 16u;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)

  const int tiles_per_batch = (p.rows_per_batch + Cfg::BM - 1) / Cfg::BM;
  const int tiles_m = tiles_per_batch * p.num_batches;
  const int tiles_n = (p.N + BN - 1) / BN;
  // work units: tiles, or pair tiles of a cluster; unit0 / units_stride: this CTA's (cluster's) first unit and stride
  const int units_m = (tiles_m + CLUSTER - 1) / CLUSTER;
  const int num_units = units_m * tiles_n;
  const int unit0 = blockIdx.x / CLUSTER;
  const int units_stride = gridDim.x / CLUSTER;
  const uint32_t rank = CLUSTER == 2 ? cluster_ctarank() : 0u;
  int nk = 0;   // k-blocks per tile
  for (int s = 0; s < p.nseg; ++s) nk += p.kblocks[s];

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nseg; ++s) {
      tma_prefetch_desc(&maps.a[s]);
      tma_prefetch_desc(&maps.w[s]);
    }
    if constexpr (SMEM_EPI) {
      tma_prefetch_desc(&maps.d);
      if constexpr (kGemmEpiReadsRows<EPI>) tma_prefetch_desc(&maps.x);
    }
    ring.init(4 * CLUSTER);   // each stage belongs to one consumer warpgroup's tile (in every CTA of the cluster)
    mbar_init(order_bars, 4);
    mbar_init(order_bars + 8, 4);
    mbar_init(epi_full_bars, 1);
    mbar_init(epi_full_bars + 8, 1);
    fence_mbar_init();
  }
  // no multicast or remote arrive may reach a CTA before its barriers exist
  if constexpr (CLUSTER == 2) cluster_sync();
  else __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer (warp 0, one elected lane issues) =====================
    reg_dealloc<40>();
    if (warp == 0) {
      for (int unit = unit0; unit < num_units; unit += units_stride) {
        int tm, tn;
        gemm_tile_coords(unit, units_m, tiles_n, tm, tn);
        tm = tm * CLUSTER + (int)rank;
        const int b = tm / tiles_per_batch;
        const int s0 = (tm - b * tiles_per_batch) * Cfg::BM;
        const int n0 = tn * BN;
        for (int seg = 0; seg < p.nseg; ++seg) {
          for (int kb = 0; kb < p.kblocks[seg]; ++kb) {
            ring.wait_empty(1);
            const uint32_t sa = smem_base + ring.stage * Cfg::STAGE_BYTES;
            const uint32_t full = ring.full_bar(ring.stage);
            if (elect_one()) {
              mbar_arrive_expect_tx(full, Cfg::STAGE_BYTES);
              if constexpr (CONV) {
                // implicit-GEMM 3x3 conv: shifted input window; TMA zero-fills the halo (x / y out of range)
                const int tap = kb / p.conv_cblocks;
                const int c0 = (kb - tap * p.conv_cblocks) * 64;
                const int img = b / p.conv_h_out, yo = b - img * p.conv_h_out;
                const int dy = tap / 3, dx = tap - dy * 3;
                tma_load_4d(sa, &maps.a[0], full, c0, s0 * p.conv_stride + dx - p.conv_pad,
                            yo * p.conv_stride + dy - p.conv_pad, img);
              } else {
                tma_load_3d(sa, &maps.a[seg], full, kb * 64, s0, b);
              }
              if constexpr (CLUSTER == 2) {
                // this CTA's half of the W tile, into both CTAs: n-columns [64 r, 64 r + 64), k-major or MN-major
                const int hn = n0 + 64 * (int)rank;
                const uint32_t hw = sa + Cfg::A_BYTES + rank * 8192u;
                if (p.w_kn[seg]) tma_load_2d_mc(hw, &maps.w[seg], full, hn, kb * 64, 0x3);
                else tma_load_2d_mc(hw, &maps.w[seg], full, kb * 64, hn, 0x3);
              } else if (p.w_kn[seg]) {
#pragma unroll
                for (int g = 0; g < BN / 64; ++g)
                  tma_load_2d(sa + Cfg::A_BYTES + g * 8192, &maps.w[seg], full, n0 + g * 64, kb * 64);
              } else {
                tma_load_2d(sa + Cfg::A_BYTES, &maps.w[seg], full, kb * 64, n0);
              }
            }
            __syncwarp();
            ring.advance();
          }
        }
      }
    }
  } else {
    // ===================== consumers: ping-pong over whole tiles =====================
    // Consumer cw takes the CTA's tiles cw, cw + 2, ...; the producer fills the ring in tile order, so each consumer
    // passes over the other's nk stages.  Its epilogue then runs while the other consumer's MMAs use the tensor pipe.
    reg_alloc<232>();
    const int cw = wg - 1;
    const int wq = warp & 3;             // warp within the warpgroup: rows 16 wq .. 16 wq + 15 of each m64 block
    uint32_t order_phase = 0;
    if (cw == 1) ring.skip(nk);
    uint32_t epi_phase = 0;   // SMEM_EPI: phase of this warpgroup's epi_full barrier
    float acc[MI][BN / 2];
    for (int unit = unit0 + cw * units_stride; unit < num_units; unit += 2 * units_stride) {
      // The other consumer has waited on every stage of the tile before this one, so the producer has filled them all
      // and this consumer's full-barrier waits are at most one lap ahead of the barriers' phases.
      if (unit != unit0) {
        mbar_wait(order_bars + 8u * cw, order_phase, 4);
        order_phase ^= 1u;
      }
      int tm, tn;
      gemm_tile_coords(unit, units_m, tiles_n, tm, tn);
      tm = tm * CLUSTER + (int)rank;
      const int b = tm / tiles_per_batch;
      const int s0 = (tm - b * tiles_per_batch) * Cfg::BM;
      const int n0 = tn * BN;
      uint32_t accumulate = 0;
      int prev_stage = -1;
      for (int seg = 0; seg < p.nseg; ++seg) {
        const bool wkn = __shfl_sync(0xffffffffu, p.w_kn[seg], 0) != 0;
        for (int kb = 0; kb < p.kblocks[seg]; ++kb) {
          ring.wait_full(3);
          const uint32_t sa = smem_base + ring.stage * Cfg::STAGE_BYTES;
          const uint32_t sw = sa + Cfg::A_BYTES;
          // K past the end of the segment is zero-filled by TMA, so the last k-block runs all four K steps too
          wg_fence();
          if (wkn) {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
              for (int mi = 0; mi < MI; ++mi)
                gemm_wgmma<BN, 1>(acc[mi], sdesc_k(sa + mi * 8192, kk * 32), sdesc_mn(sw, kk * 2048, 8192),
                                  kk > 0 ? 1u : accumulate);
            // commit and wait in each branch: a wgmma group still open where the branches join makes ptxas close it
            // with an extra HGMMA, and the wait below then drains the k-block just issued as well
            wg_commit();
            wg_wait<1>();   // keep one k-block in flight; the one before it has retired -> free its slot
          } else {
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
              for (int mi = 0; mi < MI; ++mi)
                gemm_wgmma<BN, 0>(acc[mi], sdesc_k(sa + mi * 8192, kk * 32), sdesc_k(sw, kk * 32),
                                  kk > 0 ? 1u : accumulate);
            wg_commit();
            wg_wait<1>();
          }
          accumulate = 1;
          if (prev_stage >= 0) {
            if constexpr (CLUSTER == 2) ring.release_cluster(prev_stage, rank ^ 1u);
            else ring.release(prev_stage);
          }
          if constexpr (SMEM_EPI && kGemmEpiReadsRows<EPI>) {
            // the tile's res / aux block, two 64-column boxes (past the N, row or batch end TMA fills zeros), loaded by
            // the warpgroup's first thread a few k-blocks into the mainloop, when the previous tile's stores have long
            // read the buffer
            if (seg == 0 && kb == min(3, p.kblocks[0] - 1) && (threadIdx.x & 127) == 0) {
              const uint32_t ebuf = epi_smem + cw * Cfg::EPI_BYTES, epi_full = epi_full_bars + 8u * cw;
              tma_store_wait_read<0>();   // the previous tile's stores have read the buffer
              mbar_arrive_expect_tx(epi_full, Cfg::EPI_BYTES);
              tma_load_3d(ebuf, &maps.x, epi_full, n0, s0, b);
              tma_load_3d(ebuf + Cfg::EPI_BYTES / 2, &maps.x, epi_full, n0 + 64, s0, b);
            }
            __syncwarp();
          }
          prev_stage = ring.stage;
          ring.advance();
        }
      }
      // every stage of this tile has landed: the other consumer may start on the next tile
      if (unit + units_stride < num_units && lane == 0) mbar_arrive(order_bars + 8u * (cw ^ 1));
      ring.skip(nk);
      wg_wait<0>();
#pragma unroll
      for (int mi = 0; mi < MI; ++mi) wg_fence_regs(acc[mi]);
      if constexpr (CLUSTER == 2) ring.release_cluster(prev_stage, rank ^ 1u);
      else ring.release(prev_stage);

      // accumulator layout (m64nBN): acc[mi][4 i + 2 h + j] = row 64 mi + 16 wq + lane / 4 + 8 h,
      // column 8 i + 2 (lane % 4) + j
      const bool b_ok = b < p.num_batches;
      if constexpr (SMEM_EPI) {
        // ===================== epilogue through shared memory =====================
        // The buffer holds the tile as two 64-column halves of 128 rows x 128 B in TMA's SWIZZLE_128B layout: the 16-byte
        // chunk c of row r sits at chunk position c ^ (r % 8).  Column 8 i + 2 (lane % 4) of row r is then at half i / 8,
        // chunk (i % 8) ^ (lane / 4), byte 4 (lane % 4), and a warp's 8 rows x 4 words of one column group hit all 32
        // banks once.  Every thread reads (res / aux) and writes (D, then aux) only its own words; the TMA stores clip
        // the tile at the N, row and batch ends, so tail elements are computed but never leave shared memory.  The
        // warpgroup's first thread issues the stores.
        const uint32_t ebuf = epi_smem + cw * Cfg::EPI_BYTES;
        const bool epi_leader = (threadIdx.x & 127) == 0;
        const uint32_t wrow = ebuf + (wq * 16 + (lane >> 2)) * 128 + 4 * (lane & 3);
        // fill(false): the epilogue's D over the buffer; fill(true): the aux output acc + bias
        auto fill = [&](auto aux_pass) {
          constexpr bool AUX = decltype(aux_pass)::value;
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) {
            const int n = n0 + 8 * i + 2 * (lane & 3);
            const bool col_ok = n < p.N && b_ok;
            const bool two = n + 1 < p.N;
            float b0 = 0.f, b1 = 0.f, g0 = 0.f, g1 = 0.f;
            if (p.bias && col_ok) ld_bf16x2(p.bias + n, two, b0, b1);
            if constexpr (EPI == EPI_GATE_RES && !AUX)
              if (col_ok) ld_bf16x2(p.gate + (long long)b * p.gate_batch_stride + n, two, g0, g1);
            const uint32_t wcol = wrow + (i >> 3) * (Cfg::EPI_BYTES / 2) + (((i & 7) ^ (lane >> 2)) << 4);
#pragma unroll
            for (int mi = 0; mi < MI; ++mi)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint32_t w = wcol + (mi * 64 + 8 * h) * 128;
                float f0 = acc[mi][4 * i + 2 * h] + b0, f1 = acc[mi][4 * i + 2 * h + 1] + b1;
                if constexpr (!AUX) gemm_epi_math<EPI>(p, f0, f1, g0, g1, kGemmEpiReadsRows<EPI> ? ld_shared_u32(w) : 0u);
                st_shared_u32(w, pack_bf16x2(f0, f1));
              }
          }
        };
        // the buffer's words -> global: every thread's writes made visible to the async proxy, then one thread stores
        auto store = [&](const CUtensorMap* m) {
          fence_proxy_async_smem();
          named_bar_sync(1 + cw, 128);
          if (epi_leader && b_ok) {
            tma_store_3d(m, ebuf, n0, s0, b);
            tma_store_3d(m, ebuf + Cfg::EPI_BYTES / 2, n0 + 64, s0, b);
            tma_store_commit();
          }
        };
        // before the buffer is written again: the stores issued from it have read it
        auto reuse = [&]() {
          if (epi_leader) tma_store_wait_read<0>();
          named_bar_sync(1 + cw, 128);
        };
        if constexpr (kGemmEpiReadsRows<EPI>) {
          mbar_wait(epi_full_bars + 8u * cw, epi_phase, 5);
          epi_phase ^= 1u;
        } else {
          reuse();
        }
        // GELU's aux output (the pre-activation) goes first; GATE_RES's after D, which is computed over the res it reads
        if constexpr (EPI == EPI_GELU)
          if (p.aux) {
            fill(std::true_type{});
            store(&maps.aux);
            reuse();
          }
        fill(std::false_type{});
        store(&maps.d);
        if constexpr (EPI == EPI_GATE_RES)
          if (p.aux) {
            reuse();
            fill(std::true_type{});
            store(&maps.aux);
          }
        __syncwarp();
        continue;   // next tile
      }

      // ===================== epilogue from registers =====================
      constexpr int CH = BN / 8 < 8 ? BN / 8 : 8;   // column groups whose res / aux words are loaded together
#pragma unroll
      for (int mi = 0; mi < MI; ++mi) {
        const int r_lo = s0 + mi * 64 + wq * 16 + (lane >> 2);
#pragma unroll
        for (int i0 = 0; i0 < BN / 8; i0 += CH) {
          uint32_t x[CH][2];
#pragma unroll
          for (int c = 0; c < CH; ++c) {
            const int n = n0 + 8 * (i0 + c) + 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              x[c][h] = 0;
              if constexpr (kGemmEpiReadsRows<EPI>)
                if (n < p.N && r_lo + 8 * h < p.rows_per_batch && b_ok)
                  x[c][h] = ld_pair_word(gemm_epi_row_operand<EPI>(p, b, r_lo + 8 * h, n), n + 1 < p.N);
            }
          }
#pragma unroll
          for (int c = 0; c < CH; ++c) {
            const int i = i0 + c;
            const int n = n0 + 8 * i + 2 * (lane & 3);
            if (n < p.N) {
              const bool two = n + 1 < p.N;
              float b0 = 0.f, b1 = 0.f;
              if (p.bias) ld_bf16x2(p.bias + n, two, b0, b1);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int s = r_lo + 8 * h;
                if (s < p.rows_per_batch && b_ok)
                  gemm_epi_pair<EPI>(p, b, s, n, two, acc[mi][4 * i + 2 * h] + b0, acc[mi][4 * i + 2 * h + 1] + b1,
                                     x[c][h]);
              }
            }
          }
        }
      }
    }
    // the last tile's stores have completed before the CTA's shared memory goes away
    if constexpr (SMEM_EPI)
      if ((threadIdx.x & 127) == 0) tma_store_wait<0>();
  }
  // the peer may still multicast into this CTA's stages or arrive on its empty barriers until it is done too
  if constexpr (CLUSTER == 2) cluster_sync();
}

}  // namespace stb
