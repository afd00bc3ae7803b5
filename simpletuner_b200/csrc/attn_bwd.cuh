// simpletuner_b200 — attention backward on wgmma, sm_90a (autograd of the SDPA call at reference
// flux/transformer.py:200-207).
//
//   P = exp(S*scale - LSE),  dV = P^T dO,  dP = dO V^T,  dS = P o (dP - Delta) * scale,
//   dQ = dS K,  dK = dS^T Q,   Delta_i = sum_d dO_id O_id
//
// Two deterministic kernels, no atomics; 384 threads each: warpgroup 0 is the TMA producer, warpgroups 1 and 2
// own 64 rows each of the CTA's 128 resident rows.
//   attn_bwd_dkdv_kernel : one CTA per (b, h, 128-key tile); streams 64-row query tiles.  Transposed domain
//       (accumulator row = key): S^T = K Q^T, dP^T = V dO^T in registers; P^T and dS^T become the register A operand of
//       dV += P^T dO,  dK += dS^T Q  (dO / Q tiles re-read from the same shared-memory bytes as MN-major operands).
//   attn_bwd_dq_kernel   : one CTA per (b, h, 128-row query tile); streams 64-key tiles: S = Q K^T, dP = dO V^T,
//       dS in registers, dQ += dS K.
// The accumulators are staged through shared memory (fp32) for the store, so that one thread handles contiguous
// columns of a row — the fused q / k pre-processing backward (qk_prep) needs whole-row sums.
#pragma once
#include "../../include/stb200.h"
#include "attn_fwd.cuh"
#include "common.cuh"
#include "elementwise.cuh"

namespace stb {

struct AttnBwdParams {
  int B, H, Sq, Sk;
  float scale;
  const float* lse;    // [B, H, Sq]
  const float* delta;  // [B, H, Sq]
  __nv_bfloat16 *dq, *dk, *dv;
  long long dq_b, dq_s, dq_h, dk_b, dk_s, dk_h, dv_b, dv_s, dv_h;
  // raw views of q / dO (the operands themselves go through the TMA maps)
  const __nv_bfloat16 *q, *d_o;
  long long q_b, q_s, q_h, do_b, do_s, do_h;
  // optional fused backward of the q / k pre-processing (per-head RMSNorm -> RoPE, qk_rmsnorm_rope_fwd_kernel):
  // dq / dk then receive the gradient w.r.t. the PROJECTION outputs (self-attention only: token index == row index)
  int fuse_prep;
  const __nv_bfloat16* src;          // pre-norm projection output [B, S, C]: q at column 0, k at column k_off
  long long src_b, src_s;
  int k_off;
  const __nv_bfloat16 *wq0, *wk0, *wq1, *wk1;   // RMSNorm weights (image stream | tokens s < s_split), may be null
  int s_split;
  const float *cosT, *sinT;          // [S, HD] or null
  float eps;
};

struct AttnBwdMaps {
  // 4-D (d, h, s, b) SWIZZLE_128B; box (64, 1, 128, 1) for the resident operands, (64, 1, 64, 1) for the streamed ones
  CUtensorMap q128, k128, v128, do128, q64, k64, v64, do64;
};

// ------------------------------------------------------------------------------------------------
// Delta = rowsum(dO * O), one warp per (b, s, h)
// ------------------------------------------------------------------------------------------------
template <int HD>
__global__ void __launch_bounds__(256)
attn_bwd_delta_kernel(const __nv_bfloat16* __restrict__ o, long long o_b, long long o_s, long long o_h,
                      const __nv_bfloat16* __restrict__ d_o, long long do_b, long long do_s, long long do_h,
                      float* __restrict__ delta, int B, int H, int S) {
  constexpr int EPL = HD / 32;
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (wid >= (long long)B * S * H) return;
  const int lane = threadIdx.x & 31;
  const int h = int(wid % H);
  const long long r = wid / H;
  const int s = int(r % S);
  const int b = int(r / S);
  const __nv_bfloat16* po = o + b * o_b + s * o_s + h * o_h + lane * EPL;
  const __nv_bfloat16* pg = d_o + b * do_b + s * do_s + h * do_h + lane * EPL;
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < EPL; ++i) acc += __bfloat162float(po[i]) * __bfloat162float(pg[i]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) delta[((long long)b * H + h) * S + s] = acc;
}

template <int HD>
struct AttnBwdCfg {
  static constexpr int BIG = 128 * HD * 2;   // resident 128-row tile
  static constexpr int SMALL = 64 * HD * 2;  // streamed 64-row tile
  static constexpr int STAGES = 2;
  static constexpr int SMEM_BYTES = 2 * BIG + STAGES * 2 * SMALL + 1024 + 256;
};

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// fp32 accumulator (64 x HD, wgmma layout) of this warpgroup -> shared-memory rows [64][HD + 4] (multiplied by `mul`)
template <int HD>
__device__ __forceinline__ void stage_acc(float* rows, const float (&acc)[HD / 2], float mul) {
  const int t = threadIdx.x & 127, wq = t >> 5, lane = t & 31;
#pragma unroll
  for (int i = 0; i < HD / 8; ++i)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float* r = rows + (wq * 16 + (lane >> 2) + 8 * hh) * (HD + 4) + 8 * i + 2 * (lane & 3);
      r[0] = acc[4 * i + 2 * hh] * mul;
      r[1] = acc[4 * i + 2 * hh + 1] * mul;
    }
}

// One staged row (fp32, already multiplied by the softmax scale) -> bf16 global row.  Two threads per row, HD / 2
// columns each (thread pair = lanes 2k, 2k+1).  With `prep`, the row is the gradient w.r.t. the post-RoPE q or k and
// is taken back through RoPE and the per-head RMSNorm (same math as qk_rmsnorm_rope_bwd_kernel):
//   dy = R^T go;  g = dy * w;  dx = rstd * (g - xhat * mean(g * xhat)),  xhat = x * rstd
template <int HD>
__device__ __forceinline__ void store_row_half(const float* row, int half, __nv_bfloat16* grow, bool row_ok, bool prep,
                                               const __nv_bfloat16* xrow, const __nv_bfloat16* w, const float* cs,
                                               const float* sn, float eps) {
  constexpr int NC = HD / 2;
  const int c0 = half * NC;
  if (!prep) {
    if (row_ok) {
#pragma unroll
      for (int c = 0; c < NC; c += 8) {
        float o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = row[c0 + c + i];
        *reinterpret_cast<uint4*>(grow + c0 + c) = pack8(o);
      }
    }
    return;
  }
  float ss = 0.f, sgx = 0.f;
  float g[NC];
#pragma unroll
  for (int c = 0; c < NC; c += 8) {
    float x[8], wv[8];
    unpack8(row_ok ? __ldg(reinterpret_cast<const uint4*>(xrow + c0 + c)) : make_uint4(0u, 0u, 0u, 0u), x);
    if (w) unpack8(__ldg(reinterpret_cast<const uint4*>(w + c0 + c)), wv);
#pragma unroll
    for (int i = 0; i < 8; i += 2) {
      const int j = c0 + c + i;
      const float go0 = row[j], go1 = row[j + 1];
      float dy0 = go0, dy1 = go1;
      if (cs && row_ok) {
        const float2 c2 = __ldg(reinterpret_cast<const float2*>(cs + j));
        const float2 s2 = __ldg(reinterpret_cast<const float2*>(sn + j));
        // o[i] = y[i] c[i] - y[i+1] s[i];  o[i+1] = y[i+1] c[i+1] + y[i] s[i+1]
        dy0 = go0 * c2.x + go1 * s2.y;
        dy1 = go1 * c2.y - go0 * s2.x;
      }
      const float g0 = w ? dy0 * wv[i] : dy0, g1 = w ? dy1 * wv[i + 1] : dy1;
      ss += x[i] * x[i] + x[i + 1] * x[i + 1];
      sgx += g0 * x[i] + g1 * x[i + 1];
      g[c + i] = g0;
      g[c + i + 1] = g1;
    }
  }
  ss += __shfl_xor_sync(0xffffffffu, ss, 1);
  sgx += __shfl_xor_sync(0xffffffffu, sgx, 1);
  const float rstd = rsqrtf(ss / HD + eps);
  const float m = sgx * rstd / HD;
  if (row_ok) {
#pragma unroll
    for (int c = 0; c < NC; c += 8) {
      float x[8], o[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(xrow + c0 + c)), x);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = rstd * (g[c + i] - (x[i] * rstd) * m);
      *reinterpret_cast<uint4*>(grow + c0 + c) = pack8(o);
    }
  }
}

template <int HD>
__device__ __forceinline__ void mma_kmajor_n64(float (&d)[32], uint32_t a_tile, uint32_t a_atom, uint32_t b_tile, uint32_t b_atom) {
  // d (64 x 64) = A (64 rows, K = HD, K-major boxes a_atom bytes apart) . B (64 rows, K-major boxes b_atom apart)^T
#pragma unroll
  for (int kk = 0; kk < HD / 16; ++kk)
    wgmma_ss_n64<0, 0>(d, sdesc_k(a_tile, (kk / 4) * a_atom + (kk % 4) * 32), sdesc_k(b_tile, (kk / 4) * b_atom + (kk % 4) * 32),
                       kk > 0 ? 1u : 0u);
}

// ------------------------------------------------------------------------------------------------
// dK / dV
// ------------------------------------------------------------------------------------------------
template <int HD>
__global__ void __launch_bounds__(384, 1)
attn_bwd_dkdv_kernel(const __grid_constant__ AttnBwdMaps maps, const AttnBwdParams p) {
  using Cfg = AttnBwdCfg<HD>;
  constexpr int ATOMS = HD / 64;
  constexpr int BIG_ATOM = 128 * 128, SMALL_ATOM = 64 * 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t k_smem = smem_base, v_smem = smem_base + Cfg::BIG;
  const uint32_t q_smem = smem_base + 2 * Cfg::BIG;                      // STAGES streamed Q tiles
  const uint32_t do_smem = q_smem + Cfg::STAGES * Cfg::SMALL;            // STAGES streamed dO tiles
  const uint32_t bar_base = do_smem + Cfg::STAGES * Cfg::SMALL;
  const uint32_t kv_full = bar_base;
  auto s_full = [&](int s) { return bar_base + 8u * (1 + s); };
  auto s_empty = [&](int s) { return bar_base + 8u * (1 + Cfg::STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)
  const int kv0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
  const int n_q = (p.Sq + 63) / 64;

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(s_full(s), 1);
      mbar_init(s_empty(s), 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (warp == 0) {
      if (elect_one()) {
        mbar_arrive_expect_tx(kv_full, 2 * Cfg::BIG);
        for (int a = 0; a < ATOMS; ++a) {
          tma_load_4d(k_smem + a * BIG_ATOM, &maps.k128, kv_full, a * 64, h, kv0, b);
          tma_load_4d(v_smem + a * BIG_ATOM, &maps.v128, kv_full, a * 64, h, kv0, b);
        }
      }
      __syncwarp();
      for (int j = 0; j < n_q; ++j) {
        const int stg = j % Cfg::STAGES;
        mbar_wait(s_empty(stg), ((j / Cfg::STAGES) & 1) ^ 1u, 40);
        if (elect_one()) {
          mbar_arrive_expect_tx(s_full(stg), 2 * Cfg::SMALL);
          for (int a = 0; a < ATOMS; ++a) {
            tma_load_4d(q_smem + stg * Cfg::SMALL + a * SMALL_ATOM, &maps.q64, s_full(stg), a * 64, h, j * 64, b);
            tma_load_4d(do_smem + stg * Cfg::SMALL + a * SMALL_ATOM, &maps.do64, s_full(stg), a * 64, h, j * 64, b);
          }
        }
        __syncwarp();
      }
    }
  } else {
    reg_alloc<232>();
    const int cw = wg - 1;
    const float sl2 = p.scale * 1.4426950408889634f;
    const float* lse_bh = p.lse + ((long long)b * p.H + h) * p.Sq;
    const float* del_bh = p.delta + ((long long)b * p.H + h) * p.Sq;
    float dv_acc[HD / 2], dk_acc[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dv_acc[i] = dk_acc[i] = 0.f;
    mbar_wait(kv_full, 0, 41);
    for (int j = 0; j < n_q; ++j) {
      const int stg = j % Cfg::STAGES;
      mbar_wait(s_full(stg), (j / Cfg::STAGES) & 1, 42);
      const uint32_t qa = q_smem + stg * Cfg::SMALL, da = do_smem + stg * Cfg::SMALL;
      float st[32], dpt[32];
      wg_fence();
      mma_kmajor_n64<HD>(st, k_smem + cw * 8192, BIG_ATOM, qa, SMALL_ATOM);    // S^T  = K Q^T
      mma_kmajor_n64<HD>(dpt, v_smem + cw * 8192, BIG_ATOM, da, SMALL_ATOM);   // dP^T = V dO^T
      wg_commit();
      wg_wait<0>();
      wg_fence_regs(st);
      wg_fence_regs(dpt);
      // st[4 i + 2 hh + e]: key row (16 wq + lane / 4 + 8 hh), query column 8 i + 2 (lane % 4) + e
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int q = j * 64 + 8 * i + 2 * (lane & 3) + e;
          const bool ok = q < p.Sq;
          const float l2 = ok ? __ldg(lse_bh + q) * 1.4426950408889634f : 0.f;
          const float dl = ok ? __ldg(del_bh + q) : 0.f;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int x = 4 * i + 2 * hh + e;
            const float pv = ok ? ex2f(fmaf(st[x], sl2, -l2)) : 0.f;
            st[x] = pv;                        // P^T
            dpt[x] = pv * (dpt[x] - dl);       // dS^T (softmax scale applied in the epilogue)
          }
        }
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {   // 64 queries / 16
        uint32_t a[4];
        acc_to_afrag(st, kk, a);
        wgmma_rs_mn<HD>(dv_acc, a, sdesc_mn(da, kk * 2048, SMALL_ATOM), 1u);
        acc_to_afrag(dpt, kk, a);
        wgmma_rs_mn<HD>(dk_acc, a, sdesc_mn(qa, kk * 2048, SMALL_ATOM), 1u);
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_regs(dv_acc);
      wg_fence_regs(dk_acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(s_empty(stg));
    }
    // ---- epilogue: stage dV and dK rows through the (now idle) K / V tiles, then store row-contiguously
    named_bar_sync(1, 256);
    float* stage_rows = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw))) + cw * 64 * (HD + 4);
    const int t = threadIdx.x & 127;
    const int r = t >> 1, half = t & 1;
    const int kv = kv0 + cw * 64 + r;
    const bool row_ok = kv < p.Sk;
    stage_acc<HD>(stage_rows, dv_acc, 1.f);
    named_bar_sync(2 + cw, 128);
    store_row_half<HD>(stage_rows + r * (HD + 4), half, p.dv + (long long)b * p.dv_b + (long long)kv * p.dv_s + (long long)h * p.dv_h,
                       row_ok, false, nullptr, nullptr, nullptr, nullptr, 0.f);
    named_bar_sync(2 + cw, 128);
    stage_acc<HD>(stage_rows, dk_acc, p.scale);
    named_bar_sync(2 + cw, 128);
    const __nv_bfloat16* xrow = nullptr;
    const __nv_bfloat16* wk = nullptr;
    const float *cs = nullptr, *sn = nullptr;
    if (p.fuse_prep) {   // dK row -> gradient of the k projection output (token index == key index)
      xrow = p.src + (long long)b * p.src_b + (long long)min(kv, p.Sk - 1) * p.src_s + p.k_off + h * HD;
      wk = (kv < p.s_split) ? p.wk1 : p.wk0;
      cs = p.cosT ? p.cosT + (long long)min(kv, p.Sk - 1) * HD : nullptr;
      sn = p.sinT ? p.sinT + (long long)min(kv, p.Sk - 1) * HD : nullptr;
    }
    store_row_half<HD>(stage_rows + r * (HD + 4), half, p.dk + (long long)b * p.dk_b + (long long)kv * p.dk_s + (long long)h * p.dk_h,
                       row_ok, p.fuse_prep != 0, xrow, wk, cs, sn, p.eps);
  }
}

// ------------------------------------------------------------------------------------------------
// dQ
// ------------------------------------------------------------------------------------------------
template <int HD>
__global__ void __launch_bounds__(384, 1)
attn_bwd_dq_kernel(const __grid_constant__ AttnBwdMaps maps, const AttnBwdParams p) {
  using Cfg = AttnBwdCfg<HD>;
  constexpr int ATOMS = HD / 64;
  constexpr int BIG_ATOM = 128 * 128, SMALL_ATOM = 64 * 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_smem = smem_base, do_smem = smem_base + Cfg::BIG;
  const uint32_t k_smem = smem_base + 2 * Cfg::BIG;                      // STAGES streamed K tiles
  const uint32_t v_smem = k_smem + Cfg::STAGES * Cfg::SMALL;             // STAGES streamed V tiles
  const uint32_t bar_base = v_smem + Cfg::STAGES * Cfg::SMALL;
  const uint32_t qd_full = bar_base;
  auto s_full = [&](int s) { return bar_base + 8u * (1 + s); };
  auto s_empty = [&](int s) { return bar_base + 8u * (1 + Cfg::STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)
  const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
  const int n_kv = (p.Sk + 63) / 64;

  if (threadIdx.x == 0) {
    mbar_init(qd_full, 1);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(s_full(s), 1);
      mbar_init(s_empty(s), 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (warp == 0) {
      if (elect_one()) {
        mbar_arrive_expect_tx(qd_full, 2 * Cfg::BIG);
        for (int a = 0; a < ATOMS; ++a) {
          tma_load_4d(q_smem + a * BIG_ATOM, &maps.q128, qd_full, a * 64, h, q0, b);
          tma_load_4d(do_smem + a * BIG_ATOM, &maps.do128, qd_full, a * 64, h, q0, b);
        }
      }
      __syncwarp();
      for (int j = 0; j < n_kv; ++j) {
        const int stg = j % Cfg::STAGES;
        mbar_wait(s_empty(stg), ((j / Cfg::STAGES) & 1) ^ 1u, 50);
        if (elect_one()) {
          mbar_arrive_expect_tx(s_full(stg), 2 * Cfg::SMALL);
          for (int a = 0; a < ATOMS; ++a) {
            tma_load_4d(k_smem + stg * Cfg::SMALL + a * SMALL_ATOM, &maps.k64, s_full(stg), a * 64, h, j * 64, b);
            tma_load_4d(v_smem + stg * Cfg::SMALL + a * SMALL_ATOM, &maps.v64, s_full(stg), a * 64, h, j * 64, b);
          }
        }
        __syncwarp();
      }
    }
  } else {
    reg_alloc<232>();
    const int cw = wg - 1, wq = warp & 3;
    const float sl2 = p.scale * 1.4426950408889634f;
    // this thread's two query rows
    float l2[2], dl[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int q = q0 + cw * 64 + wq * 16 + (lane >> 2) + 8 * hh;
      const long long o = ((long long)b * p.H + h) * p.Sq + min(q, p.Sq - 1);
      l2[hh] = __ldg(p.lse + o) * 1.4426950408889634f;
      dl[hh] = __ldg(p.delta + o);
    }
    float dq_acc[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dq_acc[i] = 0.f;
    mbar_wait(qd_full, 0, 51);
    for (int j = 0; j < n_kv; ++j) {
      const int stg = j % Cfg::STAGES;
      mbar_wait(s_full(stg), (j / Cfg::STAGES) & 1, 52);
      const uint32_t ka = k_smem + stg * Cfg::SMALL, va = v_smem + stg * Cfg::SMALL;
      float sc[32], dp[32];
      wg_fence();
      mma_kmajor_n64<HD>(sc, q_smem + cw * 8192, BIG_ATOM, ka, SMALL_ATOM);    // S  = Q K^T
      mma_kmajor_n64<HD>(dp, do_smem + cw * 8192, BIG_ATOM, va, SMALL_ATOM);   // dP = dO V^T
      wg_commit();
      wg_wait<0>();
      wg_fence_regs(sc);
      wg_fence_regs(dp);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool ok = j * 64 + 8 * i + 2 * (lane & 3) + e < p.Sk;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int x = 4 * i + 2 * hh + e;
            const float pv = ok ? ex2f(fmaf(sc[x], sl2, -l2[hh])) : 0.f;
            dp[x] = pv * (dp[x] - dl[hh]);   // dS (softmax scale applied in the epilogue)
          }
        }
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {   // 64 keys / 16
        uint32_t a[4];
        acc_to_afrag(dp, kk, a);
        wgmma_rs_mn<HD>(dq_acc, a, sdesc_mn(ka, kk * 2048, SMALL_ATOM), 1u);
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_regs(dq_acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(s_empty(stg));
    }
    // ---- epilogue through the (now idle) Q / dO tiles
    named_bar_sync(1, 256);
    float* stage_rows = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw))) + cw * 64 * (HD + 4);
    const int t = threadIdx.x & 127;
    const int r = t >> 1, half = t & 1;
    const int qrow = q0 + cw * 64 + r;
    const bool row_ok = qrow < p.Sq;
    stage_acc<HD>(stage_rows, dq_acc, p.scale);
    named_bar_sync(2 + cw, 128);
    const __nv_bfloat16* xrow = nullptr;
    const __nv_bfloat16* wqn = nullptr;
    const float *cs = nullptr, *sn = nullptr;
    if (p.fuse_prep) {   // dQ row -> gradient of the q projection output
      const int qc = min(qrow, p.Sq - 1);
      xrow = p.src + (long long)b * p.src_b + (long long)qc * p.src_s + h * HD;
      wqn = (qrow < p.s_split) ? p.wq1 : p.wq0;
      cs = p.cosT ? p.cosT + (long long)qc * HD : nullptr;
      sn = p.sinT ? p.sinT + (long long)qc * HD : nullptr;
    }
    store_row_half<HD>(stage_rows + r * (HD + 4), half, p.dq + (long long)b * p.dq_b + (long long)qrow * p.dq_s + (long long)h * p.dq_h,
                       row_ok, p.fuse_prep != 0, xrow, wqn, cs, sn, p.eps);
  }
}

}  // namespace stb
