// simpletuner_b200 — attention backward on wgmma, sm_90a (autograd of the SDPA call at reference
// flux/transformer.py:200-207).
//
//   P = exp(S*scale - LSE),  dV = P^T dO,  dP = dO V^T,  dS = P o (dP - Delta) * scale,
//   dQ = dS K,  dK = dS^T Q,   Delta_i = sum_d dO_id O_id
//
// Two deterministic kernels, no atomics; 384 threads each: warpgroup 0 is the TMA producer (three-stage ring),
// warpgroups 1 and 2 consume.
//   attn_bwd_dkdv_kernel : one CTA per (b, h, 64-key tile); streams 64-row query tiles.  Transposed domain
//       (accumulator row = key): warpgroup 1 forms S^T = K Q^T and P^T and runs dV += P^T dO, warpgroup 2 forms
//       dP^T = V dO^T and dS^T (with P^T handed over through shared memory) and runs dK += dS^T Q  (dO / Q tiles re-read
//       from the same shared-memory bytes as MN-major operands).
//   attn_bwd_dq_kernel   : one CTA per (b, h, 128-row query tile), warpgroups 1 and 2 own 64 rows each; streams 64-key
//       tiles: S = Q K^T, dP = dO V^T, dS in registers, dQ += dS K.
// The accumulators are staged through shared memory (fp32) for the store, so that each thread pair owns one whole row
// and writes it with 16-byte stores (in the wgmma accumulator layout a thread's columns of a row come in pairs 8 apart).
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
  // BIAS instantiations only: the forward's per-key logit bias, bias[b * bias_b + sk] (bf16, -inf = masked key)
  const __nv_bfloat16* bias;
  long long bias_b;
  // BIAS instantiations only, optional: the bias's live list (attn_fwd.cuh, kv_tile_at), rows kv_live_b apart.  The
  // dK/dV kernel writes zeros for a 64-key tile inside a dead 128-key tile; the dQ kernel iterates over live tiles only.
  const int* kv_live;
  long long kv_live_b;
};

struct AttnBwdMaps {
  // 4-D (d, h, s, b) SWIZZLE_128B; box (64, 1, 128, 1) for the dQ kernel's resident Q / dO, (64, 1, 64, 1) otherwise
  CUtensorMap q128, do128, q64, k64, v64, do64;
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
  static constexpr int STAGES = 3;
  static constexpr int STAT = 64 * 8;        // per stage (dK / dV kernel): 64 query rows x {LSE * log2(e), Delta}
  static constexpr int PT = 64 * 64 * 4;     // one fp32 P^T tile handed between the dK / dV warpgroups
  static constexpr int DKDV_SMEM_BYTES = 2 * SMALL + STAGES * (2 * SMALL + STAT) + 2 * PT + 1024 + 256;
  static constexpr int DQ_SMEM_BYTES = 2 * BIG + STAGES * 2 * SMALL + 1024 + 256;
  static constexpr int KB = 64 * 4;          // per stage (dQ kernel, BIAS): 64 keys x bias * log2(e)
};


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
// columns each (thread pair = lanes 2k, 2k+1).
template <int HD>
__device__ __forceinline__ void store_row_half(const float* row, int half, __nv_bfloat16* grow, bool row_ok) {
  constexpr int NC = HD / 2;
  const int c0 = half * NC;
  if (!row_ok) return;
#pragma unroll
  for (int c = 0; c < NC; c += 8) {
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = row[c0 + c + i];
    *reinterpret_cast<uint4*>(grow + c0 + c) = pack8(o);
  }
}

// m64n64k16, both operands K-major in shared memory, D = A B^T (scale-d = 0).  The accumulator is write-only ("=f"):
// with "+f" the compiler copies the previous tile's values into the accumulator registers at the loop back edge, and
// ptxas serializes every wgmma of a kernel in which a non-wgmma instruction defines an accumulator while MMAs are in
// flight.
__device__ __forceinline__ void wgmma_ss_n64_zero(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, "
      "%14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]),
        "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]),
        "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]),
        "=f"(d[25]), "=f"(d[26]), "=f"(d[27]), "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31])
      : "l"(a), "l"(b), "r"(0u));
}

template <int HD>
__device__ __forceinline__ void mma_kmajor_n64(float (&d)[32], uint32_t a_tile, uint32_t a_atom, uint32_t b_tile, uint32_t b_atom) {
  // d (64 x 64) = A (64 rows, K = HD, K-major boxes a_atom bytes apart) . B (64 rows, K-major boxes b_atom apart)^T
  wgmma_ss_n64_zero(d, sdesc_k(a_tile, 0), sdesc_k(b_tile, 0));
#pragma unroll
  for (int kk = 1; kk < HD / 16; ++kk)
    wgmma_ss_n64<0, 0>(d, sdesc_k(a_tile, (kk / 4) * a_atom + (kk % 4) * 32), sdesc_k(b_tile, (kk / 4) * b_atom + (kk % 4) * 32), 1u);
}

// ------------------------------------------------------------------------------------------------
// dK / dV
// ------------------------------------------------------------------------------------------------
// One CTA per (b, h, 64-key tile).  The two consumer warpgroups split the work by product, so that each holds one
// 64 x HD accumulator and one 64 x 64 product (dV and dK of 64 keys plus S^T and dP^T in one warpgroup do not fit the
// 168 registers a 384-thread CTA has per thread, and ptxas then spills and serializes the wgmma):
//   warpgroup 1: S^T = K Q^T -> P^T -> dV += P^T dO;  P^T (fp32) goes to warpgroup 2 through shared memory
//   warpgroup 2: dP^T = V dO^T;  dS^T = P^T o (dP^T - Delta) -> dK += dS^T Q
// The P^T hand-over is double-buffered (named barriers PT_FULL / PT_EMPTY + buffer), so warpgroup 1 runs up to one
// query tile ahead and the two warpgroups' MMAs interleave on the tensor pipe.
// BIAS: each thread's two key rows carry a constant bias * log2(e) in the exponent of P^T; a -inf key gets P^T = 0 and
// with it dS^T = 0, so its dK and dV are exactly 0.
template <int HD, bool BIAS = false>
__global__ void __launch_bounds__(384, 1)
attn_bwd_dkdv_kernel(const __grid_constant__ AttnBwdMaps maps, const AttnBwdParams p) {
  using Cfg = AttnBwdCfg<HD>;
  constexpr int ATOMS = HD / 64;
  constexpr int ATOM = 64 * 128;   // [64 rows x 64 elems] SW128 box
  constexpr int PT_FULL = 4, PT_EMPTY = 6;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t k_smem = smem_base, v_smem = smem_base + Cfg::SMALL;    // resident 64-key K / V tiles
  const uint32_t q_smem = smem_base + 2 * Cfg::SMALL;                    // STAGES streamed Q tiles
  const uint32_t do_smem = q_smem + Cfg::STAGES * Cfg::SMALL;            // STAGES streamed dO tiles
  const uint32_t stat_smem = do_smem + Cfg::STAGES * Cfg::SMALL;         // STAGES x 64 float2 {LSE * log2(e), Delta}
  const uint32_t pt_smem = stat_smem + Cfg::STAGES * Cfg::STAT;          // 2 x P^T tile, [32 values][128 threads] fp32
  const uint32_t bar_base = pt_smem + 2 * Cfg::PT;
  const uint32_t kv_full = bar_base;
  auto s_full = [&](int s) { return bar_base + 8u * (1 + s); };
  auto s_empty = [&](int s) { return bar_base + 8u * (1 + Cfg::STAGES + s); };
  float* smem_f = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw)));
  const float2* stat_rows = reinterpret_cast<const float2*>(smem_f + (stat_smem - smem_base) / 4);
  float* pt_rows = smem_f + (pt_smem - smem_base) / 4;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)
  const int kv0 = blockIdx.x * 64, h = blockIdx.y, b = blockIdx.z;
  const int n_q = (p.Sq + 63) / 64;
  if constexpr (BIAS) {
    // every key of a dead tile has P^T = 0, so its dK and dV are 0: write them without loading anything
    if (p.kv_live && p.kv_live[(long long)b * p.kv_live_b + 1 + (p.Sk + 127) / 128 + (kv0 >> 7)] == 0) {
      for (int i = threadIdx.x; i < 64 * (HD / 2); i += blockDim.x) {
        const int kv = kv0 + i / (HD / 2), c = 2 * (i % (HD / 2));
        if (kv < p.Sk) {
          *reinterpret_cast<uint32_t*>(p.dk + (long long)b * p.dk_b + (long long)kv * p.dk_s + (long long)h * p.dk_h + c) = 0u;
          *reinterpret_cast<uint32_t*>(p.dv + (long long)b * p.dv_b + (long long)kv * p.dv_s + (long long)h * p.dv_h + c) = 0u;
        }
      }
      return;
    }
  }

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(s_full(s), 2);   // TMA bytes + the row statistics
      mbar_init(s_empty(s), 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (warp == 0) {
      const float* lse_bh = p.lse + ((long long)b * p.H + h) * p.Sq;
      const float* del_bh = p.delta + ((long long)b * p.H + h) * p.Sq;
      if (elect_one()) {
        mbar_arrive_expect_tx(kv_full, 2 * Cfg::SMALL);
        for (int a = 0; a < ATOMS; ++a) {
          tma_load_4d(k_smem + a * ATOM, &maps.k64, kv_full, a * 64, h, kv0, b);
          tma_load_4d(v_smem + a * ATOM, &maps.v64, kv_full, a * 64, h, kv0, b);
        }
      }
      __syncwarp();
      for (int j = 0; j < n_q; ++j) {
        const int stg = j % Cfg::STAGES;
        mbar_wait(s_empty(stg), ((j / Cfg::STAGES) & 1) ^ 1u, 40);
        if (elect_one()) {
          mbar_arrive_expect_tx(s_full(stg), 2 * Cfg::SMALL);
          for (int a = 0; a < ATOMS; ++a) {
            tma_load_4d(q_smem + stg * Cfg::SMALL + a * ATOM, &maps.q64, s_full(stg), a * 64, h, j * 64, b);
            tma_load_4d(do_smem + stg * Cfg::SMALL + a * ATOM, &maps.do64, s_full(stg), a * 64, h, j * 64, b);
          }
        }
        // Queries past Sq get LSE = +inf, so that their P (and with it dS) is exactly 0.
        float2* st = const_cast<float2*>(stat_rows) + stg * 64;
#pragma unroll
        for (int r = lane; r < 64; r += 32) {
          const int q = j * 64 + r;
          st[r] = q < p.Sq ? make_float2(__ldg(lse_bh + q) * 1.4426950408889634f, __ldg(del_bh + q)) : make_float2(INFINITY, 0.f);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(s_full(stg));
      }
    }
  } else {
    reg_alloc<232>();
    const int cw = wg - 1;
    const int t = threadIdx.x & 127;
    float acc[HD / 2];   // dV (warpgroup 1) or dK (warpgroup 2) of the CTA's 64 keys; the first MMA initialises it
    mbar_wait(kv_full, 0, 41);
    // s[4 i + 2 hh + e]: key row (16 wq + lane / 4 + 8 hh), query column 8 i + 2 (lane % 4) + e;
    // stat4[4 i + lane % 4] = {LSE * log2(e), Delta} of query columns 8 i + 2 (lane % 4) + {0, 1}
    if (cw == 0) {
      const float sl2 = p.scale * 1.4426950408889634f;
      float kb[2] = {0.f, 0.f};   // bias * log2(e) of key rows 16 wq + lane / 4 + 8 hh
      if constexpr (BIAS) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int kv = kv0 + 16 * (t >> 5) + (lane >> 2) + 8 * hh;
          kb[hh] = kv < p.Sk ? __bfloat162float(p.bias[(long long)b * p.bias_b + kv]) * 1.4426950408889634f : 0.f;
        }
      }
      for (int j = 0; j < n_q; ++j) {
        const int stg = j % Cfg::STAGES, buf = j & 1;
        mbar_wait(s_full(stg), (j / Cfg::STAGES) & 1, 42);
        const uint32_t qa = q_smem + stg * Cfg::SMALL, da = do_smem + stg * Cfg::SMALL;
        const float4* stat4 = reinterpret_cast<const float4*>(stat_rows + stg * 64);
        float s[32];
        wg_fence();
        mma_kmajor_n64<HD>(s, k_smem, ATOM, qa, ATOM);   // S^T = K Q^T
        wg_commit();
        wg_wait<0>();   // S^T, and the previous tile's dV
        wg_fence_regs(s);
        if (j > 0) {   // both MMAs of this warpgroup that read the previous stage have retired
          __syncwarp();
          if (lane == 0) mbar_arrive(s_empty((j - 1) % Cfg::STAGES));
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 sv = stat4[4 * i + (lane & 3)];
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            if constexpr (BIAS) {
              s[4 * i + 2 * hh] = ex2f(fmaf(s[4 * i + 2 * hh], sl2, kb[hh] - sv.x));   // P^T
              s[4 * i + 2 * hh + 1] = ex2f(fmaf(s[4 * i + 2 * hh + 1], sl2, kb[hh] - sv.z));
            } else {
              s[4 * i + 2 * hh] = ex2f(fmaf(s[4 * i + 2 * hh], sl2, -sv.x));   // P^T
              s[4 * i + 2 * hh + 1] = ex2f(fmaf(s[4 * i + 2 * hh + 1], sl2, -sv.z));
            }
          }
        }
        if (j >= 2) named_bar_sync(PT_EMPTY + buf, 256);   // warpgroup 2 has read P^T of tile j - 2
        float* pt = pt_rows + buf * (Cfg::PT / 4);
#pragma unroll
        for (int x = 0; x < 32; ++x) pt[x * 128 + t] = s[x];
        named_bar_arrive(PT_FULL + buf, 256);
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {   // 64 queries / 16
          uint32_t a[4];
          acc_to_afrag(s, kk, a);
          wgmma_rs_mn<HD>(acc, a, sdesc_mn(da, kk * 2048, ATOM), (j > 0 || kk > 0) ? 1u : 0u);   // dV += P^T dO
        }
        wg_commit();
      }
    } else {
      for (int j = 0; j < n_q; ++j) {
        const int stg = j % Cfg::STAGES, buf = j & 1;
        mbar_wait(s_full(stg), (j / Cfg::STAGES) & 1, 43);
        const uint32_t qa = q_smem + stg * Cfg::SMALL, da = do_smem + stg * Cfg::SMALL;
        const float4* stat4 = reinterpret_cast<const float4*>(stat_rows + stg * 64);
        float s[32];
        wg_fence();
        mma_kmajor_n64<HD>(s, v_smem, ATOM, da, ATOM);   // dP^T = V dO^T
        wg_commit();
        wg_wait<0>();   // dP^T, and the previous tile's dK
        wg_fence_regs(s);
        if (j > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(s_empty((j - 1) % Cfg::STAGES));
        }
        named_bar_sync(PT_FULL + buf, 256);
        const float* pt = pt_rows + buf * (Cfg::PT / 4);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 sv = stat4[4 * i + (lane & 3)];
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {   // dS^T (softmax scale applied in the epilogue)
            const int x = 4 * i + 2 * hh;
            s[x] = pt[x * 128 + t] * (s[x] - sv.y);
            s[x + 1] = pt[(x + 1) * 128 + t] * (s[x + 1] - sv.w);
          }
        }
        if (j + 2 < n_q) named_bar_arrive(PT_EMPTY + buf, 256);
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          uint32_t a[4];
          acc_to_afrag(s, kk, a);
          wgmma_rs_mn<HD>(acc, a, sdesc_mn(qa, kk * 2048, ATOM), (j > 0 || kk > 0) ? 1u : 0u);   // dK += dS^T Q
        }
        wg_commit();
      }
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    // ---- epilogue: stage the dV (warpgroup 1) / dK (warpgroup 2) rows through the (now idle) K / V / Q tiles, then
    // store row-contiguously
    named_bar_sync(1, 256);
    float* stage_rows = smem_f + cw * 64 * (HD + 4);
    const int r = t >> 1, half = t & 1;
    const int kv = kv0 + r;
    const bool row_ok = kv < p.Sk;
    stage_acc<HD>(stage_rows, acc, cw == 0 ? 1.f : p.scale);
    named_bar_sync(2 + cw, 128);
    if (cw == 0) {
      store_row_half<HD>(stage_rows + r * (HD + 4), half, p.dv + (long long)b * p.dv_b + (long long)kv * p.dv_s + (long long)h * p.dv_h,
                         row_ok);
    } else {
      store_row_half<HD>(stage_rows + r * (HD + 4), half, p.dk + (long long)b * p.dk_b + (long long)kv * p.dk_s + (long long)h * p.dk_h,
                         row_ok);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// dQ
// ------------------------------------------------------------------------------------------------
// BIAS: the producer stages each key tile's 64 values of bias * log2(e) next to its K / V (s_full then also counts the
// producer warp's arrive); the consumers fold them into the exponent of P.
template <int HD, bool BIAS = false>
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
  const uint32_t kb_smem = v_smem + Cfg::STAGES * Cfg::SMALL;            // BIAS: STAGES x 64 fp32 key biases
  const uint32_t bar_base = kb_smem + (BIAS ? Cfg::STAGES * Cfg::KB : 0);
  float* kb_rows = reinterpret_cast<float*>(smem_raw + (kb_smem - smem_u32(smem_raw)));
  const uint32_t qd_full = bar_base;
  auto s_full = [&](int s) { return bar_base + 8u * (1 + s); };
  auto s_empty = [&](int s) { return bar_base + 8u * (1 + Cfg::STAGES + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)
  const int q0 = blockIdx.x * 128, h = blockIdx.y, b = blockIdx.z;
  int n_kv = (p.Sk + 63) / 64;
  const int* live = nullptr;   // BIAS with a live list: the 64-key halves of the live 128-key tiles only
  if constexpr (BIAS) {
    if (p.kv_live) {
      live = p.kv_live + (long long)b * p.kv_live_b;
      const int n_live = live[0];
      // the last live tile may be the tail tile with a single 64-key half
      n_kv = n_live > 0 ? 2 * n_live - (2 * live[n_live] + 1 >= n_kv ? 1 : 0) : 0;
    }
  }
  auto tile64 = [&](int t) { return live ? 2 * live[1 + (t >> 1)] + (t & 1) : t; };

  if (threadIdx.x == 0) {
    mbar_init(qd_full, 1);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(s_full(s), BIAS ? 2 : 1);
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
      for (int t = 0; t < n_kv; ++t) {
        const int j = tile64(t);
        const int stg = t % Cfg::STAGES;
        mbar_wait(s_empty(stg), ((t / Cfg::STAGES) & 1) ^ 1u, 50);
        if (elect_one()) {
          mbar_arrive_expect_tx(s_full(stg), 2 * Cfg::SMALL);
          for (int a = 0; a < ATOMS; ++a) {
            tma_load_4d(k_smem + stg * Cfg::SMALL + a * SMALL_ATOM, &maps.k64, s_full(stg), a * 64, h, j * 64, b);
            tma_load_4d(v_smem + stg * Cfg::SMALL + a * SMALL_ATOM, &maps.v64, s_full(stg), a * 64, h, j * 64, b);
          }
        }
        __syncwarp();
        if constexpr (BIAS) {   // keys past Sk: any finite value (their P is forced to 0)
#pragma unroll
          for (int r = lane; r < 64; r += 32) {
            const int kv = j * 64 + r;
            kb_rows[stg * 64 + r] =
                kv < p.Sk ? __bfloat162float(p.bias[(long long)b * p.bias_b + kv]) * 1.4426950408889634f : 0.f;
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(s_full(stg));
        }
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
    float dq_acc[HD / 2];   // the first MMA initialises it
    mbar_wait(qd_full, 0, 51);
    // Per key tile, three wgmma groups: S, dP, dQ.  The previous tile's dQ MMA retires behind this tile's S (its dS
    // fragments stay live until then, so dP is issued only after it: all of them together exceed the 168 registers of
    // a 384-thread CTA); exp(S) runs while dP is on the tensor pipe.  A stage goes back to the producer once the dQ MMA
    // reading its K has retired.
    for (int t = 0; t < n_kv; ++t) {
      const int j = tile64(t);
      const int stg = t % Cfg::STAGES;
      mbar_wait(s_full(stg), (t / Cfg::STAGES) & 1, 52);
      const uint32_t ka = k_smem + stg * Cfg::SMALL, va = v_smem + stg * Cfg::SMALL;
      float sc[32], dp[32];
      wg_fence();
      mma_kmajor_n64<HD>(sc, q_smem + cw * 8192, BIG_ATOM, ka, SMALL_ATOM);    // S  = Q K^T
      wg_commit();
      wg_wait<1>();   // the previous tile's dQ
      if (t > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(s_empty((t - 1) % Cfg::STAGES));
      }
      mma_kmajor_n64<HD>(dp, do_smem + cw * 8192, BIG_ATOM, va, SMALL_ATOM);   // dP = dO V^T
      wg_commit();
      wg_wait<1>();   // S
      wg_fence_regs(sc);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float2 kb2 = make_float2(0.f, 0.f);
        if constexpr (BIAS) kb2 = reinterpret_cast<const float2*>(kb_rows + stg * 64)[4 * i + (lane & 3)];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool ok = j * 64 + 8 * i + 2 * (lane & 3) + e < p.Sk;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int x = 4 * i + 2 * hh + e;
            if constexpr (BIAS) sc[x] = ok ? ex2f(fmaf(sc[x], sl2, (e ? kb2.y : kb2.x) - l2[hh])) : 0.f;   // P
            else sc[x] = ok ? ex2f(fmaf(sc[x], sl2, -l2[hh])) : 0.f;
          }
        }
      }
      wg_wait<0>();   // dP
      wg_fence_regs(dp);
#pragma unroll
      for (int x = 0; x < 32; ++x) dp[x] = sc[x] * (dp[x] - dl[(x >> 1) & 1]);   // dS (softmax scale applied in the epilogue)
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {   // 64 keys / 16
        uint32_t a[4];
        acc_to_afrag(dp, kk, a);
        wgmma_rs_mn<HD>(dq_acc, a, sdesc_mn(ka, kk * 2048, SMALL_ATOM), (t > 0 || kk > 0) ? 1u : 0u);
      }
      wg_commit();
    }
    wg_wait<0>();
    wg_fence_regs(dq_acc);
    // ---- epilogue through the (now idle) Q / dO tiles
    named_bar_sync(1, 256);
    float* stage_rows = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw))) + cw * 64 * (HD + 4);
    const int t = threadIdx.x & 127;
    const int r = t >> 1, half = t & 1;
    const int qrow = q0 + cw * 64 + r;
    const bool row_ok = qrow < p.Sq;
    stage_acc<HD>(stage_rows, dq_acc, p.scale);
    named_bar_sync(2 + cw, 128);
    store_row_half<HD>(stage_rows + r * (HD + 4), half, p.dq + (long long)b * p.dq_b + (long long)qrow * p.dq_s + (long long)h * p.dq_h,
                       row_ok);
  }
}

}  // namespace stb
