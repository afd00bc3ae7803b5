// simpletuner_b200 — joint (non-causal) softmax attention forward on wgmma, sm_90a.
//
// Replaces F.scaled_dot_product_attention at reference flux/transformer.py:200-207 (and the SD3 /
// PixArt call sites) for the training path: O = softmax(Q K^T * scale) V, plus the per-row
// log-sum-exp that the backward kernel consumes.
//
// One CTA owns 128 query rows of one (batch, head) and streams the whole key/value sequence in 128-key tiles:
//   warpgroup 0    : TMA producer (Q once, K / V double-buffered; one warp issues)
//   warpgroups 1, 2: 64 query rows each.  S = Q K^T (wgmma, both operands in shared memory, S in registers),
//                    online softmax in registers, O += P V (wgmma with P as the register A operand, V MN-major).
// The two consumer warpgroups run independently, so one's softmax overlaps the other's MMAs.
#pragma once
#include "common.cuh"

namespace stb {

struct AttnFwdParams {
  int B, H, Sq, Sk;
  float scale;        // softmax scale (1/sqrt(head_dim) unless overridden)
  __nv_bfloat16* O;   // [B, Sq, H, HD] via strides
  long long o_b, o_s, o_h;
  float* lse;         // [B, H, Sq] natural-log LSE of the scaled scores
  // BIAS instantiation only: additive logit bias (T5 relative position bias, CLIP causal mask, the Flux per-sample key
  // bias of masked training):
  // logit = scale * q.k + bias[b * bias_b + h * bias_h + sq * bias_q + sk]   (bf16; -inf masks; a zero stride shares the
  // bias along that dimension: bias_b = 0 across the batch, bias_h = bias_q = 0 gives one row per sample over the keys)
  const __nv_bfloat16* bias;
  long long bias_h, bias_q;
  float inv_scale;
  long long bias_b;
  // KEY instantiation only, optional: the live list of the per-key bias (kv_live_row): row b at kv_live + b * kv_live_b
  // holds {n_live, the n_live live 128-key tile indices in ascending order, ...}.  Null: every tile is processed.
  const int* kv_live;
  long long kv_live_b;
};

// Live list of a per-key bias, one row per bias row: [n_live, live tile indices ascending (n_tiles slots, the first
// n_live used), live flag per tile (n_tiles)], n_tiles = ceil(Sk / 128).  A 128-key tile is dead when every key of it
// has bias -inf (the padding past Sk counts as -inf).  Skipping a dead tile gives the bits of processing it: its keys
// have p = 0, which adds nothing to l or O, and the row max either stays (alpha = 1) or stays -inf (alpha = 0).
__device__ __forceinline__ int kv_tile_at(const int* live, int t) { return live ? live[1 + t] : t; }

struct AttnFwdMaps {
  CUtensorMap q, k, v;  // 4-D (d, h, s, b), box (64, 1, 128, 1), SWIZZLE_128B
};

template <int HD>
struct AttnFwdCfg {
  static constexpr int ATOMS = HD / 64;
  static constexpr int TILE_BYTES = 128 * HD * 2;
  static constexpr int KV_STAGES = 2;
  static constexpr int SMEM_BYTES = TILE_BYTES + KV_STAGES * 2 * TILE_BYTES + 1024 + 256;
  static constexpr int THREADS = 384;
};

// A operand (64 x 16, bf16) of k-step kk from a 64 x N fp32 accumulator in wgmma layout
template <int R>
__device__ __forceinline__ void acc_to_afrag(const float (&d)[R], int kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(d[8 * kk + 0], d[8 * kk + 1]);
  a[1] = pack_bf16x2(d[8 * kk + 2], d[8 * kk + 3]);
  a[2] = pack_bf16x2(d[8 * kk + 4], d[8 * kk + 5]);
  a[3] = pack_bf16x2(d[8 * kk + 6], d[8 * kk + 7]);
}

template <int N>
__device__ __forceinline__ void wgmma_rs_mn(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b, uint32_t accumulate) {
  if constexpr (N == 128) wgmma_rs_n128<1>(d, a, b, accumulate);
  else wgmma_rs_n64<1>(d, a, b, accumulate);
}

// BIAS = true: the bias tile is added to the raw scores (pre-divided by the softmax scale).  Every query row needs at least
// one finite logit somewhere; a 128-key tile in which a row is all -inf (at any position) contributes nothing.
// KEY = true (with BIAS; bias_h = bias_q = 0): one bias row per sample.  The producer warp stages each key tile's 128
// values in shared memory (ring b_full / b_empty next to K / V) and the consumers read them as float2: per-element global
// loads of the general form made the forward 1.7x slower at the Flux shape (DESIGN.md 1).
template <int HD, bool BIAS = false, bool KEY = false>
__global__ void __launch_bounds__(384, 1)
attn_fwd_kernel(const __grid_constant__ AttnFwdMaps maps, const AttnFwdParams p) {
  using Cfg = AttnFwdCfg<HD>;
  constexpr int ATOMS = Cfg::ATOMS;
  constexpr int TILE = Cfg::TILE_BYTES;
  constexpr int ATOM_BYTES = 128 * 64 * 2;  // [128 rows x 64 elems] SW128 box
  constexpr int NSTG = Cfg::KV_STAGES;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_smem = smem_base;
  const uint32_t k_smem = q_smem + TILE;
  const uint32_t v_smem = k_smem + NSTG * TILE;
  const uint32_t bar_base = v_smem + NSTG * TILE;
  const uint32_t q_full = bar_base;
  auto k_full = [&](int s) { return bar_base + 8u * (1 + s); };
  auto k_empty = [&](int s) { return bar_base + 8u * (1 + NSTG + s); };
  auto v_full = [&](int s) { return bar_base + 8u * (1 + 2 * NSTG + s); };
  auto v_empty = [&](int s) { return bar_base + 8u * (1 + 3 * NSTG + s); };
  auto b_full = [&](int s) { return bar_base + 8u * (1 + 4 * NSTG + s); };    // KEY only
  auto b_empty = [&](int s) { return bar_base + 8u * (1 + 5 * NSTG + s); };
  float* kb_rows = reinterpret_cast<float*>(smem_raw + (bar_base + 256 - smem_u32(smem_raw)));   // KEY: NSTG x 128 fp32

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform for the compiler (wgmma needs converged warpgroups)
  const int q0 = blockIdx.x * 128;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  int n_kv = (p.Sk + 127) / 128;
  const int* live = nullptr;   // KEY with a live list: iterate over the live tiles only
  if constexpr (KEY) {
    if (p.kv_live) {
      live = p.kv_live + (long long)b * p.kv_live_b;
      n_kv = live[0];
    }
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps.q);
    tma_prefetch_desc(&maps.k);
    tma_prefetch_desc(&maps.v);
    mbar_init(q_full, 1);
    for (int s = 0; s < NSTG; ++s) {
      mbar_init(k_full(s), 1);
      mbar_init(k_empty(s), 8);
      mbar_init(v_full(s), 1);
      mbar_init(v_empty(s), 8);
      if constexpr (KEY) {
        mbar_init(b_full(s), 1);
        mbar_init(b_empty(s), 8);
      }
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    reg_dealloc<40>();
    if (warp == 0) {
      if (elect_one()) {
        mbar_arrive_expect_tx(q_full, TILE);
        for (int a = 0; a < ATOMS; ++a) tma_load_4d(q_smem + a * ATOM_BYTES, &maps.q, q_full, a * 64, h, q0, b);
      }
      __syncwarp();
      for (int t = 0; t < n_kv; ++t) {
        const int j = kv_tile_at(live, t);
        const int stg = t % NSTG;
        const uint32_t par = ((t / NSTG) & 1) ^ 1u;
        mbar_wait(k_empty(stg), par, 10);
        if (elect_one()) {
          mbar_arrive_expect_tx(k_full(stg), TILE);
          for (int a = 0; a < ATOMS; ++a)
            tma_load_4d(k_smem + stg * TILE + a * ATOM_BYTES, &maps.k, k_full(stg), a * 64, h, j * 128, b);
        }
        __syncwarp();
        mbar_wait(v_empty(stg), par, 11);
        if (elect_one()) {
          mbar_arrive_expect_tx(v_full(stg), TILE);
          for (int a = 0; a < ATOMS; ++a)
            tma_load_4d(v_smem + stg * TILE + a * ATOM_BYTES, &maps.v, v_full(stg), a * 64, h, j * 128, b);
        }
        __syncwarp();
        if constexpr (KEY) {   // after the V issue: the bias is needed only once S is done
          mbar_wait(b_empty(stg), par, 12);
          const __nv_bfloat16* brow = p.bias + (long long)b * p.bias_b + (long long)j * 128;
#pragma unroll
          for (int r = lane; r < 128; r += 32) kb_rows[stg * 128 + r] = j * 128 + r < p.Sk ? __bfloat162float(brow[r]) : 0.f;
          __syncwarp();
          if (lane == 0) mbar_arrive(b_full(stg));
        }
      }
    }
  } else {
    // ===================== consumers: 64 query rows each =====================
    reg_alloc<232>();
    const int cw = wg - 1;
    const int wq = warp & 3;
    const int r_lo = q0 + cw * 64 + wq * 16 + (lane >> 2);   // rows r_lo and r_lo + 8
    const float sl2 = p.scale * 1.4426950408889634f;
    float s_acc[64];
    float o_acc[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o_acc[i] = 0.f;
    float m_row[2] = {-INFINITY, -INFINITY};   // raw-score row max
    float l_row[2] = {0.f, 0.f};               // this thread's share of the row sum
    const __nv_bfloat16* brow[2] = {nullptr, nullptr};
    if constexpr (BIAS && !KEY) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
        brow[hh] = p.bias + (long long)b * p.bias_b + (long long)h * p.bias_h +
                   (long long)min(r_lo + 8 * hh, p.Sq - 1) * p.bias_q;
    }
    const uint32_t qa = q_smem + cw * 8192;
    mbar_wait(q_full, 0, 20);

    for (int t = 0; t < n_kv; ++t) {
      const int j = kv_tile_at(live, t);
      const int stg = t % NSTG;
      const uint32_t par = (t / NSTG) & 1;
      // ---- S = Q K^T
      mbar_wait(k_full(stg), par, 21);
      const uint32_t ka = k_smem + stg * TILE;
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
        const uint32_t off = (kk / 4) * ATOM_BYTES + (kk % 4) * 32;
        wgmma_ss_n128<0, 0>(s_acc, sdesc_k(qa, off), sdesc_k(ka, off), kk > 0 ? 1u : 0u);
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_regs(s_acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(k_empty(stg));

      // ---- online softmax (s_acc[4 i + 2 hh + e] = row r_lo + 8 hh, key 8 i + 2 (lane % 4) + e)
      const int kv_valid = p.Sk - j * 128;
      if constexpr (KEY) mbar_wait(b_full(stg), par, 23);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float2 kb2 = make_float2(0.f, 0.f);
        if constexpr (KEY) kb2 = reinterpret_cast<const float2*>(kb_rows + stg * 128)[4 * i + (lane & 3)];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * i + 2 * (lane & 3) + e;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            float v = s_acc[4 * i + 2 * hh + e];
            if constexpr (KEY) {
              if (c < kv_valid) v = fmaf(e ? kb2.y : kb2.x, p.inv_scale, v);
            } else if constexpr (BIAS) {
              if (c < kv_valid) v = fmaf(__bfloat162float(brow[hh][j * 128 + c]), p.inv_scale, v);
            }
            if (c >= kv_valid) v = -INFINITY;
            s_acc[4 * i + 2 * hh + e] = v;
          }
        }
      }
      if constexpr (KEY) {
        __syncwarp();
        if (lane == 0) mbar_arrive(b_empty(stg));
      }
      float alpha[2], nmb[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float m = -INFINITY;
#pragma unroll
        for (int i = 0; i < 16; ++i) m = fmaxf(m, fmaxf(s_acc[4 * i + 2 * hh], s_acc[4 * i + 2 * hh + 1]));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        const float m_new = fmaxf(m_row[hh], m);
        // A row that is -inf in every key so far (a bias can do that) exponentiates against 0 instead of -inf: its
        // exponentials and alpha are then 0, not NaN.  Without a bias every tile has a finite key.
        const float m_exp = (BIAS && m_new == -INFINITY) ? 0.f : m_new;
        alpha[hh] = ex2f((m_row[hh] - m_exp) * sl2);   // 0 on the first tile
        m_row[hh] = m_new;
        nmb[hh] = -m_exp * sl2;
        l_row[hh] *= alpha[hh];
      }
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) {
        o_acc[4 * i + 0] *= alpha[0];
        o_acc[4 * i + 1] *= alpha[0];
        o_acc[4 * i + 2] *= alpha[1];
        o_acc[4 * i + 3] *= alpha[1];
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float x = ex2f(fmaf(s_acc[4 * i + 2 * hh + e], sl2, nmb[hh]));
            l_row[hh] += x;
            s_acc[4 * i + 2 * hh + e] = x;
          }
        }
      }

      // ---- O += P V
      mbar_wait(v_full(stg), par, 22);
      const uint32_t va = v_smem + stg * TILE;
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {   // 128 keys / 16
        uint32_t a[4];
        acc_to_afrag(s_acc, kk, a);
        wgmma_rs_mn<HD>(o_acc, a, sdesc_mn(va, kk * 2048, ATOM_BYTES), 1u);
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_regs(o_acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(v_empty(stg));
    }

    // ---- epilogue: O / l -> bf16 -> global; LSE
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float l = l_row[hh];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const int s = r_lo + 8 * hh;
      const float inv_l = 1.f / l;
      if (s < p.Sq) {
        __nv_bfloat16* orow = p.O + (long long)b * p.o_b + (long long)s * p.o_s + (long long)h * p.o_h;
#pragma unroll
        for (int i = 0; i < HD / 8; ++i)
          *reinterpret_cast<uint32_t*>(orow + 8 * i + 2 * (lane & 3)) =
              pack_bf16x2(o_acc[4 * i + 2 * hh] * inv_l, o_acc[4 * i + 2 * hh + 1] * inv_l);
        if (p.lse && (lane & 3) == 0) p.lse[((long long)b * p.H + h) * p.Sq + s] = m_row[hh] * p.scale + logf(l);
      }
    }
  }
}

}  // namespace stb
