// simpletuner_b200 — HBM-bound fused elementwise / row-reduction kernels of the diffusion step.
// Each one collapses a chain of eager PyTorch ops of the reference into a single pass with 16-byte
// coalesced accesses; the bf16 rounding points of the reference chain are reproduced so results
// track the reference path bit-for-bit wherever that is cheap.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace stb {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float bf16r(float x) { return __bfloat162float(__float2bfloat16(x)); }

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  return u;
}

// block-wide sum for 128-thread CTAs
__device__ __forceinline__ float block_sum_128(float v, float* red /*[4]*/) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return red[0] + red[1] + red[2] + red[3];
}

// ------------------------------------------------------------------------------------------------
// adaLN modulation:  out = LayerNorm(x; eps, no affine) * (1 + scale[b]) + shift[b]
// reference: diffusers AdaLayerNormZero / ZeroSingle / Continuous as called at
// flux/transformer.py:386-412 and the norm2 + modulation at :577-580.
// One 128-thread CTA per row; the row lives in registers (VPT x 8 bf16 per thread).
// ------------------------------------------------------------------------------------------------
template <int VPT>
__global__ void __launch_bounds__(128)
ln_modulate_fwd_kernel(const __nv_bfloat16* __restrict__ x, long long x_b, long long x_s,
                       const __nv_bfloat16* __restrict__ shift, const __nv_bfloat16* __restrict__ scale,
                       long long mod_b, __nv_bfloat16* __restrict__ out, long long o_b, long long o_s,
                       int S, int D, float eps) {
  __shared__ float red[4];
  const int row = blockIdx.x;
  const int b = row / S, s = row - b * S;
  const __nv_bfloat16* xr = x + b * x_b + s * x_s;
  float v[VPT][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = (i * 128 + threadIdx.x) * 8;
    if (c < D) {
      unpack8(*reinterpret_cast<const uint4*>(xr + c), v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[i][j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = 0.f;
    }
  }
  const float mean = block_sum_128(sum, red) / D;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = (i * 128 + threadIdx.x) * 8;
    if (c < D) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float d = v[i][j] - mean;
        sq += d * d;
      }
    }
  }
  const float rstd = rsqrtf(block_sum_128(sq, red) / D + eps);
  const __nv_bfloat16* sh = shift + b * mod_b;
  const __nv_bfloat16* sc = scale + b * mod_b;
  __nv_bfloat16* orow = out + b * o_b + s * o_s;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = (i * 128 + threadIdx.x) * 8;
    if (c < D) {
      float fs[8], fc[8], o[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(sh + c)), fs);
      unpack8(__ldg(reinterpret_cast<const uint4*>(sc + c)), fc);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float ln = bf16r((v[i][j] - mean) * rstd);   // LayerNorm output tensor (bf16)
        float t1 = bf16r(1.f + fc[j]);               // (1 + scale)
        o[j] = bf16r(ln * t1) + fs[j];               // * then + , each a bf16 tensor op
      }
      *reinterpret_cast<uint4*>(orow + c) = pack8(o);
    }
  }
}

// Backward of the above w.r.t. x only (modulation parameters are frozen in LoRA training):
//   dx = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * (1 + scale);   out = dx (+ add)
template <int VPT>
__global__ void __launch_bounds__(128)
ln_modulate_bwd_kernel(const __nv_bfloat16* __restrict__ dy, long long dy_b, long long dy_s,
                       const __nv_bfloat16* __restrict__ x, long long x_b, long long x_s,
                       const __nv_bfloat16* __restrict__ scale, long long mod_b,
                       const __nv_bfloat16* __restrict__ add, long long add_b, long long add_s,
                       __nv_bfloat16* __restrict__ dx, long long dx_b, long long dx_s, int S, int D,
                       float eps) {
  __shared__ float red[4];
  const int row = blockIdx.x;
  const int b = row / S, s = row - b * S;
  const __nv_bfloat16* xr = x + b * x_b + s * x_s;
  const __nv_bfloat16* gr = dy + b * dy_b + s * dy_s;
  const __nv_bfloat16* sc = scale + b * mod_b;
  float v[VPT][8], g[VPT][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = (i * 128 + threadIdx.x) * 8;
    if (c < D) {
      unpack8(*reinterpret_cast<const uint4*>(xr + c), v[i]);
      float fc[8];
      unpack8(*reinterpret_cast<const uint4*>(gr + c), g[i]);
      unpack8(__ldg(reinterpret_cast<const uint4*>(sc + c)), fc);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        sum += v[i][j];
        g[i][j] *= bf16r(1.f + fc[j]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = 0.f, g[i][j] = 0.f;
    }
  }
  const float mean = block_sum_128(sum, red) / D;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = (i * 128 + threadIdx.x) * 8;
    if (c < D) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float d = v[i][j] - mean;
        sq += d * d;
      }
    }
  }
  const float rstd = rsqrtf(block_sum_128(sq, red) / D + eps);
  float sg = 0.f, sgx = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = (i * 128 + threadIdx.x) * 8;
    if (c < D) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float xh = (v[i][j] - mean) * rstd;
        v[i][j] = xh;
        sg += g[i][j];
        sgx += g[i][j] * xh;
      }
    }
  }
  const float mg = block_sum_128(sg, red) / D;
  const float mgx = block_sum_128(sgx, red) / D;
  __nv_bfloat16* orow = dx + b * dx_b + s * dx_s;
  const __nv_bfloat16* arow = add ? add + b * add_b + s * add_s : nullptr;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = (i * 128 + threadIdx.x) * 8;
    if (c < D) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rstd * (g[i][j] - mg - v[i][j] * mgx);
      if (arow) {
        float a[8];
        unpack8(*reinterpret_cast<const uint4*>(arow + c), a);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += a[j];
      }
      *reinterpret_cast<uint4*>(orow + c) = pack8(o);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// QK RMSNorm + RoPE.  reference: diffusers RMSNorm (fp32 variance, cast, * weight) at
// flux/transformer.py:138-141,159-162 and _apply_rotary_emb_anyshape at :73-98.
// src: projection output, token-major [B, S, *] with q at column offset 0 and k at `k_off`
//      (fused QKV buffer) — per (token, head) a contiguous HD vector at head stride HD.
// dst: q_out / k_out [B, S, H, HD] (same strides for both).
// One warp per TOKEN: the token's cos/sin row and the four norm-weight slices are loaded once into
// registers and reused for all 2*H (q|k, head) rows, which are processed 4 at a time for ILP; lane owns
// HD/32 consecutive elements (RoPE pairs stay in-lane).  Rows s < s_split use the "added" (text
// stream) norm weights wq1/wk1, the rest wq0/wk0.
// ------------------------------------------------------------------------------------------------
template <int EPL>
__device__ __forceinline__ void ld_row(const __nv_bfloat16* p, float (&x)[EPL]) {
  if constexpr (EPL == 4) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    x[0] = bf16_lo(u.x); x[1] = bf16_hi(u.x); x[2] = bf16_lo(u.y); x[3] = bf16_hi(u.y);
  } else {
    const uint32_t u = *reinterpret_cast<const uint32_t*>(p);
    x[0] = bf16_lo(u); x[1] = bf16_hi(u);
  }
}
template <int EPL>
__device__ __forceinline__ void st_row(__nv_bfloat16* p, const float (&o)[EPL]) {
  if constexpr (EPL == 4) {
    uint2 u;
    u.x = pack_bf16x2(o[0], o[1]);
    u.y = pack_bf16x2(o[2], o[3]);
    *reinterpret_cast<uint2*>(p) = u;
  } else {
    *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(o[0], o[1]);
  }
}

template <int HD>
__global__ void __launch_bounds__(256)
qk_rmsnorm_rope_fwd_kernel(const __nv_bfloat16* __restrict__ src, long long src_b, long long src_s,
                           int k_off, const __nv_bfloat16* __restrict__ wq0,
                           const __nv_bfloat16* __restrict__ wk0, const __nv_bfloat16* __restrict__ wq1,
                           const __nv_bfloat16* __restrict__ wk1, int s_split,
                           const float* __restrict__ cosT, const float* __restrict__ sinT,
                           __nv_bfloat16* __restrict__ q_out, __nv_bfloat16* __restrict__ k_out,
                           long long dst_b, long long dst_s, int B, int S, int H, float eps) {
  constexpr int EPL = HD / 32;
  constexpr int U = 4;  // rows in flight per warp
  const long long tok = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (tok >= (long long)B * S) return;
  const int lane = threadIdx.x & 31;
  const int s = int(tok % S);
  const int b = int(tok / S);
  const bool txt = s < s_split;
  const __nv_bfloat16* wq = txt ? wq1 : wq0;
  const __nv_bfloat16* wk = txt ? wk1 : wk0;
  float wqv[EPL], wkv[EPL], cs[EPL], sn[EPL];
#pragma unroll
  for (int i = 0; i < EPL; ++i) {
    wqv[i] = wq ? __bfloat162float(wq[lane * EPL + i]) : 1.f;
    wkv[i] = wk ? __bfloat162float(wk[lane * EPL + i]) : 1.f;
    cs[i] = cosT ? cosT[(long long)s * HD + lane * EPL + i] : 1.f;
    sn[i] = sinT ? sinT[(long long)s * HD + lane * EPL + i] : 0.f;
  }
  const __nv_bfloat16* in_tok = src + b * src_b + s * src_s + lane * EPL;
  const long long out_tok = b * dst_b + s * dst_s + lane * EPL;
  const int rows = 2 * H;  // row r: which = r / H (0 = q, 1 = k), head = r % H
  for (int r0 = 0; r0 < rows; r0 += U) {
    float x[U][EPL];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u;
      if (r < rows) {
        const int which = r >= H, hh = which ? r - H : r;
        ld_row<EPL>(in_tok + (which ? k_off : 0) + hh * HD, x[u]);
      } else {
#pragma unroll
        for (int i = 0; i < EPL; ++i) x[u][i] = 0.f;
      }
    }
    float ss[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      ss[u] = 0.f;
#pragma unroll
      for (int i = 0; i < EPL; ++i) ss[u] += x[u][i] * x[u][i];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int u = 0; u < U; ++u) ss[u] += __shfl_xor_sync(0xffffffffu, ss[u], o);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u;
      if (r >= rows) continue;
      const int which = r >= H, hh = which ? r - H : r;
      const float rstd = rsqrtf(ss[u] / HD + eps);
      const bool has_w = which ? (wk != nullptr) : (wq != nullptr);
      float y[EPL], o[EPL];
#pragma unroll
      for (int i = 0; i < EPL; ++i) {
        const float n = bf16r(x[u][i] * rstd);  // fp32 normalise, cast to the weight dtype ...
        y[i] = has_w ? bf16r(n * (which ? wkv[i] : wqv[i])) : n;  // ... then * weight (bf16 tensor op)
      }
#pragma unroll
      for (int i = 0; i < EPL; i += 2) {
        o[i] = y[i] * cs[i] + (-y[i + 1]) * sn[i];
        o[i + 1] = y[i + 1] * cs[i + 1] + y[i] * sn[i + 1];
      }
      st_row<EPL>((which ? k_out : q_out) + out_tok + hh * HD, o);
    }
  }
}

// Backward: given dq/dk in post-RoPE space, produce gradient w.r.t. the projection outputs
// (written into the q / k column ranges of the fused d_qkv buffer).  RMSNorm weights are frozen.
//   dy = R^T d_out ;  g = dy * w ;  dx = rstd * (g - xhat * mean(g * xhat))
// DW = false (LoRA / frozen norms): no weight-gradient registers, no shared-memory staging — the round-1 footprint.
template <int HD, bool DW>
__global__ void __launch_bounds__(256)
qk_rmsnorm_rope_bwd_kernel(const __nv_bfloat16* __restrict__ dq, const __nv_bfloat16* __restrict__ dk,
                           long long d_b, long long d_s, const __nv_bfloat16* __restrict__ src,
                           long long src_b, long long src_s, int k_off,
                           const __nv_bfloat16* __restrict__ wq0, const __nv_bfloat16* __restrict__ wk0,
                           const __nv_bfloat16* __restrict__ wq1, const __nv_bfloat16* __restrict__ wk1,
                           int s_split, const float* __restrict__ cosT, const float* __restrict__ sinT,
                           __nv_bfloat16* __restrict__ dsrc, long long ds_b, long long ds_s, int B, int S,
                           int H, float eps, float* __restrict__ dw) {
  // dw (optional, full fine-tune): fp32 [4][HD] gradients of the RMSNorm weights (wq0, wk0, wq1, wk1), accumulated with
  // shared-memory atomics per block and one global atomic per entry per block:  dw[i] += (R^T d_out)[i] * xhat[i]
  constexpr int EPL = HD / 32;
  constexpr int U = 4;
  __shared__ float dw_s[DW ? 4 * HD : 1];
  if constexpr (DW) {
    for (int i = threadIdx.x; i < 4 * HD; i += blockDim.x) dw_s[i] = 0.f;
    __syncthreads();
  }
  const long long tok = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const bool active = tok < (long long)B * S;
  if (!active && !DW) return;
  const int lane = threadIdx.x & 31;
  if (active) {
  const int s = int(tok % S);
  const int b = int(tok / S);
  const bool txt = s < s_split;
  const __nv_bfloat16* wq = txt ? wq1 : wq0;
  const __nv_bfloat16* wk = txt ? wk1 : wk0;
  float wqv[EPL], wkv[EPL], cs[EPL], sn[EPL];
#pragma unroll
  for (int i = 0; i < EPL; ++i) {
    wqv[i] = wq ? __bfloat162float(wq[lane * EPL + i]) : 1.f;
    wkv[i] = wk ? __bfloat162float(wk[lane * EPL + i]) : 1.f;
    cs[i] = cosT ? cosT[(long long)s * HD + lane * EPL + i] : 1.f;
    sn[i] = sinT ? sinT[(long long)s * HD + lane * EPL + i] : 0.f;
  }
  const __nv_bfloat16* in_tok = src + b * src_b + s * src_s + lane * EPL;
  __nv_bfloat16* out_tok = dsrc + b * ds_b + s * ds_s + lane * EPL;
  const long long g_tok = b * d_b + s * d_s + lane * EPL;
  const int rows = 2 * H;
  float dwacc[2][EPL];
#pragma unroll
  for (int i = 0; i < EPL; ++i) dwacc[0][i] = 0.f, dwacc[1][i] = 0.f;
  for (int r0 = 0; r0 < rows; r0 += U) {
    float x[U][EPL], go[U][EPL];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u;
      if (r < rows) {
        const int which = r >= H, hh = which ? r - H : r;
        ld_row<EPL>(in_tok + (which ? k_off : 0) + hh * HD, x[u]);
        ld_row<EPL>((which ? dk : dq) + g_tok + hh * HD, go[u]);
      } else {
#pragma unroll
        for (int i = 0; i < EPL; ++i) x[u][i] = 0.f, go[u][i] = 0.f;
      }
    }
    float ss[U], sgx[U], g[U][EPL];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int which = (r0 + u) >= H;
      ss[u] = 0.f;
      sgx[u] = 0.f;
#pragma unroll
      for (int i = 0; i < EPL; i += 2) {
        // o[i] = y[i] c[i] - y[i+1] s[i];  o[i+1] = y[i+1] c[i+1] + y[i] s[i+1]
        const float dy0 = go[u][i] * cs[i] + go[u][i + 1] * sn[i + 1];
        const float dy1 = go[u][i + 1] * cs[i + 1] - go[u][i] * sn[i];
        g[u][i] = dy0 * (which ? wkv[i] : wqv[i]);
        g[u][i + 1] = dy1 * (which ? wkv[i + 1] : wqv[i + 1]);
        if constexpr (DW) {
          go[u][i] = dy0;        // keep the pre-weight gradient for dw
          go[u][i + 1] = dy1;
        }
      }
#pragma unroll
      for (int i = 0; i < EPL; ++i) {
        ss[u] += x[u][i] * x[u][i];
        sgx[u] += g[u][i] * x[u][i];  // scaled by rstd below
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        ss[u] += __shfl_xor_sync(0xffffffffu, ss[u], o);
        sgx[u] += __shfl_xor_sync(0xffffffffu, sgx[u], o);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u;
      if (r >= rows) continue;
      const int which = r >= H, hh = which ? r - H : r;
      const float rstd = rsqrtf(ss[u] / HD + eps);
      const float m = sgx[u] * rstd / HD;  // mean(g * xhat)
      float o[EPL];
#pragma unroll
      for (int i = 0; i < EPL; ++i) o[i] = rstd * (g[u][i] - (x[u][i] * rstd) * m);
      st_row<EPL>(out_tok + (which ? k_off : 0) + hh * HD, o);
      if constexpr (DW) {
#pragma unroll
        for (int i = 0; i < EPL; ++i) dwacc[which][i] += go[u][i] * (x[u][i] * rstd);
      }
    }
  }
  if constexpr (DW) {
    const int base = (txt ? 2 : 0) * HD;
#pragma unroll
    for (int i = 0; i < EPL; ++i) {
      atomicAdd(&dw_s[base + lane * EPL + i], dwacc[0][i]);
      atomicAdd(&dw_s[base + HD + lane * EPL + i], dwacc[1][i]);
    }
  }
  }  // active
  if constexpr (DW) {
    __syncthreads();
    for (int i = threadIdx.x; i < 4 * HD; i += blockDim.x)
      if (dw_s[i] != 0.f) atomicAdd(dw + i, dw_s[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// "Flat" variant of the backward kernel above for HD = 128 with frozen norm weights (the LoRA / LoKr training path): one
// thread = one 16-byte chunk (8 elements) of one head row, 16 lanes = one head row, no per-thread loop — the launch
// exposes B*S*2H*16 independent threads at 44 registers instead of one warp walking 48 head rows of a token, i.e. the
// memory-level parallelism of the plain streaming kernels.  Measured at the Flux shape (B = 4, S = 4608, 24 x 128;
// tools/one_kernel.py time_rope_bwd): backward 169 us = 4.0 TB/s against 254 us for the warp-per-token loop (and 196-586 us
// for its occupancy / unroll variants) -> the backward uses this kernel; the same scheme for the forward took 137 us
// against 114 us -> the forward keeps the loop kernel (its cos / sin registers are amortised over 48 head rows there).
// The token's cos / sin row (1 KB) is re-read per head row and hits L1 (16 head rows of a token share a block).
// g_q / g_k: gradients w.r.t. the post-RoPE q, k;  dsrc: the fused d_qkv buffer (q at column 0, k at column k_off).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
qk_rmsnorm_rope_flat128_bwd_kernel(const __nv_bfloat16* __restrict__ g_q, const __nv_bfloat16* __restrict__ g_k,
                                   long long g_b, long long g_s, const __nv_bfloat16* __restrict__ src, long long src_b,
                                   long long src_s, int k_off, const __nv_bfloat16* __restrict__ wq0,
                                   const __nv_bfloat16* __restrict__ wk0, const __nv_bfloat16* __restrict__ wq1,
                                   const __nv_bfloat16* __restrict__ wk1, int s_split, const float* __restrict__ cosT,
                                   const float* __restrict__ sinT, __nv_bfloat16* __restrict__ dsrc, long long ds_b,
                                   long long ds_s, int B, int S, int H, float eps) {
  constexpr int HD = 128;
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 4;   // (token, which, head)
  const int sub = threadIdx.x & 15;                                                   // 8-element chunk of the head row
  const long long rows = (long long)B * S * 2 * H;
  const bool live = row < rows;
  const long long rr = live ? row : rows - 1;      // dead lanes shadow the last row (the shuffles below are warp-wide)
  const int hh2 = int(rr % (2 * H));
  const long long tok = rr / (2 * H);
  const int s = int(tok % S), b = int(tok / S);
  const int which = hh2 >= H, hh = which ? hh2 - H : hh2;
  const bool txt = s < s_split;
  const __nv_bfloat16* w = which ? (txt ? wk1 : wk0) : (txt ? wq1 : wq0);
  float x[8], wv[8], cs[8], sn[8];
  unpack8(*reinterpret_cast<const uint4*>(src + b * src_b + s * src_s + (which ? k_off : 0) + hh * HD + sub * 8), x);
  if (w) unpack8(__ldg(reinterpret_cast<const uint4*>(w + sub * 8)), wv);
  else {
#pragma unroll
    for (int i = 0; i < 8; ++i) wv[i] = 1.f;
  }
  if (cosT) {
    const float4* cp = reinterpret_cast<const float4*>(cosT + (long long)s * HD + sub * 8);
    const float4* sp = reinterpret_cast<const float4*>(sinT + (long long)s * HD + sub * 8);
    const float4 c0 = __ldg(cp), c1 = __ldg(cp + 1), s0 = __ldg(sp), s1 = __ldg(sp + 1);
    cs[0] = c0.x; cs[1] = c0.y; cs[2] = c0.z; cs[3] = c0.w; cs[4] = c1.x; cs[5] = c1.y; cs[6] = c1.z; cs[7] = c1.w;
    sn[0] = s0.x; sn[1] = s0.y; sn[2] = s0.z; sn[3] = s0.w; sn[4] = s1.x; sn[5] = s1.y; sn[6] = s1.z; sn[7] = s1.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) cs[i] = 1.f, sn[i] = 0.f;
  }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss = fmaf(x[i], x[i], ss);
  float go[8], g[8];
  unpack8(*reinterpret_cast<const uint4*>((which ? g_k : g_q) + b * g_b + s * g_s + hh * HD + sub * 8), go);
  float sgx = 0.f;
#pragma unroll
  for (int i = 0; i < 8; i += 2) {
    const float dy0 = go[i] * cs[i] + go[i + 1] * sn[i + 1];
    const float dy1 = go[i + 1] * cs[i + 1] - go[i] * sn[i];
    g[i] = dy0 * wv[i];
    g[i + 1] = dy1 * wv[i + 1];
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) sgx = fmaf(g[i], x[i], sgx);
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) {
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
    sgx += __shfl_xor_sync(0xffffffffu, sgx, o);
  }
  const float rstd = rsqrtf(ss / HD + eps);
  const float m = sgx * rstd / HD;
  float o8[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o8[i] = rstd * (g[i] - (x[i] * rstd) * m);
  if (live) *reinterpret_cast<uint4*>(dsrc + b * ds_b + s * ds_s + (which ? k_off : 0) + hh * HD + sub * 8) = pack8(o8);
}

// ------------------------------------------------------------------------------------------------
// Flow-matching batch prep + Flux 2x2 patchify in one pass.
// reference: common.py:4975-4992 (_prepare_flow_noisy_latents: (1-sigma) x + sigma eps),
//            flux/__init__.py:25-30 (pack_latents).  latents/noise: [B, C, Hh, Ww] contiguous.
// noisy (bf16, reference tensor dtype) is written both unpacked [B,C,Hh,Ww] and packed
// [B, (Hh/2)(Ww/2), 4C];  packed index = ((c*2 + dy)*2 + dx).  Packed batch rows lie packed_b elements
// apart, so the tokens can land in a token range of a longer joint sequence (Flux Kontext: scene tokens, then
// each reference image's tokens).  noise == NULL: plain pack_latents of the latents, no noise and no sigma.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
flow_prep_pack_kernel(const __nv_bfloat16* __restrict__ lat, const __nv_bfloat16* __restrict__ noise,
                      const float* __restrict__ sigmas, __nv_bfloat16* __restrict__ noisy,
                      __nv_bfloat16* __restrict__ packed, long long packed_b, int B, int C, int Hh, int Ww) {
  const long long n = (long long)B * C * Hh * Ww;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int w = int(r % Ww); r /= Ww;
    const int hh = int(r % Hh); r /= Hh;
    const int c = int(r % C);
    const int b = int(r / C);
    __nv_bfloat16 vb = lat[i];
    if (noise) {
      // reference arithmetic (common.py:4953-4960, 4989-4991): the sigma grid is cast to the latent
      // dtype (bf16) first, then every op of (1 - g) * x + g * eps is a bf16 tensor op — reproduce
      // each rounding so the result is bit-identical to the eager chain.
      const float sg = bf16r(sigmas[b]);
      const float x = __bfloat162float(vb);
      const float e = __bfloat162float(noise[i]);
      const float v = bf16r(bf16r(1.f - sg) * x) + bf16r(sg * e);
      vb = __float2bfloat16(v);
      if (noisy) noisy[i] = vb;
    }
    const int ph = hh >> 1, dy = hh & 1, pw = w >> 1, dx = w & 1;
    const long long tok = (long long)ph * (Ww >> 1) + pw;
    const long long pi = (long long)b * packed_b + tok * (4 * C) + ((c * 2 + dy) * 2 + dx);
    packed[pi] = vb;
  }
}

// ------------------------------------------------------------------------------------------------
// Pointwise loss of reference `conditional_loss` (common.py:6132-6166) on d = pred - target (fp32):
//   l2        : d^2                                   grad 2 d
//   huber     : 2 c (sqrt(d^2 + c^2) - c)             grad 2 c d / sqrt(d^2 + c^2)
//   smooth_l1 : 2   (sqrt(d^2 + c^2) - c)             grad 2   d / sqrt(d^2 + c^2)
// c = huber_c of the sample (constant or scheduled per timestep, common.py:6168-6215).
// ------------------------------------------------------------------------------------------------
enum LossType : int { LOSS_L2 = 0, LOSS_HUBER = 1, LOSS_SMOOTH_L1 = 2 };

__device__ __forceinline__ void pointwise_loss(float d, int loss_type, float c, float& val, float& grad) {
  if (loss_type == LOSS_L2) {
    val = d * d;
    grad = 2.f * d;
    return;
  }
  const float k = loss_type == LOSS_HUBER ? 2.f * c : 2.f;
  const float r = sqrtf(d * d + c * c);
  val = k * (r - c);
  grad = k * d / r;
}

// ------------------------------------------------------------------------------------------------
// Loss reduction without floating-point atomics: the loss kernels run as ONE cluster of LOSS_CTAS CTAs of
// LOSS_THREADS threads (a fixed grid, so every thread sums a fixed set of elements in a fixed order); each CTA reduces
// its threads in a fixed tree, and CTA 0 adds the CTA sums in rank order through distributed shared memory.  The loss
// is therefore the same bit for bit from run to run.
// ------------------------------------------------------------------------------------------------
constexpr int LOSS_CTAS = 8;
constexpr int LOSS_THREADS = 1024;

__device__ __forceinline__ void loss_cluster_store(float acc, float scale, float* loss_out) {
  __shared__ float red[LOSS_THREADS / 32];
  __shared__ float cta_sum;
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    const float v = warp_sum(red[threadIdx.x]);
    if (threadIdx.x == 0) cta_sum = v;
  }
  cooperative_groups::cluster_group cl = cooperative_groups::this_cluster();
  cl.sync();
  if (cl.block_rank() == 0 && threadIdx.x == 0) {
    float t = 0.f;
    for (unsigned r = 0; r < cl.num_blocks(); ++r) t += *cl.map_shared_rank(&cta_sum, r);
    *loss_out = t * scale;
  }
  cl.sync();   // the other CTAs' shared memory stays alive until CTA 0 has read it
}

// ------------------------------------------------------------------------------------------------
// Loss: mean over batch of mean over (C,H,W) of (pred.float() - target.float())^2 with
// target = noise - latents (flow matching, common.py:4610-4611, 6286, 6426-6429), where pred arrives
// in the packed token layout (unpack_latents, flux/__init__.py:33-44, folded into the index math).
// Also emits d loss / d pred in the packed layout (bf16) scaled by `grad_scale`.
// loss_out[0] (fp32) is written, not accumulated; launch as one cluster (loss_cluster_store).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LOSS_THREADS)
flow_mse_loss_kernel(const __nv_bfloat16* __restrict__ pred_packed, const __nv_bfloat16* __restrict__ lat,
                     const __nv_bfloat16* __restrict__ noise, float* __restrict__ loss_out,
                     __nv_bfloat16* __restrict__ dpred_packed, float grad_scale, int B, int C, int Hh,
                     int Ww, int layout, int loss_type, const float* __restrict__ huber_c) {
  const long long n = (long long)B * C * Hh * Ww;
  const float inv = 1.f / float((long long)C * Hh * Ww) / float(B);
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int w = int(r % Ww); r /= Ww;
    const int hh = int(r % Hh); r /= Hh;
    const int c = int(r % C);
    const int b = int(r / C);
    const int ph = hh >> 1, dy = hh & 1, pw = w >> 1, dx = w & 1;
    const long long tok = (long long)ph * (Ww >> 1) + pw;
    // token features: Flux pack_latents order (c, dy, dx)  |  SD3 unpatchify order (dy, dx, c) ("nhwpqc->nchpwq")
    const int feat = layout == 0 ? ((c * 2 + dy) * 2 + dx) : ((dy * 2 + dx) * C + c);
    const long long pi = layout == 2 ? i : ((long long)b * ((Hh >> 1) * (Ww >> 1)) + tok) * (4 * C) + feat;   // 2 = NCHW (UNet output)
    // target = noise - latents computed in the latent dtype (bf16 tensor), then .float()
    const float tgt = bf16r(__bfloat162float(noise[i]) - __bfloat162float(lat[i]));
    const float d = __bfloat162float(pred_packed[pi]) - tgt;
    float lv, lg;
    pointwise_loss(d, loss_type, huber_c ? huber_c[b] : 0.f, lv, lg);
    acc += lv;
    if (dpred_packed) dpred_packed[pi] = __float2bfloat16(lg * inv * grad_scale);
  }
  loss_cluster_store(acc, inv, loss_out);
}

// ------------------------------------------------------------------------------------------------
// epsilon / v-prediction families (PixArt, SDXL): DDPM forward-noising + 2x2 patchify, and the weighted MSE.
// reference: common.py:5998-6002 — `noise_schedule.add_noise(latents.float(), input_noise.float(), timesteps)`
// (diffusers DDPMScheduler.add_noise: sqrt(acp[t]) * x + sqrt(1 - acp[t]) * eps, fp32) `.to(weight_dtype)`.
// coef_a / coef_b: fp32 [B] (the two gathered square roots).  Each fp32 op is rounded separately (no FMA
// contraction) so the bf16 result is bit-identical to the eager chain.
// packed feature order = (c, dy, dx): the flattened [D, C, 2, 2] PatchEmbed conv weight (diffusers PatchEmbed.proj).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ddpm_prep_pack_kernel(const __nv_bfloat16* __restrict__ lat, const __nv_bfloat16* __restrict__ noise,
                      const float* __restrict__ coef_a, const float* __restrict__ coef_b,
                      __nv_bfloat16* __restrict__ noisy, __nv_bfloat16* __restrict__ packed, int B, int C, int Hh,
                      int Ww) {
  const long long n = (long long)B * C * Hh * Ww;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int w = int(r % Ww); r /= Ww;
    const int hh = int(r % Hh); r /= Hh;
    const int c = int(r % C);
    const int b = int(r / C);
    const float v = __fadd_rn(__fmul_rn(coef_a[b], __bfloat162float(lat[i])),
                              __fmul_rn(coef_b[b], __bfloat162float(noise[i])));
    const __nv_bfloat16 vb = __float2bfloat16(v);
    if (noisy) noisy[i] = vb;
    if (packed) {
      const int ph = hh >> 1, dy = hh & 1, pw = w >> 1, dx = w & 1;
      const long long tok = (long long)ph * (Ww >> 1) + pw;
      packed[((long long)b * ((Hh >> 1) * (Ww >> 1)) + tok) * (4 * C) + ((c * 2 + dy) * 2 + dx)] = vb;
    }
  }
}

// loss = mean_b [ w_b * mean_chw (pred.float() - target.float())^2 ]   (common.py:6376-6398, 6426-6429)
// pred: packed tokens [B, (Hh/2)(Ww/2), 4C] (layout as flow_mse_loss_kernel); target: [B, C, Hh, Ww] bf16
// (epsilon: the noise; v-prediction: get_velocity(...)); weights: fp32 [B] min-SNR weights or nullptr.
__global__ void __launch_bounds__(LOSS_THREADS)
target_mse_loss_kernel(const __nv_bfloat16* __restrict__ pred_packed, const __nv_bfloat16* __restrict__ target,
                       const float* __restrict__ weights, float* __restrict__ loss_out,
                       __nv_bfloat16* __restrict__ dpred_packed, float grad_scale, int B, int C, int Hh, int Ww,
                       int layout, int loss_type, const float* __restrict__ huber_c) {
  const long long n = (long long)B * C * Hh * Ww;
  const float inv = 1.f / float((long long)C * Hh * Ww) / float(B);
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    const int w = int(r % Ww); r /= Ww;
    const int hh = int(r % Hh); r /= Hh;
    const int c = int(r % C);
    const int b = int(r / C);
    const int ph = hh >> 1, dy = hh & 1, pw = w >> 1, dx = w & 1;
    const long long tok = (long long)ph * (Ww >> 1) + pw;
    const int feat = layout == 0 ? ((c * 2 + dy) * 2 + dx) : ((dy * 2 + dx) * C + c);
    const long long pi = layout == 2 ? i : ((long long)b * ((Hh >> 1) * (Ww >> 1)) + tok) * (4 * C) + feat;   // 2 = NCHW (UNet output)
    const float wgt = weights ? weights[b] : 1.f;
    const float d = __bfloat162float(pred_packed[pi]) - __bfloat162float(target[i]);
    float lv, lg;
    pointwise_loss(d, loss_type, huber_c ? huber_c[b] : 0.f, lv, lg);
    acc += wgt * lv;
    if (dpred_packed) dpred_packed[pi] = __float2bfloat16(lg * wgt * inv * grad_scale);
  }
  loss_cluster_store(acc, inv, loss_out);
}

// ------------------------------------------------------------------------------------------------
// y[b, s, :] = gate[b, :] * x[b, s, :]   (backward of `gate * linear(...)`, flux/transformer.py:464,
// 584, 652 — the incoming gradient is scaled by the adaLN gate before the dgrad GEMM).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gate_mul_kernel(const __nv_bfloat16* __restrict__ x, long long x_b, long long x_s,
                const __nv_bfloat16* __restrict__ gate, long long g_b, __nv_bfloat16* __restrict__ y,
                long long y_b, long long y_s, int B, int S, int D) {
  const int vec_per_row = D >> 3;
  const long long total = (long long)B * S * vec_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % vec_per_row) * 8;
    const long long r = i / vec_per_row;
    const int s = int(r % S);
    const int b = int(r / S);
    float xv[8], gv[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(x + b * x_b + s * x_s + c), xv);
    unpack8(__ldg(reinterpret_cast<const uint4*>(gate + b * g_b + c)), gv);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = xv[j] * gv[j];
    *reinterpret_cast<uint4*>(y + b * y_b + s * y_s + c) = pack8(o);
  }
}


// ------------------------------------------------------------------------------------------------
// T5LayerNorm (text-encoder path, SURVEY.md 8f rank 4): out = w * bf16(x * rsqrt(mean(x^2) + eps)); one warp per row,
// 16-byte accesses, the row is read twice (second read hits L1 / L2: a T5-XXL row is 8 KB).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
rmsnorm_fwd_kernel(const __nv_bfloat16* __restrict__ x, long long x_b, long long x_s, const __nv_bfloat16* __restrict__ w,
                   __nv_bfloat16* __restrict__ out, long long o_b, long long o_s, int B, int S, int D, float eps) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= (long long)B * S) return;
  const int lane = threadIdx.x & 31;
  const int s = int(row % S), b = int(row / S);
  const __nv_bfloat16* xr = x + b * x_b + s * x_s;
  __nv_bfloat16* orow = out + b * o_b + s * o_s;
  float ss = 0.f;
  for (int c = lane * 8; c < D; c += 256) {
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) ss = fmaf(v[j], v[j], ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rstd = rsqrtf(ss / D + eps);
  for (int c = lane * 8; c < D; c += 256) {
    float v[8], wv[8], o8[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c), v);
    unpack8(__ldg(reinterpret_cast<const uint4*>(w + c)), wv);
#pragma unroll
    for (int j = 0; j < 8; ++j) o8[j] = wv[j] * bf16r(v[j] * rstd);
    *reinterpret_cast<uint4*>(orow + c) = pack8(o8);
  }
}


// ------------------------------------------------------------------------------------------------
// GELU(tanh) outside a GEMM epilogue — only the LoRA-on-MLP paths need it (flux_lora_target = "all+ffs" etc.,
// reference flux/model.py:1283-1338):  mode 0: y = gelu(pre)  — re-creates the bf16 activation the forward GEMM's
// EPI_GELU epilogue produced from the saved pre-activation (bit-identical: that epilogue applies gelu to the
// bf16-rounded pre-activation too), as the input of the fc2 / proj_out adapter's weight gradient;
// mode 1: y = g * gelu'(pre) — the dgrad through the activation when the LoRA dropout branch had to be added to the
// un-activated gradient first.  x / g / y: [B, S, D] views (element strides), D % 8 == 0.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gelu_tanh_kernel(const __nv_bfloat16* __restrict__ pre, long long p_b, long long p_s, const __nv_bfloat16* __restrict__ g,
                 long long g_b, long long g_s, __nv_bfloat16* __restrict__ y, long long y_b, long long y_s, int B, int S,
                 int D, int mode) {
  const int vec_per_row = D >> 3;
  const long long total = (long long)B * S * vec_per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % vec_per_row) * 8;
    const long long r = i / vec_per_row;
    const int s = int(r % S);
    const int b = int(r / S);
    float xv[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(pre + b * p_b + s * p_s + c), xv);
    if (mode == 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = gelu_tanh(xv[j]);
    } else {
      float gv[8];
      unpack8(*reinterpret_cast<const uint4*>(g + b * g_b + s * g_s + c), gv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = gv[j] * gelu_tanh_grad(xv[j]);
    }
    *reinterpret_cast<uint4*>(y + b * y_b + s * y_s + c) = pack8(o);
  }
}


// ------------------------------------------------------------------------------------------------
// LoRA dropout (PEFT `lora_dropout`: result += lora_B(lora_A(dropout(x))) * scaling, reference common.py:1094-1117 with the
// reference default lora_dropout = 0.1, field_registry/sections/lora.py:130-137).  Every adapted Linear owns its own
// nn.Dropout, so the members of one fused projection group (to_q / to_k / to_v share the input x) need INDEPENDENT masks.
// Masks are never stored: they are a pure function of (seed, stream, element index) — a counter-based generator, the
// murmur3 32-bit finaliser over a Weyl-sequenced counter — and are regenerated by the backward kernels:
//     keep(seed, stream, idx) = u24(mix32(idx * 0x9E3779B1 + stream * 0x85EBCA77 + seed)) >= p * 2^24
// `idx` = (b * S + s) * K + k on the LOGICAL [B, S, K] tensor.  (torch's own Philox stream is not reproduced: the
// distribution is the same, the draws are not; parity tests replay this mask into the oracle.)
//   dropout_expand : out[m, b, s, :] = bf16( x[b, s, :] * keep_m / (1 - p) )          m = 0 .. members-1
//   dropout_accum  : dx[b, s, :]    += sum_m keep_m / (1 - p) * d[m, b, s, :]          (backward through the same masks)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t mix32(uint32_t h) {
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}
__device__ __forceinline__ bool dropout_keep(uint32_t seed, uint32_t stream, unsigned long long idx, uint32_t thresh24) {
  const uint32_t lo = uint32_t(idx), hi = uint32_t(idx >> 32);
  const uint32_t h = mix32(lo * 0x9E3779B1u + mix32(hi + stream * 0x85EBCA77u + seed));
  return (h >> 8) >= thresh24;
}

__global__ void __launch_bounds__(256)
dropout_expand_kernel(const __nv_bfloat16* __restrict__ x, long long x_b, long long x_s, __nv_bfloat16* __restrict__ out,
                      int members, int B, int S, int K, float inv_keep, uint32_t thresh24, uint32_t seed, uint32_t stream0) {
  const int vec_per_row = K >> 3;
  const long long total = (long long)B * S * vec_per_row;
  const long long plane = (long long)B * S * K;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % vec_per_row) * 8;
    const long long r = i / vec_per_row;
    const int s = int(r % S);
    const int b = int(r / S);
    float xv[8];
    unpack8(*reinterpret_cast<const uint4*>(x + b * x_b + s * x_s + c), xv);
    const unsigned long long idx0 = (unsigned long long)r * K + c;
    for (int m = 0; m < members; ++m) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = dropout_keep(seed, stream0 + m, idx0 + j, thresh24) ? xv[j] * inv_keep : 0.f;
      *reinterpret_cast<uint4*>(out + m * plane + r * K + c) = pack8(o);
    }
  }
}

__global__ void __launch_bounds__(256)
dropout_accum_kernel(const __nv_bfloat16* __restrict__ d, __nv_bfloat16* __restrict__ dx, long long dx_b, long long dx_s,
                     int members, int B, int S, int K, float inv_keep, uint32_t thresh24, uint32_t seed, uint32_t stream0) {
  const int vec_per_row = K >> 3;
  const long long total = (long long)B * S * vec_per_row;
  const long long plane = (long long)B * S * K;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % vec_per_row) * 8;
    const long long r = i / vec_per_row;
    const int s = int(r % S);
    const int b = int(r / S);
    float acc[8];
    __nv_bfloat16* dst = dx + b * dx_b + s * dx_s + c;
    unpack8(*reinterpret_cast<const uint4*>(dst), acc);
    const unsigned long long idx0 = (unsigned long long)r * K + c;
    for (int m = 0; m < members; ++m) {
      float dv[8];
      unpack8(*reinterpret_cast<const uint4*>(d + m * plane + r * K + c), dv);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (dropout_keep(seed, stream0 + m, idx0 + j, thresh24)) acc[j] += dv[j] * inv_keep;
    }
    *reinterpret_cast<uint4*>(dst) = pack8(acc);
  }
}

// fp32 -> bf16 cast with optional transpose-free accumulate into an existing bf16 grad
__global__ void __launch_bounds__(256)
cast_f32_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16(in[i]);
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
