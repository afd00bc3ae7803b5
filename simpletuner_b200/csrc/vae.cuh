// simpletuner_b200 — non-GEMM kernels of the VAE latent-encode path (AutoencoderKL encoder), sm_90a.
// Activations are NHWC bf16 so that every 3x3 / 1x1 conv is a wgmma GEMM over pixels
// (gemm.cuh, CONV mode: 9 shifted K-segments whose halo TMA zero-fills).  Here: the HBM-bound pieces.
//   conv_in_3ch_kernel     : 3 -> C conv3x3 on the NCHW pixel tensor (K = 27: CUDA cores), writes NHWC
//   groupnorm_stats_kernel : per (image, group) sum / sum-of-squares of x - pivot over H*W*(C/G)   (fp32 atomics)
//   groupnorm_apply_kernel : (x - mean) * rstd * gamma + beta, optional SiLU, bf16 NHWC
//   softmax_rows_kernel    : in-place row softmax of the mid-block attention scores (fp32 math)
//   gaussian_sample_scale  : z = (mean + exp(0.5 clamp(logvar)) * eps - shift) * scale -> NCHW latents; shift and scale
//                            are scalars (AutoencoderKL) or [L] vectors (Wan 2.1 / Qwen-Image latents_mean, 1 / latents_std)
//   channel_rmsnorm_kernel : Wan 2.1 channel RMS norm F.normalize(x, dim=C) * sqrt(C) * gamma (+ bias), optional SiLU
// reference: diffusers AutoencoderKL.encode as called at common.py:2766-2772, sampling at caching/vae.py:1337,
// scaling at foundation_mixins.py:68-81.
#pragma once
#include "common.cuh"
#include "elementwise.cuh"

namespace stb {

// pixels: [B, 3, H, W] bf16 (NCHW, as the reference hands them to vae.encode); w: [C, 3, 3, 3] (OIHW); out NHWC.
// one thread = one output pixel x 8 output channels
__global__ void __launch_bounds__(256)
conv_in_3ch_kernel(const __nv_bfloat16* __restrict__ px, const __nv_bfloat16* __restrict__ w,
                   const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ out, int B, int H, int W, int C) {
  extern __shared__ float sw[];  // [C][27] + [C]
  for (int i = threadIdx.x; i < C * 27; i += blockDim.x) sw[i] = __bfloat162float(w[i]);
  for (int i = threadIdx.x; i < C; i += blockDim.x) sw[C * 27 + i] = __bfloat162float(bias[i]);
  __syncthreads();
  const int cgroups = C / 8;
  const long long total = (long long)B * H * W * cgroups;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int cg = int(idx % cgroups);
    long long pix = idx / cgroups;
    const int x = int(pix % W);
    pix /= W;
    const int y = int(pix % H);
    const int b = int(pix / H);
    float in[27];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          const int yy = y + dy - 1, xx = x + dx - 1;
          in[(c * 3 + dy) * 3 + dx] = (yy >= 0 && yy < H && xx >= 0 && xx < W)
                                          ? __bfloat162float(px[(((long long)b * 3 + c) * H + yy) * W + xx])
                                          : 0.f;
        }
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int co = cg * 8 + j;
      float acc = sw[C * 27 + co];
#pragma unroll
      for (int t = 0; t < 27; ++t) acc += in[t] * sw[co * 27 + t];
      o[j] = acc;
    }
    *reinterpret_cast<uint4*>(out + (((long long)b * H + y) * W + x) * C + cg * 8) = pack8(o);
  }
}

// Tensor-core version of the RGB stem conv: per 128-pixel tile an im2col A tile [128 px x 32] (k = (c, dy, dx): 27
// taps + 5 zeros) is built in shared memory in the SWIZZLE_128B K-major layout the wgmma descriptors expect, the padded
// weights [C x 32] sit next to it, and two K = 16 wgmma produce the [128 x C] outputs in registers.
// Persistent CTAs of two warpgroups; warpgroup w builds and multiplies pixels [64 w, 64 w + 64) of each tile.
__device__ __forceinline__ uint32_t sw128_row_chunk(uint32_t tile, int row, int chunk) {
  return tile + uint32_t(row >> 3) * 1024u + uint32_t(row & 7) * 128u + uint32_t((chunk ^ (row & 7)) << 4);
}

template <int C>
__global__ void __launch_bounds__(256, 1)
conv_in_3ch_mma_kernel(const __nv_bfloat16* __restrict__ px, const __nv_bfloat16* __restrict__ w,
                       const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ out, int B, int H, int W) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_smem = base;                       // [C rows x 128 B]
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const uint32_t a_smem = base + 32768u + uint32_t(wg) * 8192u;   // [64 rows x 128 B] per warpgroup
  const int warp = t >> 5, lane = t & 31;
  const int tiles_x = (W + 127) / 128;
  const long long num_tiles = (long long)B * H * tiles_x;

  // weights: row = output channel, 27 taps then zeros up to k = 32, swizzled like a TMA box would be
  for (int o = threadIdx.x; o < C; o += blockDim.x) {
    const unsigned short* wr = reinterpret_cast<const unsigned short*>(w) + o * 27;
    uint32_t v[16];
#pragma unroll
    for (int k = 0; k < 32; k += 2) {
      const uint32_t lo = k < 27 ? uint32_t(wr[k]) : 0u, hi = (k + 1) < 27 ? uint32_t(wr[k + 1]) : 0u;
      v[k / 2] = lo | (hi << 16);
    }
#pragma unroll
    for (int c4 = 0; c4 < 4; ++c4)
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sw128_row_chunk(w_smem, o, c4)), "r"(v[c4 * 4 + 0]),
                   "r"(v[c4 * 4 + 1]), "r"(v[c4 * 4 + 2]), "r"(v[c4 * 4 + 3]) : "memory");
  }
  fence_proxy_async_smem();
  __syncthreads();

  float acc[C / 2];
  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int tx = int(tile % tiles_x);
    const long long row = tile / tiles_x;   // b * H + y
    const int y = int(row % H);
    const int b = int(row / H);
    if (t < 64) {
      const int x = tx * 128 + wg * 64 + t;
      uint32_t pk[16];
#pragma unroll
      for (int k = 0; k < 32; k += 2) {
        float f2[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int kk = k + e;
          float val = 0.f;
          if (kk < 27) {
            const int c = kk / 9, dy = (kk % 9) / 3, dx = kk % 3;
            const int yy = y + dy - 1, xx = x + dx - 1;
            if (yy >= 0 && yy < H && xx >= 0 && xx < W) val = __bfloat162float(px[(((long long)b * 3 + c) * H + yy) * W + xx]);
          }
          f2[e] = val;
        }
        pk[k / 2] = pack_bf16x2(f2[0], f2[1]);
      }
#pragma unroll
      for (int c4 = 0; c4 < 4; ++c4)
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sw128_row_chunk(a_smem, t, c4)), "r"(pk[c4 * 4 + 0]),
                     "r"(pk[c4 * 4 + 1]), "r"(pk[c4 * 4 + 2]), "r"(pk[c4 * 4 + 3]) : "memory");
      fence_proxy_async_smem();
    }
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      if constexpr (C == 256) wgmma_ss_n256<0, 0>(acc, sdesc_k(a_smem, kk * 32), sdesc_k(w_smem, kk * 32), kk > 0 ? 1u : 0u);
      else if constexpr (C == 128) wgmma_ss_n128<0, 0>(acc, sdesc_k(a_smem, kk * 32), sdesc_k(w_smem, kk * 32), kk > 0 ? 1u : 0u);
      else wgmma_ss_n64<0, 0>(acc, sdesc_k(a_smem, kk * 32), sdesc_k(w_smem, kk * 32), kk > 0 ? 1u : 0u);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_regs(acc);
    // every warp of the warpgroup is past its MMAs before the A rows are rebuilt for the next tile
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
    // acc[4 i + 2 hh + e] = pixel 16 warp + lane / 4 + 8 hh of this warpgroup, channel 8 i + 2 (lane % 4) + e
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int x = tx * 128 + wg * 64 + warp * 16 + (lane >> 2) + 8 * hh;
      if (x >= W) continue;
      __nv_bfloat16* orow = out + (row * W + x) * C;
#pragma unroll
      for (int i = 0; i < C / 8; ++i) {
        const int c = 8 * i + 2 * (lane & 3);
        const uint32_t bv = __ldg(reinterpret_cast<const uint32_t*>(bias + c));
        *reinterpret_cast<uint32_t*>(orow + c) = pack_bf16x2(acc[4 * i + 2 * hh] + bf16_lo(bv), acc[4 * i + 2 * hh + 1] + bf16_hi(bv));
      }
    }
  }
}

// x: NHWC [B, HW, C]; stats: fp32 [B, G, 2] (zeroed by the caller).  grid = (chunks, B); each CTA reduces a
// contiguous chunk of pixels for all channels; C <= 512, channels-per-group cpg = C / G in {1, 2, 4} or a multiple of 8.
// The sums are taken around a pivot p per (image, group), the group's first channel at pixel 0: stats hold sum (x - p)
// and sum (x - p)^2.  A single-pass E[x^2] - mean^2 loses about log2(1 + (mean / sigma)^2) bits of the variance to
// cancellation (12 of fp32's 24 at mean / sigma = 64); around p the factor is 1 + (mean - p)^2 / sigma^2, a few units
// for any group whose first element is a typical member.  groupnorm_apply_kernel reads the same pivot to form the mean.
__device__ __forceinline__ void groupnorm_pivots(const __nv_bfloat16* __restrict__ xb, int v, int cpg, float (&pv)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) pv[j] = __bfloat162float(xb[((v * 8 + j) / cpg) * cpg]);
}

__global__ void __launch_bounds__(256)
groupnorm_stats_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ stats, int HW, int C, int G,
                       int pix_per_cta) {
  __shared__ float s_sum[64], s_sq[64];
  const int b = blockIdx.y;
  if (threadIdx.x < G) s_sum[threadIdx.x] = 0.f, s_sq[threadIdx.x] = 0.f;
  __syncthreads();
  const int vec_per_pix = C / 8;
  const int cpg = C / G;
  const long long p0 = (long long)blockIdx.x * pix_per_cta;
  const long long p1 = min((long long)HW, p0 + pix_per_cta);
  const __nv_bfloat16* xb = x + (long long)b * HW * C;
  // thread -> one fixed 8-channel vector column (its group(s) are fixed), striding over the chunk's pixels
  const int rows_par = blockDim.x / vec_per_pix;  // vec_per_pix <= 64 (C <= 512)
  const int r0 = threadIdx.x / vec_per_pix;
  if (r0 < rows_par) {
    const int v = threadIdx.x % vec_per_pix;
    float f[8], a[8], q[8], pv[8];
    groupnorm_pivots(xb, v, cpg, pv);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = 0.f, q[j] = 0.f;
    // unrolled so that several independent 16-byte loads are in flight; each lane still adds its pixels in order
#pragma unroll 4
    for (long long pix = p0 + r0; pix < p1; pix += rows_par) {
      unpack8(*reinterpret_cast<const uint4*>(xb + pix * C + v * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float t = f[j] - pv[j];
        a[j] += t, q[j] += t * t;
      }
    }
    if (cpg >= 8) {  // the whole 8-vector belongs to one group
      float sa = 0.f, sq = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) sa += a[j], sq += q[j];
      atomicAdd(&s_sum[(v * 8) / cpg], sa);
      atomicAdd(&s_sq[(v * 8) / cpg], sq);
    } else {  // cpg in {1, 2, 4}
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        atomicAdd(&s_sum[(v * 8 + j) / cpg], a[j]);
        atomicAdd(&s_sq[(v * 8 + j) / cpg], q[j]);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < G) {
    atomicAdd(&stats[((long long)b * G + threadIdx.x) * 2 + 0], s_sum[threadIdx.x]);
    atomicAdd(&stats[((long long)b * G + threadIdx.x) * 2 + 1], s_sq[threadIdx.x]);
  }
}

// grid = (chunks, B): like the stats kernel, a thread owns one fixed 8-channel vector column, so the per-channel
// affine (a = rstd * gamma, b = beta - mean * a, mean = p + (mean - p)) is computed once per thread and the streaming loop
// is one FMA + SiLU per element — no integer division or rsqrt in the inner loop (the first version spent 4x the HBM time there).
__global__ void __launch_bounds__(256)
groupnorm_apply_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ stats,
                       const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ beta,
                       __nv_bfloat16* __restrict__ out, int B, int HW, int C, int G, float eps, int silu,
                       int pix_per_cta) {
  const int b = blockIdx.y;
  const int vec_per_pix = C / 8;
  const int cpg = C / G;
  const int rows_par = blockDim.x / vec_per_pix;
  const int r0 = threadIdx.x / vec_per_pix;
  if (r0 >= rows_par) return;
  const int v = threadIdx.x - r0 * vec_per_pix;
  const float inv_n = 1.f / (float(HW) * float(cpg));
  float sc[8], sh[8], gm[8], bt[8], pv[8];   // pv: the stats kernel's pivots
  groupnorm_pivots(x + (long long)b * HW * C, v, cpg, pv);
  unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + v * 8)), gm);
  unpack8(__ldg(reinterpret_cast<const uint4*>(beta + v * 8)), bt);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int g = (v * 8 + j) / cpg;
    const float s1 = stats[((long long)b * G + g) * 2 + 0];
    const float q1 = stats[((long long)b * G + g) * 2 + 1];
    const float dm = s1 * inv_n;                       // mean - p
    const float var = fmaxf(q1 * inv_n - dm * dm, 0.f);
    const float rstd = rsqrtf(var + eps);
    sc[j] = rstd * gm[j];
    sh[j] = bt[j] - (pv[j] + dm) * sc[j];
  }
  const long long p0 = (long long)blockIdx.x * pix_per_cta;
  const long long p1 = min((long long)HW, p0 + pix_per_cta);
  const __nv_bfloat16* xb = x + (long long)b * HW * C + v * 8;
  __nv_bfloat16* ob = out + (long long)b * HW * C + v * 8;
  // four independent 16-byte loads in flight per thread (a single load per iteration left the kernel latency-bound at about
  // a third of the stats kernel's bandwidth)
  constexpr int UN = 4;
  for (long long pix = p0 + r0; pix < p1; pix += (long long)rows_par * UN) {
    uint4 raw[UN];
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const long long pp = pix + (long long)u * rows_par;
      if (pp < p1) raw[u] = *reinterpret_cast<const uint4*>(xb + pp * C);
    }
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const long long pp = pix + (long long)u * rows_par;
      if (pp >= p1) break;
      float f[8], o[8];
      unpack8(raw[u], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float y = fmaf(f[j], sc[j], sh[j]);
        if (silu) {
          y = bf16r(y);                 // GroupNorm output tensor (bf16), then nn.SiLU
          y = __fdividef(y, 1.f + __expf(-y));
        }
        o[j] = y;
      }
      *reinterpret_cast<uint4*>(ob + pp * C) = pack8(o);
    }
  }
}

// in-place softmax over the last dimension of s [rows, cols] (bf16 storage, fp32 math), logits pre-scaled by `scale`
__global__ void __launch_bounds__(256)
softmax_rows_kernel(__nv_bfloat16* __restrict__ s, long long row_stride, int cols, float scale) {
  __shared__ float red[8];
  __nv_bfloat16* row = s + (long long)blockIdx.x * row_stride;
  float m = -INFINITY;
  for (int c = threadIdx.x * 8; c < cols; c += blockDim.x * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(row + c), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) m = fmaxf(m, f[j]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int c = threadIdx.x * 8; c < cols; c += blockDim.x * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(row + c), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) sum += __expf((f[j] - m) * scale);
  }
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = red[0] + red[1] + red[2] + red[3] + red[4] + red[5] + red[6] + red[7];
  const float inv = 1.f / sum;
  for (int c = threadIdx.x * 8; c < cols; c += blockDim.x * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(row + c), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = __expf((f[j] - m) * scale) * inv;
    *reinterpret_cast<uint4*>(row + c) = pack8(f);
  }
}

// moments: NHWC [B, h*w, 2L] (mean | logvar); eps: NCHW [B, L, h, w]; out: NCHW [B, L, h, w] (bf16).
// shift_c / scale_c (both or neither): bf16 [L] vectors that replace the scalars, as in Qwen-Image's
// post_vae_encode_transform_sample, bf16(bf16(z - latents_mean[c]) * (1 / latents_std)[c]).
__global__ void __launch_bounds__(256)
gaussian_sample_scale_kernel(const __nv_bfloat16* __restrict__ moments, const __nv_bfloat16* __restrict__ eps,
                             __nv_bfloat16* __restrict__ out, int B, int L, int hw, float shift, float scale,
                             int has_shift, const __nv_bfloat16* __restrict__ shift_c,
                             const __nv_bfloat16* __restrict__ scale_c) {
  const long long total = (long long)B * L * hw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = int(i % hw);
    const long long r = i / hw;
    const int c = int(r % L);
    const int b = int(r / L);
    const __nv_bfloat16* mrow = moments + ((long long)b * hw + p) * (2 * L);
    const float mean = __bfloat162float(mrow[c]);
    const float logvar = fminf(fmaxf(__bfloat162float(mrow[L + c]), -30.f), 20.f);
    // DiagonalGaussianDistribution: std = exp(0.5 * logvar) (bf16 tensor), sample = mean + std * eps (bf16 ops)
    const float std = bf16r(__expf(0.5f * bf16r(logvar)));
    float z = bf16r(mean + bf16r(std * __bfloat162float(eps[i])));
    const float sh = shift_c ? __bfloat162float(shift_c[c]) : shift, sc = scale_c ? __bfloat162float(scale_c[c]) : scale;
    z = has_shift ? bf16r(bf16r(z - sh) * sc) : bf16r(z * sc);
    out[i] = __float2bfloat16(z);
  }
}

// Wan 2.1 channel RMS norm over the rows of x [rows, C] (NHWC pixels), C a multiple of 8 up to 512:
// diffusers QwenImageRMS_norm, F.normalize(x, dim=C) * self.scale * self.gamma + self.bias, then (silu) the encoder's
// separate SiLU.  Every step is a bf16 tensor in the eager module, so the kernel rounds after each one, in this order:
//   n = bf16(sqrt(sum_c x_c^2))      the norm's fp32 sum of squares (overflows to inf as torch's does), one rounding
//   n = max(n, bf16(eps))            clamp_min(eps) of F.normalize, eps = 1e-12 there (a NaN norm stays NaN)
//   q = bf16(x / n)                  IEEE fp32 division
//   s = bf16(q * scale)              scale = fp32(sqrt(C)), the Python float dim ** 0.5 as torch passes it
//   g = bf16(s * gamma[c])
//   y = bf16(g + bias[c])            without a bias module attribute the reference adds the Python float 0.0: y = g + 0
//                                    (which turns -0 into +0)
//   out = bf16(y / (1 + expf(-y)))   silu: torch's SiLU kernel, IEEE division and the accurate expf
// Only the sum of squares is taken in another order than torch's; it moves n by at most (C + 4) 2^-24 relative before
// the bf16 rounding.  A group of TPR lanes (the power of two >= C / 8, at most 32) owns a row; lane j holds the 8-channel
// vector j (and j + 32 when TPR = 32), and a warp takes 32 / TPR rows at a time, so every lane of the warp takes part in the shuffles.
template <int TPR>
__global__ void __launch_bounds__(256)
channel_rmsnorm_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
                       const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ out, long long rows, int C,
                       float scale, float eps, int silu) {
  constexpr int RPW = 32 / TPR;             // rows per warp and step
  constexpr int VPL = TPR == 32 ? 2 : 1;     // 8-channel vectors per lane (C / 8 <= 64)
  const int lane = threadIdx.x & 31, sub = lane / TPR, j = lane % TPR;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int nvec = C / 8;
  const float n_min = bf16r(eps);           // torch casts the clamp_min scalar to the tensor's dtype
  for (long long base = warp * RPW; base < rows; base += nwarps * RPW) {
    const long long row = base + sub;
    const bool live = row < rows;
    float f[VPL][8];
    float ss = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c8 = j + v * TPR;
      if (live && c8 < nvec) unpack8(*reinterpret_cast<const uint4*>(x + row * C + c8 * 8), f[v]);
      else
#pragma unroll
        for (int e = 0; e < 8; ++e) f[v][e] = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) ss += f[v][e] * f[v][e];
    }
#pragma unroll
    for (int o = TPR / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    float n = bf16r(sqrtf(ss));
    if (!(n != n)) n = fmaxf(n, n_min);      // a NaN norm stays NaN (fmaxf would return n_min)
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c8 = j + v * TPR;
      if (!live || c8 >= nvec) continue;
      float o[8], gm[8], bs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + c8 * 8)), gm);
      if (bias) unpack8(__ldg(reinterpret_cast<const uint4*>(bias + c8 * 8)), bs);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float q = bf16r(__fdiv_rn(f[v][e], n));
        const float g = bf16r(bf16r(q * scale) * gm[e]);
        float y = bf16r(g + bs[e]);
        if (silu) y = __fdiv_rn(y, 1.f + expf(-y));
        o[e] = y;
      }
      *reinterpret_cast<uint4*>(out + row * C + c8 * 8) = pack8(o);
    }
  }
}

}  // namespace stb
