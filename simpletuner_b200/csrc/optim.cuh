// simpletuner_b200 — multi-tensor AdamW-bf16 with stochastic rounding (the reference's default optimizer `adamw_bf16`),
// one launch per optimizer step for every trainable tensor.
// reference: helpers/training/optimizers/adamw_bfloat16/__init__.py:54-180 (`AdamWBF16.step`, `_make_step`) and
//            .../stochastic/__init__.py:48-121 — ~25 tiny eager kernels per parameter tensor there.
// Every rounding point of the eager chain is reproduced (bf16 tensors between ops, fp32 `result` buffers before each
// stochastic rounding, CUDA scalar semantics: fp32 alpha / eps, addcdiv = fma(value, t1 / t2, self)); including the
// reference's quirk that the first moment is `grad + (1 - beta1) * (beta1 * exp_avg)` (oracle/adamw_bf16_oracle.py).
// Stochastic rounding: add a 16-bit random integer to the fp32 bit pattern, keep the upper 16 bits.  The integers come
// either from a caller-supplied stream (parity tests) or from a counter-based hash of (seed, element, draw).
#pragma once
#include "common.cuh"
#include "elementwise.cuh"

namespace stb {

__device__ __forceinline__ uint32_t hash_u32(uint64_t x) {   // splitmix64 finaliser -> upper bits
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return uint32_t((x ^ (x >> 31)) >> 32);
}
__device__ __forceinline__ float stochastic_bf16(float x, uint32_t rnd16) {
  return __uint_as_float((__float_as_uint(x) + rnd16) & 0xFFFF0000u);
}

constexpr int OPT_CHUNK = 256 * 8;   // elements per block

// ptrs: [5][T] device pointers (p, grad, exp_avg, exp_avg_sq, shift), all bf16 with sizes[t] elements
// Two neighbours of the optimizer step ride along, each an extra pass over the same tensors in the reference:
//   grad_clamp > 0 : the default `grad_clip_method = "value"` element clamp (trainer.py:7188-7195, clip_grad_value_)
//                    applied to the gradient as it is read (bf16 result of clamp(g, -c, c), NaN kept);
//   ema != nullptr : EMAModel.step's foreach update `shadow -= (1 - decay) * (shadow - p_new)` (ema.py:352-420) on
//                    bf16 shadows, rounding points of the two eager kernels kept (bf16 difference, then fma).
__global__ void __launch_bounds__(256)
adamw_bf16_multi_kernel(const long long* __restrict__ ptrs, const long long* __restrict__ sizes, const float* __restrict__ decay,
                        const int* __restrict__ blk_tensor, const long long* __restrict__ blk_off, int T, float beta1,
                        float beta2, float alpha1, float alpha2, float value, float eps, const int* __restrict__ rnd,
                        const long long* __restrict__ rnd_off, long long rnd_plane, unsigned long long seed, float grad_clamp,
                        const long long* __restrict__ ema, float ema_alpha) {
  const int t = blk_tensor[blockIdx.x];
  const long long n = sizes[t];
  const long long i0 = blk_off[blockIdx.x];
  __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(ptrs[0 * T + t]);
  const __nv_bfloat16* g = reinterpret_cast<const __nv_bfloat16*>(ptrs[1 * T + t]);
  __nv_bfloat16* m = reinterpret_cast<__nv_bfloat16*>(ptrs[2 * T + t]);
  __nv_bfloat16* v = reinterpret_cast<__nv_bfloat16*>(ptrs[3 * T + t]);
  __nv_bfloat16* s = reinterpret_cast<__nv_bfloat16*>(ptrs[4 * T + t]);
  __nv_bfloat16* e = ema ? reinterpret_cast<__nv_bfloat16*>(ema[t]) : nullptr;
  const float dec = decay[t];
  // per-tensor keys: t is the index within this launch, so the host gives every launch of one step its own seed
  // (training/optim.py launch_seed: optimizer seed, step, `only=` chunk salt and param-group ordinal)
  const uint32_t key0 = hash_u32(seed ^ (uint64_t(uint32_t(t)) << 40)), key1 = hash_u32((seed + 0x632BE59BD9B4E019ull) ^ (uint64_t(uint32_t(t)) << 17));
  const long long roff = rnd_off ? rnd_off[t] : 0;
  // one element of the update, shared by the vector and the scalar path
  auto clampg = [&](float gv) {
    return (grad_clamp > 0.f && gv == gv) ? bf16r(fminf(fmaxf(gv, -grad_clamp), grad_clamp)) : gv;
  };
  auto ema_update = [&](float ev, float p_new) { return bf16r(fmaf(-ema_alpha, bf16r(__fsub_rn(ev, p_new)), ev)); };
  auto update = [&](long long i, float gv, float pv, float mv, float vv, float sv, float& p_o, float& m_o, float& v_o, float& s_o) {
    uint32_t r0, r1, r2, r3;
    gv = clampg(gv);
    if (rnd) {
      r0 = uint32_t(rnd[0 * rnd_plane + roff + i]), r1 = uint32_t(rnd[1 * rnd_plane + roff + i]);
      r2 = uint32_t(rnd[2 * rnd_plane + roff + i]), r3 = uint32_t(rnd[3 * rnd_plane + roff + i]);
    } else {
      // two murmur3 finalisers over a Weyl-sequenced element counter, keyed per (launch seed, tensor): 64 random bits for
      // ~14 integer instructions (the splitmix64 pair this replaces made the kernel instruction-bound, 3.2 TB/s)
      const uint32_t c = uint32_t(i) * 0x9E3779B1u + uint32_t(uint64_t(i) >> 32) * 0x7FEB352Du;
      const uint32_t h0 = mix32(c ^ key0), h1 = mix32(c + key1);
      r0 = h0 & 0xFFFFu, r1 = h0 >> 16, r2 = h1 & 0xFFFFu, r3 = h1 >> 16;
    }
    // exp_avg.mul_(beta1); add_stochastic_(exp_avg, grad, alpha = 1 - beta1)  ->  grad + alpha * exp_avg
    const float m1 = bf16r(mv * beta1);
    const float m2 = stochastic_bf16(fmaf(alpha1, m1, gv), r0);
    // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value = 1 - beta2): torch's CUDA addcmul is a + value * (b * c), so
    // g * g is rounded on its own (exact unless it under- or overflows) and then one FMA (the CPU kernel's (value * b) * c
    // differs in about 6 of 10^4 elements and makes g^2 = inf only where (value * g) * g overflows)
    const float v1 = bf16r(vv * beta2);
    const float v2 = bf16r(fmaf(alpha2, __fmul_rn(gv, gv), v1));
    // addcdiv_stochastic_(shift, exp_avg, sqrt(exp_avg_sq) + eps, value = -lr * sqrt(1 - beta2^step))
    const float den = bf16r(bf16r(sqrtf(v2)) + eps);
    const float s1 = stochastic_bf16(fmaf(value, __fdiv_rn(m2, den), sv), r1);
    // p += shift (stochastic); shift += (p_old - p_new) (stochastic): the part of the update bf16 could not hold
    const float p1 = stochastic_bf16(__fadd_rn(s1, pv), r2);
    const float diff = bf16r(__fsub_rn(pv, p1));
    float s2 = stochastic_bf16(__fadd_rn(diff, s1), r3);
    if (dec > 0.f) s2 = bf16r(fmaf(-dec, p1, s2));   // delayed weight decay goes into the remainder
    p_o = p1, m_o = m2, v_o = v2, s_o = s2;
  };
  const long long i_end = min(n, i0 + (long long)OPT_CHUNK);
  const bool vec_ok = (((ptrs[0 * T + t] | ptrs[1 * T + t] | ptrs[2 * T + t] | ptrs[3 * T + t] | ptrs[4 * T + t] | (ema ? ema[t] : 0)) & 15) == 0);
  const long long iv = i0 + (long long)threadIdx.x * 8;
  if (vec_ok && iv + 8 <= i_end) {
    // 16-byte accesses: the step is pure HBM streaming (5 reads + 4 writes of 2 B per parameter)
    float gv[8], pv[8], mv[8], vv[8], sv[8], po[8], mo[8], vo[8], so[8];
    unpack8(*reinterpret_cast<const uint4*>(g + iv), gv);
    unpack8(*reinterpret_cast<const uint4*>(p + iv), pv);
    unpack8(*reinterpret_cast<const uint4*>(m + iv), mv);
    unpack8(*reinterpret_cast<const uint4*>(v + iv), vv);
    unpack8(*reinterpret_cast<const uint4*>(s + iv), sv);
#pragma unroll
    for (int j = 0; j < 8; ++j) update(iv + j, gv[j], pv[j], mv[j], vv[j], sv[j], po[j], mo[j], vo[j], so[j]);
    *reinterpret_cast<uint4*>(p + iv) = pack8(po);
    *reinterpret_cast<uint4*>(m + iv) = pack8(mo);
    *reinterpret_cast<uint4*>(v + iv) = pack8(vo);
    *reinterpret_cast<uint4*>(s + iv) = pack8(so);
    if (e) {
      float ev[8];
      unpack8(*reinterpret_cast<const uint4*>(e + iv), ev);
#pragma unroll
      for (int j = 0; j < 8; ++j) ev[j] = ema_update(ev[j], po[j]);
      *reinterpret_cast<uint4*>(e + iv) = pack8(ev);
    }
  } else {
    for (long long i = iv; i < min(i_end, iv + 8); ++i) {
      float po, mo, vo, so;
      update(i, __bfloat162float(g[i]), __bfloat162float(p[i]), __bfloat162float(m[i]), __bfloat162float(v[i]), __bfloat162float(s[i]),
             po, mo, vo, so);
      p[i] = __float2bfloat16(po);
      m[i] = __float2bfloat16(mo);
      v[i] = __float2bfloat16(vo);
      s[i] = __float2bfloat16(so);
      if (e) e[i] = __float2bfloat16(ema_update(__bfloat162float(e[i]), po));
    }
  }
}

}  // namespace stb
