/* stb200.h — C ABI of libstb200.so: the sm_90a (H100) kernels of the SimpleTuner diffusion training step.
 *
 * Plain pointers, sizes and element strides only; every pointer is a CUDA device pointer unless
 * noted, every tensor is bf16 unless noted, `stream` is a cudaStream_t.  All functions return 0 on
 * success and a negative code on failure; stb_last_error() returns the message of the last failure
 * on the calling thread.  There is no CPU fallback: without an sm_90 (H100) device every launch fails.
 *
 * The reference (bghira/SimpleTuner) has no FFI for this path — its seams are Python-level
 * (SURVEY.md §8b).  Each entry point below names the reference call site it replaces; the Python
 * host layer (simpletuner_b200/) binds these through ctypes and mirrors the reference's module /
 * processor interfaces on top.  INTEGRATION.md shows the reference-side binding.
 */
#ifndef STB200_H
#define STB200_H
#ifdef __cplusplus
extern "C" {
#endif

#define STB_OK 0
#define STB_ERR_ARG (-1)
#define STB_ERR_CUDA (-2)
#define STB_ERR_UNSUPPORTED (-3)

const char* stb_last_error(void);
int stb_version(void);
/* number of kernel launches issued by this library since load / last reset (bench gpu_launches) */
long long stb_launch_count(void);
void stb_reset_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * Linear layers.  Replaces nn.Linear / PEFT lora.Linear / torch.cat+Linear call sites:
 *   flux/transformer.py:127-129,146-148 (q/k/v + added projections), :218-221 (out projections),
 *   :460-464 (single-block proj_mlp / GELU / cat / proj_out / gate / residual),
 *   :581-586 (FeedForward + gate + residual), :1001,1064,1506 (embedders, proj_out),
 *   common.py:1094-1117 (LoRA: y = x W^T + b + s (x A^T) B^T as an extra K-segment).
 *
 *   D[b, s, n] = epi( sum_seg  A_seg[b, s, :K_seg] . W_seg[n, :K_seg]  + bias[n] )
 *
 * A_seg: [num_batches, rows_per_batch, K] with element strides (a_batch_stride, a_row_stride, 1).
 * W_seg: [N, K] with row stride w_row_stride (K contiguous) — nn.Linear weight layout.
 * Alignment: base pointers 16 B; strides multiples of 8 elements.
 * ------------------------------------------------------------------------------------------- */
enum stb_gemm_epilogue {
  STB_EPI_STORE = 0,     /* D = acc + bias                                                     */
  STB_EPI_GELU = 1,      /* D = gelu_tanh(acc + bias); aux (optional, written) = acc + bias    */
  STB_EPI_GATE_RES = 2,  /* D = res + gate[b, n] * (acc + bias); nan_to_num optional           */
  STB_EPI_MUL_DGELU = 3, /* D = acc * gelu_tanh'(aux[b, s, n])      (aux read)                 */
  STB_EPI_ADD_RES = 4,   /* D = acc + bias + res                                               */
  STB_EPI_MUL = 5,       /* D = bf16(acc + bias) * aux[b, s, n]  (aux read) — T5 gated-GELU feed-forward, transformers
                            T5DenseGatedActDense (called through flux/pipeline.py:1085)             */
  STB_EPI_QUICK_GELU = 6, /* D = y * sigmoid(1.702 y), y = bf16(acc + bias) — CLIP text MLP (flux/pipeline.py:1127) */
  STB_EPI_SILU = 7        /* D = y * sigmoid(y), y = bf16(acc + bias) — Chroma approximator layers, PixArtAlphaTextProjection
                             with act_fn "silu" (chroma/transformer.py:297-313)                                       */
};

typedef struct {
  const void* a;
  long long a_batch_stride, a_row_stride;
  const void* w;
  long long w_row_stride;
  int K;
  int w_kn;  /* 0: w is [N, K] row-major (nn.Linear layout); 1: w is [K, N] row-major, i.e. the contraction index is the ROW
                of w — the dgrad of a Linear reads the forward weight itself (dx = dy W), no transposed copy.  N % 8 == 0. */
} stb_gemm_seg;

typedef struct {
  int num_batches, rows_per_batch, N, nseg;
  stb_gemm_seg seg[3];
  void* d;
  long long d_batch_stride, d_row_stride;
  const void* bias; /* [N] or NULL */
  int epi;
  int nan_to_num;   /* STB_EPI_GATE_RES: nan->0, +-inf->+-65504 (flux/transformer.py:467,601) */
  const void* gate; /* [num_batches, N] with batch stride */
  long long gate_batch_stride;
  const void* res;
  long long res_batch_stride, res_row_stride;
  void* aux;
  long long aux_batch_stride, aux_row_stride;
  int tile_mt, tile_bn; /* 0 = pick automatically; else BN in {64,128,256} (tiles of 128 rows, 64 at BN 256).
                           MT: 1 = single CTAs, 2 = 2-CTA clusters multicasting the shared W tile (BN 128 only; other
                           widths run single CTAs), 0 = automatic (clusters for the GELU / dGELU epilogues at 16 or
                           more 128-row tiles).  The results are the same bits either way. */
} stb_gemm_args;

int stb_gemm_bf16(const stb_gemm_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Attention.  Replaces F.scaled_dot_product_attention (non-causal, no mask, dropout 0) at
 * flux/transformer.py:200-207 and its autograd backward.  q/k/v/o are [B, S, H, HD] views given by
 * element strides (batch, token, head; HD contiguous).  lse: fp32 [B, H, Sq].  HD in {64, 128}.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  int B, H, Sq, Sk, HD;
  float scale;
  const void *q, *k, *v;
  long long q_b, q_s, q_h, k_b, k_s, k_h, v_b, v_s, v_h;
  void* o;
  long long o_b, o_s, o_h;
  float* lse;
  /* optional additive logit bias: logit = scale * q.k + bias[b * bias_b + h * bias_h + sq * bias_q + sk], bf16,
   * -inf = masked; NULL = none.  A zero stride shares the bias along that dimension.  Two forms:
   *  - bias_q >= Sk: a [B or 1, H or 1, Sq, Sk] bias (text encoders: T5 relative position bias T5Attention.compute_bias,
   *    CLIP causal mask — transformers classes called at flux/pipeline.py:1085, 1127);
   *  - bias_q = bias_h = 0: one row per sample over the keys, [B or 1, Sk] (Flux masked training: the float mask
   *    `(expand_flux_attention_mask(...) > 0).to(dtype)` that FluxAttnProcessor2_0 adds to the logits, reference
   *    flux/transformer.py:170-173, 200-207, 227-242).
   * Every query row must keep at least one finite logit. */
  const void* bias;
  long long bias_h, bias_q;
  long long bias_b;
  /* optional, per-key bias only: its live list, int32 rows kv_live_b elements apart (0 = one row for the batch), each
   * {n_live, the indices of the n_live live 128-key tiles in ascending order padded to n_tiles slots, one 0/1 live flag
   * per tile}, n_tiles = ceil(Sk / 128).  A tile is dead when the bias of every key in it is -inf (past Sk counts as
   * -inf).  The kernels then skip the dead tiles, with the same results; a row with no live tile is outside the contract
   * above.  NULL = process every tile.  Built on the device by simpletuner_b200.ops.key_bias_live_list. */
  const int* kv_live;
  long long kv_live_b;
} stb_attn_fwd_args;
int stb_attn_fwd(const stb_attn_fwd_args* args, void* stream);

typedef struct {
  int B, H, Sq, Sk, HD;
  float scale;
  const void *q, *k, *v, *o, *d_o;
  long long q_b, q_s, q_h, k_b, k_s, k_h, v_b, v_s, v_h, o_b, o_s, o_h, do_b, do_s, do_h;
  const float* lse;  /* [B, H, Sq] from the forward */
  float* delta;      /* [B, H, Sq] fp32 scratch: rowsum(dO * O) */
  void *dq, *dk, *dv;
  long long dq_b, dq_s, dq_h, dk_b, dk_s, dk_h, dv_b, dv_s, dv_h;
  /* the forward's per-key bias (bias_q = bias_h = 0 form of stb_attn_fwd_args; reference flux/transformer.py:170-173,
   * 200-207): bf16 bias[b * bias_b + sk], bias_b = 0 shares one row across the batch; NULL = none.  Any other form
   * returns STB_ERR_UNSUPPORTED.  Keys whose bias is -inf get dk = dv = 0. */
  const void* bias;
  long long bias_b;
  /* optional: the forward's live list (stb_attn_fwd_args.kv_live).  dk = dv = 0 is written for the keys of dead tiles
   * without computing them, and dq iterates over the live tiles only.  NULL = process every tile. */
  const int* kv_live;
  long long kv_live_b;
} stb_attn_bwd_args;
int stb_attn_bwd(const stb_attn_bwd_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * adaLN modulation: out = LayerNorm(x, eps, no affine) * (1 + scale[b]) + shift[b]
 * Replaces diffusers AdaLayerNormZero/ZeroSingle/Continuous + the norm2 modulation, as called at
 * flux/transformer.py:386-412, 577-580, 589-593.  Backward is w.r.t. x only (+ optional residual
 * gradient `add`), the modulation linears being frozen under LoRA training.
 * ------------------------------------------------------------------------------------------- */
int stb_ln_modulate_fwd(const void* x, long long x_b, long long x_s, const void* shift, const void* scale,
                        long long mod_b, void* out, long long o_b, long long o_s, int B, int S, int D,
                        float eps, void* stream);
int stb_ln_modulate_bwd(const void* dy, long long dy_b, long long dy_s, const void* x, long long x_b,
                        long long x_s, const void* scale, long long mod_b, const void* add, long long add_b,
                        long long add_s, void* dx, long long dx_b, long long dx_s, int B, int S, int D,
                        float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Per-head RMSNorm (fp32 variance, learned weight) + rotary embedding on q and k.
 * Replaces attn.norm_q/norm_k/norm_added_q/norm_added_k + _apply_rotary_emb_anyshape
 * (flux/transformer.py:73-98, 138-141, 159-162, 189-190).  src is the projection output
 * [B, S, ...] holding q at column 0 and k at column k_off (head stride HD); rows s < s_split use
 * the *_added weights (text stream), the rest the image-stream weights.  cos/sin: fp32 [S, HD] or NULL.
 * ------------------------------------------------------------------------------------------- */
int stb_qk_rmsnorm_rope_fwd(const void* src, long long src_b, long long src_s, int k_off, const void* wq,
                            const void* wk, const void* wq_added, const void* wk_added, int s_split,
                            const float* cos_t, const float* sin_t, void* q_out, void* k_out,
                            long long dst_b, long long dst_s, int B, int S, int H, int HD, float eps,
                            void* stream);
int stb_qk_rmsnorm_rope_bwd(const void* dq, const void* dk, long long d_b, long long d_s, const void* src,
                            long long src_b, long long src_s, int k_off, const void* wq, const void* wk,
                            const void* wq_added, const void* wk_added, int s_split, const float* cos_t,
                            const float* sin_t, void* dsrc, long long ds_b, long long ds_s, int B, int S,
                            int H, int HD, float eps, float* dw /* optional fp32 [4][HD], accumulated: d(wq, wk, wq_added, wk_added) */,
                            void* stream);

/* ---------------------------------------------------------------------------------------------
 * Flow-matching batch prep and loss (Flux 2x2 patchify folded into the index math).
 *   stb_flow_prep_pack : noisy = (1 - sigma) * latents + sigma * noise  (common.py:4975-4992),
 *                        written unpacked (optional) and packed (flux/__init__.py:25-30).  Packed batch rows
 *                        are packed_b elements apart (>= (Hh/2)(Ww/2)*4C; offset `packed` to start at a token), so
 *                        the tokens can fill a range of a joint sequence.  noise = sigmas = noisy = NULL: a plain
 *                        pack_latents (Flux Kontext reference latents, flux/__init__.py:64-172).
 *   stb_flow_mse_loss  : mean_b mean_chw (pred.float() - (noise - latents).float())^2
 *                        (common.py:4610-4611, 6286, 6426-6429) with pred in packed layout
 *                        (layout 0: Flux unpack_latents order, flux/__init__.py:33-44; layout 1: SD3
 *                        unpatchify order "nhwpqc->nchpwq", sd3/transformer.py:894); optional d loss/d pred.
 * latents/noise: bf16 [B, C, Hh, Ww] contiguous; sigmas fp32 [B]; loss_out fp32 [1] (written; the reduction has a fixed
 * order, so the loss is the same bit for bit from run to run).
 * loss_type (both loss entry points): 0 = l2, 1 = huber, 2 = smooth_l1 as `conditional_loss` defines them
 * (common.py:6132-6166): huber = 2c(sqrt(d^2+c^2)-c), smooth_l1 = 2(sqrt(d^2+c^2)-c); huber_c = fp32 [B]
 * per-sample c (constant or the scheduled value of common.py:6168-6215), may be NULL for l2.
 * ------------------------------------------------------------------------------------------- */
int stb_flow_prep_pack(const void* latents, const void* noise, const float* sigmas, void* noisy,
                       void* packed, long long packed_b, int B, int C, int Hh, int Ww, void* stream);
int stb_flow_mse_loss(const void* pred_packed, const void* latents, const void* noise, float* loss_out,
                      void* dpred_packed, float grad_scale, int B, int C, int Hh, int Ww, int layout, int loss_type,
                      const float* huber_c, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Optimizer (SURVEY.md 8f rank 1): the reference's default `adamw_bf16` — AdamWBF16.step / _make_step,
 * helpers/training/optimizers/adamw_bfloat16/__init__.py:54-180, with the stochastic-rounding helpers of
 * .../stochastic/__init__.py:48-121 — for EVERY trainable tensor in one launch.
 *   ptrs      : device int64 [5][T] = pointers to p, grad, exp_avg, exp_avg_sq, shift (bf16, sizes[t] elements each)
 *   decay     : device fp32 [T] `decay_this_iteration` per tensor (0 = none; __init__.py:96-99 delayed weight decay)
 *   blk_tensor / blk_off : device [num_blocks] block -> (tensor, first element); a block covers stb_adamw_bf16_chunk() elements
 *   step, lr  : the reference's `state["step"]` (after the increment) and group lr; betas / eps as in the group — all as
 *               doubles (Python floats): the derived fp32 scalars are formed exactly as the eager path forms them
 *   rnd       : optional device int32 [4][rnd_plane] 16-bit random integers in the reference's draw order (exp_avg, shift,
 *               p, shift) with per-tensor offsets rnd_off[T] — parity tests; NULL = counter-based generator keyed by `seed`
 *   grad_clamp: > 0 fuses the default element clamp of the gradients (`grad_clip_method = "value"`, trainer.py:7188-7195)
 *               into the read of `grad` (the stored gradient is left untouched); 0 = off
 *   ema_shadow: optional device int64 [T] pointers to bf16 EMA shadows; with it the kernel also applies EMAModel.step's
 *               `shadow -= ema_one_minus_decay * (shadow - p_new)` (helpers/training/ema.py:352-420); NULL = off
 * ------------------------------------------------------------------------------------------- */
int stb_adamw_bf16_multi(const long long* ptrs, const long long* sizes, const float* decay, const int* blk_tensor,
                         const long long* blk_off, int num_blocks, int T, double beta1, double beta2, double step, double lr,
                         double eps, const int* rnd, const long long* rnd_off, long long rnd_plane, unsigned long long seed,
                         double grad_clamp, const long long* ema_shadow, double ema_one_minus_decay, void* stream);
int stb_adamw_bf16_chunk(void);

/* ---------------------------------------------------------------------------------------------
 * Epsilon / v-prediction families (PixArt, SDXL).
 *   stb_ddpm_prep_pack  : noisy = (coef_a[b] * latents.float() + coef_b[b] * noise.float()).to(bf16), the
 *                         DDPMScheduler.add_noise the reference calls in fp32 at common.py:5998-6002
 *                         (coef_a = sqrt(alphas_cumprod[t]), coef_b = sqrt(1 - alphas_cumprod[t]), fp32 [B]);
 *                         written unpacked [B,C,Hh,Ww] (optional) and 2x2-patchified [B, Hh/2*Ww/2, 4C]
 *                         in (c, dy, dx) feature order = the flattened PatchEmbed conv weight (optional).
 *   stb_target_mse_loss : mean_b [ w_b * mean_chw (pred.float() - target.float())^2 ]  (common.py:6376-6398,
 *                         6426-6429; w = min-SNR weights or NULL) with pred in packed layout (layout as above:
 *                         0 = (c,dy,dx), 1 = (dy,dx,c) "nhwpqc->nchpwq", pixart/transformer.py:763-782);
 *                         target bf16 [B,C,Hh,Ww]; optional d loss / d pred (packed, bf16).
 * ------------------------------------------------------------------------------------------- */
int stb_ddpm_prep_pack(const void* latents, const void* noise, const float* coef_a, const float* coef_b, void* noisy,
                       void* packed, int B, int C, int Hh, int Ww, void* stream);
int stb_target_mse_loss(const void* pred_packed, const void* target, const float* weights, float* loss_out,
                        void* dpred_packed, float grad_scale, int B, int C, int Hh, int Ww, int layout, int loss_type,
                        const float* huber_c, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LyCORIS LoKr (lora_type = "lycoris", algo = "lokr": helpers/training/trainer.py:3390-3505; module attributes lokr_w1 /
 * lokr_w2 / org_weight as used by helpers/training/peft_init.py:34-38; algorithm from the third-party lycoris-lora, setup.py:319):
 *   delta W = kron(w1 [a, c], w2 [b, d]) * scale on a Linear of shape [a*b, c*d];  y = linear(x, W + delta W).
 *   stb_lokr_rebuild     : out = bf16(W + delta W) (row stride out_row_stride) and, when out_t != NULL, its transpose
 *                          (row stride out_t_row_stride) in the same pass — once per optimizer step, straight into the fused
 *                          q|k|v / dgrad layouts the GEMMs read.
 *   stb_lokr_factor_grads: dw1 [a, c], dw2 [b, d] (fp32, overwritten) from the full weight gradient dW [a*b, c*d] (bf16):
 *                          dw1[i,k] = scale * sum_{j,l} dW[ib+j, kd+l] w2[j,l];  dw2[j,l] = scale * sum_{i,k} dW[ib+j, kd+l] w1[i,k]
 *                          — what autograd computes through torch.kron in the reference.  d % 8 == 0.
 * ------------------------------------------------------------------------------------------- */
int stb_lokr_rebuild(const void* W, long long w_row_stride, const void* w1, const void* w2, float scale, void* out,
                     long long out_row_stride, void* out_t, long long out_t_row_stride, int a, int b, int c, int d, void* stream);
int stb_lokr_factor_grads(const void* dW, long long dw_row_stride, const void* w1, const void* w2, float scale, float* dw1,
                          float* dw2, int a, int b, int c, int d, void* stream);

/* T5LayerNorm (RMS norm without mean subtraction or bias; transformers T5LayerNorm.forward, the text encoder the reference
 * runs at flux/pipeline.py:1085):  out = w * bf16(x * rsqrt(mean_d(x^2) + eps)), statistics in fp32.
 * x / out: [B, S, D] views (element strides, D contiguous, D % 8 == 0); w: bf16 [D]. */
int stb_rmsnorm_fwd(const void* x, long long x_b, long long x_s, const void* w, void* out, long long o_b, long long o_s,
                    int B, int S, int D, float eps, void* stream);

/* GELU(tanh) outside a GEMM epilogue, for the adapters on the MLP projections (flux_lora_target "all+ffs", "context+ffs",
 * "tiny" ...: reference flux/model.py:1272-1376; activation: flux/transformer.py:447, diffusers FeedForward
 * "gelu-approximate").  mode 0: y = gelu(pre) (the activation the forward epilogue produced, re-created from the saved
 * pre-activation); mode 1: y = g * gelu'(pre).  [B, S, D] views with element strides, D % 8 == 0. */
int stb_gelu_tanh(const void* pre, long long p_b, long long p_s, const void* g, long long g_b, long long g_s, void* y,
                  long long y_b, long long y_s, int B, int S, int D, int mode, void* stream);

/* y[b, s, :] = gate[b, :] * x[b, s, :]  — gradient of `gate * linear(...)` w.r.t. the linear output
 * (flux/transformer.py:464, 584, 652), applied before the dgrad GEMM. */
int stb_gate_mul(const void* x, long long x_b, long long x_s, const void* gate, long long g_b, void* y,
                 long long y_b, long long y_s, int B, int S, int D, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LoRA dropout (PEFT `lora_dropout`, reference common.py:1094-1117; default 0.1: field_registry/sections/lora.py:130-137).
 * Masks are a counter-based function of (seed, stream0 + member, element index of the logical [B,S,K] tensor) and are
 * regenerated in backward, never stored.
 *   stb_dropout_expand: out[m, b, s, :] = bf16(x[b, s, :] * keep_m / (1 - p)), out contiguous [members, B, S, K]
 *   stb_dropout_accum : dx[b, s, :] += sum_m keep_m / (1 - p) * d[m, b, s, :],  d contiguous [members, B, S, K]
 * K multiple of 8, 0 <= p < 1. */
int stb_dropout_expand(const void* x, long long x_b, long long x_s, void* out, int members, int B, int S, int K, float p,
                       unsigned int seed, unsigned int stream0, void* stream);
int stb_dropout_accum(const void* d, void* dx, long long dx_b, long long dx_s, int members, int B, int S, int K, float p,
                      unsigned int seed, unsigned int stream0, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Full-rank weight gradient (full fine-tune, BASELINE config 3; autograd of nn.Linear.weight under
 * `accelerator.backward`, reference trainer.py:7126, sd3/transformer.py:145-241):
 *   dW[n, k] = alpha * sum_{b,s} dY[b, s, n] * X[b, s, k]  (+ dW[n, k] if accumulate)     bf16 [N, K], row stride dw_row_stride
 * dY [B, S, N] / X [B, S, K] bf16 views (last dim contiguous; strides in elements, multiples of 8); N, K multiples of 8.
 *
 * stb_colsum2: per-(batch, column) token reductions for the adaLN / gate / bias gradients:
 *   sum[b, d] = sum_s dy[b, s, d];   dot[b, d] = sum_s dy[b, s, d] * z[b, s, d]     fp32 [B, D], either may be NULL. */
int stb_wgrad_full(const void* dy, long long dy_b, long long dy_s, const void* x, long long x_b, long long x_s, void* dw,
                   long long dw_row_stride, int B, int S, int N, int K, float alpha, int accumulate, void* stream);
int stb_colsum2(const void* dy, long long dy_b, long long dy_s, const void* z, long long z_b, long long z_s, float* sum,
                float* dot, int B, int S, int D, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LoRA weight gradients: out[r, n] += alpha * sum_m L[m, r] * Rm[m, n]   (fp32 out [R, N])
 *   dA = s * (dY B)^T X   (L = dY B [M, r], Rm = X  [M, K])
 *   dB^T = s * (X A^T)^T dY (L = X A^T [M, r], Rm = dY [M, N])
 * Autograd of peft lora.Linear (reference common.py:1094-1117).
 * R is a multiple of 8 up to 128 and N a multiple of 8; L and Rm are 16-byte aligned with row strides (and, when B > 1,
 * batch strides) that are multiples of 8 elements.  Every (batch, row-split) CTA writes its partial [R, N] into
 * `workspace` (fp32, at least stb_skinny_tn_workspace(B, S, R, N) elements) with plain stores and a second kernel adds
 * the slabs to `out` in index order, so the result is the same bit for bit from run to run.  Anything else, a NULL or
 * short workspace included, returns STB_ERR_ARG before any launch.
 * ------------------------------------------------------------------------------------------- */
long long stb_skinny_tn_workspace(int B, int S, int R, int N);
int stb_skinny_tn(const void* L, long long l_b, long long l_s, const void* Rm, long long r_b, long long r_s,
                  float* out, int B, int S, int R, int N, float alpha, float* workspace, long long workspace_elems,
                  void* stream);

/* ---------------------------------------------------------------------------------------------
 * VAE latent encode (diffusers AutoencoderKL.encode as called at reference common.py:2766-2772 from
 * caching/vae.py:1311; sampling caching/vae.py:1337; scaling foundation_mixins.py:68-81).
 * Activations are NHWC bf16; every 3x3 conv is a wgmma implicit GEMM (9 shifted K-segments, the halo
 * is zero-filled by TMA); 1x1 convs / attention projections are stb_gemm_bf16 over pixels.
 *   stb_conv3x3_nhwc : out[B,Ho,Wo,Co] = conv3x3(x[B,H,W,Ci]; w[Co, 9*Cp] tap-major (dy,dx,ci)) + bias (+ res)
 *                      stride 1: padding 1;  stride 2: F.pad(x,(0,1,0,1)) then stride-2 (Downsample2D)
 *                      Ci and Co multiples of 8; Cp = Ci rounded up to a multiple of 64, each tap's columns
 *                      [Ci, Cp) of w zero (Cp = Ci when Ci % 64 == 0)
 *   stb_conv_in_3ch  : conv_in on the NCHW pixel tensor [B,3,H,W] (w OIHW [C,3,3,3]) -> NHWC [B,H,W,C]
 *   stb_groupnorm_nhwc : GroupNorm(G, eps, affine) (+ SiLU) over NHWC; stats = fp32 scratch [B*G*2]
 *   stb_softmax_rows : in-place softmax(scale * s) over rows of the mid-block attention scores (scale > 0)
 *   stb_gaussian_sample_scale : z = (mean + exp(.5 clamp(logvar,-30,20)) * eps - shift) * scale, NHWC moments
 *                      [B,h*w,2L] + NCHW eps [B,L,h,w] -> NCHW latents [B,L,h,w]
 *   stb_gaussian_sample_channel_norm : the same sample, then bf16(bf16(z - shift[c]) * inv_std[c]) with bf16 [L]
 *                      vectors (Qwen-Image latents_mean and 1 / latents_std)
 *   stb_channel_rmsnorm_nhwc : Wan 2.1 channel RMS norm over the contiguous rows of x [rows, C]:
 *                      F.normalize(x, dim=C, eps) * sqrt(C) * gamma (+ bias, may be NULL) (+ SiLU); C a multiple of 8
 *                      in [8, 512], finite eps >= 0, 16-byte aligned pointers; the eager module's bf16 rounding after
 *                      every op (csrc/vae.cuh)
 * ------------------------------------------------------------------------------------------- */
int stb_conv3x3_nhwc(const void* x, const void* w, const void* bias, const void* res, void* out, int B, int H, int W,
                     int C_in, int C_out, int stride, void* stream);
int stb_conv_in_3ch(const void* pixels, const void* w, const void* bias, void* out, int B, int H, int W, int C,
                    void* stream);
int stb_groupnorm_nhwc(const void* x, const void* gamma, const void* beta, void* out, float* stats, int B, int HW,
                       int C, int G, float eps, int silu, void* stream);
int stb_softmax_rows(void* s, long long row_stride, int rows, int cols, float scale, void* stream);
int stb_gaussian_sample_scale(const void* moments, const void* eps, void* out, int B, int L, int hw, float shift,
                              float scale, int has_shift, void* stream);
int stb_gaussian_sample_channel_norm(const void* moments, const void* eps, void* out, int B, int L, int hw,
                                     const void* shift, const void* inv_std, void* stream);
int stb_channel_rmsnorm_nhwc(const void* x, const void* gamma, const void* bias, void* out, long long rows, int C,
                             float eps, int silu, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STB200_H */
