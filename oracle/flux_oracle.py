"""CPU oracle for the Flux training step — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module; the product path (simpletuner_b200/) never does.

What this is: a plain-PyTorch restatement, written from the reference sources cited on every
function, of the arithmetic that SimpleTuner's Flux training step performs:
  * FluxTransformer2DModel.forward           reference flux/transformer.py:940-1515
  * FluxTransformerBlock / Single block      reference flux/transformer.py:416-510, 514-687
  * FluxAttnProcessor2_0                     reference flux/transformer.py:116-224
  * Flux._model_predict_single               reference flux/model.py:707-864
  * flow-matching batch prep / target / loss reference common.py:4975-4992, 4610-4611, 6286, 6426-6429
The layer classes that the reference imports from the third-party `diffusers` package
(diffusers>=0.36.0, reference setup.py:287 — NOT vendored in the reference and not installed
here) are restated from their published semantics: Attention + RMSNorm, AdaLayerNormZero /
ZeroSingle / Continuous, FeedForward("gelu-approximate"), FluxPosEmbed (get_1d_rotary_pos_embed),
CombinedTimestep(Guidance)TextProjEmbeddings, PEFT lora.Linear.

PARITY STATUS: the index / schedule / RoPE-application / pack-unpack functions are pinned against
the reference's own source executed verbatim (oracle/ref_extract.py, tests/golden/); the
diffusers-owned layer arithmetic is **parity unpinned** — the reference's tests hold no golden
vector for the denoiser forward/backward (SURVEY.md §4, §8c).

The code is dtype-agnostic: run it on fp32 tensors for the "truth" the CUDA path is compared with,
or on bf16 tensors to emulate the eager bf16 tensor-op chain of the reference.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


@dataclass
class FluxConfig:
    """Mirror of FluxTransformer2DModel.__init__ arguments (reference flux/transformer.py:727-743)."""
    patch_size: int = 1
    in_channels: int = 64
    num_layers: int = 19
    num_single_layers: int = 38
    attention_head_dim: int = 128
    num_attention_heads: int = 24
    joint_attention_dim: int = 4096
    pooled_projection_dim: int = 768
    guidance_embeds: bool = True
    axes_dims_rope: Tuple[int, int, int] = (16, 56, 56)

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim


# --------------------------------------------------------------------------------------------------
# parameter inventory (names follow the diffusers / reference state_dict so checkpoints map 1:1)
# --------------------------------------------------------------------------------------------------
def flux_param_shapes(cfg: FluxConfig) -> Dict[str, Tuple[int, ...]]:
    D, hd = cfg.inner_dim, cfg.attention_head_dim
    shapes: Dict[str, Tuple[int, ...]] = {}

    def lin(name, out_f, in_f):
        shapes[name + ".weight"] = (out_f, in_f)
        shapes[name + ".bias"] = (out_f,)

    lin("x_embedder", D, cfg.in_channels)
    lin("context_embedder", D, cfg.joint_attention_dim)
    lin("time_text_embed.timestep_embedder.linear_1", D, 256)
    lin("time_text_embed.timestep_embedder.linear_2", D, D)
    if cfg.guidance_embeds:
        lin("time_text_embed.guidance_embedder.linear_1", D, 256)
        lin("time_text_embed.guidance_embedder.linear_2", D, D)
    lin("time_text_embed.text_embedder.linear_1", D, cfg.pooled_projection_dim)
    lin("time_text_embed.text_embedder.linear_2", D, D)
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}."
        lin(p + "norm1.linear", 6 * D, D)
        lin(p + "norm1_context.linear", 6 * D, D)
        for n in ("to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj", "to_out.0", "to_add_out"):
            lin(p + "attn." + n, D, D)
        for n in ("norm_q", "norm_k", "norm_added_q", "norm_added_k"):
            shapes[p + f"attn.{n}.weight"] = (hd,)
        lin(p + "ff.net.0.proj", 4 * D, D)
        lin(p + "ff.net.2", D, 4 * D)
        lin(p + "ff_context.net.0.proj", 4 * D, D)
        lin(p + "ff_context.net.2", D, 4 * D)
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}."
        lin(p + "norm.linear", 3 * D, D)
        lin(p + "proj_mlp", 4 * D, D)
        lin(p + "proj_out", D, 5 * D)
        for n in ("to_q", "to_k", "to_v"):
            lin(p + "attn." + n, D, D)
        for n in ("norm_q", "norm_k"):
            shapes[p + f"attn.{n}.weight"] = (hd,)
    lin("norm_out.linear", 2 * D, D)
    lin("proj_out", cfg.patch_size * cfg.patch_size * cfg.in_channels, D)
    return shapes


def init_flux_params(cfg: FluxConfig, seed: int = 0, dtype=torch.float32, std: float = 0.02) -> Dict[str, Tensor]:
    """Deterministic synthetic weights (SURVEY.md §8d): Linear ~ N(0, std^2), biases ~ N(0, (std/2)^2)
    so that bias paths are exercised, RMSNorm weights = 1 + N(0, 0.05^2)."""
    g = torch.Generator().manual_seed(seed)
    out: Dict[str, Tensor] = {}
    for name, shape in flux_param_shapes(cfg).items():
        if name.endswith("norm_q.weight") or name.endswith("norm_k.weight") or name.endswith("norm_added_q.weight") or name.endswith("norm_added_k.weight"):
            t = 1.0 + 0.05 * torch.randn(shape, generator=g)
        elif name.endswith(".bias"):
            t = 0.5 * std * torch.randn(shape, generator=g)
        else:
            t = std * torch.randn(shape, generator=g)
        out[name] = t.to(dtype)
    return out


FLUX_LORA_TARGETS_ALL = ("to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj", "to_out.0", "to_add_out")
"""flux_lora_target="all" (reference flux/model.py:1249-1262; to_qkv/add_qkv_proj only exist when fused)."""


FLUX_LORA_TARGETS_FFS = FLUX_LORA_TARGETS_ALL + ("ff.net.0.proj", "ff.net.2", "ff_context.net.0.proj", "ff_context.net.2",
                                                 "proj_mlp", "proj_out")
"""flux_lora_target="all+ffs" (reference flux/model.py:1283-1301); "+embedder" adds x_embedder (:1320-1338)."""


def lora_target_names(cfg: FluxConfig, targets=FLUX_LORA_TARGETS_ALL):
    """PEFT's target_modules rule: a Linear is adapted when its qualified name equals a target or ends with ".<target>"
    (so "proj_out" selects every single block's proj_out AND the model's final proj_out)."""
    names = []
    for key in flux_param_shapes(cfg):
        if not key.endswith(".weight"):
            continue
        mod = key[: -len(".weight")]
        if any(mod == t or mod.endswith("." + t) for t in targets) and len(flux_param_shapes(cfg)[key]) == 2:
            names.append(mod)
    return names


def init_lora_params(cfg: FluxConfig, rank: int, seed: int = 1, dtype=torch.float32, b_std: float = 0.02,
                     targets=FLUX_LORA_TARGETS_ALL) -> Dict[str, Tensor]:
    """PEFT default init: A ~ kaiming_uniform(a=sqrt(5)), B = 0; b_std > 0 gives a non-zero B so that
    gradients w.r.t. A are exercised (SURVEY.md §8d)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    shapes = flux_param_shapes(cfg)
    for n in lora_target_names(cfg, targets):
        n_out, k_in = shapes[n + ".weight"]
        bound = 1.0 / math.sqrt(k_in)  # kaiming_uniform(a=sqrt(5)) on [r, K]: bound = sqrt(6/((1+5) K)) = 1/sqrt(K)
        out[n + ".lora_A.weight"] = ((torch.rand((rank, k_in), generator=g) * 2 - 1) * bound).to(dtype)
        out[n + ".lora_B.weight"] = (b_std * torch.randn((n_out, rank), generator=g)).to(dtype)
    return out


# --------------------------------------------------------------------------------------------------
# layer restatements (diffusers semantics)
# --------------------------------------------------------------------------------------------------
# PEFT lora_dropout replay (tests only): {linear name: mask [B, S, K] already divided by (1 - p)}.  PEFT applies
# `lora_B(lora_A(dropout(x)))` with one nn.Dropout per adapted Linear; the CUDA path draws its masks from its own
# counter-based generator, so parity tests materialise those masks and replay them here.
DROPOUT_MASKS: Optional[Dict[str, Tensor]] = None
# LyCORIS LoKr settings used when the adapter dict carries `<linear>.lokr_w1` entries (reference documentation/LYCORIS.md default)
LOKR: Dict[str, float] = {"linear_dim": 10000, "linear_alpha": 1, "multiplier": 1.0}


def linear(x: Tensor, P: Dict[str, Tensor], name: str, lora: Optional[Dict[str, Tensor]] = None,
           lora_scale: float = 1.0) -> Tensor:
    """nn.Linear, optionally wrapped by PEFT lora.Linear (reference common.py:1094-1117):
    result = base(x) + lora_B(lora_A(dropout(x))) * scaling   (dropout = identity unless DROPOUT_MASKS replays a mask)."""
    if lora is not None and (name + ".lokr_w1") in lora:
        # LyCORIS LoKr (oracle/lokr_oracle.py): the adapted weight is rebuilt, y = linear(x, W + kron(w1, w2) * scale)
        from .lokr_oracle import lokr_linear
        return lokr_linear(x, P[name + ".weight"], P.get(name + ".bias"), lora, name, LOKR["linear_dim"], LOKR["linear_alpha"],
                           LOKR.get("multiplier", 1.0))
    y = F.linear(x, P[name + ".weight"], P.get(name + ".bias"))
    if lora is not None and (name + ".lora_A.weight") in lora:
        a = lora[name + ".lora_A.weight"]
        b = lora[name + ".lora_B.weight"]
        xa = x
        if DROPOUT_MASKS is not None and name in DROPOUT_MASKS:
            xa = (x * DROPOUT_MASKS[name].to(x.dtype)).to(x.dtype)
        y = y + F.linear(F.linear(xa, a), b) * lora_scale
    return y


def rms_norm(x: Tensor, weight: Tensor, eps: float) -> Tensor:
    """diffusers RMSNorm.forward: fp32 variance, scale, cast to the weight dtype, multiply."""
    in_dtype = x.dtype
    var = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
    x = x * torch.rsqrt(var + eps)
    if weight.dtype in (torch.float16, torch.bfloat16):
        x = x.to(weight.dtype)
    x = x * weight
    return x.to(in_dtype) if weight.dtype == in_dtype else x


def layer_norm_noaffine(x: Tensor, eps: float = 1e-6) -> Tensor:
    return F.layer_norm(x, (x.shape[-1],), None, None, eps)


def timestep_embedding(t: Tensor, dim: int = 256, max_period: int = 10000) -> Tensor:
    """diffusers get_timestep_embedding(flip_sin_to_cos=True, downscale_freq_shift=0, scale=1)."""
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32, device=t.device) / half
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    return torch.cat([emb[:, half:], emb[:, :half]], dim=-1)  # flip: [cos, sin]


def time_text_embed(P, cfg: FluxConfig, timestep: Tensor, guidance: Optional[Tensor], pooled: Tensor) -> Tensor:
    """CombinedTimestep(Guidance)TextProjEmbeddings.forward (reference call flux/transformer.py:1048)."""
    dt = pooled.dtype
    pre = "time_text_embed."

    def mlp(x, name):
        h = F.silu(F.linear(x, P[pre + name + ".linear_1.weight"], P[pre + name + ".linear_1.bias"]))
        return F.linear(h, P[pre + name + ".linear_2.weight"], P[pre + name + ".linear_2.bias"])

    emb = mlp(timestep_embedding(timestep).to(dt), "timestep_embedder")
    if cfg.guidance_embeds:
        emb = emb + mlp(timestep_embedding(guidance).to(dt), "guidance_embedder")
    return emb + mlp(pooled, "text_embedder")


def rope_tables(ids: Tensor, axes_dim=(16, 56, 56), theta: float = 10000.0) -> Tuple[Tensor, Tensor]:
    """FluxPosEmbed.forward -> get_1d_rotary_pos_embed(use_real=True, repeat_interleave_real=True,
    freqs_dtype=float64): cos/sin [S, sum(axes_dim)] float32."""
    pos = ids.float()
    cos_out, sin_out = [], []
    for i, d in enumerate(axes_dim):
        freqs = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.float64)[: d // 2] / d))
        f = torch.outer(pos[:, i].to(torch.float64), freqs)
        cos_out.append(f.cos().repeat_interleave(2, dim=1).float())
        sin_out.append(f.sin().repeat_interleave(2, dim=1).float())
    return torch.cat(cos_out, dim=-1), torch.cat(sin_out, dim=-1)


def apply_rope(x: Tensor, cos: Tensor, sin: Tensor) -> Tensor:
    """reference flux/transformer.py:73-98 (use_real=True, unbind_dim=-1); x [B,H,S,D], cos/sin [S,D]."""
    cos, sin = cos[None, None], sin[None, None]
    xr, xi = x.reshape(*x.shape[:-1], -1, 2).unbind(-1)
    rot = torch.stack([-xi, xr], dim=-1).flatten(3)
    return (x.float() * cos + rot.float() * sin).to(x.dtype)


def sdpa(q: Tensor, k: Tensor, v: Tensor) -> Tensor:
    """F.scaled_dot_product_attention(dropout 0, non-causal, no mask) — explicit math, fp32 softmax."""
    scale = q.shape[-1] ** -0.5
    s = (q.float() @ k.float().transpose(-1, -2)) * scale
    return (torch.softmax(s, dim=-1) @ v.float()).to(q.dtype)


def flux_attention(P, cfg, prefix, x, enc, rope, lora, lora_scale):
    """FluxAttnProcessor2_0.__call__ (reference flux/transformer.py:116-224)."""
    H, hd = cfg.num_attention_heads, cfg.attention_head_dim
    B = x.shape[0]

    def heads(t):
        return t.view(B, -1, H, hd).transpose(1, 2)

    q = heads(linear(x, P, prefix + "to_q", lora, lora_scale))
    k = heads(linear(x, P, prefix + "to_k", lora, lora_scale))
    v = heads(linear(x, P, prefix + "to_v", lora, lora_scale))
    q = rms_norm(q, P[prefix + "norm_q.weight"], 1e-6)
    k = rms_norm(k, P[prefix + "norm_k.weight"], 1e-6)
    if enc is not None:
        eq = heads(linear(enc, P, prefix + "add_q_proj", lora, lora_scale))
        ek = heads(linear(enc, P, prefix + "add_k_proj", lora, lora_scale))
        ev = heads(linear(enc, P, prefix + "add_v_proj", lora, lora_scale))
        eq = rms_norm(eq, P[prefix + "norm_added_q.weight"], 1e-6)
        ek = rms_norm(ek, P[prefix + "norm_added_k.weight"], 1e-6)
        q = torch.cat([eq, q], dim=2)  # Flux order: [text, image]
        k = torch.cat([ek, k], dim=2)
        v = torch.cat([ev, v], dim=2)
    cos, sin = rope
    q = apply_rope(q, cos, sin)
    k = apply_rope(k, cos, sin)
    o = sdpa(q, k, v)
    o = o.transpose(1, 2).reshape(B, -1, H * hd).to(q.dtype)
    if enc is not None:
        n_txt = enc.shape[1]
        eo, o = o[:, :n_txt], o[:, n_txt:]
        o = linear(o, P, prefix + "to_out.0", lora, lora_scale)
        eo = linear(eo, P, prefix + "to_add_out", lora, lora_scale)
        return o, eo
    return o


def nan_to_num_(x: Tensor) -> Tensor:
    return torch.nan_to_num(x, nan=0.0, posinf=65504, neginf=-65504)


def flux_double_block(P, cfg, i, x, enc, temb, rope, lora, lora_scale):
    """FluxTransformerBlock.forward + _ffn_forward (reference flux/transformer.py:563-687)."""
    p = f"transformer_blocks.{i}."
    D = cfg.inner_dim
    mod = F.linear(F.silu(temb), P[p + "norm1.linear.weight"], P[p + "norm1.linear.bias"])
    sh_a, sc_a, g_a, sh_m, sc_m, g_m = mod.chunk(6, dim=1)
    cmod = F.linear(F.silu(temb), P[p + "norm1_context.linear.weight"], P[p + "norm1_context.linear.bias"])
    csh_a, csc_a, cg_a, csh_m, csc_m, cg_m = cmod.chunk(6, dim=1)
    nx = layer_norm_noaffine(x) * (1 + sc_a[:, None]) + sh_a[:, None]
    nenc = layer_norm_noaffine(enc) * (1 + csc_a[:, None]) + csh_a[:, None]
    ao, eo = flux_attention(P, cfg, p + "attn.", nx, nenc, rope, lora, lora_scale)
    x = x + g_a.unsqueeze(1) * ao
    enc = enc + cg_a.unsqueeze(1) * eo
    nx = layer_norm_noaffine(x) * (1 + sc_m[:, None]) + sh_m[:, None]
    ff = linear(F.gelu(linear(nx, P, p + "ff.net.0.proj", lora, lora_scale), approximate="tanh"), P, p + "ff.net.2", lora, lora_scale)
    x = x + g_m.unsqueeze(1) * ff
    nenc = layer_norm_noaffine(enc) * (1 + csc_m[:, None]) + csh_m[:, None]
    cff = linear(F.gelu(linear(nenc, P, p + "ff_context.net.0.proj", lora, lora_scale), approximate="tanh"), P,
                 p + "ff_context.net.2", lora, lora_scale)
    enc = nan_to_num_(enc + cg_m.unsqueeze(1) * cff)
    return enc, x


def flux_single_block(P, cfg, i, x, temb, rope, lora, lora_scale):
    """FluxSingleTransformerBlock.forward + _ffn_forward (reference flux/transformer.py:453-510)."""
    p = f"single_transformer_blocks.{i}."
    mod = F.linear(F.silu(temb), P[p + "norm.linear.weight"], P[p + "norm.linear.bias"])
    sh, sc, gate = mod.chunk(3, dim=1)
    nx = layer_norm_noaffine(x) * (1 + sc[:, None]) + sh[:, None]
    ao = flux_attention(P, cfg, p + "attn.", nx, None, rope, lora, lora_scale)
    mlp = F.gelu(linear(nx, P, p + "proj_mlp", lora, lora_scale), approximate="tanh")
    h = torch.cat([ao, mlp], dim=2)
    h = gate.unsqueeze(1) * linear(h, P, p + "proj_out", lora, lora_scale)
    return nan_to_num_(x + h)


def flux_forward(P: Dict[str, Tensor], cfg: FluxConfig, hidden_states: Tensor, encoder_hidden_states: Tensor,
                 pooled_projections: Tensor, timestep: Tensor, img_ids: Tensor, txt_ids: Tensor,
                 guidance: Optional[Tensor] = None, lora: Optional[Dict[str, Tensor]] = None,
                 lora_scale: float = 1.0) -> Tensor:
    """FluxTransformer2DModel.forward (reference flux/transformer.py:940-1515), default path only
    (no mask / TREAD / controlnet / token-wise timesteps).  timestep and guidance arrive divided by
    1000 and are multiplied back inside (reference :1003-1007, quirk Q8)."""
    x = linear(hidden_states, P, "x_embedder", lora, lora_scale)
    t = timestep.to(torch.float32) * 1000
    g = guidance.to(torch.float32) * 1000 if guidance is not None else None
    temb = time_text_embed(P, cfg, t, g, pooled_projections)
    enc = F.linear(encoder_hidden_states, P["context_embedder.weight"], P["context_embedder.bias"])
    if txt_ids.ndim == 3:
        txt_ids = txt_ids[0]
    if img_ids.ndim == 3:
        img_ids = img_ids[0]
    ids = torch.cat((txt_ids, img_ids), dim=0)
    rope = rope_tables(ids, cfg.axes_dims_rope)
    for i in range(cfg.num_layers):
        enc, x = flux_double_block(P, cfg, i, x, enc, temb, rope, lora, lora_scale)
    h = torch.cat([enc, x], dim=1)
    for i in range(cfg.num_single_layers):
        h = flux_single_block(P, cfg, i, h, temb, rope, lora, lora_scale)
    x = h[:, enc.shape[1]:]
    emb = F.linear(F.silu(temb).to(x.dtype), P["norm_out.linear.weight"], P["norm_out.linear.bias"])
    scale, shift = torch.chunk(emb, 2, dim=1)
    x = layer_norm_noaffine(x) * (1 + scale)[:, None, :] + shift[:, None, :]
    return linear(x, P, "proj_out", lora, lora_scale)


# --------------------------------------------------------------------------------------------------
# Flux wrapper + flow-matching step (restated from reference flux/__init__.py, flux/model.py, common.py)
# --------------------------------------------------------------------------------------------------
def pack_latents(latents, batch_size, num_channels_latents, height, width):
    """reference flux/__init__.py:25-30 (restated; pinned against the source in tests/golden)."""
    latents = latents.view(batch_size, num_channels_latents, height // 2, 2, width // 2, 2)
    latents = latents.permute(0, 2, 4, 1, 3, 5)
    return latents.reshape(batch_size, (height // 2) * (width // 2), num_channels_latents * 4)


def unpack_latents(latents, height, width, vae_scale_factor):
    """reference flux/__init__.py:33-44."""
    batch_size, num_patches, channels = latents.shape
    height = height // vae_scale_factor
    width = width // vae_scale_factor
    latents = latents.view(batch_size, height, width, channels // 4, 2, 2)
    latents = latents.permute(0, 3, 1, 4, 2, 5)
    return latents.reshape(batch_size, channels // 4, height * 2, width * 2)


def prepare_latent_image_ids(height, width):
    """reference flux/__init__.py:47-61 (batch dimension dropped, as the reference returns [0])."""
    ids = torch.zeros(height // 2, width // 2, 3)
    ids[..., 1] = ids[..., 1] + torch.arange(height // 2)[:, None]
    ids[..., 2] = ids[..., 2] + torch.arange(width // 2)[None, :]
    return ids.reshape(-1, 3).to(torch.float32)


def apply_flow_schedule_shift(sigmas: Tensor, shift: float = 3.0) -> Tensor:
    """reference custom_schedule.py:443-477, static-shift branch: s*sigma / (1 + (s-1)*sigma)."""
    return (sigmas * shift) / (1 + (shift - 1) * sigmas)


def sample_flow_sigmas(bsz: int, generator: Optional[torch.Generator] = None, sigmoid_scale: float = 1.0,
                       shift: float = 3.0, device="cpu") -> Tuple[Tensor, Tensor]:
    """reference common.py:5062-5073, 5089-5090 (default branch)."""
    normal = torch.randn((bsz,), device=device, generator=generator)
    sigmas = torch.sigmoid(sigmoid_scale * normal)
    sigmas = apply_flow_schedule_shift(sigmas, shift)
    return sigmas, sigmas * 1000.0


def flow_noisy_latents(latents: Tensor, noise: Tensor, sigmas: Tensor) -> Tensor:
    """reference common.py:4953-4960, 4975-4992: the sigma grid is cast to the latent dtype first."""
    grid = sigmas.reshape(sigmas.shape[0], -1)[:, 0].view(-1, 1, 1, 1).to(dtype=latents.dtype)
    return (1.0 - grid) * latents + grid * noise


def flow_target(latents: Tensor, noise: Tensor) -> Tensor:
    """reference common.py:4610-4611."""
    return noise - latents


def flow_loss(pred: Tensor, target: Tensor) -> Tensor:
    """reference common.py:6286, 6426-6429: fp32 MSE, mean over (C,H,W) then over the batch."""
    loss = F.mse_loss(pred.float(), target.float(), reduction="none")
    return loss.mean(dim=list(range(1, loss.dim()))).mean()


def flux_model_predict(P, cfg, noisy_latents, timesteps, prompt_embeds, pooled, guidance_value=1.0,
                       lora=None, lora_scale=1.0):
    """Flux._model_predict_single, default path (reference flux/model.py:707-864): pack, constant
    guidance, img_ids, timesteps/1000, zero txt_ids, transformer, unpack (height=latent*8 with
    vae_scale_factor=16, reference flux/model.py:856-861)."""
    B, Cc, Hh, Ww = noisy_latents.shape
    packed = pack_latents(noisy_latents, B, Cc, Hh, Ww)
    guidance = torch.full((B,), float(guidance_value), dtype=torch.float32) if cfg.guidance_embeds else None
    img_ids = prepare_latent_image_ids(Hh, Ww)
    txt_ids = torch.zeros(prompt_embeds.shape[1], 3)
    t = timesteps.to(torch.float32) / 1000.0
    out = flux_forward(P, cfg, packed, prompt_embeds, pooled, t, img_ids, txt_ids, guidance, lora, lora_scale)
    return unpack_latents(out, Hh * 8, Ww * 8, 16)


def flux_train_step_loss(P, cfg, batch, lora=None, lora_scale=1.0):
    """prepare (noisy latents) -> model_predict -> loss; `batch` carries latents, noise, sigmas,
    prompt_embeds, pooled (all in the dtype the run should emulate)."""
    noisy = flow_noisy_latents(batch["latents"], batch["noise"], batch["sigmas"])
    timesteps = batch["sigmas"].float() * 1000.0
    pred = flux_model_predict(P, cfg, noisy, timesteps, batch["prompt_embeds"], batch["pooled"],
                              batch.get("guidance", 1.0), lora, lora_scale)
    return flow_loss(pred, flow_target(batch["latents"], batch["noise"])), pred


# --------------------------------------------------------------------------------------------------
# loss family (reference common.py:6132-6215, 6217-6430) — pinned against the reference's own `loss` executed
# verbatim: tests/golden/loss_golden.pt (oracle/make_golden_loss.py), tests/test_loss_golden.py
# --------------------------------------------------------------------------------------------------
def conditional_loss(pred: Tensor, target: Tensor, loss_type: str = "l2", huber_c=0.1) -> Tensor:
    """common.py:6132-6166 with reduction="none"; `huber_c` scalar or [B] (broadcast over the sample)."""
    if loss_type == "l2":
        return F.mse_loss(pred, target, reduction="none")
    c = huber_c if not torch.is_tensor(huber_c) else huber_c.view(-1, *([1] * (pred.dim() - 1)))
    k = 2 * c if loss_type == "huber" else 2.0
    if loss_type not in ("huber", "smooth_l1"):
        raise NotImplementedError(loss_type)
    return k * (torch.sqrt((pred - target) ** 2 + c ** 2) - c)


def scheduled_huber_c(timesteps: Tensor, base: float, schedule: str, prediction_type: str,
                      alphas_cumprod: Optional[Tensor] = None, num_train_timesteps: int = 1000) -> Tensor:
    """common.py:6168-6215."""
    if schedule == "constant":
        return torch.full((timesteps.numel(),), base)
    if schedule == "exponential":
        return torch.exp(-(-math.log(base) / num_train_timesteps) * timesteps).float()
    if schedule == "snr":
        if prediction_type == "flow_matching":
            sig = timesteps / 1000
            sig = ((1.0 - sig) / (sig + 0.0001)) ** 0.5
        else:
            sig = ((1.0 - alphas_cumprod[timesteps]) / alphas_cumprod[timesteps]) ** 0.5
        return ((1 - base) / (1 + sig) ** 2 + base).float()
    raise NotImplementedError(schedule)


def model_loss(pred: Tensor, target: Tensor, loss_type: str = "l2", huber_c=0.1, weights: Optional[Tensor] = None,
               snr_weight: float = 1.0) -> Tensor:
    """common.py:6286 / 6376-6398 / 6426-6429: pointwise loss in fp32, optional per-sample (min-SNR) weights,
    mean over (C, H, W) then over the batch."""
    l = conditional_loss(pred.float(), target.float(), loss_type, huber_c)
    if weights is not None:
        l = l * weights.view(-1, 1, 1, 1)
    elif loss_type == "l2":
        l = snr_weight * l
    return l.mean(dim=list(range(1, l.dim()))).mean()
