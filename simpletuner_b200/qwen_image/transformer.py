"""QwenImageTransformer2DModel on libstb200: the H100 drop-in for reference
simpletuner/helpers/models/qwen_image/transformer.py:1000-1500 (text-to-image flavours v1.0 / v2.0, LoRA training).

A Qwen-Image block is op for op a Flux double block (reference :825-997 against flux/transformer.py:514-687): non-affine
LayerNorm (eps 1e-6) then x (1 + scale) + shift, (shift, scale, gate) x 2 from a Linear(SiLU(temb), 6D) per stream, q/k/v
with bias, per-head RMSNorm, interleaved-pair RoPE, joint attention over [text | image], gated residuals and a tanh-GELU
FeedForward per stream.  So every block runs flux/blocks.DoubleBlockFn through flux/transformer.run_double_block, the
tail is TailFn over the image rows and the loss is FlowLossFn with the Flux (c, dy, dx) packing.  Only the edges are
Qwen's own: `txt_norm` (RMSNorm over the text features) + `txt_in`, `img_in`, a timestep-only embedding, the centred RoPE
positions of QwenEmbedRope(scale_rope=True), and the prompt mask, which becomes a -inf per-key logit bias.

Memory layout of the frozen weights (20.4 B parameters, 40.8 GB in bf16 for Qwen-Image): each stream's q, k and v
parameters are row views of one [3D, D] tensor owned by the attention module, so the fused q|k|v projection reads the
parameters themselves, and every dgrad GEMM reads its weight in place as an MN-major operand (ops.WT).  No transposed or
concatenated copy of any frozen weight exists; a copy would add 34 GB and the model would not train on an 80 GB card.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Any, Dict, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..flux.blocks import AttnPlan, MlpPlan, TailFn
from ..flux.transformer import (AdapterModelAPI, AttnProcessorAPI, Linear, LoraDropoutAPI, RMSNormWeight, _AdaNorm,
                                _FeedForward, _TimestepEmbedding, run_double_block)

_ATTN = ["to_q", "to_k", "to_v", "to_out.0", "add_q_proj", "add_k_proj", "add_v_proj", "to_add_out"]
_MLP = ["img_mlp.net.0.proj", "img_mlp.net.2", "txt_mlp.net.0.proj", "txt_mlp.net.2"]
QWEN_DEFAULT_LORA_TARGETS = ["to_k", "to_q", "to_v", "to_out.0"]      # reference qwen_image/model.py:111
_ADAPTABLE_SUFFIXES = tuple("." + t for t in (_ATTN + _MLP))


class QwenAttention(nn.Module):
    """Parameter container of diffusers Attention as the reference configures it (:841-853): to_q/k/v, add_q/k/v_proj,
    to_out.0, to_add_out (all with bias), norm_q / norm_k / norm_added_q / norm_added_k (RMSNorm over head_dim).

    The q, k, v weights (and biases) of each stream are row views of one [3D, D] ([3D]) tensor, `fused["img"]` /
    `fused["txt"]`.  load_state_dict copies into the views.  Whatever splits the storage (`_apply`: .to / .cuda / .half
    move parameters one by one; load_state_dict(assign=True) or accelerate replace them) is caught by `fused_qkv()`, which
    every forward reads: it re-fuses from the current parameters, keeping every Parameter object."""

    def __init__(self, dim, heads, head_dim, dtype):
        super().__init__()
        self.heads, self.head_dim = heads, head_dim
        for n in ("to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj"):
            setattr(self, n, Linear(dim, dim, dtype=dtype))
        self.to_out = nn.ModuleList([Linear(dim, dim, dtype=dtype), nn.Identity()])
        self.to_add_out = Linear(dim, dim, dtype=dtype)
        for n in ("norm_q", "norm_k", "norm_added_q", "norm_added_k"):
            setattr(self, n, RMSNormWeight(head_dim, dtype))
        self.__dict__["fused"] = {}
        self._fuse()

    def streams(self):
        return {"img": (self.to_q, self.to_k, self.to_v), "txt": (self.add_q_proj, self.add_k_proj, self.add_v_proj)}

    def _fuse(self):
        for name, lins in self.streams().items():
            w0 = lins[0].weight
            n = w0.shape[0]
            w = torch.empty((3 * n, w0.shape[1]), device=w0.device, dtype=w0.dtype)
            b = torch.empty((3 * n,), device=w0.device, dtype=w0.dtype)
            for m, lin in enumerate(lins):
                w[m * n:(m + 1) * n].copy_(lin.weight.data)
                b[m * n:(m + 1) * n].copy_(lin.bias.data)
                lin.weight.data = w[m * n:(m + 1) * n]
                lin.bias.data = b[m * n:(m + 1) * n]
            self.fused[name] = (w, b)

    def _is_fused(self) -> bool:
        for name, lins in self.streams().items():
            w, b = self.fused[name]
            n, k = lins[0].weight.shape
            for m, lin in enumerate(lins):
                lw, lb = lin.weight, lin.bias
                if (lw.device != w.device or lw.dtype != w.dtype or tuple(lw.shape) != (n, k) or lw.stride() != (k, 1)
                        or lw.data_ptr() != w.data_ptr() + m * n * k * w.element_size()
                        or lb.device != b.device or lb.dtype != b.dtype or lb.data_ptr() != b.data_ptr() + m * n * b.element_size()):
                    return False
        return True

    def fused_qkv(self):
        """{"img" | "txt": (w [3D, D], b [3D])} backing the current q / k / v parameters (re-fused if they were split)."""
        if not self._is_fused():
            self._fuse()
        return self.fused

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self.fused_qkv()
        return out


class QwenImageTransformerBlock(nn.Module):
    """reference qwen_image/transformer.py:825-997"""

    def __init__(self, dim, heads, head_dim, dtype):
        super().__init__()
        self.dim, self.heads, self.head_dim = dim, heads, head_dim
        self.img_mod = nn.ModuleList([nn.Identity(), Linear(dim, 6 * dim, dtype=dtype)])     # Sequential(SiLU, Linear)
        self.attn = QwenAttention(dim, heads, head_dim, dtype)
        self.img_mlp = _FeedForward(dim, dtype)
        self.txt_mod = nn.ModuleList([nn.Identity(), Linear(dim, 6 * dim, dtype=dtype)])
        self.txt_mlp = _FeedForward(dim, dtype)

    def plans(self):
        """Every operand is a parameter read in place: w_qkv IS the fused [3D, D] tensor and each dgrad operand is ops.WT
        of its forward weight, so building the plans allocates no weight-sized tensor.  They are built per forward (a few
        views), so they always describe the current parameters."""
        a = self.attn
        pl = {}
        fused = a.fused_qkv()
        for name, out in (("img", a.to_out[0]), ("txt", a.to_add_out)):
            w, b = fused[name]
            nq, nk = (a.norm_q, a.norm_k) if name == "img" else (a.norm_added_q, a.norm_added_k)
            wo = out.weight.detach()
            pl[name + "_attn"] = AttnPlan(w.detach(), b.detach(), ops.WT(w.detach()), w_out=wo, b_out=out.bias.detach(),
                                          w_out_t=ops.WT(wo), norm_q=nq.weight.detach(), norm_k=nk.weight.detach())
        for name, ff in (("img", self.img_mlp), ("txt", self.txt_mlp)):
            w1, w2 = ff.net[0].proj.weight.detach(), ff.net[2].weight.detach()
            pl[name + "_mlp"] = MlpPlan(w1, ff.net[0].proj.bias.detach(), ops.WT(w1), w2, ff.net[2].bias.detach(), ops.WT(w2))
        return pl

    def forward(self, h, silu_temb, cos, sin, S_txt, lora_scaling, key_bias=None):
        mod_img = self.img_mod[1](silu_temb)
        mod_txt = self.txt_mod[1](silu_temb)
        a = self.attn
        attn_l = [a.to_q, a.to_k, a.to_v, a.to_out[0], a.add_q_proj, a.add_k_proj, a.add_v_proj, a.to_add_out]
        mlp_l = [self.img_mlp.net[0].proj, self.img_mlp.net[2], self.txt_mlp.net[0].proj, self.txt_mlp.net[2]]
        # the reference clips only fp16 activations (:991-995); bf16 text rows pass through unchanged
        return run_double_block(self, h, mod_img, mod_txt, cos, sin, S_txt, lora_scaling, key_bias, None, attn_l, mlp_l,
                                nan_to_num_txt=False)


class _TimeEmbed(nn.Module):
    """QwenTimestepProjEmbeddings (reference :397-528) without TwinFlow / FlowMap: only `timestep_embedder`."""

    def __init__(self, dim, dtype):
        super().__init__()
        self.timestep_embedder = _TimestepEmbedding(256, dim, dtype)


def qwen_timestep_proj(t: torch.Tensor, dim: int = 256, max_period: int = 10000) -> torch.Tensor:
    """The reference's `time_proj` input chain (:1295, :401, :493): t rounded to bf16, then diffusers
    get_timestep_embedding(flip_sin_to_cos=True, downscale_freq_shift=0, scale=1000), which scales AFTER t * freq."""
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32, device=t.device) / half
    emb = t.to(torch.bfloat16)[:, None].float() * torch.exp(exponent)[None, :]
    emb = 1000 * emb
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


def _rope_freqs(index: torch.Tensor, dim: int, theta: float) -> torch.Tensor:
    """QwenEmbedRope.rope_params (:559-567): fp32 frequencies, complex via torch.polar."""
    freqs = torch.outer(index, 1.0 / torch.pow(theta, torch.arange(0, dim, 2).to(torch.float32).div(dim)))
    return torch.polar(torch.ones_like(freqs), freqs)


def qwen_rope_tables(h: int, w: int, S_txt: int, axes_dim=(16, 56, 56), theta: float = 10000.0):
    """cos, sin fp32 [S_txt + h w, sum(axes_dim)] in joint [text | image] order: QwenEmbedRope(scale_rope=True).forward for
    one frame + precompute_real_rope_qwen (:351-368, :569-644).  Image rows: frame index 0, row / column indices
    [-(n - n//2), n//2 - 1] (centred); text rows: max(h//2, w//2) + i on all three axes."""
    f0, fh, fw = axes_dim
    frame = _rope_freqs(torch.zeros(1, dtype=torch.long), f0, theta).expand(h, w, -1)
    rows = _rope_freqs(torch.arange(-(h - h // 2), h // 2), fh, theta)[:, None, :].expand(h, w, -1)
    cols = _rope_freqs(torch.arange(-(w - w // 2), w // 2), fw, theta)[None, :, :].expand(h, w, -1)
    img = torch.cat([frame, rows, cols], dim=-1).reshape(h * w, -1)
    pos = torch.arange(max(h // 2, w // 2), max(h // 2, w // 2) + S_txt)
    txt = torch.cat([_rope_freqs(pos, d, theta) for d in axes_dim], dim=1)
    f = torch.cat([txt, img], dim=0)
    return f.real.repeat_interleave(2, dim=-1).contiguous(), f.imag.repeat_interleave(2, dim=-1).contiguous()


def qwen_key_bias(mask: torch.Tensor, S_img: int, dtype=torch.bfloat16) -> torch.Tensor:
    """[B, S_txt + S_img] per-key logit bias of the reference's prompt mask (:721-821, :1353-1366), device ops only.
    The mask is read as bool (compute_text_seq_len_from_mask, :387-388).  B == 1: text key j is kept where mask[0, j] is
    set, whatever the pattern (joint SDPA with the bool mask).  B > 1: text key j is kept when j < max(sum(mask[b]), 1)
    (the reference slices each sample's first `sum` tokens, so a non-prefix mask acts as that prefix).  Kept keys and every
    image key get 0, the others -inf."""
    B, L = mask.shape
    m = mask != 0
    if B > 1:
        n = m.sum(dim=1, keepdim=True).clamp_min(1)
        m = torch.arange(L, device=mask.device)[None, :] < n
    bias = torch.zeros((B, L + S_img), device=mask.device, dtype=dtype)
    bias[:, :L].masked_fill_(~m, float("-inf"))
    return bias


def mask_hides_keys(mask: torch.Tensor) -> bool:
    """Host-side: whether `qwen_key_bias(mask)` has any -inf key (so the biased attention kernels are needed)."""
    m = mask.reshape(mask.shape[0], -1) != 0
    if m.shape[0] == 1:
        return not bool(m.all())
    return bool((m.sum(dim=1) < m.shape[1]).any())


class QwenImageTransformer2DModel(AdapterModelAPI, AttnProcessorAPI, LoraDropoutAPI, nn.Module):
    _no_split_modules = ["QwenImageTransformerBlock"]
    _supports_gradient_checkpointing = True
    _DEFAULT_LORA_TARGETS = QWEN_DEFAULT_LORA_TARGETS

    def __init__(self, patch_size: int = 2, in_channels: int = 64, out_channels: Optional[int] = 16, num_layers: int = 60,
                 attention_head_dim: int = 128, num_attention_heads: int = 24, joint_attention_dim: int = 3584,
                 guidance_embeds: bool = False, axes_dims_rope: Tuple[int, ...] = (16, 56, 56), dtype=torch.bfloat16,
                 **unused):
        super().__init__()
        if attention_head_dim not in (64, 128):
            raise NotImplementedError("libstb200 attention supports head_dim 64 / 128")
        if guidance_embeds:
            raise NotImplementedError("Qwen-Image with guidance_embeds is not supported by the libstb200 path")
        if patch_size != 2 or in_channels != 64 or (out_channels or in_channels) != 16:
            raise NotImplementedError("libstb200 Qwen-Image packs 16-channel latents in 2x2 patches (in_channels 64)")
        for k in ("musubi_blocks_to_swap", "enable_time_sign_embed", "deltatime_type"):
            if unused.get(k):
                raise NotImplementedError(f"Qwen-Image with {k}={unused[k]!r} is not supported by the libstb200 path")
        self.config = SimpleNamespace(patch_size=patch_size, in_channels=in_channels, out_channels=out_channels,
                                      num_layers=num_layers, attention_head_dim=attention_head_dim,
                                      num_attention_heads=num_attention_heads, joint_attention_dim=joint_attention_dim,
                                      guidance_embeds=guidance_embeds, axes_dims_rope=tuple(axes_dims_rope))
        self.out_channels = out_channels or in_channels
        self.inner_dim = D = num_attention_heads * attention_head_dim
        self.time_text_embed = _TimeEmbed(D, dtype)
        self.txt_norm = RMSNormWeight(joint_attention_dim, dtype)
        self.img_in = Linear(in_channels, D, dtype=dtype)
        self.txt_in = Linear(joint_attention_dim, D, dtype=dtype)
        self.transformer_blocks = nn.ModuleList(
            [QwenImageTransformerBlock(D, num_attention_heads, attention_head_dim, dtype) for _ in range(num_layers)])
        self.norm_out = _AdaNorm(D, 2, dtype)
        self.proj_out = Linear(D, patch_size * patch_size * self.out_channels, dtype=dtype)
        self.gradient_checkpointing = False
        self._rope_cache: Dict[Any, Tuple[torch.Tensor, torch.Tensor]] = {}
        self._lora_scaling = 1.0
        self.peft_config: Dict[str, Any] = {}

    @staticmethod
    def _lora_adaptable(name: str) -> bool:
        return name.endswith(_ADAPTABLE_SUFFIXES)

    def invalidate_plans(self):
        """The plans are built per forward; what is kept is the RoPE tables and the fused q|k|v storage, which
        load_state_dict(assign=True) splits by replacing the q / k / v parameters."""
        self._rope_cache.clear()
        for blk in self.transformer_blocks:
            blk.attn.fused_qkv()

    def _rope(self, h: int, w: int, S_txt: int, device):
        key = (h, w, S_txt, str(device))
        hit = self._rope_cache.get(key)
        if hit is None:
            cos, sin = qwen_rope_tables(h, w, S_txt, self.config.axes_dims_rope)
            if len(self._rope_cache) > 64:
                self._rope_cache.clear()
            hit = self._rope_cache[key] = (cos.to(device), sin.to(device))
        return hit

    def forward(self, hidden_states: torch.Tensor, encoder_hidden_states: torch.Tensor = None,
                encoder_hidden_states_mask: Optional[torch.Tensor] = None, timestep: torch.Tensor = None,
                img_shapes: Optional[Sequence] = None, txt_seq_lens=None, guidance=None, attention_kwargs=None,
                return_dict: bool = True, timestep_sign=None, r_timestep=None, controlnet_block_samples=None,
                force_keep_mask=None, hidden_states_buffer=None, modulate_index=None):
        """hidden_states [B, h w, 64] packed latents, encoder_hidden_states [B, S_txt, joint_attention_dim], the prompt
        mask [B, S_txt] (or None: every key kept), timestep [B] in [0, 1], img_shapes [(1, h, w)] * B.  Returns
        (Tensor[B, h w, 64],).  txt_seq_lens is ignored, as by the reference: RoPE spans the padded text length."""
        for nm, v in (("guidance", guidance), ("timestep_sign", timestep_sign), ("r_timestep", r_timestep),
                      ("controlnet_block_samples", controlnet_block_samples), ("force_keep_mask", force_keep_mask),
                      ("hidden_states_buffer", hidden_states_buffer), ("modulate_index", modulate_index)):
            if v is not None:
                raise NotImplementedError(f"libstb200 Qwen-Image path does not support `{nm}`; use the reference module")
        if attention_kwargs and set(attention_kwargs) - {"scale"}:
            raise NotImplementedError(f"attention_kwargs {sorted(attention_kwargs)} are not supported by the libstb200 path")
        # attention_kwargs["scale"] multiplies every adapter's scaling for this call (reference :1255-1263, scale_lora_layers)
        lora_scale = float((attention_kwargs or {}).get("scale", 1.0))
        if timestep.ndim != 1:
            raise NotImplementedError("token-wise timesteps are not supported by the libstb200 Qwen-Image path")
        if hidden_states.ndim != 3:
            raise NotImplementedError("libstb200 Qwen-Image takes packed latent tokens [B, S_img, 64]")
        if not hidden_states.is_cuda:
            from .._lib import StbError
            raise StbError("QwenImageTransformer2DModel (libstb200) needs CUDA tensors; there is no CPU fallback")
        B, S_img, _ = hidden_states.shape
        shp = img_shapes[0] if img_shapes else None
        if isinstance(shp, list):
            shp = shp[0]
        if shp is None or len(shp) != 3 or shp[0] != 1 or shp[1] * shp[2] != S_img:
            raise ValueError(f"img_shapes must describe one frame of {S_img} tokens, got {img_shapes!r}")
        gh, gw = int(shp[1]), int(shp[2])
        dt = self.img_in.weight.dtype
        dev = hidden_states.device
        S_txt = encoder_hidden_states.shape[1]
        D = self.inner_dim
        h = torch.empty((B, S_txt + S_img, D), device=dev, dtype=dt)       # joint buffer [text | image]
        self._begin_lora_dropout(list(self.transformer_blocks))
        ops.gemm([hidden_states.to(dt).contiguous()], [self.img_in.weight], self.img_in.bias, out=h[:, S_txt:])
        # txt_norm (diffusers RMSNorm, bf16 weight = T5LayerNorm) then txt_in; nothing upstream trains
        ntxt = ops.rmsnorm_fwd(encoder_hidden_states.to(dt).contiguous(), self.txt_norm.weight, 1e-6)
        ops.gemm([ntxt], [self.txt_in.weight], self.txt_in.bias, out=h[:, :S_txt])
        del ntxt
        temb = self.time_text_embed.timestep_embedder(qwen_timestep_proj(timestep.to(dev)).to(dt))
        silu_temb = F.silu(temb).contiguous()
        cos, sin = self._rope(gh, gw, S_txt, dev)
        key_bias = None
        if encoder_hidden_states_mask is not None:
            mask = encoder_hidden_states_mask
            if mask.dim() == 3 and mask.shape[1] == 1:
                mask = mask.squeeze(1)
            if tuple(mask.shape) != (B, S_txt):
                raise ValueError(f"encoder_hidden_states_mask must be [{B}, {S_txt}], got {tuple(mask.shape)}")
            # one bias for every block, passed as an argument so that checkpoint re-runs see it
            key_bias = qwen_key_bias(mask.to(dev, non_blocking=True), S_img, dt)
        scaling = self._lora_scaling * lora_scale
        for i, blk in enumerate(self.transformer_blocks):
            h = self._run_block(i, blk, h, silu_temb, cos, sin, S_txt, scaling, key_bias)
        w = self.proj_out.weight.detach()
        tail = {"w_proj": w, "b_proj": self.proj_out.bias.detach(), "w_proj_t": ops.WT(w)}
        mod = self.norm_out.linear(silu_temb)          # AdaLayerNormContinuous: (scale | shift)
        out = TailFn.apply(h, mod, {"S_txt": S_txt, "lora_scaling": scaling, "lora_drop": None, **tail})
        if not return_dict:
            return (out,)
        return SimpleNamespace(sample=out)
