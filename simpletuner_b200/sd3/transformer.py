"""SD3Transformer2DModel on libstb200 — B200-native drop-in for reference
simpletuner/helpers/models/sd3/transformer.py:244-909 (class SD3Transformer2DModel), LoRA-training path.

Same constructor arguments / `.config`, forward kwargs (`hidden_states [B,C,H,W]`, `encoder_hidden_states`,
`pooled_projections`, `timestep`, `return_dict=False`) and `(Tensor[B,C_out,H,W],)` return as the reference;
diffusers / PEFT parameter names (`transformer_blocks.N.attn.to_q.weight`, `…attn2.to_out.0.lora_A.default.weight`,
`pos_embed.proj.weight`, the persistent `pos_embed.pos_embed` buffer …).

The joint blocks run on the shared `DoubleBlockFn` schedule (flux/blocks.py): SD3 has no RoPE, so the joint
attention is order-invariant and the [text | image] joint buffer of the Flux path is reused unchanged; SD3.5's
image-only `attn2` (dual_attention_layers) and the `context_pre_only` last block are flags of that schedule.
The 2x2 stride-2 PatchEmbed conv is a K=64 GEMM on the patchified latents (same (c, dy, dx) feature order as
Flux `pack_latents`) with the cropped positional table added in the epilogue.
Unsupported: TREAD routing, controlnet residuals, token-wise timesteps, flow-map / TwinFlow inputs, full
— they raise so a shim can keep the reference module.  Full fine-tune (model_type=full, BASELINE configs[2]), after
`enable_full_finetune()`, runs the same `DoubleBlockFn` / `TailFn` schedules with every Linear's (weight, bias) in the
adapter slots (`JointTransformerBlock.block_slots`); only the patch / context embedding has a Function of its own.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Dict, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..flux.blocks import DoubleBlockFn, TailFn, _wt
from ..flux.transformer import (_ATTN, AdapterModelAPI, AttnProcessorAPI, LoraDropoutAPI, Linear, RMSNormWeight, _AdaNorm,
                                _FeedForward, _TimestepEmbedding, _attn_plan, _mlp_plan, _sinusoid)
from ..pretrained import ModelConfig, PretrainedIOAPI

SD3_LORA_TARGETS = ["to_k", "to_q", "to_v", "to_out.0"]  # SD3.DEFAULT_LORA_TARGET, reference sd3/model.py:122
_ADAPTABLE_SUFFIXES = tuple("." + t for t in _ATTN)


class _JointAttention(nn.Module):
    def __init__(self, dim, heads, head_dim, joint: bool, pre_only: bool, qk_norm: bool, dtype):
        super().__init__()
        self.to_q = Linear(dim, dim, dtype=dtype)
        self.to_k = Linear(dim, dim, dtype=dtype)
        self.to_v = Linear(dim, dim, dtype=dtype)
        self.to_out = nn.ModuleList([Linear(dim, dim, dtype=dtype), nn.Identity()])
        if qk_norm:
            self.norm_q = RMSNormWeight(head_dim, dtype)
            self.norm_k = RMSNormWeight(head_dim, dtype)
        if joint:
            self.add_q_proj = Linear(dim, dim, dtype=dtype)
            self.add_k_proj = Linear(dim, dim, dtype=dtype)
            self.add_v_proj = Linear(dim, dim, dtype=dtype)
            if not pre_only:
                self.to_add_out = Linear(dim, dim, dtype=dtype)
            if qk_norm:
                self.norm_added_q = RMSNormWeight(head_dim, dtype)
                self.norm_added_k = RMSNormWeight(head_dim, dtype)


class JointTransformerBlock(nn.Module):
    """diffusers JointTransformerBlock as configured at reference sd3/transformer.py:360-367."""

    def __init__(self, dim, heads, head_dim, context_pre_only: bool, qk_norm: Optional[str], use_dual_attention: bool, dtype):
        super().__init__()
        self.dim, self.heads, self.head_dim = dim, heads, head_dim
        self.context_pre_only, self.use_dual_attention, self.qk_norm = context_pre_only, use_dual_attention, bool(qk_norm)
        self.norm1 = _AdaNorm(dim, 9 if use_dual_attention else 6, dtype)
        self.norm1_context = _AdaNorm(dim, 2 if context_pre_only else 6, dtype)
        self.attn = _JointAttention(dim, heads, head_dim, True, context_pre_only, bool(qk_norm), dtype)
        if use_dual_attention:
            self.attn2 = _JointAttention(dim, heads, head_dim, False, False, bool(qk_norm), dtype)
        self.ff = _FeedForward(dim, dtype)
        if not context_pre_only:
            self.ff_context = _FeedForward(dim, dtype)
        self._plans = None

    def plans(self):
        if self._plans is None:
            a = self.attn
            g = lambda m, n: getattr(m, n, None)
            dyn = bool(getattr(self, "_full_ft", False))      # full fine-tune: the weights change every step
            pl = {
                "img_attn": _attn_plan(a.to_q, a.to_k, a.to_v, a.to_out[0], g(a, "norm_q"), g(a, "norm_k"), dyn),
                "txt_attn": _attn_plan(a.add_q_proj, a.add_k_proj, a.add_v_proj, g(a, "to_add_out"), g(a, "norm_added_q"),
                                       g(a, "norm_added_k"), dyn),
                "img_mlp": _mlp_plan(self.ff.net[0].proj, self.ff.net[2], dyn),
            }
            if not self.context_pre_only:
                pl["txt_mlp"] = _mlp_plan(self.ff_context.net[0].proj, self.ff_context.net[2], dyn)
            if self.use_dual_attention:
                b = self.attn2
                pl["img_attn2"] = _attn_plan(b.to_q, b.to_k, b.to_v, b.to_out[0], g(b, "norm_q"), g(b, "norm_k"), dyn)
            self._plans = pl
        return self._plans

    def block_slots(self):
        """DoubleBlockFn's flat slot list.  LoRA: the (A, B) of the adapted attention projections.  Full fine-tune: every
        Linear's (weight, bias) in the same slots, the FeedForwards' too, then the q / k RMSNorm weights; the adaLN linears
        (`norm1*`) train through torch autograd on the modulation vectors instead."""
        a, b = self.attn, getattr(self, "attn2", None)
        g = lambda m, n: getattr(m, n, None)
        lins = [a.to_q, a.to_k, a.to_v, a.to_out[0], a.add_q_proj, a.add_k_proj, a.add_v_proj, g(a, "to_add_out")]
        lins += [b.to_q, b.to_k, b.to_v, b.to_out[0]] if b is not None else [None] * 4
        if not getattr(self, "_full_ft", False):
            return [t for lin in lins for t in (lin.lora_tensors() if lin is not None else (None, None))]
        ffc = g(self, "ff_context")
        lins += [self.ff.net[0].proj, self.ff.net[2], ffc.net[0].proj if ffc else None, ffc.net[2] if ffc else None]
        norms = [g(a, "norm_q"), g(a, "norm_k"), g(a, "norm_added_q"), g(a, "norm_added_k"), g(b, "norm_q"), g(b, "norm_k")]
        return [t for lin in lins for t in ((lin.weight, lin.bias) if lin is not None else (None, None))] + \
            [n.weight if n is not None else None for n in norms]

    def forward(self, h, silu_temb, S_txt, lora_scaling):
        mod_img = self.norm1.linear(silu_temb)
        mod_txt = self.norm1_context.linear(silu_temb)
        st = {"S_txt": S_txt, "H": self.heads, "hd": self.head_dim, "plans": self.plans(), "lora_scaling": lora_scaling,
              "nan_to_num_txt": False, "context_pre_only": self.context_pre_only, "dual": self.use_dual_attention,
              "lora_drop": getattr(self, "_lora_drop", None), "full": bool(getattr(self, "_full_ft", False))}
        return DoubleBlockFn.apply(h, mod_img, mod_txt, None, None, st, *self.block_slots())


class EmbedFullFn(torch.autograd.Function):
    """Joint hidden buffer [text | image] from the patchified latents and the text states, with weight gradients:
    h[:, S_txt:] = patches W_pe^T + b_pe + pos;  h[:, :S_txt] = enc W_ctx^T + b_ctx  (reference sd3/transformer.py:600-640)."""

    @staticmethod
    def forward(ctx, patches, enc, pos, w_pe, b_pe, w_ctx, b_ctx):
        B, S_img, _ = patches.shape
        S_txt = enc.shape[1]
        D = w_pe.shape[0]
        h = torch.empty((B, S_txt + S_img, D), device=patches.device, dtype=torch.bfloat16)
        ops.gemm([patches], [w_pe.detach().reshape(D, -1)], b_pe.detach(), out=h[:, S_txt:], epi=ops.EPI_ADD_RES, res=pos)
        ops.gemm([enc], [w_ctx.detach()], b_ctx.detach(), out=h[:, :S_txt])
        ctx.save_for_backward(patches, enc)
        ctx.S_txt, ctx.w_pe_shape = S_txt, tuple(w_pe.shape)
        return h

    @staticmethod
    def backward(ctx, dh):
        patches, enc = ctx.saved_tensors
        S_txt = ctx.S_txt
        dh = dh.contiguous()
        d_img, d_txt = dh[:, S_txt:], dh[:, :S_txt]
        dw_pe = ops.wgrad_full(d_img, patches).reshape(ctx.w_pe_shape)
        db_pe = ops.colsum2(d_img)[0].sum(0).to(torch.bfloat16)
        dw_ctx = ops.wgrad_full(d_txt, enc)
        db_ctx = ops.colsum2(d_txt)[0].sum(0).to(torch.bfloat16)
        return None, None, None, dw_pe, db_pe, dw_ctx, db_ctx


class _PatchEmbed(nn.Module):
    """diffusers PatchEmbed(patch_size=2, pos_embed_max_size=...): conv `proj` + persistent sincos `pos_embed` buffer."""

    def __init__(self, in_channels, dim, patch_size, max_size, dtype):
        super().__init__()
        self.patch_size, self.max_size = patch_size, max_size
        self.proj = nn.Conv2d(in_channels, dim, kernel_size=patch_size, stride=patch_size, bias=True, dtype=dtype)
        for p in self.proj.parameters():
            p.requires_grad_(False)
        self.register_buffer("pos_embed", torch.zeros(1, max_size * max_size, dim, dtype=torch.float32), persistent=True)


class _TimeTextEmbed(nn.Module):
    def __init__(self, dim, pooled_dim, dtype):
        super().__init__()
        self.timestep_embedder = _TimestepEmbedding(256, dim, dtype)
        self.text_embedder = _TimestepEmbedding(pooled_dim, dim, dtype)


class SD3Transformer2DModel(AdapterModelAPI, AttnProcessorAPI, LoraDropoutAPI, PretrainedIOAPI, nn.Module):
    _no_split_modules = ["JointTransformerBlock"]
    _DEFAULT_LORA_TARGETS = SD3_LORA_TARGETS

    def __init__(self, sample_size: int = 128, patch_size: int = 2, in_channels: int = 16, num_layers: int = 18,
                 attention_head_dim: int = 64, num_attention_heads: int = 18, joint_attention_dim: int = 4096,
                 caption_projection_dim: int = 1152, pooled_projection_dim: int = 2048, out_channels: int = 16,
                 pos_embed_max_size: int = 96, dual_attention_layers: Tuple[int, ...] = (), qk_norm: Optional[str] = None,
                 dtype=torch.bfloat16, **unused):
        super().__init__()
        if patch_size != 2:
            raise NotImplementedError("libstb200 SD3 path supports patch_size=2")
        if attention_head_dim not in (64, 128):
            raise NotImplementedError("libstb200 attention supports head_dim 64 / 128")
        self.config = ModelConfig(sample_size=sample_size, patch_size=patch_size, in_channels=in_channels,
                                  num_layers=num_layers, attention_head_dim=attention_head_dim,
                                  num_attention_heads=num_attention_heads, joint_attention_dim=joint_attention_dim,
                                  caption_projection_dim=caption_projection_dim, pooled_projection_dim=pooled_projection_dim,
                                  out_channels=out_channels, pos_embed_max_size=pos_embed_max_size,
                                  dual_attention_layers=tuple(dual_attention_layers), qk_norm=qk_norm)
        self.out_channels = out_channels if out_channels is not None else in_channels
        self.inner_dim = D = num_attention_heads * attention_head_dim
        if caption_projection_dim != D:
            raise ValueError("caption_projection_dim must equal the inner dim (as in every released SD3 checkpoint)")
        self.pos_embed = _PatchEmbed(in_channels, D, patch_size, pos_embed_max_size, dtype)
        self.time_text_embed = _TimeTextEmbed(D, pooled_projection_dim, dtype)
        self.context_embedder = Linear(joint_attention_dim, caption_projection_dim, dtype=dtype)
        self.transformer_blocks = nn.ModuleList([
            JointTransformerBlock(D, num_attention_heads, attention_head_dim, i == num_layers - 1, qk_norm,
                                  i in self.config.dual_attention_layers, dtype) for i in range(num_layers)])
        self.norm_out = _AdaNorm(D, 2, dtype)
        self.proj_out = Linear(D, patch_size * patch_size * self.out_channels, dtype=dtype)
        self._lora_scaling = 1.0
        self._tail_plan = None
        self._pos_cache: Dict[Any, torch.Tensor] = {}
        self.peft_config: Dict[str, Any] = {}
        self.gradient_checkpointing = False

    # ---- reference-facing utilities -------------------------------------------------------------
    @staticmethod
    def _lora_adaptable(name: str) -> bool:
        # the attention projections of `attn` / `attn2`; the FeedForward and adaLN linears are not in the LoRA schedule
        return (".attn." in name or ".attn2." in name) and name.endswith(_ADAPTABLE_SUFFIXES)

    def invalidate_plans(self):
        for blk in self.transformer_blocks:
            blk._plans = None
        self._tail_plan = None
        self._pos_cache.clear()

    def enable_full_finetune(self, enabled: bool = True):
        """model_type=full (BASELINE configs[2]): every parameter trains.  The joint blocks run DoubleBlockFn in its full
        fine-tune mode; fused / transposed weight layouts are rebuilt after every optimizer step
        (`after_optimizer_step`, called by TrainStep) because the base weights now change."""
        if enabled and self.lora_linears():
            raise NotImplementedError("full fine-tune and LoRA adapters are mutually exclusive on the libstb200 path")
        self._full_ft = bool(enabled)
        for p in self.parameters():
            p.requires_grad_(bool(enabled))
        for blk in self.transformer_blocks:
            blk._full_ft = bool(enabled)
        self.invalidate_plans()
        return self

    def after_optimizer_step(self):
        if getattr(self, "_full_ft", False):
            self.invalidate_plans()

    def before_graph_capture(self):
        """training.step.GraphedTrainStep: in full fine-tune the fused / transposed layouts are rebuilt INSIDE the captured
        step (they depend on weights the optimizer changes between replays)."""
        if getattr(self, "_full_ft", False):
            self.invalidate_plans()

    # ---- forward --------------------------------------------------------------------------------
    def _cropped_pos(self, h: int, w: int, dtype) -> torch.Tensor:
        """diffusers PatchEmbed.cropped_pos_embed: centre crop of the [max, max] table to the (h, w) patch grid."""
        key = (h, w, dtype)
        hit = self._pos_cache.get(key)
        if hit is None:
            mx = self.pos_embed.max_size
            if h > mx or w > mx:
                raise ValueError(f"patch grid {h}x{w} exceeds pos_embed_max_size {mx}")
            top, left = (mx - h) // 2, (mx - w) // 2
            pe = self.pos_embed.pos_embed.reshape(1, mx, mx, -1)[:, top:top + h, left:left + w, :]
            hit = pe.reshape(1, h * w, -1).to(dtype).contiguous()
            self._pos_cache[key] = hit
        return hit

    def forward(self, hidden_states: torch.Tensor, encoder_hidden_states: torch.Tensor = None,
                pooled_projections: torch.Tensor = None, timestep: torch.Tensor = None, timestep_sign=None, r_timestep=None,
                block_controlnet_hidden_states=None, joint_attention_kwargs: Optional[Dict[str, Any]] = None,
                return_dict: bool = True, skip_layers=None, force_keep_mask=None, hidden_states_buffer=None,
                grounding_kwargs=None, _packed_latents: Optional[torch.Tensor] = None, _packed_output: bool = False):
        for nm, v in (("timestep_sign", timestep_sign), ("r_timestep", r_timestep), ("skip_layers", skip_layers),
                      ("block_controlnet_hidden_states", block_controlnet_hidden_states),
                      ("force_keep_mask", force_keep_mask), ("grounding_kwargs", grounding_kwargs)):
            if v is not None:
                raise NotImplementedError(f"libstb200 SD3 path does not support `{nm}`; use the reference module")
        if timestep.ndim != 1:
            raise NotImplementedError("token-wise timesteps are not supported by the libstb200 SD3 path")
        if not hidden_states.is_cuda:
            from .._lib import StbError
            raise StbError("SD3Transformer2DModel (libstb200) needs CUDA tensors; there is no CPU fallback")
        dt = self.context_embedder.weight.dtype
        B, C, Hh, Ww = hidden_states.shape
        hp, wp = Hh // 2, Ww // 2
        S_img, S_txt, D = hp * wp, encoder_hidden_states.shape[1], self.inner_dim
        dev = hidden_states.device
        if _packed_latents is None:
            x = hidden_states.to(dt).view(B, C, hp, 2, wp, 2).permute(0, 2, 4, 1, 3, 5).reshape(B, S_img, C * 4)
        else:
            x = _packed_latents
        full = getattr(self, "_full_ft", False) and torch.is_grad_enabled()
        pos = self._cropped_pos(hp, wp, dt).expand(B, S_img, D)
        if full:
            h = EmbedFullFn.apply(x.contiguous(), encoder_hidden_states.to(dt).contiguous(), pos, self.pos_embed.proj.weight,
                                  self.pos_embed.proj.bias, self.context_embedder.weight, self.context_embedder.bias)
        else:
            h = torch.empty((B, S_txt + S_img, D), device=dev, dtype=dt)
            # PatchEmbed: conv2x2/s2 == GEMM over (c, dy, dx) features; + cropped pos table in the epilogue
            w_pe = self.pos_embed.proj.weight.detach().reshape(D, C * 4)
            ops.gemm([x.contiguous()], [w_pe], self.pos_embed.proj.bias.detach(), out=h[:, S_txt:], epi=ops.EPI_ADD_RES, res=pos)
            ops.gemm([encoder_hidden_states.to(dt).contiguous()], [self.context_embedder.weight], self.context_embedder.bias,
                     out=h[:, :S_txt])
        tte = self.time_text_embed
        temb = tte.timestep_embedder(_sinusoid(timestep.to(dev).float()).to(dt)) + tte.text_embedder(pooled_projections.to(dt).contiguous())
        silu_temb = F.silu(temb).contiguous()
        self._begin_lora_dropout(list(self.transformer_blocks))
        for i, blk in enumerate(self.transformer_blocks):
            h = self._run_block(i, blk, h, silu_temb, S_txt, self._lora_scaling)
        if self._tail_plan is None:
            self._tail_plan = {"w_proj": self.proj_out.weight.detach(), "b_proj": self.proj_out.bias.detach(),
                               "w_proj_t": _wt(self.proj_out.weight.detach())}
        mod = self.norm_out.linear(silu_temb)
        slot = (self.proj_out.weight, self.proj_out.bias) if full else ()
        out = TailFn.apply(h, mod, {"S_txt": S_txt, "full": full, **self._tail_plan}, *slot)  # [B, S_img, p*p*C_out], (dy, dx, c)
        if not _packed_output:
            Co = self.out_channels
            out = torch.einsum("nhwpqc->nchpwq", out.reshape(B, hp, wp, 2, 2, Co)).reshape(B, Co, hp * 2, wp * 2)
        if not return_dict:
            return (out,)
        return SimpleNamespace(sample=out)
