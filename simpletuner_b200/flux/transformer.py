"""FluxTransformer2DModel on libstb200 — the B200-native drop-in for reference
simpletuner/helpers/models/flux/transformer.py:690-1515 (class FluxTransformer2DModel).

Interface kept from the reference (SURVEY.md §8b, seam B1):
  * constructor arguments (`patch_size`, `in_channels`, `num_layers`, `num_single_layers`,
    `attention_head_dim`, `num_attention_heads`, `joint_attention_dim`, `pooled_projection_dim`,
    `guidance_embeds`, `axes_dims_rope`) and the `.config` namespace read by the wrapper
    (flux/model.py:724-728);
  * `forward(hidden_states, encoder_hidden_states, pooled_projections, timestep, img_ids, txt_ids,
    guidance, joint_attention_kwargs=None, return_dict=False, attention_mask=None, ...)`
    returning the tuple `(Tensor[B, S_img, in_channels],)`;
  * parameter names of the diffusers / reference state_dict (transformer_blocks.N.attn.to_q.weight …)
    and PEFT adapter names (….to_q.lora_A.default.weight / lora_B.default.weight) so that
    `get_peft_model_state_dict`-style saving and DDP see the same nn.Parameters;
  * `add_adapter(...)` (PeftAdapterMixin) with flux_lora_target groups (flux/model.py:1235-1383).
Unsupported options raise (attention masks — quirk Q2 —, token-wise timesteps, TREAD routing,
controlnet residuals, hidden-state capture): the shim must fall back to the reference module then.

Arithmetic: every dense op is a libstb200 kernel (blocks.py); torch provides parameters,
allocation and the autograd graph between blocks.  The tiny per-sample conditioning path
(sinusoidal timestep embedding + SiLU on [B, 3072] vectors) uses torch elementwise ops.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from .blocks import AttnPlan, DoubleBlockFn, LoraDrop, LoraLinearFn, MlpPlan, SingleBlockFn, TailFn, _t, _wt

_ATTN = ["to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj", "to_out.0", "to_add_out"]
_FFS = ["ff.net.0.proj", "ff.net.2", "ff_context.net.0.proj", "ff_context.net.2", "proj_mlp", "proj_out"]
FLUX_LORA_TARGETS = {
    # reference flux/model.py:1235-1383 (names that exist un-fused; PEFT selects a Linear whose qualified name equals a
    # target or ends with ".<target>", so "proj_out" covers every single block's proj_out and the model's final proj_out)
    "all": _ATTN,
    "mmdit": _ATTN,
    "context": ["add_q_proj", "add_k_proj", "add_v_proj", "to_add_out"],
    "context+ffs": ["add_q_proj", "add_k_proj", "add_v_proj", "to_add_out", "ff_context.net.0.proj", "ff_context.net.2"],
    "all+ffs": _ATTN + _FFS,
    "all+ffs+embedder": ["x_embedder"] + _ATTN + _FFS,
    "tiny": ["single_transformer_blocks.7.proj_out", "single_transformer_blocks.20.proj_out"],
    "nano": ["single_transformer_blocks.7.proj_out"],
}
# Linears the block schedules can adapt; "ai-toolkit" additionally adapts the adaLN linears (norm.linear, norm1.linear,
# norm1_context.linear), whose gradients need d loss / d modulation — not produced by the LoRA schedules
_ADAPTABLE_SUFFIXES = tuple("." + t for t in (_ATTN + _FFS))


def _peft_match(name: str, targets) -> bool:
    return any(name == t or name.endswith("." + t) for t in targets)


class _Weight(nn.Module):
    """Holds `weight` (and nothing else) so that `lora_A.default.weight` resolves like PEFT's ModuleDict."""

    def __init__(self, shape, dtype):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(shape, dtype=dtype))


class Linear(nn.Module):
    """Parameter holder with nn.Linear naming; optionally carries one PEFT-style LoRA adapter."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, dtype=torch.bfloat16):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty((out_features, in_features), dtype=dtype), requires_grad=False)
        self.bias = nn.Parameter(torch.empty((out_features,), dtype=dtype), requires_grad=False) if bias else None
        self.lora_A: Optional[nn.ModuleDict] = None
        self.lora_B: Optional[nn.ModuleDict] = None
        self.scaling: Dict[str, float] = {}
        self.lora_enabled = True
        self.__dict__["lokr"] = None   # simpletuner_b200.lycoris.LokrModule (owned by the LycorisNetwork, not a sub-module)

    def add_lora(self, rank: int, alpha: float, adapter_name: str = "default", init_lora_weights: bool = True):
        dt = self.weight.dtype
        a = _Weight((rank, self.in_features), dt)
        b = _Weight((self.out_features, rank), dt)
        with torch.no_grad():
            nn.init.kaiming_uniform_(a.weight, a=math.sqrt(5))  # PEFT default ("default" init style)
            nn.init.zeros_(b.weight)
        a.to(self.weight.device)
        b.to(self.weight.device)
        self.lora_A = nn.ModuleDict({adapter_name: a})
        self.lora_B = nn.ModuleDict({adapter_name: b})
        self.scaling[adapter_name] = alpha / rank

    _lokr_capable = False           # set on the Linears of Attention / FeedForward modules (the LyCORIS preset targets)

    def lora_tensors(self, adapter_name: str = "default"):
        """The two trainable tensors the block schedules differentiate: LoRA (A, B) or the LoKr factors (w1, w2)."""
        if self.lokr is not None:
            return self.lokr.factors()
        if self.lora_A is None or not self.lora_enabled:
            return None, None
        return self.lora_A[adapter_name].weight, self.lora_B[adapter_name].weight

    def lokr_scale(self) -> Optional[float]:
        return None if self.lokr is None else self.lokr.scale * self.lokr.multiplier

    def effective_weight(self) -> torch.Tensor:
        """The weight the projection GEMMs read: W, or W + kron(w1, w2) * scale with a LoKr adapter (rebuilt per step)."""
        return self.weight.detach() if self.lokr is None else self.lokr.effective_weight()

    def forward(self, x):  # small-M helper path (embedders / conditioning MLPs on [B, D] vectors)
        if self.weight.requires_grad and torch.is_grad_enabled():
            # full fine-tune: the conditioning path trains through plain torch autograd (< 0.1 % of the step's work)
            return F.linear(x, self.weight, self.bias)
        return ops.gemm([x.contiguous()], [self.weight], self.bias)


class RMSNormWeight(nn.Module):
    def __init__(self, dim, dtype=torch.bfloat16):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim, dtype=dtype), requires_grad=False)


class FluxAttention(nn.Module):
    """Parameter container mirroring diffusers Attention as configured at flux/transformer.py:440-451, 539-551."""

    def __init__(self, dim, heads, head_dim, joint: bool, dtype):
        super().__init__()
        self.heads, self.head_dim = heads, head_dim
        self.to_q = Linear(dim, dim, dtype=dtype)
        self.to_k = Linear(dim, dim, dtype=dtype)
        self.to_v = Linear(dim, dim, dtype=dtype)
        self.norm_q = RMSNormWeight(head_dim, dtype)
        self.norm_k = RMSNormWeight(head_dim, dtype)
        if joint:
            self.add_q_proj = Linear(dim, dim, dtype=dtype)
            self.add_k_proj = Linear(dim, dim, dtype=dtype)
            self.add_v_proj = Linear(dim, dim, dtype=dtype)
            self.norm_added_q = RMSNormWeight(head_dim, dtype)
            self.norm_added_k = RMSNormWeight(head_dim, dtype)
            self.to_out = nn.ModuleList([Linear(dim, dim, dtype=dtype), nn.Identity()])
            self.to_add_out = Linear(dim, dim, dtype=dtype)
        for m in self.modules():
            if isinstance(m, Linear):
                m._lokr_capable = True

    _lycoris_class_name = "Attention"       # diffusers class name the LyCORIS presets select (documentation/LYCORIS.md)


class _AdaNorm(nn.Module):
    def __init__(self, dim, mult, dtype):
        super().__init__()
        self.linear = Linear(dim, mult * dim, dtype=dtype)


class _GELUProj(nn.Module):
    def __init__(self, dim, inner, dtype):
        super().__init__()
        self.proj = Linear(dim, inner, dtype=dtype)


class _FeedForward(nn.Module):
    """diffusers FeedForward(dim, dim_out=dim, activation_fn="gelu-approximate"): net.0.proj, net.2."""

    def __init__(self, dim, dtype):
        super().__init__()
        self.net = nn.ModuleList([_GELUProj(dim, 4 * dim, dtype), nn.Identity(), Linear(4 * dim, dim, dtype=dtype)])
        self.net[0].proj._lokr_capable = True
        self.net[2]._lokr_capable = True

    _lycoris_class_name = "FeedForward"


def _fill_weight(lin: Linear, out: torch.Tensor) -> None:
    """Write `lin`'s effective weight into (a slice of) a plan's layout; with a LoKr adapter it comes out of one
    `stb_lokr_rebuild` pass over W."""
    if lin.lokr is None:
        out.copy_(lin.weight.detach())
    else:
        lin.lokr.rebuild_into(out)


def _weight_pair(lin: Linear, dynamic: bool = False):
    """(forward weight, dgrad operand) of one Linear.  dynamic: the weight is rewritten every optimizer step (full
    fine-tune); a LoKr weight is rebuilt every step, so it is dynamic too."""
    if lin.lokr is None:
        w = lin.weight.detach()
        return w, _wt(w, dynamic)
    w = torch.empty_like(lin.weight)
    _fill_weight(lin, w)
    return w, _wt(w, True)


def _attn_plan(q: Linear, k: Linear, v: Linear, out: Optional[Linear], nq, nk, dynamic: bool = False) -> AttnPlan:
    """Fused q|k|v and output layouts of one attention stream; nq / nk None: no QK norm (SD3 without qk_norm)."""
    b_qkv = torch.cat([q.bias.detach(), k.bias.detach(), v.bias.detach()], 0).contiguous()
    if q.lokr is None and k.lokr is None and v.lokr is None:
        w_qkv = torch.cat([q.weight.detach(), k.weight.detach(), v.weight.detach()], 0).contiguous()
        w_qkv_t = _wt(w_qkv, dynamic)
    else:
        n = q.out_features
        w_qkv = torch.empty((3 * n, q.in_features), device=q.weight.device, dtype=q.weight.dtype)
        for m, lin in enumerate((q, k, v)):
            _fill_weight(lin, w_qkv[m * n:(m + 1) * n])
        w_qkv_t = _wt(w_qkv, True)
    p = AttnPlan(w_qkv, b_qkv, w_qkv_t, norm_q=None if nq is None else nq.weight.detach(),
                 norm_k=None if nk is None else nk.weight.detach())
    if out is not None:
        p.w_out, p.w_out_t = _weight_pair(out, dynamic)
        p.b_out = out.bias.detach()
    return p


def _mlp_plan(fc1: Linear, fc2: Linear, dynamic: bool = False) -> MlpPlan:
    (w1, w1_t), (w2, w2_t) = _weight_pair(fc1, dynamic), _weight_pair(fc2, dynamic)
    return MlpPlan(w1, fc1.bias.detach(), w1_t, w2, fc2.bias.detach(), w2_t)


def _lora_list(linears: Sequence[Linear]) -> List[Optional[torch.Tensor]]:
    out: List[Optional[torch.Tensor]] = []
    for lin in linears:
        a, b = lin.lora_tensors()
        out += [a, b]
    return out


def _lokr_scales(linears: Sequence[Optional[Linear]]) -> Optional[List[Optional[float]]]:
    """Per (A, B) slot of the flat adapter list: the LoKr scale of that Linear (None = LoRA / not adapted)."""
    sc = [None if lin is None else lin.lokr_scale() for lin in linears]
    return sc if any(x is not None for x in sc) else None


class FluxTransformerBlock(nn.Module):
    """reference flux/transformer.py:514-687"""

    def __init__(self, dim, heads, head_dim, dtype):
        super().__init__()
        self.dim, self.heads, self.head_dim = dim, heads, head_dim
        self.norm1 = _AdaNorm(dim, 6, dtype)
        self.norm1_context = _AdaNorm(dim, 6, dtype)
        self.attn = FluxAttention(dim, heads, head_dim, True, dtype)
        self.ff = _FeedForward(dim, dtype)
        self.ff_context = _FeedForward(dim, dtype)
        self._plans = None

    def _plan_linears(self):
        a = self.attn
        return {"img_attn": (a.to_q, a.to_k, a.to_v, a.to_out[0]), "txt_attn": (a.add_q_proj, a.add_k_proj, a.add_v_proj, a.to_add_out),
                "img_mlp": (self.ff.net[0].proj, self.ff.net[2]), "txt_mlp": (self.ff_context.net[0].proj, self.ff_context.net[2])}

    def plans(self):
        if self._plans is None:
            self._plans = {}
        pl = self._plans
        a = self.attn
        if "img_attn" not in pl:
            pl["img_attn"] = _attn_plan(a.to_q, a.to_k, a.to_v, a.to_out[0], a.norm_q, a.norm_k)
        if "txt_attn" not in pl:
            pl["txt_attn"] = _attn_plan(a.add_q_proj, a.add_k_proj, a.add_v_proj, a.to_add_out, a.norm_added_q, a.norm_added_k)
        if "img_mlp" not in pl:
            pl["img_mlp"] = _mlp_plan(self.ff.net[0].proj, self.ff.net[2])
        if "txt_mlp" not in pl:
            pl["txt_mlp"] = _mlp_plan(self.ff_context.net[0].proj, self.ff_context.net[2])
        return pl

    def drop_adapted_plans(self):
        """LoKr: only the layouts that embed an adapted weight follow the optimizer; the rest stay as built."""
        if self._plans:
            for key, lins in self._plan_linears().items():
                if any(l.lokr is not None for l in lins):
                    self._plans.pop(key, None)

    def forward(self, h, silu_temb, cos, sin, S_txt, lora_scaling, key_bias=None, segs=None):
        """segs (Flux Kontext): (scene, conditioning) token counts of the image stream; silu_temb then stacks the
        [text | scene | conditioning] rows [3B, D] (FluxTransformer2DModel.forward)."""
        if segs is None:
            mod_img = self.norm1.linear(silu_temb)
            mod_txt = self.norm1_context.linear(silu_temb)
        else:
            B = silu_temb.shape[0] // 3
            mod_img = self.norm1.linear(silu_temb[B:])            # [2B, 6D]: scene rows, conditioning rows
            mod_txt = self.norm1_context.linear(silu_temb[:B])
        a = self.attn
        attn_l = [a.to_q, a.to_k, a.to_v, a.to_out[0], a.add_q_proj, a.add_k_proj, a.add_v_proj, a.to_add_out]
        mlp_l = [self.ff.net[0].proj, self.ff.net[2], self.ff_context.net[0].proj, self.ff_context.net[2]]
        return run_double_block(self, h, mod_img, mod_txt, cos, sin, S_txt, lora_scaling, key_bias, segs, attn_l, mlp_l)


def run_double_block(blk, h, mod_img, mod_txt, cos, sin, S_txt, lora_scaling, key_bias, segs, attn_l, mlp_l, **flags):
    """DoubleBlockFn over one joint block: `attn_l` = the image q, k, v, out then text q, k, v, out Linears, `mlp_l` = the
    image fc1, fc2 then text fc1, fc2 Linears; `blk` provides heads, head_dim, plans() and the step's dropout state.
    Shared by the Flux and Qwen-Image double blocks; `flags` are DoubleBlockFn's `st` switches (e.g. nan_to_num_txt)."""
    st = {"S_txt": S_txt, "H": blk.heads, "hd": blk.head_dim, "plans": blk.plans(), "lora_scaling": lora_scaling,
          "lora_drop": getattr(blk, "_lora_drop", None), "key_bias": key_bias, "img_segs": segs, **flags}
    lora = _lora_list(attn_l)
    mlp = _lora_list(mlp_l)
    st["lokr_scales"] = _lokr_scales(attn_l + [None] * 4 + mlp_l)
    if any(t is not None for t in mlp):
        lora = lora + [None] * 8 + mlp          # [16..23] = the SD3.5 second attention, unused here
    return DoubleBlockFn.apply(h, mod_img, mod_txt, cos, sin, st, *lora)


class FluxSingleTransformerBlock(nn.Module):
    """reference flux/transformer.py:416-510"""

    def __init__(self, dim, heads, head_dim, dtype):
        super().__init__()
        self.dim, self.heads, self.head_dim = dim, heads, head_dim
        self.norm = _AdaNorm(dim, 3, dtype)
        self.proj_mlp = Linear(dim, 4 * dim, dtype=dtype)
        self.proj_out = Linear(5 * dim, dim, dtype=dtype)
        self.attn = FluxAttention(dim, heads, head_dim, False, dtype)
        self._plans = None

    def plans(self):
        if self._plans is None:
            self._plans = {}
        pl = self._plans
        a = self.attn
        if "attn" not in pl:
            pl["attn"] = _attn_plan(a.to_q, a.to_k, a.to_v, None, a.norm_q, a.norm_k)
        if "mlp" not in pl:
            pl["mlp"] = _mlp_plan(self.proj_mlp, self.proj_out)
        return pl

    def drop_adapted_plans(self):
        a = self.attn
        if self._plans and any(l.lokr is not None for l in (a.to_q, a.to_k, a.to_v)):
            self._plans.pop("attn", None)

    def forward(self, h, silu_temb, cos, sin, lora_scaling, key_bias=None, segs=None):
        """segs (Flux Kontext): (text, scene, conditioning) token counts; silu_temb then holds those rows [3B, D]."""
        return run_single_block(self, h, self.norm.linear(silu_temb), cos, sin, lora_scaling, key_bias, segs)


def run_single_block(blk, h, mod, cos, sin, lora_scaling, key_bias, segs):
    """SingleBlockFn over one single-stream block with its modulation rows `mod` [B, 3D] (shift | scale | gate); shared by
    the Flux and Chroma single blocks."""
    st = {"H": blk.heads, "hd": blk.head_dim, "plans": blk.plans(), "lora_scaling": lora_scaling,
          "lora_drop": getattr(blk, "_lora_drop", None), "key_bias": key_bias, "segs": segs}
    a = blk.attn
    lora = _lora_list([a.to_q, a.to_k, a.to_v])
    st["lokr_scales"] = _lokr_scales([a.to_q, a.to_k, a.to_v])
    mlp = _lora_list([blk.proj_mlp, blk.proj_out])
    if any(t is not None for t in mlp):
        lora = lora + mlp
    return SingleBlockFn.apply(h, mod, cos, sin, st, *lora)


class _TimestepEmbedding(nn.Module):
    def __init__(self, in_ch, dim, dtype):
        super().__init__()
        self.linear_1 = Linear(in_ch, dim, dtype=dtype)
        self.linear_2 = Linear(dim, dim, dtype=dtype)

    def forward(self, x):
        return self.linear_2(F.silu(self.linear_1(x)))


class _TimeTextEmbed(nn.Module):
    """diffusers CombinedTimestep(Guidance)TextProjEmbeddings (reference flux/transformer.py:765-771)."""

    def __init__(self, dim, pooled_dim, guidance: bool, dtype):
        super().__init__()
        self.timestep_embedder = _TimestepEmbedding(256, dim, dtype)
        if guidance:
            self.guidance_embedder = _TimestepEmbedding(256, dim, dtype)
        self.text_embedder = _TimestepEmbedding(pooled_dim, dim, dtype)
        self.guidance = guidance


def _sinusoid(t: torch.Tensor, dim: int = 256, max_period: int = 10000) -> torch.Tensor:
    """diffusers get_timestep_embedding(flip_sin_to_cos=True, downscale_freq_shift=0)."""
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32, device=t.device) / half
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


def rope_tables(ids: torch.Tensor, axes_dim, theta: float = 10000.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """diffusers FluxPosEmbed (reference flux/transformer.py:764, 1094): float64 frequencies,
    repeat_interleave(2), returned as float32 [S, sum(axes_dim)].  Index math on the host (exact)."""
    pos = ids.detach().to("cpu", torch.float64)
    cos_out, sin_out = [], []
    for i, d in enumerate(axes_dim):
        freqs = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.float64)[: d // 2] / d))
        f = torch.outer(pos[:, i], freqs)
        cos_out.append(f.cos().repeat_interleave(2, dim=1).float())
        sin_out.append(f.sin().repeat_interleave(2, dim=1).float())
    return torch.cat(cos_out, dim=-1).contiguous(), torch.cat(sin_out, dim=-1).contiguous()


def flux_key_bias(attention_mask: torch.Tensor, B: int, S: int, dtype, device) -> torch.Tensor:
    """The per-key logit bias [B, S] of Flux masked training: `expand_flux_attention_mask` (ones over the joint
    [text | image] sequence, the text mask written into its first L columns) then `(mask > 0).to(dtype)` as
    FluxAttnProcessor2_0 does before SDPA adds it to the logits (reference flux/transformer.py:170-173, 227-242).  So kept
    text keys and every image key get +1 and padded text keys +0.  Device ops only: no host sync, CUDA-graph capturable."""
    if attention_mask.dim() != 2 or attention_mask.shape[0] != B or attention_mask.shape[1] > S:
        raise ValueError(f"attention_mask must be [B, L] with B = {B} and L <= {S}, got {tuple(attention_mask.shape)}")
    bias = torch.ones((B, S), device=device, dtype=dtype)
    bias[:, :attention_mask.shape[1]] = (attention_mask.to(device, non_blocking=True) > 0).to(dtype)
    return bias


class B200FusedAttnProcessor:
    """Marker processor: the attention of this module runs inside the libstb200 block schedule (blocks.py)."""

    def __call__(self, *a, **k):
        raise RuntimeError("B200FusedAttnProcessor is a marker; the attention runs inside the fused block schedule")


# processors whose arithmetic the fused block schedule reproduces (plain un-masked SDPA attention with the model's own
# projections / QK-norm / RoPE): reference flux/transformer.py:116-224, flux/attention.py:309-579, diffusers
# JointAttnProcessor2_0 / AttnProcessor2_0
_EQUIVALENT_PROCESSORS = {
    "B200FusedAttnProcessor", "FluxAttnProcessor2_0", "FluxAttnProcessor", "FluxFusedSDPAProcessor",
    "FluxFusedFlashAttnProcessor3", "FluxSingleFusedFlashAttnProcessor3", "FusedFluxAttnProcessor2_0",
    "JointAttnProcessor2_0", "FusedJointAttnProcessor2_0", "AttnProcessor2_0", "AttnProcessor", "FusedAttnProcessor2_0",
}


class AttnProcessorAPI:
    """`attn_processors` / `set_attn_processor` of the reference denoisers (seam B2: flux/transformer.py:880-912, sd3
    :483, pixart :404).  The B200 modules have no pluggable processor: setting one whose arithmetic the fused schedule
    reproduces is recorded and accepted; anything else (IP-adapter, masked, custom) raises NotImplementedError so that the
    caller keeps the reference module for that feature."""

    def _attention_modules(self):
        return {n: m for n, m in self.named_modules() if n.endswith(("attn", "attn1", "attn2")) and hasattr(m, "to_q")}

    @property
    def attn_processors(self):
        store = self.__dict__.setdefault("_attn_processor_store", {})
        return {f"{n}.processor": store.get(n, B200FusedAttnProcessor()) for n in self._attention_modules()}

    def set_attn_processor(self, processor):
        mods = self._attention_modules()
        if isinstance(processor, dict):
            if len(processor) != len(mods):
                raise ValueError(f"A dict of processors was passed, but the number of processors {len(processor)} does not "
                                 f"match the number of attention layers: {len(mods)}. Please make sure to pass {len(mods)} "
                                 "processor classes.")
            items = {k[: -len(".processor")] if k.endswith(".processor") else k: v for k, v in processor.items()}
        else:
            items = {n: processor for n in mods}
        for n, proc in items.items():
            name = type(proc).__name__
            if name not in _EQUIVALENT_PROCESSORS:
                raise NotImplementedError(f"attention processor {name} is not reproduced by the libstb200 "
                                          "block schedule; use the reference module for it")
            if getattr(self, "attention_masked_training", False) and "Flash" in name:
                # the flash processors mask by key padding (varlen), not by the additive bias the blocks apply
                raise NotImplementedError(f"attention processor {name} with flux_attention_masked_training applies "
                                          "key-padding semantics the libstb200 block schedule does not reproduce")
        self.__dict__.setdefault("_attn_processor_store", {}).update(items)

    def fuse_qkv_projections(self):
        """diffusers `fuse_qkv_projections` (reference common.py:3547 calls the family hook after load): the fused
        [3D, D] projection already IS the internal layout (blocks.AttnPlan.w_qkv); parameters keep their un-fused names so
        that LoRA files stay PEFT / ComfyUI compatible.  Nothing to do."""
        return None

    def unfuse_qkv_projections(self):
        return None


class LoraDropoutAPI:
    """PEFT `lora_dropout` for the fused LoRA path (reference common.py:1094-1117; default 0.1,
    field_registry/sections/lora.py:130-137).  Active only in training mode (`module.training`, like nn.Dropout).  One seed
    is drawn per forward from torch's CPU default generator (no device sync; seeded runs are reproducible); every block gets
    16 mask streams (one per adapted Linear), regenerated — not stored — by the backward kernels (csrc/elementwise.cuh)."""

    _lora_dropout_p: float = 0.0
    STREAMS_PER_BLOCK = 16

    def _begin_lora_dropout(self, blocks) -> None:
        p = float(getattr(self, "_lora_dropout_p", 0.0) or 0.0)
        active = p > 0.0 and self.training and torch.is_grad_enabled()
        seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item()) if active else 0
        for i, blk in enumerate(blocks):
            blk._lora_drop = LoraDrop(p, seed, i * self.STREAMS_PER_BLOCK) if active else None

    @staticmethod
    def _check_dropout_p(p) -> float:
        p = float(p or 0.0)
        if not 0.0 <= p < 1.0:
            raise ValueError(f"lora_dropout must be in [0, 1), got {p}")
        return p


class AdapterModelAPI:
    """Gradient checkpointing, the PEFT adapter surface and the parameter lifecycle shared by every denoiser built on the
    Flux blocks.  A model sets `_DEFAULT_LORA_TARGETS`, `_lora_adaptable(name)` (the Linears its block schedules can
    adapt) and `invalidate_plans()` (drops what it derived from the parameters; run after `.to()` / `load_state_dict`)."""

    _DEFAULT_LORA_TARGETS: Sequence[str] = ()

    @staticmethod
    def _lora_adaptable(name: str) -> bool:
        raise NotImplementedError

    def invalidate_plans(self):
        raise NotImplementedError

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self.invalidate_plans()
        return out

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        self.invalidate_plans()
        return out

    def enable_gradient_checkpointing(self):
        """common.py:3550-3636 / flux/transformer.py:1240-1287: blocks selected by `gradient_checkpointing_interval`
        (every block when None) are re-run in backward instead of keeping their saved set (block input only is kept),
        through torch.utils.checkpoint like the reference.  Off by default: the block schedules already keep a minimal
        activation set; on an 80 GB H100 that holds one 1024^2 sample next to the Flux.1-dev weights, and larger batches need
        recompute."""
        self.gradient_checkpointing = True

    def disable_gradient_checkpointing(self):
        self.gradient_checkpointing = False

    def _run_block(self, index: int, blk, *args):
        interval = getattr(self, "gradient_checkpointing_interval", None)
        if self.gradient_checkpointing and torch.is_grad_enabled() and (interval is None or index % interval == 0):
            from torch.utils.checkpoint import checkpoint
            return checkpoint(blk, *args, use_reentrant=False)
        return blk(*args)

    def set_gradient_checkpointing_interval(self, value: int):
        self.gradient_checkpointing_interval = value

    def lora_linears(self) -> Dict[str, Linear]:
        return {n: m for n, m in self.named_modules() if isinstance(m, Linear) and m.lora_A is not None}

    def add_adapter(self, lora_config=None, adapter_name: str = "default", *, rank: Optional[int] = None,
                    lora_alpha: Optional[float] = None, target_modules: Optional[Sequence[str]] = None,
                    lora_dropout: float = 0.0):
        """PeftAdapterMixin.add_adapter (reference common.py:1117).  Accepts a peft.LoraConfig-like object
        (attributes r, lora_alpha, target_modules, lora_dropout) or keyword arguments."""
        if lora_config is not None:
            rank = getattr(lora_config, "r", rank)
            lora_alpha = getattr(lora_config, "lora_alpha", lora_alpha)
            target_modules = getattr(lora_config, "target_modules", target_modules)
            lora_dropout = getattr(lora_config, "lora_dropout", lora_dropout)
        if rank is None:
            raise ValueError("LoRA rank is required")
        if getattr(self, "_lycoris_network", None) is not None:
            raise NotImplementedError("a LyCORIS network is attached: PEFT LoRA and LoKr adapters cannot be mixed on this path")
        lora_dropout = self._check_dropout_p(lora_dropout)
        if not 1 <= rank <= 128:
            raise NotImplementedError("fused LoRA path supports rank 1..128 (one 128-wide rank block per adapted Linear)")
        lora_alpha = float(lora_alpha) if lora_alpha is not None else float(rank)  # common.py:1090-1093
        targets = list(target_modules) if target_modules is not None else list(self._DEFAULT_LORA_TARGETS)
        chosen = self.lora_target_linears(targets)
        if not chosen:
            raise ValueError(f"no module matched LoRA targets {targets}")
        for mod in chosen.values():
            mod.add_lora(rank, lora_alpha, adapter_name)
        self._lora_scaling = lora_alpha / rank
        self._lora_dropout_p = lora_dropout
        self.peft_config[adapter_name] = SimpleNamespace(r=rank, lora_alpha=lora_alpha, target_modules=targets,
                                                         lora_dropout=lora_dropout)
        return len(chosen)

    def lora_target_linears(self, targets: Sequence[str]) -> Dict[str, Linear]:
        """The Linears PEFT's suffix rule selects for `targets` (a qualified name equal to a target or ending with
        ".<target>").  Raises NotImplementedError naming the first one the block schedules cannot adapt; the shim calls
        this at load time so that such a run keeps the reference module."""
        chosen = {}
        for name, mod in self.named_modules():
            if not isinstance(mod, Linear) or not _peft_match(name, targets):
                continue
            if not self._lora_adaptable(name):
                raise NotImplementedError(f"LoRA target {name} is not supported by the fused path (use the reference "
                                          "module, e.g. for the adaLN linears of flux_lora_target=ai-toolkit)")
            chosen[name] = mod
        return chosen

    def disable_lora(self):
        for m in self.lora_linears().values():
            m.lora_enabled = False

    def enable_lora(self):
        for m in self.lora_linears().values():
            m.lora_enabled = True

    def trainable_parameters(self):
        return [p for p in self.parameters() if p.requires_grad]


class FluxTransformer2DModel(AdapterModelAPI, AttnProcessorAPI, LoraDropoutAPI, nn.Module):
    _no_split_modules = ["FluxTransformerBlock", "FluxSingleTransformerBlock"]
    _supports_gradient_checkpointing = True

    def __init__(self, patch_size: int = 1, in_channels: int = 64, num_layers: int = 19, num_single_layers: int = 38,
                 attention_head_dim: int = 128, num_attention_heads: int = 24, joint_attention_dim: int = 4096,
                 pooled_projection_dim: int = 768, guidance_embeds: bool = False,
                 axes_dims_rope: Tuple[int, ...] = (16, 56, 56), dtype=torch.bfloat16, **unused):
        super().__init__()
        if attention_head_dim not in (64, 128):
            raise NotImplementedError("libstb200 attention supports head_dim 64 / 128")
        self.config = SimpleNamespace(patch_size=patch_size, in_channels=in_channels, num_layers=num_layers,
                                      num_single_layers=num_single_layers, attention_head_dim=attention_head_dim,
                                      num_attention_heads=num_attention_heads, joint_attention_dim=joint_attention_dim,
                                      pooled_projection_dim=pooled_projection_dim, guidance_embeds=guidance_embeds,
                                      axes_dims_rope=tuple(axes_dims_rope))
        self.out_channels = in_channels
        self.inner_dim = D = num_attention_heads * attention_head_dim
        self.time_text_embed = _TimeTextEmbed(D, pooled_projection_dim, guidance_embeds, dtype)
        self.context_embedder = Linear(joint_attention_dim, D, dtype=dtype)
        self.x_embedder = Linear(in_channels, D, dtype=dtype)
        self.transformer_blocks = nn.ModuleList(
            [FluxTransformerBlock(D, num_attention_heads, attention_head_dim, dtype) for _ in range(num_layers)])
        self.single_transformer_blocks = nn.ModuleList(
            [FluxSingleTransformerBlock(D, num_attention_heads, attention_head_dim, dtype) for _ in range(num_single_layers)])
        self.norm_out = _AdaNorm(D, 2, dtype)
        self.proj_out = Linear(D, patch_size * patch_size * self.out_channels, dtype=dtype)
        self.gradient_checkpointing = False
        self._rope_cache: Dict[Any, Tuple[torch.Tensor, ...]] = {}
        self._tail_plan = None
        self._lora_scaling = 1.0
        self.peft_config: Dict[str, Any] = {}

    _DEFAULT_LORA_TARGETS = FLUX_LORA_TARGETS["all"]

    @staticmethod
    def _lora_adaptable(name: str) -> bool:
        # adaLN linears ("ai-toolkit") stay on the reference module: their gradients need d loss / d modulation
        return name.endswith(_ADAPTABLE_SUFFIXES) or name in ("proj_out", "x_embedder")

    def invalidate_plans(self):
        """Call after base weights change (load_state_dict / .to()); derived layouts are rebuilt lazily."""
        for blk in list(self.transformer_blocks) + list(self.single_transformer_blocks):
            blk._plans = None
        self._tail_plan = None
        self._rope_cache.clear()

    def after_optimizer_step(self):
        """TrainStep hook: with a LyCORIS LoKr network attached the projection layouts embed W + kron(w1, w2) and must follow
        the factors the optimizer just updated."""
        if getattr(self, "_lycoris_network", None) is not None:
            for blk in list(self.transformer_blocks) + list(self.single_transformer_blocks):
                blk.drop_adapted_plans()

    # ---- forward ------------------------------------------------------------------------------
    def _rope(self, txt_ids, img_ids, device):
        # keyed on the id CONTENT: a sum (or the shape) does not identify a bucket — the (128, 64) and (64, 128) latent
        # grids have the same shape and the same id sum but different (row, col) tables
        ti, ii = txt_ids.detach().to("cpu", torch.float32).contiguous(), img_ids.detach().to("cpu", torch.float32).contiguous()
        key = (tuple(ti.shape), tuple(ii.shape), hash(ti.numpy().tobytes()), hash(ii.numpy().tobytes()), str(device))
        hit = self._rope_cache.get(key)
        if hit is not None and not (torch.equal(hit[2], ti) and torch.equal(hit[3], ii)):   # hash collision
            hit = None
        if hit is None:
            cos, sin = rope_tables(torch.cat((ti, ii), dim=0), self.config.axes_dims_rope)
            hit = (cos.to(device), sin.to(device), ti, ii)
            if len(self._rope_cache) > 64:
                self._rope_cache.clear()
            self._rope_cache[key] = hit
        return hit

    def _embed_image(self, x: torch.Tensor, out: torch.Tensor) -> None:
        """out (the image rows of the joint buffer) = x_embedder(x), with its LoRA adapter when one is attached."""
        xa, xb = self.x_embedder.lora_tensors()
        if xa is None or not torch.is_grad_enabled():
            ops.gemm([x.contiguous()], [self.x_embedder.weight], self.x_embedder.bias, out=out)
            if xa is not None:          # inference with the adapter attached
                out += F.linear(F.linear(x, xa), xb) * self._lora_scaling
        else:
            y = LoraLinearFn.apply(x.contiguous(), self.x_embedder.weight, self.x_embedder.bias,
                                   self._lora_scaling, getattr(self.x_embedder, "_lora_drop", None), xa, xb)
            out.copy_(y)                # autograd routes the image rows of dh to the adapter

    def _tail(self, h, mod, S_txt: int, S_end: int, scaling: float) -> torch.Tensor:
        """norm_out (mod [B, 2D] = scale | shift) and proj_out over the image rows [S_txt, S_end) of the joint buffer."""
        if self._tail_plan is None:
            self._tail_plan = {"w_proj": self.proj_out.weight.detach(), "b_proj": self.proj_out.bias.detach(),
                               "w_proj_t": _wt(self.proj_out.weight.detach())}
        pa, pb = self.proj_out.lora_tensors()
        tail_lora = () if pa is None else (pa, pb)
        return TailFn.apply(h, mod, {"S_txt": S_txt, "S_end": S_end, "lora_scaling": scaling,
                                     "lora_drop": getattr(self.proj_out, "_lora_drop", None), **self._tail_plan}, *tail_lora)

    def _temb(self, timestep, guidance, pooled):
        tte = self.time_text_embed
        dt = pooled.dtype
        emb = tte.timestep_embedder(_sinusoid(timestep).to(dt))
        if tte.guidance:
            emb = emb + tte.guidance_embedder(_sinusoid(guidance).to(dt))
        return emb + tte.text_embedder(pooled)

    def forward(self, hidden_states: torch.Tensor, encoder_hidden_states: torch.Tensor = None,
                pooled_projections: torch.Tensor = None, timestep: torch.Tensor = None, img_ids: torch.Tensor = None,
                txt_ids: torch.Tensor = None, guidance: torch.Tensor = None, timestep_sign=None, r_timestep=None,
                joint_attention_kwargs: Optional[Dict[str, Any]] = None, controlnet_block_samples=None,
                controlnet_single_block_samples=None, return_dict: bool = True, attention_mask=None,
                controlnet_blocks_repeat: bool = False, force_keep_mask=None, hidden_states_buffer=None,
                grounding_kwargs=None, conditioning_tokens: int = 0):
        """conditioning_tokens (Flux Kontext): the last `conditioning_tokens` rows of `hidden_states` / `img_ids` are
        reference-image tokens.  They are conditioned at timestep 0 while `timestep` [B] conditions the scene tokens, as the
        reference does with its 2-D timesteps (flux/model.py:602-618, flux/transformer.py:245-294, 1068-1085), and the
        output holds the scene tokens only ([B, S_img - conditioning_tokens, C]; the reference slices them off in
        model_predict, flux/model.py:846-848)."""
        for nm, v in (("timestep_sign", timestep_sign), ("r_timestep", r_timestep),
                      ("controlnet_block_samples", controlnet_block_samples),
                      ("controlnet_single_block_samples", controlnet_single_block_samples),
                      ("force_keep_mask", force_keep_mask), ("grounding_kwargs", grounding_kwargs)):
            if v is not None:
                raise NotImplementedError(f"libstb200 Flux path does not support `{nm}`; use the reference module")
        if timestep.ndim != 1:
            raise NotImplementedError("token-wise timesteps are not supported by the libstb200 Flux path (Kontext passes "
                                      "per-sample timesteps and `conditioning_tokens`)")
        if not hidden_states.is_cuda:
            from .._lib import StbError
            raise StbError("FluxTransformer2DModel (libstb200) needs CUDA tensors; there is no CPU fallback")
        dt = self.x_embedder.weight.dtype
        B, S_img, _ = hidden_states.shape
        S_txt = encoder_hidden_states.shape[1]
        S_c = int(conditioning_tokens or 0)
        if not 0 <= S_c < S_img:
            raise ValueError(f"conditioning_tokens must be in [0, {S_img}), got {S_c}")
        S_scene = S_img - S_c
        D = self.inner_dim
        dev = hidden_states.device
        # joint hidden buffer: [text | image]
        h = torch.empty((B, S_txt + S_img, D), device=dev, dtype=dt)
        blocks = list(self.transformer_blocks) + list(self.single_transformer_blocks)
        self._begin_lora_dropout(blocks + [self.proj_out, self.x_embedder])      # one mask-stream slot each
        self._embed_image(hidden_states.to(dt), h[:, S_txt:])
        ops.gemm([encoder_hidden_states.to(dt).contiguous()], [self.context_embedder.weight], self.context_embedder.bias,
                 out=h[:, :S_txt])
        # reference :1003-1007 — timestep / guidance arrive in [0,1] and are scaled by 1000 here
        t = timestep.to(device=dev, dtype=torch.float32) * 1000
        g = guidance.to(device=dev, dtype=torch.float32) * 1000 if guidance is not None else None
        if self.config.guidance_embeds and g is None:
            raise ValueError("guidance is required when guidance_embeds=True")
        pooled = pooled_projections.to(dt)
        if S_c == 0:
            temb = self._temb(t, g, pooled)
            silu_temb = F.silu(temb).contiguous()
        else:
            # _flux_tokenwise_conditioning has two distinct rows per sample, temb(t) over the scene tokens and temb(0) over
            # the conditioning tokens (same guidance and pooled projection): one pass over 2B rows.  The text stream's
            # temb.mean(dim=1) over all image tokens is the fp32 mean of those rows with their token counts, rounded once
            # to bf16 as the reference's bf16 mean is; [B, S, D] is never formed.
            temb2 = self._temb(torch.cat([t, torch.zeros_like(t)]), None if g is None else torch.cat([g, g]),
                               torch.cat([pooled, pooled]))
            temb_txt = ((temb2[:B].float() * S_scene + temb2[B:].float() * S_c) / S_img).to(dt)
            silu_temb = F.silu(torch.cat([temb_txt, temb2])).contiguous()     # [3B, D]: text, scene, conditioning rows
        if txt_ids.ndim == 3:
            txt_ids = txt_ids[0]
        if img_ids.ndim == 3:
            img_ids = img_ids[0]
        cos, sin = self._rope(txt_ids, img_ids, dev)[:2]
        scaling = self._lora_scaling
        # masked training: one per-key bias for every attention of the step (an argument of each block, so the re-run
        # under gradient checkpointing sees it too)
        key_bias = None if attention_mask is None else flux_key_bias(attention_mask, B, S_txt + S_img, dt, dev)
        # Kontext token segments: host ints, block arguments like key_bias
        img_segs = (S_scene, S_c) if S_c else None
        single_segs = (S_txt, S_scene, S_c) if S_c else None
        for i, blk in enumerate(self.transformer_blocks):
            h = self._run_block(i, blk, h, silu_temb, cos, sin, S_txt, scaling, key_bias, img_segs)
        for i, blk in enumerate(self.single_transformer_blocks):
            h = self._run_block(i, blk, h, silu_temb, cos, sin, scaling, key_bias, single_segs)
        mod = self.norm_out.linear(silu_temb[B:2 * B] if S_c else silu_temb)     # norm_out uses temb_img: the scene rows
        out = self._tail(h, mod, S_txt, S_txt + S_scene, scaling)
        if not return_dict:
            return (out,)
        return SimpleNamespace(sample=out)
