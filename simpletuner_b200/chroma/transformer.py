"""ChromaTransformer2DModel on libstb200: the H100 drop-in for reference simpletuner/helpers/models/chroma/transformer.py
(Chroma 1 base / HD / flash, LoRA training).

Chroma is Flux with the per-block adaLN linears pruned away.  One frozen MLP, `distilled_guidance_layer` (the
"approximator", :297-313), maps a [B, 344, 64] input (16 timestep channels, 16 guidance channels at guidance 0, then the
32-channel `mod_proj` row embedding, :263-294) to `pooled_temb` [B, 344, D], and every block reads its shift / scale /
gate rows from it (:966-1300):
  * single block i:  rows 3 i .. 3 i + 2            (shift, scale, gate: Flux's AdaLayerNormZeroSingle chunk order)
  * double block i:  image rows 114 + 6 i .. + 5, text rows 228 + 6 i .. + 5   (Flux's AdaLayerNormZero chunk order)
  * norm_out:        the last two rows, (shift, scale) — the reverse of Flux's AdaLayerNormContinuous (scale, shift).
(114 = 3 x 38 and 228 = 114 + 6 x 19 at the Chroma 1 depth; the offsets follow num_layers / num_single_layers.)

So the blocks run the Flux schedules (flux/blocks.DoubleBlockFn / SingleBlockFn / TailFn) with modulation views of
`pooled_temb`, the approximator runs on the GEMM and RMSNorm kernels with the SiLU epilogue (ops.EPI_SILU), and the
prompt mask is a per-key -inf logit bias.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Any, Dict, Optional, Tuple

import torch
import torch.nn as nn

from .. import ops
from ..flux.transformer import (FluxAttention, FluxSingleTransformerBlock, FluxTransformer2DModel, FluxTransformerBlock,
                                Linear, RMSNormWeight, _FeedForward, run_double_block, run_single_block)

_ALL = ["to_k", "to_q", "to_v", "to_qkv", "add_qkv_proj", "add_k_proj", "add_q_proj", "add_v_proj", "to_out.0", "to_add_out"]
_CTX = ["add_k_proj", "add_q_proj", "add_v_proj", "add_qkv_proj", "to_add_out"]
_FF = ["ff.net.0.proj", "ff.net.2", "ff_context.net.0.proj", "ff_context.net.2", "proj_mlp", "proj_out"]
_TINY = ["to_q", "to_k", "to_v", "to_out.0", "ff.net.0.proj"]
# reference chroma/model.py:54, 472-592.  `to_qkv` / `add_qkv_proj` only exist on fused projections and the adaLN linears
# (`norm.linear`, `norm1.linear`, `norm1_context.linear`) are pruned from Chroma, so those names match no module: PEFT
# ignores them and so does add_adapter.  "ai-toolkit" therefore adapts exactly what "all+ffs" does.
CHROMA_DEFAULT_LORA_TARGET = ["to_k", "to_q", "to_v", "to_out.0", "to_qkv"]
CHROMA_LORA_TARGETS = {
    "all": _ALL,
    "context": _CTX,
    "context+ffs": _CTX + ["ff_context.net.0.proj", "ff_context.net.2"],
    "all+ffs": _ALL + _FF,
    "all+ffs+embedder": ["x_embedder"] + _ALL + _FF,
    "ai-toolkit": _ALL + _FF[:4] + ["norm.linear", "norm1.linear", "norm1_context.linear"] + _FF[4:],
    "tiny": _TINY,
    "tiny+embedder": ["x_embedder"] + _TINY,
}


def _timestep_embedding(t: torch.Tensor, dim: int, max_period: int = 10000) -> torch.Tensor:
    """diffusers get_timestep_embedding(t, dim, flip_sin_to_cos=True, downscale_freq_shift=0), fp32."""
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32, device=t.device) / half
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


def chroma_mod_proj(rows: int, num_channels: int) -> torch.Tensor:
    """The `mod_proj` buffer of ChromaCombinedTimestepTextProjEmbeddings (:270-276): fp32 [rows, 2 num_channels] on the
    host, the sinusoidal embedding of row index x 1000."""
    return _timestep_embedding(torch.arange(rows) * 1000, 2 * num_channels)


def chroma_input_vec(timestep: torch.Tensor, mod_proj: torch.Tensor) -> torch.Tensor:
    """ChromaCombinedTimestepTextProjEmbeddings.forward (:278-294) for 1-D timesteps: [B, rows, 4 C] in timestep's dtype,
    per row [time_proj(t) | guidance_proj(0) | mod_proj[row]].  `timestep` is what the model's forward made of its
    argument, `timestep.to(dtype) * 1000` (:857); `mod_proj` [rows, 2 C]."""
    B, dt = timestep.shape[0], timestep.dtype
    rows, C = mod_proj.shape[0], mod_proj.shape[1] // 2
    tg = torch.cat([_timestep_embedding(timestep, C).to(dt),
                    _timestep_embedding(torch.zeros_like(timestep), C).to(dt)], dim=1)
    return torch.cat([tg[:, None, :].expand(B, rows, 2 * C),
                      mod_proj.to(device=timestep.device, dtype=dt)[None].expand(B, rows, 2 * C)], dim=-1)


def chroma_key_bias(attention_mask: torch.Tensor, B: int, S: int, dtype) -> torch.Tensor:
    """[B, S] per-key logit bias of the joint bool mask the reference's model_predict builds (chroma/model.py:649-665):
    0 where the mask is set (> 0), -inf elsewhere.  Device ops only.  The reference's attention mask is the outer product
    mask[:, None, :] * mask[:, :, None] (:389, :536): it also blanks the padded text query rows.  Those rows reach
    neither the loss nor any LoRA gradient (their keys are -inf for every query, and text rows are dropped before
    norm_out), so the per-key bias gives the same loss and gradients."""
    if attention_mask.dim() != 2 or tuple(attention_mask.shape) != (B, S):
        raise ValueError(f"attention_mask must be the joint [B, S_txt + S_img] = [{B}, {S}] mask, "
                         f"got {tuple(attention_mask.shape)}")
    keep = attention_mask if attention_mask.dtype == torch.bool else attention_mask > 0
    bias = torch.zeros((B, S), device=attention_mask.device, dtype=dtype)
    return bias.masked_fill_(~keep, float("-inf"))


def adjust_chroma_sigmas(sigmas: torch.Tensor) -> torch.Tensor:
    """Chroma._adjust_chroma_sigmas (chroma/model.py:309-314), in the dtype of `sigmas`."""
    return torch.where(sigmas < 0.5, sigmas.square(), 1 - (1 - sigmas).square())


class _ApproxLayer(nn.Module):
    """PixArtAlphaTextProjection(hidden, hidden, act_fn="silu"): linear_1 -> SiLU -> linear_2."""

    def __init__(self, dim, dtype):
        super().__init__()
        self.linear_1 = Linear(dim, dim, dtype=dtype)
        self.linear_2 = Linear(dim, dim, dtype=dtype)


class ChromaApproximator(nn.Module):
    """reference ChromaApproximator (:297-313): in_proj, `n_layers` x (x + linear_2(silu(linear_1(rmsnorm(x))))),
    out_proj.  Frozen; runs once per forward, without autograd, on B x rows rows."""

    def __init__(self, in_dim, out_dim, hidden_dim, n_layers, dtype):
        super().__init__()
        self.in_proj = Linear(in_dim, hidden_dim, dtype=dtype)
        self.layers = nn.ModuleList([_ApproxLayer(hidden_dim, dtype) for _ in range(n_layers)])
        self.norms = nn.ModuleList([RMSNormWeight(hidden_dim, dtype) for _ in range(n_layers)])
        self.out_proj = Linear(hidden_dim, out_dim, dtype=dtype)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [B, rows, in_dim] bf16 -> [B, rows, out_dim]."""
        # nn.RMSNorm(hidden_dim) has eps=None: torch then takes the epsilon of the float accumulation type, 2^-23, for
        # bf16 input too (pinned by tests/golden/chroma_golden.pt).  torch multiplies by the norm weight before its one
        # bf16 rounding; rmsnorm_fwd rounds the normalised value first (T5LayerNorm order), one rounding step apart.
        eps = torch.finfo(torch.float32).eps
        B, R, _ = x.shape
        h = ops.gemm([x.reshape(1, B * R, -1)], [self.in_proj.weight], self.in_proj.bias)
        nxt = torch.empty_like(h)
        # x + bf16(linear_2(...)) rounded once more, the reference's bf16 residual add: GATE_RES with a gate of ones
        ones = torch.ones((1, h.shape[-1]), device=h.device, dtype=h.dtype)
        for layer, norm in zip(self.layers, self.norms):
            n = ops.rmsnorm_fwd(h, norm.weight, eps)
            a = ops.gemm([n], [layer.linear_1.weight], layer.linear_1.bias, epi=ops.EPI_SILU)
            ops.gemm([a], [layer.linear_2.weight], layer.linear_2.bias, out=nxt, epi=ops.EPI_GATE_RES, gate=ones, res=h)
            h, nxt = nxt, h
        return ops.gemm([h], [self.out_proj.weight], self.out_proj.bias).view(B, R, -1)


class ChromaTransformerBlock(FluxTransformerBlock):
    """reference ChromaTransformerBlock (:447-616): a Flux double block without norm1.linear / norm1_context.linear."""

    def __init__(self, dim, heads, head_dim, dtype):
        nn.Module.__init__(self)
        self.dim, self.heads, self.head_dim = dim, heads, head_dim
        self.attn = FluxAttention(dim, heads, head_dim, True, dtype)
        self.ff = _FeedForward(dim, dtype)
        self.ff_context = _FeedForward(dim, dtype)
        self._plans = None

    def forward(self, h, mod_img, mod_txt, cos, sin, S_txt, lora_scaling, key_bias=None):
        a = self.attn
        attn_l = [a.to_q, a.to_k, a.to_v, a.to_out[0], a.add_q_proj, a.add_k_proj, a.add_v_proj, a.to_add_out]
        mlp_l = [self.ff.net[0].proj, self.ff.net[2], self.ff_context.net[0].proj, self.ff_context.net[2]]
        return run_double_block(self, h, mod_img, mod_txt, cos, sin, S_txt, lora_scaling, key_bias, None, attn_l, mlp_l)


class ChromaSingleTransformerBlock(FluxSingleTransformerBlock):
    """reference ChromaSingleTransformerBlock (:316-444): a Flux single block without norm.linear."""

    def __init__(self, dim, heads, head_dim, dtype):
        nn.Module.__init__(self)
        self.dim, self.heads, self.head_dim = dim, heads, head_dim
        self.proj_mlp = Linear(dim, 4 * dim, dtype=dtype)
        self.proj_out = Linear(5 * dim, dim, dtype=dtype)
        self.attn = FluxAttention(dim, heads, head_dim, False, dtype)
        self._plans = None

    def forward(self, h, mod, cos, sin, lora_scaling, key_bias=None):
        return run_single_block(self, h, mod, cos, sin, lora_scaling, key_bias, None)


class ChromaTransformer2DModel(FluxTransformer2DModel):
    """Constructor arguments and state-dict names of the reference ChromaTransformer2DModel (:650-762).  The reference's
    `time_text_embed` holds only the non-persistent `mod_proj` buffer, and `pos_embed` / `norm_out` hold no parameters, so
    none of them appears here; `mod_proj` is rebuilt on the host at first use."""

    _no_split_modules = ["ChromaTransformerBlock", "ChromaSingleTransformerBlock"]
    _DEFAULT_LORA_TARGETS = CHROMA_DEFAULT_LORA_TARGET

    def __init__(self, patch_size: int = 1, in_channels: int = 64, out_channels: Optional[int] = None, num_layers: int = 19,
                 num_single_layers: int = 38, attention_head_dim: int = 128, num_attention_heads: int = 24,
                 joint_attention_dim: int = 4096, axes_dims_rope: Tuple[int, ...] = (16, 56, 56),
                 approximator_num_channels: int = 64, approximator_hidden_dim: int = 5120, approximator_layers: int = 5,
                 enable_time_sign_embed: bool = False, musubi_blocks_to_swap: int = 0, musubi_block_swap_device: str = "cpu",
                 gate_value: Optional[float] = None, deltatime_type: Optional[str] = None, dtype=torch.bfloat16, **unused):
        nn.Module.__init__(self)
        if attention_head_dim not in (64, 128):
            raise NotImplementedError("libstb200 attention supports head_dim 64 / 128")
        if patch_size != 1 or in_channels != 64 or (out_channels or in_channels) != in_channels:
            raise NotImplementedError("libstb200 Chroma takes 2x2-packed 16-channel latents (patch_size 1, in_channels 64)")
        if enable_time_sign_embed:
            raise NotImplementedError("Chroma with enable_time_sign_embed (TwinFlow) is not supported by the libstb200 path")
        if musubi_blocks_to_swap:
            raise NotImplementedError("musubi block swap is not supported by the libstb200 path")
        if deltatime_type is not None:
            raise NotImplementedError("Chroma FlowMap time conditioning is not supported by the libstb200 path")
        if approximator_num_channels % 8:
            raise NotImplementedError("libstb200 Chroma needs approximator_num_channels to be a multiple of 8")
        self.config = SimpleNamespace(patch_size=patch_size, in_channels=in_channels, out_channels=in_channels,
                                      num_layers=num_layers, num_single_layers=num_single_layers,
                                      attention_head_dim=attention_head_dim, num_attention_heads=num_attention_heads,
                                      joint_attention_dim=joint_attention_dim, axes_dims_rope=tuple(axes_dims_rope),
                                      approximator_num_channels=approximator_num_channels,
                                      approximator_hidden_dim=approximator_hidden_dim,
                                      approximator_layers=approximator_layers, enable_time_sign_embed=False,
                                      musubi_blocks_to_swap=0, musubi_block_swap_device=musubi_block_swap_device,
                                      gate_value=gate_value, deltatime_type=None, guidance_embeds=False)
        self.out_channels = in_channels
        self.inner_dim = D = num_attention_heads * attention_head_dim
        self.mod_rows = 3 * num_single_layers + 2 * 6 * num_layers + 2
        self.distilled_guidance_layer = ChromaApproximator(approximator_num_channels, D, approximator_hidden_dim,
                                                           approximator_layers, dtype)
        self.context_embedder = Linear(joint_attention_dim, D, dtype=dtype)
        self.x_embedder = Linear(in_channels, D, dtype=dtype)
        self.transformer_blocks = nn.ModuleList(
            [ChromaTransformerBlock(D, num_attention_heads, attention_head_dim, dtype) for _ in range(num_layers)])
        self.single_transformer_blocks = nn.ModuleList(
            [ChromaSingleTransformerBlock(D, num_attention_heads, attention_head_dim, dtype) for _ in range(num_single_layers)])
        self.proj_out = Linear(D, patch_size * patch_size * self.out_channels, dtype=dtype)
        self.gradient_checkpointing = False
        self._rope_cache: Dict[Any, Tuple[torch.Tensor, ...]] = {}
        self._mod_proj: Optional[torch.Tensor] = None
        self._tail_plan = None
        self._lora_scaling = 1.0
        self.peft_config: Dict[str, Any] = {}

    def mod_proj(self) -> torch.Tensor:
        if self._mod_proj is None:
            self._mod_proj = chroma_mod_proj(self.mod_rows, self.config.approximator_num_channels // 4)
        return self._mod_proj

    def pooled_temb(self, timestep: torch.Tensor) -> torch.Tensor:
        """The approximator output [B, rows, D] for the model-dtype timesteps `timestep.to(dtype) * 1000` (:857-864)."""
        with torch.no_grad():
            return self.distilled_guidance_layer(chroma_input_vec(timestep, self.mod_proj()))

    def modulations(self, pooled: torch.Tensor):
        """The modulation rows of every block from pooled_temb [B, rows, D] (reference :966-979, :1136-1148, :1337-1339):
        ([(image [B, 6D], text [B, 6D]) per double block], [[B, 3D] per single block], norm_out [B, 2D]).  The block rows
        are views (batch stride rows x D); norm_out's rows are (shift, scale) and TailFn reads (scale | shift), so that
        one is a [B, 2D] copy."""
        B, D = pooled.shape[0], pooled.shape[2]
        n_single = len(self.single_transformer_blocks)
        img0, txt0 = 3 * n_single, 3 * n_single + 6 * len(self.transformer_blocks)
        double = [(pooled[:, img0 + 6 * i:img0 + 6 * i + 6].flatten(1, 2), pooled[:, txt0 + 6 * i:txt0 + 6 * i + 6].flatten(1, 2))
                  for i in range(len(self.transformer_blocks))]
        single = [pooled[:, 3 * i:3 * i + 3].flatten(1, 2) for i in range(n_single)]
        return double, single, pooled[:, -2:].flip(1).reshape(B, 2 * D)

    def forward(self, hidden_states: torch.Tensor, encoder_hidden_states: torch.Tensor = None,
                timestep: torch.Tensor = None, timestep_sign=None, r_timestep=None, img_ids: torch.Tensor = None,
                txt_ids: torch.Tensor = None, attention_mask: Optional[torch.Tensor] = None,
                joint_attention_kwargs: Optional[Dict[str, Any]] = None, controlnet_block_samples=None,
                controlnet_single_block_samples=None, return_dict: bool = True, controlnet_blocks_repeat: bool = False,
                force_keep_mask=None, hidden_states_buffer=None, skip_layers=None, grounding_kwargs=None):
        """hidden_states [B, S_img, 64] packed latents, encoder_hidden_states [B, S_txt, joint_attention_dim] (T5),
        timestep [B] in [0, 1], attention_mask the joint bool [B, S_txt + S_img] mask (None: nothing masked).
        Returns (Tensor[B, S_img, 64],)."""
        for nm, v in (("timestep_sign", timestep_sign), ("r_timestep", r_timestep),
                      ("controlnet_block_samples", controlnet_block_samples),
                      ("controlnet_single_block_samples", controlnet_single_block_samples),
                      ("force_keep_mask", force_keep_mask), ("hidden_states_buffer", hidden_states_buffer),
                      ("skip_layers", skip_layers), ("grounding_kwargs", grounding_kwargs)):
            if v is not None:
                raise NotImplementedError(f"libstb200 Chroma path does not support `{nm}`; use the reference module")
        if joint_attention_kwargs and set(joint_attention_kwargs) - {"scale"}:
            raise NotImplementedError(f"joint_attention_kwargs {sorted(joint_attention_kwargs)} are not supported by the "
                                      "libstb200 path")
        # joint_attention_kwargs["scale"] multiplies every adapter's scaling for this call (:841-848, scale_lora_layers)
        lora_scale = float((joint_attention_kwargs or {}).get("scale", 1.0))
        if timestep.ndim != 1:
            raise NotImplementedError("token-wise timesteps are not supported by the libstb200 Chroma path")
        if not hidden_states.is_cuda:
            from .._lib import StbError
            raise StbError("ChromaTransformer2DModel (libstb200) needs CUDA tensors; there is no CPU fallback")
        dt = self.x_embedder.weight.dtype
        B, S_img, _ = hidden_states.shape
        S_txt = encoder_hidden_states.shape[1]
        D = self.inner_dim
        dev = hidden_states.device
        h = torch.empty((B, S_txt + S_img, D), device=dev, dtype=dt)      # joint buffer [text | image]
        blocks = list(self.transformer_blocks) + list(self.single_transformer_blocks)
        self._begin_lora_dropout(blocks + [self.proj_out, self.x_embedder])
        self._embed_image(hidden_states.to(dt), h[:, S_txt:])
        ops.gemm([encoder_hidden_states.to(dt).contiguous()], [self.context_embedder.weight], self.context_embedder.bias,
                 out=h[:, :S_txt])
        pooled = self.pooled_temb(timestep.to(device=dev).to(dt) * 1000)
        if txt_ids.ndim == 3:
            txt_ids = txt_ids[0]
        if img_ids.ndim == 3:
            img_ids = img_ids[0]
        cos, sin = self._rope(txt_ids, img_ids, dev)[:2]
        # one bias for every block, passed as an argument so that checkpoint re-runs see it
        key_bias = None if attention_mask is None else chroma_key_bias(attention_mask.to(dev, non_blocking=True), B,
                                                                       S_txt + S_img, dt)
        scaling = self._lora_scaling * lora_scale
        double, single, tail = self.modulations(pooled)
        for i, blk in enumerate(self.transformer_blocks):
            h = self._run_block(i, blk, h, *double[i], cos, sin, S_txt, scaling, key_bias)
        for i, blk in enumerate(self.single_transformer_blocks):
            h = self._run_block(i, blk, h, single[i], cos, sin, scaling, key_bias)
        out = self._tail(h, tail, S_txt, S_txt + S_img, scaling)
        if not return_dict:
            return (out,)
        return SimpleNamespace(sample=out)
