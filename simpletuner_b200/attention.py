"""Autograd wrapper around the libstb200 attention kernels: the training-capable replacement for
`F.scaled_dot_product_attention` / flash-attn's packed functions at the reference's attention seams
(flux/transformer.py:200-207; helpers/training/attention_backend.py:236-254, 479-554, 1554-1574)."""
from __future__ import annotations

from typing import Optional

import torch

from . import ops


class _AttnFn(torch.autograd.Function):
    """q, k, v: [B, S, H, HD] bf16 views (HD contiguous) -> o [B, Sq, H, HD].  key_bias: bf16 [B or 1, Sk] or None
    (no gradient: it is a mask)."""

    @staticmethod
    def forward(ctx, q, k, v, scale, key_bias=None):
        o, lse = ops.attn_fwd(q, k, v, scale, key_bias=key_bias)
        ctx.save_for_backward(q, k, v, o, lse, key_bias)
        ctx.scale = scale
        return o

    @staticmethod
    def backward(ctx, d_o):
        q, k, v, o, lse, key_bias = ctx.saved_tensors
        if d_o.stride(-1) != 1:
            d_o = d_o.contiguous()
        dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse, ctx.scale, key_bias=key_bias)
        return dq, dk, dv, None, None


class _AttnPackedFn(torch.autograd.Function):
    """qkv: [B, S, 3, H, HD]; gradients are written straight into one [B, S, 3, H, HD] buffer (strided outputs)."""

    @staticmethod
    def forward(ctx, qkv, scale, key_bias=None):
        q, k, v = qkv.unbind(2)
        o, lse = ops.attn_fwd(q, k, v, scale, key_bias=key_bias)
        ctx.save_for_backward(qkv, o, lse, key_bias)
        ctx.scale = scale
        return o

    @staticmethod
    def backward(ctx, d_o):
        qkv, o, lse, key_bias = ctx.saved_tensors
        q, k, v = qkv.unbind(2)
        if d_o.stride(-1) != 1:
            d_o = d_o.contiguous()
        d_qkv = torch.empty_like(qkv)
        dq, dk, dv = d_qkv.unbind(2)
        ops.attn_bwd(q, k, v, o, d_o, lse, ctx.scale, dq=dq, dk=dk, dv=dv, key_bias=key_bias)
        return d_qkv, None, None


def _check(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise ops._lib.StbError(f"{name} must be a CUDA tensor (libstb200 has no CPU path)")
    if t.dtype != torch.bfloat16:
        raise NotImplementedError(f"libstb200 attention computes in bf16; {name} is {t.dtype}")
    if t.shape[-1] not in (64, 128):
        raise NotImplementedError(f"libstb200 attention supports head_dim 64 / 128, got {t.shape[-1]}")


def _check_key_bias(key_bias: Optional[torch.Tensor]):
    if key_bias is not None and (not key_bias.is_cuda or key_bias.dtype != torch.bfloat16):
        raise NotImplementedError(f"key_bias must be a bf16 CUDA tensor, got {key_bias.dtype} on {key_bias.device}")


def attention_bshd(q, k, v, softmax_scale: Optional[float] = None, key_bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q/k/v [B, S, H, HD] -> [B, Sq, H, HD], differentiable in q, k, v.  key_bias: bf16 [B or 1, Sk] added to the scaled
    logits of every head and query (SDPA's float `attn_mask` of shape [B, 1, 1, Sk])."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _check(t, n)
    _check_key_bias(key_bias)
    return _AttnFn.apply(q, k, v, softmax_scale, key_bias)


def attention_qkvpacked(qkv, softmax_scale: Optional[float] = None, key_bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    _check(qkv, "qkv")
    if qkv.dim() != 5 or qkv.shape[2] != 3:
        raise ValueError(f"qkv must be [B, S, 3, H, HD], got {tuple(qkv.shape)}")
    _check_key_bias(key_bias)
    return _AttnPackedFn.apply(qkv, softmax_scale, key_bias)
