"""PixArt-Sigma full fine-tune (model_type=full) block schedule on libstb200.

The LoRA schedule (transformer.py::PixArtBlockFn) differentiates w.r.t. the hidden state and the adapter matrices only.
Here every parameter of the block receives its gradient, as `loss.backward()` through diffusers' BasicTransformerBlock
(norm_type="ada_norm_single") produces it in the reference:

  * weights of attn1 q | k | v, attn2 q, attn2 k | v (over the caption tokens), both output projections and both
    FeedForward linears: `ops.wgrad_full`, dW = dY^T X over the token rows;
  * their biases: per-(batch, column) token sums `ops.colsum2(dy)[0]`, summed over the batch;
  * the modulation mod = scale_shift_table + t6 [B, 6D]: d shift / d scale = colsum2(d_nh, LayerNorm(x)), d gate =
    colsum2(dh, pre-gate output), the pre-gate output kept through the GATE_RES aux output.  The block returns d mod; torch
    autograd turns it into d scale_shift_table (the sum over the batch) and d t6 (summed over the blocks by the engine);
  * d ctx from the k | v dgrad, so that the caption projection trains too (CaptionProjectionFullFn).

Padded heads: the q / k / v / out weights live in the head_dim 72 -> 128 zero-padded layout the forward uses.  Their
gradients are computed on that layout and the real rows (q / k / v) or columns (out) are gathered with the model's
`_pad_index`; gradients of padding entries are dropped, including the query-side mask column of the padded to_q bias and
the -10000 / scale key column of cross attention.  The padded layouts are derived data, rebuilt after every optimizer step.

The forward is PixArtBlockFn's without adapters: same kernels, same padded per-head layouts, same key mask in the first
padding column; only the two gated linears also write their pre-gate outputs.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from .. import ops
from ..flux.blocks import EPS, MlpPlan

# the block-local parameters PixArtBlockFullFn differentiates, in its argument order (scale_shift_table is reached
# through `mod` instead)
BLOCK_PARAMS = [f"{a}.{p}.{w}" for a in ("attn1", "attn2") for p in ("to_q", "to_k", "to_v", "to_out.0")
                for w in ("weight", "bias")] + [f"ff.{p}.{w}" for p in ("net.0.proj", "net.2") for w in ("weight", "bias")]


def _bias_grad(dy: torch.Tensor) -> torch.Tensor:
    return ops.colsum2(dy)[0].sum(0).to(torch.bfloat16)


def _ln(x: torch.Tensor, zero: torch.Tensor) -> torch.Tensor:
    """LayerNorm(x) without affine (bf16), via the modulate kernel with zero shift / scale."""
    return ops.ln_modulate_fwd(x, zero, zero, EPS)


class PixArtBlockFullFn(torch.autograd.Function):
    """h3 = BasicTransformerBlock(h) with gradients for every block parameter.

    inputs: h [B, S, D], enc [B, St, Dc] (projected caption), kbias [B, St] bf16 or None, mod [B, 6D], st, then the block's
    parameters in BLOCK_PARAMS order (the padded / fused / transposed layouts come from st["plans"])."""

    @staticmethod
    def forward(ctx_, h, enc, kbias, mod, st, *params):
        B, S, D = h.shape
        H, hd, hdp = st["H"], st["hd"], st["hdp"]
        Hp = H * hdp
        pl = st["plans"]
        scale = hd ** -0.5
        dev = h.device
        y_attn = torch.empty_like(h)      # pre-gate outputs of the two gated linears: the gate gradients need them
        y_mlp = torch.empty_like(h)
        # ---- self attention
        nh = ops.ln_modulate_fwd(h, mod[:, 0:D], mod[:, D:2 * D], EPS)
        qkv = ops.gemm([nh], [pl["w_qkv1"]], pl["b_qkv1"])
        del nh
        q5 = qkv.view(B, S, 3, H, hdp)
        o, lse = ops.attn_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], scale=scale)
        o = o.view(B, S, Hp)
        h1 = ops.gemm([o], [pl["w_out1"]], pl["b_out1"], epi=ops.EPI_GATE_RES, gate=mod[:, 2 * D:3 * D], res=h, aux=y_attn)
        # ---- cross attention on the un-normed stream
        q2 = ops.gemm([h1], [pl["w_q2"]], pl["b_q2"])
        kv2 = ops.gemm([enc], [pl["w_kv2"]], pl["b_kv2"])
        St = enc.shape[1]
        kv5 = kv2.view(B, St, 2, H, hdp)
        if kbias is not None:
            kv5[:, :, 0, :, hd] = kbias[:, :, None]          # mask column (transformer.py module docstring)
        o2, lse2 = ops.attn_fwd(q2.view(B, S, H, hdp), kv5[:, :, 0], kv5[:, :, 1], scale=scale)
        o2 = o2.view(B, S, Hp)
        h2 = ops.gemm([o2], [pl["w_out2"]], pl["b_out2"], epi=ops.EPI_ADD_RES, res=h1)
        # ---- feed forward
        mp: MlpPlan = pl["mlp"]
        nh2 = ops.ln_modulate_fwd(h2, mod[:, 3 * D:4 * D], mod[:, 4 * D:5 * D], EPS)
        pre = torch.empty((B, S, mp.w1.shape[0]), device=dev, dtype=torch.bfloat16)
        act = ops.gemm([nh2], [mp.w1], mp.b1, epi=ops.EPI_GELU, aux=pre)
        del nh2
        h3 = ops.gemm([act], [mp.w2], mp.b2, epi=ops.EPI_GATE_RES, gate=mod[:, 5 * D:6 * D], res=h2, aux=y_mlp)
        del act
        ctx_.st = st
        ctx_.save_for_backward(h, enc, mod, qkv, o, lse, h1, q2, kv2, o2, lse2, h2, pre, y_attn, y_mlp)
        return h3

    @staticmethod
    def backward(ctx_, dh3):
        h, enc, mod, qkv, o, lse, h1, q2, kv2, o2, lse2, h2, pre, y_attn, y_mlp = ctx_.saved_tensors
        st = ctx_.st
        B, S, D = h.shape
        H, hd, hdp = st["H"], st["hd"], st["hdp"]
        St = enc.shape[1]
        pl = st["plans"]
        mp: MlpPlan = pl["mlp"]
        scale = hd ** -0.5
        ridx = st["pad_index"]                     # real row / column of each un-padded feature (None: no padding)
        rows = (lambda g: g) if ridx is None else (lambda g: g.index_select(0, ridx))
        cols = (lambda g: g) if ridx is None else (lambda g: g.index_select(1, ridx))
        G: Dict[str, torch.Tensor] = {}
        dm = torch.empty((B, 6 * D), device=h.device, dtype=torch.float32)
        zero = torch.zeros((B, D), device=h.device, dtype=torch.bfloat16)
        dh3 = dh3.contiguous()
        # ---- feed forward: h3 = h2 + gate_mlp * fc2(gelu(fc1(LNmod(h2))))
        dm[:, 5 * D:6 * D] = ops.colsum2(dh3, y_mlp, want_sum=False)[1]
        g = ops.gate_mul(dh3, mod[:, 5 * D:6 * D])
        G["ff.net.2.weight"] = ops.wgrad_full(g, ops.gelu_tanh(pre))
        G["ff.net.2.bias"] = _bias_grad(g)
        d_pre = ops.gemm([g], [mp.w2_t], None, epi=ops.EPI_MUL_DGELU, aux=pre)
        del g
        nh2 = ops.ln_modulate_fwd(h2, mod[:, 3 * D:4 * D], mod[:, 4 * D:5 * D], EPS)
        G["ff.net.0.proj.weight"] = ops.wgrad_full(d_pre, nh2)
        G["ff.net.0.proj.bias"] = _bias_grad(d_pre)
        del nh2
        d_nh2 = ops.gemm([d_pre], [mp.w1_t], None)
        del d_pre
        dm[:, 3 * D:4 * D], dm[:, 4 * D:5 * D] = ops.colsum2(d_nh2, _ln(h2, zero))
        dh2 = ops.ln_modulate_bwd(d_nh2, h2, mod[:, 4 * D:5 * D], add=dh3, eps=EPS)
        del d_nh2
        # ---- cross attention: h2 = h1 + to_out2(attn(q2(h1), kv2(ctx)))
        G["attn2.to_out.0.weight"] = cols(ops.wgrad_full(dh2, o2))
        G["attn2.to_out.0.bias"] = _bias_grad(dh2)
        d_o2 = ops.gemm([dh2], [pl["w_out2_t"]], None)
        kv5 = kv2.view(B, St, 2, H, hdp)
        d_q2 = torch.empty_like(q2)
        d_kv2 = torch.empty_like(kv2)
        dkv5 = d_kv2.view(B, St, 2, H, hdp)
        ops.attn_bwd(q2.view(B, S, H, hdp), kv5[:, :, 0], kv5[:, :, 1], o2.view(B, S, H, hdp), d_o2.view(B, S, H, hdp), lse2,
                     scale=scale, dq=d_q2.view(B, S, H, hdp), dk=dkv5[:, :, 0], dv=dkv5[:, :, 1])
        del d_o2
        G["attn2.to_q.weight"] = rows(ops.wgrad_full(d_q2, h1))
        G["attn2.to_q.bias"] = rows(_bias_grad(d_q2))
        dh1 = ops.gemm([d_q2], [pl["w_q2_t"]], None, epi=ops.EPI_ADD_RES, res=dh2)
        del d_q2, dh2
        Hp = H * hdp
        dw_kv = ops.wgrad_full(d_kv2, enc)
        db_kv = _bias_grad(d_kv2)
        for m, n in enumerate(("to_k", "to_v")):
            G[f"attn2.{n}.weight"] = rows(dw_kv[m * Hp:(m + 1) * Hp])
            G[f"attn2.{n}.bias"] = rows(db_kv[m * Hp:(m + 1) * Hp])
        del dw_kv
        # padded k / v rows of w_kv2 are zero, so the mask column's dk does not reach d ctx
        d_enc = ops.gemm([d_kv2], [pl["w_kv2_t"]], None)
        del d_kv2
        # ---- self attention: h1 = h + gate_msa * to_out1(attn(qkv(LNmod(h))))
        dm[:, 2 * D:3 * D] = ops.colsum2(dh1, y_attn, want_sum=False)[1]
        g1 = ops.gate_mul(dh1, mod[:, 2 * D:3 * D])
        G["attn1.to_out.0.weight"] = cols(ops.wgrad_full(g1, o))
        G["attn1.to_out.0.bias"] = _bias_grad(g1)
        d_o = ops.gemm([g1], [pl["w_out1_t"]], None)
        del g1
        q5 = qkv.view(B, S, 3, H, hdp)
        d_qkv = torch.empty_like(qkv)
        dq5 = d_qkv.view(B, S, 3, H, hdp)
        ops.attn_bwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], o.view(B, S, H, hdp), d_o.view(B, S, H, hdp), lse, scale=scale,
                     dq=dq5[:, :, 0], dk=dq5[:, :, 1], dv=dq5[:, :, 2])
        del d_o
        nh = ops.ln_modulate_fwd(h, mod[:, 0:D], mod[:, D:2 * D], EPS)
        dw_qkv = ops.wgrad_full(d_qkv, nh)
        db_qkv = _bias_grad(d_qkv)
        del nh
        for m, n in enumerate(("to_q", "to_k", "to_v")):
            G[f"attn1.{n}.weight"] = rows(dw_qkv[m * Hp:(m + 1) * Hp])
            G[f"attn1.{n}.bias"] = rows(db_qkv[m * Hp:(m + 1) * Hp])
        del dw_qkv
        d_nh = ops.gemm([d_qkv], [pl["w_qkv1_t"]], None)
        del d_qkv
        dm[:, 0:D], dm[:, D:2 * D] = ops.colsum2(d_nh, _ln(h, zero))
        dh = ops.ln_modulate_bwd(d_nh, h, mod[:, D:2 * D], add=dh1, eps=EPS)
        grads: List[Optional[torch.Tensor]] = [G[n] for n in BLOCK_PARAMS]
        return (dh, d_enc, None, dm.to(mod.dtype), None, *grads)


class PatchEmbedFullFn(torch.autograd.Function):
    """PatchEmbed as the forward runs it (a GEMM over the (c, dy, dx) patch features, + the sincos table in the epilogue)
    with gradients for the conv weight [D, C, 2, 2] and bias.  No input gradient: the latents are data."""

    @staticmethod
    def forward(ctx, x, pos, w_pe, b_pe):
        D = w_pe.shape[0]
        h = ops.gemm([x], [w_pe.detach().reshape(D, -1)], b_pe.detach(), epi=ops.EPI_ADD_RES, res=pos)
        ctx.save_for_backward(x)
        ctx.w_shape = tuple(w_pe.shape)
        return h

    @staticmethod
    def backward(ctx, dh):
        (x,) = ctx.saved_tensors
        dh = dh.contiguous()
        return None, None, ops.wgrad_full(dh, x).reshape(ctx.w_shape), _bias_grad(dh)


class CaptionProjectionFullFn(torch.autograd.Function):
    """PixArtAlphaTextProjection: linear_2(gelu_tanh(linear_1(x))) with gradients for both linears.  Its input gradient
    d ctx is the sum of the blocks' k / v dgrads; the caption embeddings themselves are data."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2):
        B, St, _ = x.shape
        pre = torch.empty((B, St, w1.shape[0]), device=x.device, dtype=torch.bfloat16)
        act = ops.gemm([x], [w1.detach()], b1.detach(), epi=ops.EPI_GELU, aux=pre)
        out = ops.gemm([act], [w2.detach()], b2.detach())
        ctx.save_for_backward(x, pre, w2)
        return out

    @staticmethod
    def backward(ctx, d_out):
        x, pre, w2 = ctx.saved_tensors
        d_out = d_out.contiguous()
        dw2 = ops.wgrad_full(d_out, ops.gelu_tanh(pre))
        db2 = _bias_grad(d_out)
        d_pre = ops.gemm([d_out], [ops.WT(w2.detach())], None, epi=ops.EPI_MUL_DGELU, aux=pre)
        return None, ops.wgrad_full(d_pre, x), _bias_grad(d_pre), dw2, db2
