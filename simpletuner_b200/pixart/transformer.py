"""PixArtTransformer2DModel on libstb200 — B200-native drop-in for reference
simpletuner/helpers/models/pixart/transformer.py:148-853 (class PixArtTransformer2DModel), LoRA-training path.

Same constructor arguments / `.config`, forward signature (`hidden_states [B,4,H,W]`, `encoder_hidden_states`,
`timestep [B]`, `added_cond_kwargs{resolution, aspect_ratio}`, `encoder_attention_mask [B,S_txt]`,
`return_dict`) and `(Tensor[B,8,H,W],)` return; diffusers / PEFT parameter names
(`transformer_blocks.N.attn2.to_k.lora_A.default.weight`, `adaln_single.emb.resolution_embedder.linear_1.weight`,
`caption_projection.linear_1.weight`, `scale_shift_table`, `pos_embed.proj.weight` ...).

Block schedule (reference :57-145 -> diffusers BasicTransformerBlock, norm_type="ada_norm_single"), one
torch.autograd.Function per block, every arithmetic step a libstb200 kernel:
    mod = scale_shift_table + t           [B, 6D]
    LN-modulate -> fused QKV GEMM (+LoRA K-segment) -> wgmma attention -> to_out GEMM, gate + residual epilogue
    to_q GEMM | to_k,to_v GEMM on the projected caption -> wgmma cross attention -> to_out GEMM + residual epilogue
    LN-modulate -> FF GEMM (GELU epilogue) -> FF GEMM, gate + residual epilogue
head_dim 72 is not an MMA-K multiple: the projection weights are zero-padded per head to 128 once (derived,
frozen layouts), so q/k/v come out of the GEMM already in the [B,S,H,128] layout the attention kernel wants, the
padded columns contribute exact zeros, and to_out reads the padded layout through zero weight columns.
The additive -10000 key mask of cross attention (reference :562-564) rides in the first padding column:
q[..., 72] = 1 (a bias entry of the padded to_q), k[b, j, :, 72] = -10000 / scale for masked keys — masked keys get
probability exactly 0 like the reference's fp32 softmax, with no mask operand in the kernel.
Unsupported (raise): token-wise timesteps, TREAD routes, controlnet residuals, flow-map `r_timestep`, GLIGEN,
self-attention masks.  Full fine-tune (model_type=full), after `enable_full_finetune()`, runs the same `PixArtBlockFn` /
`TailFn` schedules with every Linear's (weight, bias) in the adapter slots (`PixArtTransformerBlock.block_slots`); the
patch embedding and the caption projection have Functions of their own (`PatchEmbedFullFn`, `CaptionProjectionFullFn`).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..flux.blocks import (EPS, MlpPlan, TailFn, _dmod_gate, _dmod_shift_scale, _linear_lora_dgrad, _linear_lora_fwd, _lora_grads,
                           _t, _wt, make_pack)
from ..flux.transformer import (AdapterModelAPI, AttnProcessorAPI, LoraDropoutAPI, Linear, _FeedForward, _lora_list, _sinusoid,
                                _TimestepEmbedding)
from ..pretrained import ModelConfig, PretrainedIOAPI

PIXART_LORA_TARGETS = ["to_k", "to_q", "to_v", "to_out.0"]  # PixartSigma.DEFAULT_LORA_TARGET, reference pixart/model.py:59
MASK_BIAS = -10000.0


def _pad_rows(w: torch.Tensor, H: int, hd: int, hdp: int) -> torch.Tensor:
    """[H*hd, K] -> [H*hdp, K] with zero rows after each head."""
    if hd == hdp:
        return w.contiguous()
    out = w.new_zeros((H, hdp) + tuple(w.shape[1:]))
    out[:, :hd] = w.view((H, hd) + tuple(w.shape[1:]))
    return out.view((H * hdp,) + tuple(w.shape[1:]))


def _pad_cols(w: torch.Tensor, H: int, hd: int, hdp: int) -> torch.Tensor:
    """[N, H*hd] -> [N, H*hdp]."""
    if hd == hdp:
        return w.contiguous()
    out = w.new_zeros((w.shape[0], H, hdp))
    out[:, :, :hd] = w.view(w.shape[0], H, hd)
    return out.view(w.shape[0], H * hdp)


class _Attention(nn.Module):
    """diffusers Attention(query_dim=D, cross_attention_dim=kdim, heads, dim_head, bias=True, out_bias=True)."""

    def __init__(self, dim, kdim, dtype):
        super().__init__()
        self.to_q = Linear(dim, dim, dtype=dtype)
        self.to_k = Linear(kdim, dim, dtype=dtype)
        self.to_v = Linear(kdim, dim, dtype=dtype)
        self.to_out = nn.ModuleList([Linear(dim, dim, dtype=dtype), nn.Identity()])


class PixArtBlockFn(torch.autograd.Function):
    """inputs: h [B,S,D], ctx [B,St,Dc] (projected caption), kbias [B,St] bf16 or None, mod [B,6D], st, then the
    flat LoRA tensors: attn1 to_q.A,B to_k.A,B to_v.A,B to_out.A,B [0..7]; attn2 likewise [8..15].

    Full fine-tune (st["full"]): each (A, B) slot holds that Linear's (weight, bias), slots [16..19] hold the FeedForward's
    net.0.proj and net.2 (weight, bias), and every one of them gets its gradient from its group's dW (WgradPack; padded
    heads are gathered back to the real rows / columns).  The block also returns d mod (shift / scale / gate column sums;
    the GATE_RES epilogues write the pre-gate outputs for the gates) and d ctx, through the k | v dgrad."""

    @staticmethod
    def forward(ctx_, h, enc, kbias, mod, st, *lora):
        B, S, D = h.shape
        H, hd, hdp = st["H"], st["hd"], st["hdp"]
        Hp = H * hdp
        pl = st["plans"]
        scaling, scale = st["lora_scaling"], hd ** -0.5
        ridx = st["pad_index"]
        dev = h.device
        drop = st.get("lora_drop")
        dr = (lambda off: drop.at(off)) if drop is not None else (lambda off: None)
        full = st.get("full", False)
        assert not (full and drop is not None), "full fine-tune: no LoRA dropout"
        mp: MlpPlan = pl["mlp"]

        def lp(base, n, n_out, k_in, rows):
            ps = []
            for m in range(n):
                a, b = lora[base + 2 * m], lora[base + 2 * m + 1]
                ps.append(None if a is None else (a, b))
            return make_pack(ps, n_out, k_in, scaling, dev, full=full, row_index=ridx if rows else None,
                             col_index=None if rows else ridx)

        pk = {"qkv1": lp(0, 3, Hp, D, True), "out1": lp(6, 1, D, Hp, False), "q2": lp(8, 1, Hp, D, True),
              "kv2": lp(10, 2, Hp, enc.shape[2], True), "out2": lp(14, 1, D, Hp, False)}
        if full:
            pk["fc1"] = make_pack([(lora[16], lora[17])], mp.w1.shape[0], D, scaling, dev, full=True)
            pk["fc2"] = make_pack([(lora[18], lora[19])], D, mp.w1.shape[0], scaling, dev, full=True)
        y_attn = torch.empty_like(h) if full else None      # pre-gate outputs of the gated linears: the gate gradients
        y_mlp = torch.empty_like(h) if full else None
        # ---- self attention
        nh = ops.ln_modulate_fwd(h, mod[:, 0:D], mod[:, D:2 * D], EPS)
        qkv, t_qkv = _linear_lora_fwd(nh, pl["w_qkv1"], pl["b_qkv1"], pk["qkv1"], dr(0))
        del nh
        q5 = qkv.view(B, S, 3, H, hdp)
        o, lse = ops.attn_fwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], scale=scale)
        o = o.view(B, S, Hp)
        h1, t_out1 = _linear_lora_fwd(o, pl["w_out1"], pl["b_out1"], pk["out1"], dr(3), epi=ops.EPI_GATE_RES,
                                      gate=mod[:, 2 * D:3 * D], res=h, aux=y_attn)
        # ---- cross attention on the un-normed stream (ada_norm_single: no norm2 before attn2)
        q2, t_q2 = _linear_lora_fwd(h1, pl["w_q2"], pl["b_q2"], pk["q2"], dr(4))
        kv2, t_kv2 = _linear_lora_fwd(enc, pl["w_kv2"], pl["b_kv2"], pk["kv2"], dr(5))
        St = enc.shape[1]
        kv5 = kv2.view(B, St, 2, H, hdp)
        if kbias is not None:
            kv5[:, :, 0, :, hd] = kbias[:, :, None]          # mask column (see module docstring)
        o2, lse2 = ops.attn_fwd(q2.view(B, S, H, hdp), kv5[:, :, 0], kv5[:, :, 1], scale=scale)
        o2 = o2.view(B, S, Hp)
        h2, t_out2 = _linear_lora_fwd(o2, pl["w_out2"], pl["b_out2"], pk["out2"], dr(7), epi=ops.EPI_ADD_RES, res=h1)
        # ---- feed forward
        nh2 = ops.ln_modulate_fwd(h2, mod[:, 3 * D:4 * D], mod[:, 4 * D:5 * D], EPS)
        pre = torch.empty((B, S, mp.w1.shape[0]), device=dev, dtype=torch.bfloat16)
        act = ops.gemm([nh2], [mp.w1], mp.b1, epi=ops.EPI_GELU, aux=pre)
        del nh2
        h3 = ops.gemm([act], [mp.w2], mp.b2, epi=ops.EPI_GATE_RES, gate=mod[:, 5 * D:6 * D], res=h2, aux=y_mlp)
        del act
        ctx_.st, ctx_.pk = st, pk
        ctx_.lora_present = [x is not None for x in lora]
        E = h.new_empty(0)
        keep = lambda t: t if t is not None else E
        ctx_.save_for_backward(h, enc, mod, qkv, o, lse, h1, q2, kv2, o2, lse2, h2, pre, keep(t_qkv), keep(t_out1),
                               keep(t_q2), keep(t_kv2), keep(t_out2), keep(y_attn), keep(y_mlp))
        return h3

    @staticmethod
    def backward(ctx_, dh3):
        (h, enc, mod, qkv, o, lse, h1, q2, kv2, o2, lse2, h2, pre, t_qkv, t_out1, t_q2, t_kv2, t_out2, y_attn,
         y_mlp) = ctx_.saved_tensors
        st, pk = ctx_.st, ctx_.pk
        B, S, D = h.shape
        H, hd, hdp = st["H"], st["hd"], st["hdp"]
        Hp = H * hdp
        St = enc.shape[1]
        pl = st["plans"]
        mp: MlpPlan = pl["mlp"]
        scale = hd ** -0.5
        grads: List[Optional[torch.Tensor]] = [None] * len(ctx_.lora_present)
        drop = st.get("lora_drop")
        dr = (lambda off: drop.at(off)) if drop is not None else (lambda off: None)
        full = st.get("full", False)
        dm = torch.empty((B, 6 * D), device=h.device, dtype=torch.float32) if full else None   # every chunk is written
        dh3 = dh3.contiguous()
        # ---- feed forward: h3 = h2 + gate_mlp * fc2(gelu(fc1(LNmod(h2))))
        if full:
            _dmod_gate(dm, dh3, y_mlp, 5)
        g = ops.gate_mul(dh3, mod[:, 5 * D:6 * D])
        if full:
            (grads[18], grads[19]), = _lora_grads(pk["fc2"], ops.gelu_tanh(pre), None, g, None)
        d_pre = ops.gemm([g], [mp.w2_t], None, epi=ops.EPI_MUL_DGELU, aux=pre)
        del g
        if full:
            nh2 = ops.ln_modulate_fwd(h2, mod[:, 3 * D:4 * D], mod[:, 4 * D:5 * D], EPS)
            (grads[16], grads[17]), = _lora_grads(pk["fc1"], nh2, None, d_pre, None)
            del nh2
        d_nh2 = ops.gemm([d_pre], [mp.w1_t], None)
        del d_pre
        if full:
            _dmod_shift_scale(dm, d_nh2, h2, 3, 4)
        dh2 = ops.ln_modulate_bwd(d_nh2, h2, mod[:, 4 * D:5 * D], add=dh3, eps=EPS)
        del d_nh2
        # ---- cross attention: h2 = h1 + to_out2(attn(q2(h1), kv2(ctx)))
        d_o2, t_up = _linear_lora_dgrad(dh2, pl["w_out2_t"], pk["out2"], dr(7))
        if pk["out2"] is not None:
            (grads[14], grads[15]), = _lora_grads(pk["out2"], o2, t_out2, dh2, t_up, dr(7))
        kv5 = kv2.view(B, St, 2, H, hdp)
        d_q2 = torch.empty_like(q2)
        d_kv2 = torch.empty_like(kv2)
        dkv5 = d_kv2.view(B, St, 2, H, hdp)
        ops.attn_bwd(q2.view(B, S, H, hdp), kv5[:, :, 0], kv5[:, :, 1], o2.view(B, S, H, hdp), d_o2.view(B, S, H, hdp), lse2,
                     scale=scale, dq=d_q2.view(B, S, H, hdp), dk=dkv5[:, :, 0], dv=dkv5[:, :, 1])
        del d_o2
        dh1, t_up = _linear_lora_dgrad(d_q2, pl["w_q2_t"], pk["q2"], dr(4), epi=ops.EPI_ADD_RES, res=dh2)
        if pk["q2"] is not None:
            (grads[8], grads[9]), = _lora_grads(pk["q2"], h1, t_q2, d_q2, t_up, dr(4))
        del d_q2
        if pk["kv2"] is not None:
            t_up = None if full else ops.gemm([d_kv2], [pk["kv2"].b_ext_t])
            for m, (da, db) in enumerate(_lora_grads(pk["kv2"], enc, t_kv2, d_kv2, t_up, dr(5))):
                grads[10 + 2 * m], grads[11 + 2 * m] = da, db
        # d ctx in full fine-tune only: otherwise the caption projection is frozen and carries no adapter.  The padded k / v
        # rows of w_kv2 are zero, so the mask column's dk does not reach it.
        d_enc = ops.gemm([d_kv2], [pl["w_kv2_t"]], None) if full else None
        del d_kv2
        # ---- self attention: h1 = h + gate_msa * to_out1(attn(qkv(LNmod(h))))
        if full:
            _dmod_gate(dm, dh1, y_attn, 2)
        g1 = ops.gate_mul(dh1, mod[:, 2 * D:3 * D])
        d_o, t_up = _linear_lora_dgrad(g1, pl["w_out1_t"], pk["out1"], dr(3))
        if pk["out1"] is not None:
            (grads[6], grads[7]), = _lora_grads(pk["out1"], o, t_out1, g1, t_up, dr(3))
        del g1
        q5 = qkv.view(B, S, 3, H, hdp)
        d_qkv = torch.empty_like(qkv)
        dq5 = d_qkv.view(B, S, 3, H, hdp)
        ops.attn_bwd(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], o.view(B, S, H, hdp), d_o.view(B, S, H, hdp), lse, scale=scale,
                     dq=dq5[:, :, 0], dk=dq5[:, :, 1], dv=dq5[:, :, 2])
        del d_o
        d_nh, t_up = _linear_lora_dgrad(d_qkv, pl["w_qkv1_t"], pk["qkv1"], dr(0))
        if pk["qkv1"] is not None:
            nh = ops.ln_modulate_fwd(h, mod[:, 0:D], mod[:, D:2 * D], EPS)
            for m, (da, db) in enumerate(_lora_grads(pk["qkv1"], nh, t_qkv, d_qkv, t_up, dr(0))):
                grads[2 * m], grads[2 * m + 1] = da, db
            del nh
        del d_qkv
        if full:
            _dmod_shift_scale(dm, d_nh, h, 0, 1)
        dh = ops.ln_modulate_bwd(d_nh, h, mod[:, D:2 * D], add=dh1, eps=EPS)
        out = [grads[i] if ctx_.lora_present[i] else None for i in range(len(ctx_.lora_present))]
        return (dh, d_enc, None, dm.to(mod.dtype) if full else None, None, *out)


class PixArtTransformerBlock(nn.Module):
    """BasicTransformerBlock(ada_norm_single) as configured at reference pixart/transformer.py:312-330."""

    def __init__(self, dim, heads, head_dim, cross_dim, dtype):
        super().__init__()
        self.dim, self.heads, self.head_dim = dim, heads, head_dim
        self.hdp = 64 if head_dim <= 64 else 128
        self.scale_shift_table = nn.Parameter(torch.randn(6, dim, dtype=torch.float32).div(dim ** 0.5).to(dtype), requires_grad=False)
        self.attn1 = _Attention(dim, dim, dtype)
        self.attn2 = _Attention(dim, cross_dim, dtype)
        self.ff = _FeedForward(dim, dtype)
        self._plans = None

    def plans(self):
        if self._plans is None:
            H, hd, hdp = self.heads, self.head_dim, self.hdp
            dyn = bool(getattr(self, "_full_ft", False))      # full fine-tune: the weights change every step
            wt = lambda w: _wt(w, dyn)
            pr = lambda lin: (_pad_rows(lin.weight.detach(), H, hd, hdp), _pad_rows(lin.bias.detach(), H, hd, hdp))
            a1, a2 = self.attn1, self.attn2
            (wq, bq), (wk, bk), (wv, bv) = pr(a1.to_q), pr(a1.to_k), pr(a1.to_v)
            w_qkv1 = torch.cat([wq, wk, wv], 0).contiguous()
            w_q2, b_q2 = pr(a2.to_q)
            if hdp > hd:
                b_q2 = b_q2.clone()
                b_q2.view(H, hdp)[:, hd] = 1.0           # the query side of the mask column
            (wk2, bk2), (wv2, bv2) = pr(a2.to_k), pr(a2.to_v)
            w_kv2 = torch.cat([wk2, wv2], 0).contiguous()
            w_out1 = _pad_cols(a1.to_out[0].weight.detach(), H, hd, hdp)
            w_out2 = _pad_cols(a2.to_out[0].weight.detach(), H, hd, hdp)
            ff = self.ff
            self._plans = {
                "w_qkv1": w_qkv1, "b_qkv1": torch.cat([bq, bk, bv], 0).contiguous(), "w_qkv1_t": wt(w_qkv1),
                "w_out1": w_out1, "b_out1": a1.to_out[0].bias.detach(), "w_out1_t": wt(w_out1),
                "w_q2": w_q2, "b_q2": b_q2, "w_q2_t": wt(w_q2),
                "w_kv2": w_kv2, "b_kv2": torch.cat([bk2, bv2], 0).contiguous(), "w_kv2_t": wt(w_kv2) if dyn else None,
                "w_out2": w_out2, "b_out2": a2.to_out[0].bias.detach(), "w_out2_t": wt(w_out2),
                "mlp": MlpPlan(ff.net[0].proj.weight.detach(), ff.net[0].proj.bias.detach(), wt(ff.net[0].proj.weight.detach()),
                               ff.net[2].weight.detach(), ff.net[2].bias.detach(), wt(ff.net[2].weight.detach())),
            }
        return self._plans

    def forward(self, h, ctx, kbias, t6, lora_scaling, pad_index):
        B, _, D = h.shape
        # reference :98-102 / diffusers: (scale_shift_table[None] + timestep.reshape(B, 6, -1)) in the weight dtype
        mod = (self.scale_shift_table[None] + t6.reshape(B, 6, D)).reshape(B, 6 * D)
        full = bool(getattr(self, "_full_ft", False))
        st = {"H": self.heads, "hd": self.head_dim, "hdp": self.hdp, "plans": self.plans(), "lora_scaling": lora_scaling,
              "pad_index": pad_index, "lora_drop": getattr(self, "_lora_drop", None), "full": full}
        return PixArtBlockFn.apply(h, ctx, kbias, mod, st, *self.block_slots())

    def block_slots(self):
        """PixArtBlockFn's flat slot list: the (A, B) of both attentions' projections, or in full fine-tune every Linear's
        (weight, bias), the FeedForward's included.  `scale_shift_table` trains through torch autograd on `mod`."""
        a1, a2 = self.attn1, self.attn2
        lins = [a1.to_q, a1.to_k, a1.to_v, a1.to_out[0], a2.to_q, a2.to_k, a2.to_v, a2.to_out[0]]
        if not getattr(self, "_full_ft", False):
            return _lora_list(lins)
        return [t for lin in lins + [self.ff.net[0].proj, self.ff.net[2]] for t in (lin.weight, lin.bias)]


def _bias_grad(dy: torch.Tensor) -> torch.Tensor:
    return ops.colsum2(dy)[0].sum(0).to(torch.bfloat16)


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


class _PatchEmbed(nn.Module):
    """diffusers PatchEmbed(patch_size=2, interpolation_scale=..., pos_embed_max_size=None): conv `proj`; the sincos
    table is rebuilt for the input grid (the persistent `pos_embed` buffer only serves the native sample_size)."""

    def __init__(self, in_channels, dim, patch_size, dtype):
        super().__init__()
        self.proj = nn.Conv2d(in_channels, dim, kernel_size=patch_size, stride=patch_size, bias=True, dtype=dtype)
        for p in self.proj.parameters():
            p.requires_grad_(False)


class _SizeEmbeddings(nn.Module):
    """diffusers PixArtAlphaCombinedTimestepSizeEmbeddings."""

    def __init__(self, dim, size_dim, additional: bool, dtype):
        super().__init__()
        self.timestep_embedder = _TimestepEmbedding(256, dim, dtype)
        if additional:
            self.resolution_embedder = _TimestepEmbedding(256, size_dim, dtype)
            self.aspect_ratio_embedder = _TimestepEmbedding(256, size_dim, dtype)


class _AdaLayerNormSingle(nn.Module):
    def __init__(self, dim, additional: bool, dtype):
        super().__init__()
        self.emb = _SizeEmbeddings(dim, dim // 3, additional, dtype)
        self.linear = Linear(dim, 6 * dim, dtype=dtype)


class _TextProjection(nn.Module):
    """diffusers PixArtAlphaTextProjection(act_fn="gelu_tanh")."""

    def __init__(self, in_features, dim, dtype):
        super().__init__()
        self.linear_1 = Linear(in_features, dim, dtype=dtype)
        self.linear_2 = Linear(dim, dim, dtype=dtype)

    def forward(self, x):
        return ops.gemm([ops.gemm([x], [self.linear_1.weight], self.linear_1.bias, epi=ops.EPI_GELU)],
                        [self.linear_2.weight], self.linear_2.bias)


def sincos_pos_embed_2d(dim: int, grid_h: int, grid_w: int, base_size: int, interpolation_scale: float, device) -> torch.Tensor:
    """diffusers get_2d_sincos_pos_embed for a (grid_h, grid_w) grid -> [h*w, dim] fp32; first half of the channels
    encodes the column, second half the row (meshgrid(w, h) ordering), each [sin | cos] (fp64 phase like numpy)."""
    gh = torch.arange(grid_h, dtype=torch.float32) / (grid_h / base_size) / interpolation_scale
    gw = torch.arange(grid_w, dtype=torch.float32) / (grid_w / base_size) / interpolation_scale
    col = gw[None, :].expand(grid_h, grid_w).reshape(-1).double()
    row = gh[:, None].expand(grid_h, grid_w).reshape(-1).double()
    d = dim // 2
    omega = 1.0 / 10000 ** (torch.arange(d // 2, dtype=torch.float64) / (d / 2.0))
    parts = []
    for pos in (col, row):
        ph = pos[:, None] * omega[None, :]
        parts += [torch.sin(ph), torch.cos(ph)]
    return torch.cat(parts, dim=1).float().to(device)


class PixArtTransformer2DModel(AdapterModelAPI, AttnProcessorAPI, LoraDropoutAPI, PretrainedIOAPI, nn.Module):
    _no_split_modules = ["BasicTransformerBlock", "PatchEmbed"]
    _DEFAULT_LORA_TARGETS = PIXART_LORA_TARGETS

    def __init__(self, num_attention_heads: int = 16, attention_head_dim: int = 72, in_channels: int = 4,
                 out_channels: Optional[int] = 8, num_layers: int = 28, dropout: float = 0.0, norm_num_groups: int = 32,
                 cross_attention_dim: Optional[int] = 1152, attention_bias: bool = True, sample_size: int = 128,
                 patch_size: int = 2, activation_fn: str = "gelu-approximate", num_embeds_ada_norm: Optional[int] = 1000,
                 upcast_attention: bool = False, norm_type: str = "ada_norm_single", norm_elementwise_affine: bool = False,
                 norm_eps: float = 1e-6, interpolation_scale: Optional[int] = None,
                 use_additional_conditions: Optional[bool] = None, caption_channels: Optional[int] = None,
                 attention_type: Optional[str] = "default", dtype=torch.bfloat16, **unused):
        super().__init__()
        if norm_type != "ada_norm_single":
            raise NotImplementedError(f"Forward pass is not implemented when `patch_size` is not None and `norm_type` is '{norm_type}'.")
        if patch_size != 2 or activation_fn != "gelu-approximate" or not attention_bias or dropout or norm_elementwise_affine:
            raise NotImplementedError("libstb200 PixArt path: patch_size=2, gelu-approximate, attention_bias, no dropout / affine norms")
        if attention_head_dim > 128 or attention_head_dim % 8:
            raise NotImplementedError("libstb200 attention supports head_dim <= 128 (multiple of 8)")
        if use_additional_conditions is None:
            use_additional_conditions = sample_size == 128
        out_channels = in_channels if out_channels is None else out_channels
        D = num_attention_heads * attention_head_dim
        if cross_attention_dim is None:
            cross_attention_dim = D
        self.config = ModelConfig(num_attention_heads=num_attention_heads, attention_head_dim=attention_head_dim,
                                  in_channels=in_channels, out_channels=out_channels, num_layers=num_layers,
                                  cross_attention_dim=cross_attention_dim, sample_size=sample_size, patch_size=patch_size,
                                  interpolation_scale=interpolation_scale, use_additional_conditions=use_additional_conditions,
                                  caption_channels=caption_channels, norm_type=norm_type, norm_eps=norm_eps,
                                  activation_fn=activation_fn, attention_bias=attention_bias)
        self.inner_dim, self.out_channels, self.use_additional_conditions = D, out_channels, use_additional_conditions
        self.attention_head_dim = attention_head_dim
        self.interpolation_scale = interpolation_scale if interpolation_scale is not None else max(sample_size // 64, 1)
        self.pos_embed = _PatchEmbed(in_channels, D, patch_size, dtype)
        self.transformer_blocks = nn.ModuleList([
            PixArtTransformerBlock(D, num_attention_heads, attention_head_dim, cross_attention_dim, dtype) for _ in range(num_layers)])
        self.scale_shift_table = nn.Parameter(torch.randn(2, D, dtype=torch.float32).div(D ** 0.5).to(dtype), requires_grad=False)
        self.proj_out = Linear(D, patch_size * patch_size * out_channels, dtype=dtype)
        self.adaln_single = _AdaLayerNormSingle(D, use_additional_conditions, dtype)
        self.caption_projection = _TextProjection(caption_channels, D, dtype) if caption_channels is not None else None
        self._lora_scaling = 1.0
        self._tail_plan: Dict[Any, Any] = {}
        self._pos_cache: Dict[Any, torch.Tensor] = {}
        self._pad_index: Optional[torch.Tensor] = None
        self.peft_config: Dict[str, Any] = {}
        self.gradient_checkpointing = False

    # ---- reference-facing utilities -------------------------------------------------------------
    @staticmethod
    def _lora_adaptable(name: str) -> bool:
        # the block schedule adapts the projections of both attentions only
        return ".attn1." in name or ".attn2." in name

    def invalidate_plans(self):
        self._drop_weight_layouts()
        self._pos_cache.clear()
        self._pad_index = None

    def _drop_weight_layouts(self):
        for blk in self.transformer_blocks:
            blk._plans = None
        self._tail_plan = {}

    def enable_full_finetune(self, enabled: bool = True):
        """model_type=full: every parameter trains, the blocks' `scale_shift_table` included.  The blocks run PixArtBlockFn in
        its full fine-tune mode; the padded / fused / transposed weight layouts are rebuilt after every
        optimizer step (`after_optimizer_step`) because the base weights now change."""
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
            self._drop_weight_layouts()

    def before_graph_capture(self):
        """training.step.GraphedTrainStep: in full fine-tune the weight layouts are rebuilt INSIDE the captured step.  The
        positional tables and the pad index do not depend on the weights and stay (building them copies from the host)."""
        if getattr(self, "_full_ft", False):
            self._drop_weight_layouts()

    # ---- forward --------------------------------------------------------------------------------
    def _pos(self, hp: int, wp: int, dtype, device) -> torch.Tensor:
        key = (hp, wp, dtype)
        hit = self._pos_cache.get(key)
        if hit is None:
            base = self.config.sample_size // self.config.patch_size
            hit = sincos_pos_embed_2d(self.inner_dim, hp, wp, base, self.interpolation_scale, device).to(dtype)[None].contiguous()
            self._pos_cache[key] = hit
        return hit

    def _conditioning(self, timestep, added_cond_kwargs, B, dt):
        """AdaLayerNormSingle.forward == reference :803-853 (1-D timesteps) -> (t6 [B,6D], embedded [B,D])."""
        emb = self.adaln_single.emb
        t = emb.timestep_embedder(_sinusoid(timestep.float()).to(dt))
        if self.use_additional_conditions:
            res, ar = added_cond_kwargs["resolution"], added_cond_kwargs["aspect_ratio"]
            r = emb.resolution_embedder(_sinusoid(res.flatten().float()).to(dt)).reshape(B, -1)
            a = emb.aspect_ratio_embedder(_sinusoid(ar.flatten().float()).to(dt)).reshape(B, -1)
            t = t + torch.cat([r, a], dim=1)
        return self.adaln_single.linear(F.silu(t).contiguous()), t

    def forward(self, hidden_states: torch.Tensor, encoder_hidden_states: Optional[torch.Tensor] = None,
                timestep: Optional[torch.Tensor] = None, added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
                cross_attention_kwargs: Optional[Dict[str, Any]] = None, attention_mask: Optional[torch.Tensor] = None,
                encoder_attention_mask: Optional[torch.Tensor] = None, controlnet_block_samples=None,
                controlnet_conditioning_scale: float = 1.0, return_dict: bool = True, force_keep_mask=None,
                hidden_states_buffer=None, r_timestep=None, _packed_latents: Optional[torch.Tensor] = None,
                _packed_output: bool = False):
        for nm, v in (("attention_mask", attention_mask), ("controlnet_block_samples", controlnet_block_samples),
                      ("force_keep_mask", force_keep_mask), ("r_timestep", r_timestep)):
            if v is not None:
                raise NotImplementedError(f"libstb200 PixArt path does not support `{nm}`; use the reference module")
        if cross_attention_kwargs:
            raise NotImplementedError("cross_attention_kwargs (GLIGEN / scale) are not supported by the libstb200 PixArt path")
        if self.use_additional_conditions and added_cond_kwargs is None:
            raise ValueError("`added_cond_kwargs` cannot be None when using additional conditions for `adaln_single`.")
        if timestep.ndim != 1:
            raise NotImplementedError("token-wise timesteps are not supported by the libstb200 PixArt path")
        if not hidden_states.is_cuda:
            from .._lib import StbError
            raise StbError("PixArtTransformer2DModel (libstb200) needs CUDA tensors; there is no CPU fallback")
        dt = self.proj_out.weight.dtype
        dev = hidden_states.device
        B, C, Hh, Ww = hidden_states.shape
        hp, wp = Hh // 2, Ww // 2
        S, D = hp * wp, self.inner_dim
        H, hd = self.config.num_attention_heads, self.attention_head_dim
        hdp = self.transformer_blocks[0].hdp
        # 1. input: PatchEmbed conv2x2/s2 == GEMM over (c, dy, dx) features, + sincos table in the epilogue
        x = _packed_latents if _packed_latents is not None else \
            hidden_states.to(dt).view(B, C, hp, 2, wp, 2).permute(0, 2, 4, 1, 3, 5).reshape(B, S, C * 4).contiguous()
        full = getattr(self, "_full_ft", False) and torch.is_grad_enabled()
        pos = self._pos(hp, wp, dt, dev).expand(B, S, D)
        if full:
            h = PatchEmbedFullFn.apply(x, pos, self.pos_embed.proj.weight, self.pos_embed.proj.bias)
        else:
            w_pe = self.pos_embed.proj.weight.detach().reshape(D, C * 4)
            h = ops.gemm([x], [w_pe], self.pos_embed.proj.bias.detach(), epi=ops.EPI_ADD_RES, res=pos)
        t6, embedded = self._conditioning(timestep.to(dev), added_cond_kwargs, B, dt)
        ctx = encoder_hidden_states.to(dt).contiguous()
        if self.caption_projection is not None:
            cp = self.caption_projection
            ctx = CaptionProjectionFullFn.apply(ctx, cp.linear_1.weight, cp.linear_1.bias, cp.linear_2.weight,
                                                cp.linear_2.bias) if full else cp(ctx)
        # 2. cross-attention key mask -> the padded q/k column (module docstring)
        kbias = None
        if encoder_attention_mask is not None:
            if encoder_attention_mask.ndim != 2:
                raise NotImplementedError("pass encoder_attention_mask as a [B, S_txt] keep-mask")
            if hdp == hd:
                if not bool((encoder_attention_mask != 0).all()):
                    raise NotImplementedError("masked cross attention needs head_dim < 64 or 64 < head_dim < 128")
            else:
                bias = (1 - encoder_attention_mask.to(device=dev, dtype=dt)) * MASK_BIAS     # reference :563 (bf16: -9984)
                kbias = (bias.float() / hd ** -0.5).to(dt).contiguous()
        if self._pad_index is None and hdp != hd:
            self._pad_index = (torch.arange(H, device=dev)[:, None] * hdp + torch.arange(hd, device=dev)[None, :]).reshape(-1)
        self._begin_lora_dropout(list(self.transformer_blocks))
        for i, blk in enumerate(self.transformer_blocks):
            h = self._run_block(i, blk, h, ctx, kbias, t6, self._lora_scaling, self._pad_index)
        # 3. output: LN -> (scale_shift_table + embedded) modulate -> proj_out  (reference :749-760)
        mod = (self.scale_shift_table[None] + embedded[:, None].to(self.scale_shift_table.dtype)).to(dt)  # [B, 2, D] (shift | scale)
        mod = torch.cat([mod[:, 1], mod[:, 0]], dim=1).contiguous()                                         # TailFn wants (scale | shift)
        keep = self.out_channels // 2 if _packed_output == "eps_half" else self.out_channels
        out = self._tail(h, mod, keep, full)
        if not _packed_output:
            Co = self.out_channels
            out = torch.einsum("nhwpqc->nchpwq", out.reshape(B, hp, wp, 2, 2, Co)).reshape(B, Co, hp * 2, wp * 2)
        if not return_dict:
            return (out,)
        return SimpleNamespace(sample=out)

    def _tail_rows(self, keep: int, dev) -> Optional[torch.Tensor]:
        """The proj_out rows of the first `keep` output channels ((dy, dx, c) row order); None: every row."""
        if keep == self.out_channels:
            return None
        return (torch.arange(4, device=dev)[:, None] * self.out_channels + torch.arange(keep, device=dev)[None, :]).reshape(-1)

    def _tail(self, h, mod, keep, full):
        """full: proj_out's kept rows are TailFn's slot, so proj_out and the modulation get gradients; the gather hands the
        learned-sigma rows an explicit zero gradient, as the reference's `.chunk(2, dim=1)[0]` does."""
        tp = self._tail_plan.get(keep)
        sel = self._tail_rows(keep, h.device) if tp is None or full else None
        if tp is None:
            w, b = self.proj_out.weight.detach(), self.proj_out.bias.detach()
            if sel is not None:   # PixartSigma keeps `.chunk(2, dim=1)[0]` only (pixart/model.py:313): skip the rest
                w, b = w[sel].contiguous(), b[sel].contiguous()
            tp = {"w_proj": w, "b_proj": b, "w_proj_t": _wt(w)}
            self._tail_plan[keep] = tp
        slot = ()
        if full:
            w, b = self.proj_out.weight, self.proj_out.bias
            slot = (w, b) if sel is None else (w[sel], b[sel])
        return TailFn.apply(h, mod, {"S_txt": 0, "full": full, **tp}, *slot)          # [B, S, 4 * keep] in (dy, dx, c) order
