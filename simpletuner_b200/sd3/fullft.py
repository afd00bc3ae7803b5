"""Full fine-tune (model_type=full, BASELINE configs[2]: SD3 MMDiT full FT) block schedules on libstb200.

The LoRA schedule (flux/blocks.py::DoubleBlockFn) only differentiates w.r.t. the hidden state and the adapter matrices.
Here EVERY parameter of the joint block receives its gradient — what `accelerator.backward(loss)` produces through
diffusers' JointTransformerBlock in the reference (trainer.py:7126; sd3/transformer.py:145-241):

  * weights of the fused q|k|v projections, the output projections and both FeedForward linears: `ops.wgrad_full`
    (wgmma, both operands MN-major; csrc/wgrad.cuh) — dW = dY^T X over the token rows, 2 M N K flops each, i.e.
    the full-FT step is 3x the forward's linear work (BASELINE.md 3: 6.8 TF per SD3.5-medium sample);
  * biases and the adaLN chunks (shift / scale / gate of norm1, norm1_context, the dual-attention norm): per-(batch, column)
    token reductions `ops.colsum2` (sum_s dy, sum_s dy * z with z = LayerNorm(x) or the gated linear output that the
    GATE_RES epilogue now also writes);
  * the per-head RMSNorm weights of q / k (SD3.5 qk_norm="rms_norm"): 4 x [head_dim] vectors per attention, accumulated
    inside the RMSNorm backward kernel (`ops.qk_rmsnorm_rope_bwd(dw=...)`, shared-memory atomics per block);
  * mod_img / mod_txt receive gradients, so norm1.linear / norm1_context.linear and the timestep / pooled-text embedders
    train through plain torch autograd on [B, D] tensors (the conditioning path is < 0.1 % of the step).

Activations saved per block: the LoRA set plus the two gated linear outputs per stream.  No LoRA in this mode.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from .. import ops
from ..flux.blocks import EPS, AttnPlan, MlpPlan, _qk_fwd


def _zeros_mod(B, D, dev):
    return torch.zeros((B, D), device=dev, dtype=torch.bfloat16)


def _ln(x, zero):
    """LayerNorm(x) without affine (bf16), via the modulate kernel with zero shift / scale."""
    return ops.ln_modulate_fwd(x, zero, zero, EPS)


class JointBlockFullFn(torch.autograd.Function):
    """h_out = JointTransformerBlock(h) with gradients for every parameter.

    inputs: h [B, S_txt + S_img, D], mod_img [B, 6D | 9D], mod_txt [B, 6D | 2D], st, then the block's parameters in the
    order of `param_order(st)` (weights / biases of the un-fused reference modules; the fused / transposed layouts come
    from st["plans"]).  Returns h_out; backward returns gradients in the same order (fused q|k|v gradients are split
    back into the three reference parameters)."""

    @staticmethod
    def forward(ctx, h, mod_img, mod_txt, st, *params):
        B, S, D = h.shape
        S_txt, H, hd = st["S_txt"], st["H"], st["hd"]
        plans: Dict[str, object] = st["plans"]
        pre_only = st.get("context_pre_only", False)
        dual = st.get("dual", False)
        dev = h.device
        streams = (("txt", slice(0, S_txt), mod_txt), ("img", slice(S_txt, S), mod_img))

        def shift_scale(name, mod):
            if name == "txt" and pre_only:       # AdaLayerNormContinuous chunks (scale | shift)
                return mod[:, D:2 * D], mod[:, 0:D]
            return mod[:, 0:D], mod[:, D:2 * D]

        qkv = torch.empty((B, S, 3 * D), device=dev, dtype=torch.bfloat16)
        for name, sl, mod in streams:
            ap: AttnPlan = plans[name + "_attn"]
            sh, sc = shift_scale(name, mod)
            nh = ops.ln_modulate_fwd(h[:, sl], sh, sc, EPS)
            ops.gemm([nh], [ap.w_qkv], ap.b_qkv, out=qkv[:, sl])
        ia, ta = plans["img_attn"], plans["txt_attn"]
        q, k = _qk_fwd(qkv, D, H, hd, ia, ta, S_txt, None, None)
        o, lse = ops.attn_fwd(q, k, qkv[:, :, 2 * D:].unflatten(-1, (H, hd)))
        del q, k
        o = o.view(B, S, D)
        h1 = torch.empty_like(h)
        h2 = torch.empty_like(h)
        y_attn = torch.empty_like(h)     # gated linear outputs (pre-gate): the gate gradients need them
        y_mlp = torch.empty_like(h)
        pre: Dict[str, Optional[torch.Tensor]] = {}
        for name, sl, mod in streams:
            ap = plans[name + "_attn"]
            if name == "txt" and pre_only:
                h1[:, sl].copy_(h[:, sl])
                h2[:, sl].copy_(h[:, sl])
                pre[name] = None
                continue
            ops.gemm([o[:, sl]], [ap.w_out], ap.b_out, out=h1[:, sl], epi=ops.EPI_GATE_RES, gate=mod[:, 2 * D:3 * D], res=h[:, sl],
                     aux=y_attn[:, sl])
        qkv2 = o2 = lse2 = y_attn2 = None
        if dual:
            isl = slice(S_txt, S)
            a2: AttnPlan = plans["img_attn2"]
            nh2a = ops.ln_modulate_fwd(h[:, isl], mod_img[:, 6 * D:7 * D], mod_img[:, 7 * D:8 * D], EPS)
            qkv2 = ops.gemm([nh2a], [a2.w_qkv], a2.b_qkv)
            del nh2a
            q2, k2 = _qk_fwd(qkv2, D, H, hd, a2, None, 0, None, None)
            o2, lse2 = ops.attn_fwd(q2, k2, qkv2[:, :, 2 * D:].unflatten(-1, (H, hd)))
            del q2, k2
            o2 = o2.view(B, S - S_txt, D)
            y_attn2 = torch.empty((B, S - S_txt, D), device=dev, dtype=torch.bfloat16)
            ops.gemm([o2], [a2.w_out], a2.b_out, out=h1[:, isl], epi=ops.EPI_GATE_RES, gate=mod_img[:, 8 * D:9 * D], res=h1[:, isl],
                     aux=y_attn2)
        for name, sl, mod in streams:
            if name == "txt" and pre_only:
                continue
            mp: MlpPlan = plans[name + "_mlp"]
            nh2 = ops.ln_modulate_fwd(h1[:, sl], mod[:, 3 * D:4 * D], mod[:, 4 * D:5 * D], EPS)
            p_ = torch.empty((B, sl.stop - sl.start, 4 * D), device=dev, dtype=torch.bfloat16)
            act = ops.gemm([nh2], [mp.w1], mp.b1, epi=ops.EPI_GELU, aux=p_)
            del nh2
            ops.gemm([act], [mp.w2], mp.b2, out=h2[:, sl], epi=ops.EPI_GATE_RES, gate=mod[:, 5 * D:6 * D], res=h1[:, sl],
                     aux=y_mlp[:, sl])
            del act
            pre[name] = p_
        ctx.st = st
        E = h.new_empty(0)
        keep = lambda t: t if t is not None else E
        ctx.save_for_backward(h, mod_img, mod_txt, qkv, o, lse, h1, keep(pre["txt"]), pre["img"], y_attn, y_mlp,
                              keep(qkv2), keep(o2), keep(lse2), keep(y_attn2))
        ctx.n_params = len(params)
        return h2

    @staticmethod
    def backward(ctx, dh2):
        h, mod_img, mod_txt, qkv, o, lse, h1, pre_txt, pre_img, y_attn, y_mlp, qkv2, o2, lse2, y_attn2 = ctx.saved_tensors
        st = ctx.st
        B, S, D = h.shape
        S_txt, H, hd = st["S_txt"], st["H"], st["hd"]
        plans = st["plans"]
        pre_only = st.get("context_pre_only", False)
        dual = st.get("dual", False)
        qk_norm = plans["img_attn"].norm_q is not None
        dev = h.device
        dh2 = dh2.contiguous()
        zero = _zeros_mod(B, D, dev)
        G: Dict[str, torch.Tensor] = {}                         # parameter name (block-local) -> gradient
        dm_img = torch.zeros_like(mod_img, dtype=torch.float32)
        dm_txt = torch.zeros_like(mod_txt, dtype=torch.float32)
        streams = (("txt", slice(0, S_txt), mod_txt, dm_txt, pre_txt), ("img", slice(S_txt, S), mod_img, dm_img, pre_img))
        dh1 = torch.empty_like(h)
        d_o = torch.empty_like(o)

        def bias_grad(colsum_bd: torch.Tensor) -> torch.Tensor:
            return colsum_bd.sum(0).to(torch.bfloat16)

        for name, sl, mod, dm, pre in streams:
            ap: AttnPlan = plans[name + "_attn"]
            if name == "txt" and pre_only:
                dh1[:, sl].copy_(dh2[:, sl])
                d_o[:, sl].zero_()
                continue
            mp: MlpPlan = plans[name + "_mlp"]
            pfx = "ff." if name == "img" else "ff_context."
            # ---- MLP branch: h2 = h1 + gate_mlp * fc2(gelu(fc1(LNmod(h1))))
            dm[:, 5 * D:6 * D] = ops.colsum2(dh2[:, sl], y_mlp[:, sl], want_sum=False)[1]           # d gate_mlp
            g2 = ops.gate_mul(dh2[:, sl], mod[:, 5 * D:6 * D])
            act = F.gelu(pre, approximate="tanh")                                                   # bf16, as the forward rounded it
            G[pfx + "net.2.weight"] = ops.wgrad_full(g2, act)
            G[pfx + "net.2.bias"] = bias_grad(ops.colsum2(g2)[0])
            del act
            d_pre = ops.gemm([g2], [mp.w2_t], None, epi=ops.EPI_MUL_DGELU, aux=pre)
            del g2
            nh2 = ops.ln_modulate_fwd(h1[:, sl], mod[:, 3 * D:4 * D], mod[:, 4 * D:5 * D], EPS)
            G[pfx + "net.0.proj.weight"] = ops.wgrad_full(d_pre, nh2)
            G[pfx + "net.0.proj.bias"] = bias_grad(ops.colsum2(d_pre)[0])
            del nh2
            d_nh2 = ops.gemm([d_pre], [mp.w1_t], None)
            del d_pre
            ln1 = _ln(h1[:, sl], zero)
            s_, d_ = ops.colsum2(d_nh2, ln1)
            dm[:, 3 * D:4 * D], dm[:, 4 * D:5 * D] = s_, d_                                          # d shift_mlp, d scale_mlp
            del ln1
            ops.ln_modulate_bwd(d_nh2, h1[:, sl], mod[:, 4 * D:5 * D], add=dh2[:, sl], eps=EPS, out=dh1[:, sl])
            del d_nh2
        # ---- image-only second attention (SD3.5 dual attention): h1_img += gate_msa2 * to_out2(attn2(...))
        d_nh2a = None
        if dual:
            isl = slice(S_txt, S)
            a2: AttnPlan = plans["img_attn2"]
            dm_img[:, 8 * D:9 * D] = ops.colsum2(dh1[:, isl], y_attn2, want_sum=False)[1]
            g = ops.gate_mul(dh1[:, isl], mod_img[:, 8 * D:9 * D])
            G["attn2.to_out.0.weight"] = ops.wgrad_full(g, o2)
            G["attn2.to_out.0.bias"] = bias_grad(ops.colsum2(g)[0])
            d_o2 = ops.gemm([g], [a2.w_out_t], None)
            del g
            d_qkv2, nq2 = _attn_bwd_full(qkv2, o2, d_o2, lse2, D, H, hd, a2, None, 0)
            del d_o2
            if qk_norm:
                G["attn2.norm_q.weight"], G["attn2.norm_k.weight"] = nq2["q_img"], nq2["k_img"]
            nh2a = ops.ln_modulate_fwd(h[:, isl], mod_img[:, 6 * D:7 * D], mod_img[:, 7 * D:8 * D], EPS)
            _split_qkv_grads(G, "attn2.", ("to_q", "to_k", "to_v"), ops.wgrad_full(d_qkv2, nh2a), bias_grad(ops.colsum2(d_qkv2)[0]), D)
            del nh2a
            d_nh2a = ops.gemm([d_qkv2], [a2.w_qkv_t], None)
            del d_qkv2
            lnh = _ln(h[:, isl], zero)
            s_, d_ = ops.colsum2(d_nh2a, lnh)
            dm_img[:, 6 * D:7 * D], dm_img[:, 7 * D:8 * D] = s_, d_
            del lnh
        # ---- attention output projections: h1 = h + gate_msa * to_out(o)
        for name, sl, mod, dm, pre in streams:
            ap = plans[name + "_attn"]
            if name == "txt" and pre_only:
                continue
            oname = "attn.to_out.0." if name == "img" else "attn.to_add_out."
            dm[:, 2 * D:3 * D] = ops.colsum2(dh1[:, sl], y_attn[:, sl], want_sum=False)[1]            # d gate_msa
            g1 = ops.gate_mul(dh1[:, sl], mod[:, 2 * D:3 * D])
            G[oname + "weight"] = ops.wgrad_full(g1, o[:, sl])
            G[oname + "bias"] = bias_grad(ops.colsum2(g1)[0])
            ops.gemm([g1], [ap.w_out_t], None, out=d_o[:, sl])
            del g1
        # ---- joint attention core
        d_qkv, nq = _attn_bwd_full(qkv, o, d_o, lse, D, H, hd, plans["img_attn"], plans["txt_attn"], S_txt)
        if qk_norm:
            G["attn.norm_q.weight"], G["attn.norm_k.weight"] = nq["q_img"], nq["k_img"]
            G["attn.norm_added_q.weight"], G["attn.norm_added_k.weight"] = nq["q_txt"], nq["k_txt"]
        dh = torch.empty_like(h)
        for name, sl, mod, dm, pre in streams:
            ap = plans[name + "_attn"]
            if name == "txt" and pre_only:
                sh_, sc_, i_sh, i_sc = mod[:, D:2 * D], mod[:, 0:D], slice(D, 2 * D), slice(0, D)
            else:
                sh_, sc_, i_sh, i_sc = mod[:, 0:D], mod[:, D:2 * D], slice(0, D), slice(D, 2 * D)
            names = ("to_q", "to_k", "to_v") if name == "img" else ("add_q_proj", "add_k_proj", "add_v_proj")
            nh = ops.ln_modulate_fwd(h[:, sl], sh_, sc_, EPS)
            _split_qkv_grads(G, "attn.", names, ops.wgrad_full(d_qkv[:, sl], nh), bias_grad(ops.colsum2(d_qkv[:, sl])[0]), D)
            del nh
            d_nh = ops.gemm([d_qkv[:, sl]], [ap.w_qkv_t], None)
            lnh = _ln(h[:, sl], zero)
            s_, d_ = ops.colsum2(d_nh, lnh)
            dm[:, i_sh], dm[:, i_sc] = s_, d_
            del lnh
            ops.ln_modulate_bwd(d_nh, h[:, sl], sc_, add=dh1[:, sl], eps=EPS, out=dh[:, sl])
            del d_nh
        if dual:
            isl = slice(S_txt, S)
            ops.ln_modulate_bwd(d_nh2a, h[:, isl], mod_img[:, 7 * D:8 * D], add=dh[:, isl], eps=EPS, out=dh[:, isl])
        grads = [G.get(n) for n in st["param_names"]]
        return (dh, dm_img.to(mod_img.dtype), dm_txt.to(mod_txt.dtype), None, *grads)


def _split_qkv_grads(G: Dict[str, torch.Tensor], prefix: str, names, dw: torch.Tensor, db: torch.Tensor, D: int) -> None:
    for i, n in enumerate(names):
        G[f"{prefix}{n}.weight"] = dw[i * D:(i + 1) * D]
        G[f"{prefix}{n}.bias"] = db[i * D:(i + 1) * D]


def _attn_bwd_full(qkv, o, d_o, lse, D, H, hd, img_plan: AttnPlan, txt_plan: Optional[AttnPlan], S_txt: int):
    """d_qkv [B, S, 3D] and (when the model has QK-norm) the RMSNorm weight gradients per stream."""
    B, S, _ = qkv.shape
    q, k = _qk_fwd(qkv, D, H, hd, img_plan, txt_plan, S_txt, None, None)
    v = qkv[:, :, 2 * D:].unflatten(-1, (H, hd))
    d_qkv = torch.empty_like(qkv)
    dv = d_qkv[:, :, 2 * D:].unflatten(-1, (H, hd))
    if img_plan.norm_q is None:
        ops.attn_bwd(q, k, v, o.view(B, S, H, hd), d_o.view(B, S, H, hd), lse,
                     dq=d_qkv[:, :, 0:D].unflatten(-1, (H, hd)), dk=d_qkv[:, :, D:2 * D].unflatten(-1, (H, hd)), dv=dv)
        return d_qkv, {}
    dq = torch.empty_like(q)
    dk = torch.empty_like(k)
    ops.attn_bwd(q, k, v, o.view(B, S, H, hd), d_o.view(B, S, H, hd), lse, dq=dq, dk=dk, dv=dv)
    del q, k
    tq = txt_plan.norm_q if txt_plan is not None else None
    tk = txt_plan.norm_k if txt_plan is not None else None
    dw = torch.zeros((4, hd), device=qkv.device, dtype=torch.float32)     # d(norm_q, norm_k, norm_added_q, norm_added_k)
    ops.qk_rmsnorm_rope_bwd(dq, dk, qkv, D, H, hd, img_plan.norm_q, img_plan.norm_k, tq, tk, S_txt, None, None, EPS, dsrc=d_qkv, dw=dw)
    dwb = dw.to(torch.bfloat16)
    nq = {"q_img": dwb[0], "k_img": dwb[1]}
    if txt_plan is not None and S_txt > 0:
        nq["q_txt"], nq["k_txt"] = dwb[2], dwb[3]
    return d_qkv, nq


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


class TailFullFn(torch.autograd.Function):
    """AdaLayerNormContinuous + proj_out with gradients for proj_out and the modulation (mod = scale | shift)."""

    @staticmethod
    def forward(ctx, h, mod, w_proj, b_proj, S_txt):
        D = h.shape[2]
        x = h[:, S_txt:]
        nx = ops.ln_modulate_fwd(x, mod[:, D:2 * D], mod[:, 0:D], EPS)
        out = ops.gemm([nx], [w_proj.detach()], b_proj.detach())
        ctx.save_for_backward(h, mod, w_proj)
        ctx.S_txt = S_txt
        return out

    @staticmethod
    def backward(ctx, d_out):
        h, mod, w_proj = ctx.saved_tensors
        S_txt = ctx.S_txt
        B, _, D = h.shape
        d_out = d_out.contiguous()
        x = h[:, S_txt:]
        nx = ops.ln_modulate_fwd(x, mod[:, D:2 * D], mod[:, 0:D], EPS)
        dw = ops.wgrad_full(d_out, nx)
        db = ops.colsum2(d_out)[0].sum(0).to(torch.bfloat16)
        del nx
        d_nx = ops.gemm([d_out], [w_proj.detach().t().contiguous()], None)
        zero = _zeros_mod(B, D, h.device)
        s_, d_ = ops.colsum2(d_nx, _ln(x, zero))
        dmod = torch.cat([d_, s_], dim=1).to(mod.dtype)              # (scale | shift)
        dh = torch.zeros_like(h) if S_txt > 0 else torch.empty_like(h)
        ops.ln_modulate_bwd(d_nx, x, mod[:, 0:D], add=None, eps=EPS, out=dh[:, S_txt:])
        return dh, dmod, dw, db, None
