"""Flux MMDiT blocks as explicit forward/backward kernel schedules (torch.autograd.Function).

Mirrors, for the training path, reference flux/transformer.py:
  * FluxTransformerBlock.forward + _ffn_forward         (:563-687)  -> DoubleBlockFn
  * FluxSingleTransformerBlock.forward + _ffn_forward   (:453-510)  -> SingleBlockFn
  * FluxAttnProcessor2_0.__call__                       (:116-224)  (inlined in both)
  * PEFT lora.Linear on the attention projections       (common.py:1094-1117, flux/model.py:1249-1262)

Every arithmetic step is a libstb200 kernel (ops.*); torch only allocates, slices and carries the
autograd graph between blocks.  Activations saved per block: block input, fused pre-norm QKV, the
post-norm / post-RoPE q and k, attention output + LSE, post-attention stream, MLP pre-activation, the
rank-r LoRA down-projections and, when a q/k/v adapter is present, the LayerNorm-modulated block input.
Keeping q and k costs 2 B S D bytes per block (Flux.1-dev: 3.2 GB per 1024^2 sample over 57 blocks) and
saves one HBM-bound RMSNorm + RoPE pass per block in backward; the modulated input (0.11 GB per block
at B = 4, 1024^2) saves one LayerNorm-modulate pass.  GELU is recomputed inside the backward kernels.
Gradient checkpointing with an interval is the way to trade this memory for compute.

The hidden state travels as ONE joint buffer [B, S_txt + S_img, D] (text tokens first, as the
reference concatenates them for attention, :166-168) so no torch.cat / split copies are needed.

In LoRA training (BASELINE config 2) the base weights are frozen: gradients are produced for the LoRA
A/B matrices and for the hidden state only; no gradient flows to temb / the adaLN linears because
none of their parameters is trainable in that configuration.  Full fine-tune (`st["full"]`, SD3 and PixArt) runs the
same schedules with each Linear's (weight, bias) in its adapter slots (WgradPack) and also returns the modulation
gradients.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch

from .. import ops

EPS = 1e-6


# ------------------------------------------------------------------------------------------------
# derived (frozen) weight layouts
# ------------------------------------------------------------------------------------------------
@dataclass
class AttnPlan:
    """Fused / transposed copies of one attention's projection weights (one per stream)."""
    w_qkv: torch.Tensor      # [3D, D]   rows: q | k | v
    b_qkv: torch.Tensor      # [3D]
    w_qkv_t: torch.Tensor    # [D, 3D]   dgrad weight
    w_out: Optional[torch.Tensor] = None    # [D, D]  (None for single blocks: pre_only attention)
    b_out: Optional[torch.Tensor] = None
    w_out_t: Optional[torch.Tensor] = None  # [D, D]
    norm_q: Optional[torch.Tensor] = None   # [hd]
    norm_k: Optional[torch.Tensor] = None


@dataclass
class MlpPlan:
    w1: torch.Tensor     # [4D, D]
    b1: torch.Tensor
    w1_t: torch.Tensor   # [D, 4D]
    w2: torch.Tensor     # [D, 4D]  (single block: proj_out [D, 5D], mlp part = columns D:)
    b2: torch.Tensor
    w2_t: torch.Tensor   # [4D, D]  (single block: [5D, D])


def _t(w: torch.Tensor) -> torch.Tensor:
    return w.t().contiguous()


def _wt(w: torch.Tensor, dynamic: bool = False):
    """The dgrad operand of a base weight.  A dgrad GEMM wants W^T in nn.Linear layout; it can get it as a real transposed
    copy (K-major B operand, the fastest tile path: Flux LoRA step 362 ms of GEMM) or as a zero-copy view of the forward
    weight (ops.WT: the kernel stages W as an MN-major B operand; +1.7 % GEMM time, but no second copy of the weights).
    Frozen weights get the copy; weights rewritten every optimizer step (`dynamic`: full fine-tune, LoKr) get the view,
    so no step spends a transpose on them."""
    return ops.WT(w) if dynamic else _t(w)


@dataclass
class LoraPack:
    """Per-step packed view of the LoRA matrices of one fused projection group.

    a_stack  [R, K]   rows: A of each member (R = n_members * r)
    a_stack_t [K, R]
    b_ext    [N, R]   block structured: member m owns rows n_m and columns [m r, (m+1) r); scaling folded in
    b_ext_t  [R, N]
    """
    a_stack: torch.Tensor
    a_stack_t: torch.Tensor
    b_ext: torch.Tensor
    b_ext_t: torch.Tensor
    rank: int
    scaling: float
    members: List[Optional[int]]  # index into the flat (A, B) parameter list, None = member not adapted
    n_out: int                    # rows per member
    rank_padded: int = 0          # per-member column block inside the stacks (rank rounded up to 8)
    row_index: Optional[torch.Tensor] = None  # member-local output row -> row of the (head-dim padded) projection
    col_index: Optional[torch.Tensor] = None  # input feature -> column of the (head-dim padded) activation


def pack_lora(params: List[Optional[Tuple[torch.Tensor, torch.Tensor]]], n_out: int, k_in: int, scaling: float,
              device, dtype=torch.bfloat16, row_index: Optional[torch.Tensor] = None,
              col_index: Optional[torch.Tensor] = None) -> Optional[LoraPack]:
    """params[m] = (A [r, K], B [n_out, r]) or None for each member of the fused projection.

    `n_out` / `k_in` are the sizes of the projection as the GEMM sees it; when heads are zero-padded (PixArt
    head_dim 72 -> 128) `row_index` / `col_index` scatter the un-padded LoRA rows / columns into that layout."""
    present = [p for p in params if p is not None]
    if not present:
        return None
    r = present[0][0].shape[0]
    rp = (r + 7) // 8 * 8   # rank padded with zero rows/columns so every TMA row stride is 16-byte aligned
    M = len(params)
    if rp > 128:
        raise NotImplementedError(f"LoRA rank {r} exceeds the 128-wide rank block of the weight-gradient kernel")
    a_stack = torch.zeros((M * rp, k_in), device=device, dtype=dtype)
    b_ext = torch.zeros((M * n_out, M * rp), device=device, dtype=dtype)
    members: List[Optional[int]] = []
    for m, p in enumerate(params):
        if p is None:
            members.append(None)
            continue
        a, b = p
        if col_index is None:
            a_stack[m * rp:m * rp + r].copy_(a.detach())
        else:
            a_stack[m * rp:m * rp + r, col_index] = a.detach().to(dtype)
        bs = b.detach().to(dtype) * scaling if scaling != 1.0 else b.detach().to(dtype)
        if row_index is None:
            b_ext[m * n_out:(m + 1) * n_out, m * rp:m * rp + r].copy_(bs)
        else:
            b_ext[m * n_out + row_index, m * rp:m * rp + r] = bs
        members.append(m)
    return LoraPack(a_stack, _t(a_stack), b_ext, _t(b_ext), r, scaling, members, n_out, rp, row_index, col_index)


@dataclass
class WgradPack:
    """Members of one fused projection group whose gradients come from the group's full weight gradient dW = dy^T x: LyCORIS
    LoKr factor pairs (simpletuner_b200/lycoris.py) or, in full fine-tune, the member's own (weight, bias).  Either way the
    weights the GEMMs read are already the plan's projection matrices, so forward / dgrad are adapter-free."""
    members: List[Optional[tuple]]   # LoKr: (w1 [a, c], w2 [b, d], scale * multiplier); full: (weight, bias)
    n_out: int                       # rows per member
    full: bool = False
    row_index: Optional[torch.Tensor] = None  # as LoraPack: member-local output row -> row of the (head-dim padded) projection
    col_index: Optional[torch.Tensor] = None  # input feature -> column of the (head-dim padded) activation


def make_pack(params, n_out: int, k_in: int, scaling: float, device, lokr_scales=None, full: bool = False,
              row_index: Optional[torch.Tensor] = None, col_index: Optional[torch.Tensor] = None):
    """LoRA pack (pack_lora) or a WgradPack: of LoKr factors when `lokr_scales[m]` is set for the present members, of
    (weight, bias) pairs when `full`."""
    if full or (lokr_scales is not None and any(s is not None for s in lokr_scales)):
        mem = list(params) if full else [None if p is None else (p[0], p[1], float(sc)) for p, sc in zip(params, lokr_scales)]
        return WgradPack(mem, n_out, full, row_index, col_index) if any(m is not None for m in mem) else None
    return pack_lora(params, n_out, k_in, scaling, device, row_index=row_index, col_index=col_index)


def _wgrad_grads(pack: WgradPack, x: torch.Tensor, dy: torch.Tensor):
    """The full weight gradient of the group (one MN-major wgmma GEMM, dy^T x), split per member: a full member takes its
    rows of dW and of the bias gradient (gathered back to the real rows / columns of padded heads), a LoKr member contracts
    its rows against the other Kronecker factor (delta W = kron(w1, w2) * scale)."""
    from ..lycoris import lokr_factor_grads
    dW = ops.wgrad_full(dy, x)                       # [members * n_out, K] bf16
    db = ops.colsum2(dy)[0].sum(0).to(torch.bfloat16) if pack.full else None
    out = []
    for m, mem in enumerate(pack.members):
        rows = slice(m * pack.n_out, (m + 1) * pack.n_out)
        if mem is None:
            out.append((None, None))
        elif not pack.full:
            out.append(lokr_factor_grads(dW[rows], *mem))
        else:
            dw, dbm = dW[rows], db[rows]
            if pack.row_index is not None:
                dw, dbm = dw.index_select(0, pack.row_index), dbm.index_select(0, pack.row_index)
            if pack.col_index is not None:
                dw = dw.index_select(1, pack.col_index)
            out.append((dw, dbm))
    return out


@dataclass
class LoraDrop:
    """PEFT `lora_dropout` state of one forward pass: probability, the step's seed and the first mask stream of the block
    (every adapted Linear of the model owns one stream, so q / k / v of one fused group draw independent masks)."""
    p: float
    seed: int
    stream: int = 0

    def at(self, offset: int) -> "LoraDrop":
        return LoraDrop(self.p, self.seed, self.stream + offset)


def _member_slices(pack: LoraPack):
    rp = pack.rank_padded or pack.rank
    return [(m, slice(m * rp, (m + 1) * rp)) for m, idx in enumerate(pack.members) if idx is not None]


def _lora_down(x: torch.Tensor, pack: LoraPack, drop: Optional[LoraDrop] = None) -> torch.Tensor:
    """T = x A_stack^T  [B, S, R];  with dropout member m sees its own masked copy: T_m = (x o keep_m / (1 - p)) A_m^T."""
    if drop is None:
        return ops.gemm([x], [pack.a_stack])
    B, S, _ = x.shape
    xm = ops.dropout_expand(x, len(pack.members), drop.p, drop.seed, drop.stream)
    t = torch.zeros((B, S, pack.a_stack.shape[0]), device=x.device, dtype=torch.bfloat16)
    for m, sl in _member_slices(pack):
        ops.gemm([xm[m]], [pack.a_stack[sl]], out=t[:, :, sl])
    return t


def _lora_grads(pack: LoraPack, x: torch.Tensor, t_down: torch.Tensor, dy: torch.Tensor, t_up: torch.Tensor,
                drop: Optional[LoraDrop] = None):
    """dA_stack [R, K] = T'^T x  (T' = dy B_ext, scaling already inside);  dB_ext^T [R, N] = T^T dy.
    With dropout dA_m contracts T'_m with the SAME masked copy of x the forward used (masks regenerated, not stored)."""
    if isinstance(pack, WgradPack):
        assert drop is None and not isinstance(x, (tuple, list))
        return _wgrad_grads(pack, x, dy)
    R = pack.a_stack.shape[0]
    wide = R > 128        # ranks above 40: the fused q|k|v rank block no longer fits one 128-wide weight-gradient tile
    if isinstance(x, (tuple, list)):        # the adapted Linear reads cat(x, -1) (single-block proj_out): one product per part
        assert drop is None and not wide
        d_a = torch.cat([ops.skinny_tn(t_up, part) for part in x], 1)
    elif drop is None and not wide:
        d_a = ops.skinny_tn(t_up, x)        # [R, K] fp32
    elif drop is None:
        d_a = torch.zeros((R, x.shape[-1]), device=x.device, dtype=torch.float32)
        for m, sl in _member_slices(pack):
            ops.skinny_tn(t_up[:, :, sl], x, out=d_a[sl])
    else:
        d_a = torch.zeros((R, x.shape[-1]), device=x.device, dtype=torch.float32)
        xm = ops.dropout_expand(x, len(pack.members), drop.p, drop.seed, drop.stream)
        for m, sl in _member_slices(pack):
            ops.skinny_tn(t_up[:, :, sl], xm[m], out=d_a[sl])
        del xm
    r, rp = pack.rank, (pack.rank_padded or pack.rank)
    if not wide:
        d_bt = ops.skinny_tn(t_down, dy)    # [R, N] fp32 (only the block diagonal is used)
    else:                                   # per member, against its own n_out columns of dy only
        d_bt = torch.zeros((R, dy.shape[-1]), device=dy.device, dtype=torch.float32)
        for m, sl in _member_slices(pack):
            blk = torch.zeros((rp, pack.n_out), device=dy.device, dtype=torch.float32)
            ops.skinny_tn(t_down[:, :, sl], dy[:, :, m * pack.n_out:(m + 1) * pack.n_out], out=blk)
            d_bt[sl, m * pack.n_out:(m + 1) * pack.n_out] = blk
    out = []
    for m, idx in enumerate(pack.members):
        if idx is None:
            out.append((None, None))
            continue
        da = d_a[m * rp:m * rp + r]
        dbt = d_bt[m * rp:m * rp + r, m * pack.n_out:(m + 1) * pack.n_out]
        if pack.col_index is not None:
            da = da[:, pack.col_index]
        if pack.row_index is not None:
            dbt = dbt[:, pack.row_index]
        db = dbt.t()
        if pack.scaling != 1.0:
            db = db * pack.scaling
        out.append((da.to(torch.bfloat16), db.to(torch.bfloat16).contiguous()))
    return out


def _lora_dgrad_dropout(dx: torch.Tensor, t_up: torch.Tensor, pack: LoraPack, drop: LoraDrop) -> None:
    """dx += sum_m keep_m / (1 - p) o (T'_m A_m): the LoRA branch of the input gradient through the dropout masks."""
    B, S, K = dx.shape
    M = len(pack.members)
    d = torch.zeros((M, B, S, K), device=dx.device, dtype=torch.bfloat16) if any(i is None for i in pack.members) \
        else torch.empty((M, B, S, K), device=dx.device, dtype=torch.bfloat16)
    for m, sl in _member_slices(pack):
        ops.gemm([t_up[:, :, sl]], [pack.a_stack_t[:, sl]], out=d[m])
    ops.dropout_accum_(dx, d, drop.p, drop.seed, drop.stream)


# ------------------------------------------------------------------------------------------------
# shared pieces
# ------------------------------------------------------------------------------------------------
def _linear_lora_fwd(x, w, b, pack: Optional[LoraPack], drop: Optional[LoraDrop] = None, **kw):
    """y = x W^T + b (+ T B_ext^T as an extra K-segment).  Returns (y, T or None)."""
    if pack is None or isinstance(pack, WgradPack):
        return ops.gemm([x], [w], b, **kw), None
    t = _lora_down(x, pack, drop)
    return ops.gemm([x, t], [w, pack.b_ext], b, **kw), t


def _linear_lora_dgrad(dy, w_t, pack: Optional[LoraPack], drop: Optional[LoraDrop] = None, **kw):
    """dx = dy W (+ (dy B_ext) A_stack).  Returns (dx, T' or None)."""
    if pack is None or isinstance(pack, WgradPack):
        return ops.gemm([dy], [w_t], None, **kw), None
    t_up = ops.gemm([dy], [pack.b_ext_t])
    if drop is None:
        return ops.gemm([dy, t_up], [w_t, pack.a_stack_t], None, **kw), t_up
    dx = ops.gemm([dy], [w_t], None, **kw)
    _lora_dgrad_dropout(dx, t_up, pack, drop)
    return dx, t_up


def _pack1(a, b, n_out: int, k_in: int, scaling: float, device, lokr_scale=None, full: bool = False):
    """Pack of a single adapted Linear (MLP projections, proj_out, x_embedder); full: (a, b) = (weight, bias)."""
    return None if a is None else make_pack([(a, b)], n_out, k_in, scaling, device, [lokr_scale], full)


def _dgrad_through_gelu(dy, w_t, pack: Optional[LoraPack], drop: Optional[LoraDrop], pre):
    """d_pre = (dy W (+ LoRA branch)) * gelu'(pre).  Returns (d_pre, T' or None).  Without dropout the LoRA branch is one more
    K-segment and the activation gradient stays in the GEMM epilogue; with dropout the masked branch is added to the
    un-activated gradient first."""
    if pack is None or drop is None or isinstance(pack, WgradPack):
        return _linear_lora_dgrad(dy, w_t, pack, None, epi=ops.EPI_MUL_DGELU, aux=pre)
    d_act, t_up = _linear_lora_dgrad(dy, w_t, pack, drop)
    return ops.mul_dgelu_tanh(d_act, pre, out=d_act), t_up


# ------------------------------------------------------------------------------------------------
# token segments (Flux Kontext): a stream whose tokens fall into segments with their own modulation rows
# ------------------------------------------------------------------------------------------------
def _segments(mod: torch.Tensor, counts, n: int):
    """[(token slice of the stream, modulation rows [B, kD])].  counts None: one segment, `mod` [B, kD]; otherwise `mod`
    stacks one [B, kD] block per segment (segment-major) and counts[i] tokens follow each other."""
    if counts is None:
        return [(slice(0, n), mod)]
    B = mod.shape[0] // len(counts)
    out, s0 = [], 0
    for i, c in enumerate(counts):
        out.append((slice(s0, s0 + c), mod[i * B:(i + 1) * B]))
        s0 += c
    assert s0 == n, (counts, n)
    return out


def _chunk(mod: torch.Tensor, i: int, D: int) -> torch.Tensor:
    return mod[:, i * D:(i + 1) * D]


def _out(x: torch.Tensor, out: Optional[torch.Tensor]) -> torch.Tensor:
    return out if out is not None else torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)


# Each output row of the LayerNorm-modulate, gate and GATE_RES kernels depends on its own row and its sample's
# modulation row only, so one launch per segment gives the bits of a per-token modulation (reference
# flux/transformer.py:386-412, the 3-D branches of the adaLN helpers).
def _lnm_fwd(x, segs, ish: int, isc: int, out=None):
    if len(segs) == 1:
        m = segs[0][1]
        return ops.ln_modulate_fwd(x, _chunk(m, ish, x.shape[2]), _chunk(m, isc, x.shape[2]), EPS, out=out)
    out = _out(x, out)
    for sl, m in segs:
        ops.ln_modulate_fwd(x[:, sl], _chunk(m, ish, x.shape[2]), _chunk(m, isc, x.shape[2]), EPS, out=out[:, sl])
    return out


def _lnm_bwd(d, x, segs, isc: int, add=None, out=None):
    out = _out(x, out)
    for sl, m in segs:
        ops.ln_modulate_bwd(d[:, sl], x[:, sl], _chunk(m, isc, x.shape[2]), add=None if add is None else add[:, sl], eps=EPS,
                            out=out[:, sl])
    return out


def _dmod_gate(dm, dy, y, ig: int):
    """Full fine-tune: d gate (chunk ig of dm [B, kD] fp32) of out = res + gate * y, as sum_s dy * y."""
    D = y.shape[2]
    dm[:, ig * D:(ig + 1) * D] = ops.colsum2(dy, y, want_sum=False)[1]


def _dmod_shift_scale(dm, d_nx, x, ish: int, isc: int):
    """Full fine-tune: d shift / d scale (chunks ish / isc of dm) of nx = LayerNorm(x) (1 + scale) + shift, as sum_s d_nx and
    sum_s d_nx * LayerNorm(x); LayerNorm(x) comes from the modulate kernel with zero shift / scale."""
    B, _, D = x.shape
    zero = torch.zeros((B, D), device=x.device, dtype=torch.bfloat16)
    dm[:, ish * D:(ish + 1) * D], dm[:, isc * D:(isc + 1) * D] = ops.colsum2(d_nx, ops.ln_modulate_fwd(x, zero, zero, EPS))


def _gate_mul(x, segs, ig: int):
    if len(segs) == 1:
        return ops.gate_mul(x, _chunk(segs[0][1], ig, x.shape[2]))
    out = _out(x, None)
    for sl, m in segs:
        ops.gate_mul(x[:, sl], _chunk(m, ig, x.shape[2]), out=out[:, sl])
    return out


def _gemm_gate_res(a_list, w_list, bias, segs, ig: int, res, out=None, nan_to_num=False):
    """ops.gemm with the GATE_RES epilogue, one launch per segment (each segment gates with its own rows)."""
    D = res.shape[2]
    if len(segs) == 1:
        return ops.gemm(a_list, w_list, bias, out=out, epi=ops.EPI_GATE_RES, gate=_chunk(segs[0][1], ig, D), res=res,
                        nan_to_num=nan_to_num)
    out = _out(res, out)
    for sl, m in segs:
        ops.gemm([a[:, sl] for a in a_list], w_list, bias, out=out[:, sl], epi=ops.EPI_GATE_RES, gate=_chunk(m, ig, D),
                 res=res[:, sl], nan_to_num=nan_to_num)
    return out


def _linear_lora_gate_res(x, w, b, pack, drop, segs, ig: int, res, out, nan_to_num=False, aux=None):
    """_linear_lora_fwd with the GATE_RES epilogue over segments: the LoRA down-projection (and its dropout mask) spans
    the whole stream, the base GEMM runs per segment.  aux (one segment only): receives the pre-gate output.  Returns T
    or None."""
    if len(segs) == 1:
        return _linear_lora_fwd(x, w, b, pack, drop, out=out, epi=ops.EPI_GATE_RES, gate=_chunk(segs[0][1], ig, res.shape[2]),
                                res=res, nan_to_num=nan_to_num, aux=aux)[1]
    assert aux is None
    if pack is None or isinstance(pack, WgradPack):
        _gemm_gate_res([x], [w], b, segs, ig, res, out, nan_to_num)
        return None
    t = _lora_down(x, pack, drop)
    _gemm_gate_res([x, t], [w, pack.b_ext], b, segs, ig, res, out, nan_to_num)
    return t


class LoraLinearFn(torch.autograd.Function):
    """y = x W^T + b + scaling * B A dropout(x) for an adapted Linear outside the block schedules (x_embedder,
    flux_lora_target = "all+ffs+embedder", reference flux/model.py:1320-1338).  x carries no gradient (model input)."""

    @staticmethod
    def forward(ctx, x, w, b, scaling, drop, lora_a, lora_b):
        pk = _pack1(lora_a, lora_b, w.shape[0], w.shape[1], scaling, x.device)
        y, t = _linear_lora_fwd(x, w, b, pk, drop)
        ctx.pack, ctx.drop = pk, drop
        ctx.save_for_backward(x, t)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, t = ctx.saved_tensors
        pk, drop = ctx.pack, ctx.drop
        dy = dy if dy.stride(-1) == 1 else dy.contiguous()
        t_up = ops.gemm([dy], [pk.b_ext_t])
        (da, db), = _lora_grads(pk, x, t, dy, t_up, drop)
        return None, None, None, None, None, da, db


# ------------------------------------------------------------------------------------------------
# shared: q / k preparation (per-head RMSNorm + RoPE, or plain views when the model has neither)
# ------------------------------------------------------------------------------------------------
def _qk_fwd(qkv, D, H, hd, img_plan: AttnPlan, txt_plan: Optional[AttnPlan], S_txt, cos, sin):
    if img_plan.norm_q is None and cos is None:  # SD3-medium (qk_norm=None): nothing to compute
        return qkv[:, :, 0:D].unflatten(-1, (H, hd)), qkv[:, :, D:2 * D].unflatten(-1, (H, hd))
    tq = txt_plan.norm_q if txt_plan is not None else None
    tk = txt_plan.norm_k if txt_plan is not None else None
    return ops.qk_rmsnorm_rope_fwd(qkv, D, H, hd, img_plan.norm_q, img_plan.norm_k, tq, tk, S_txt, cos, sin, EPS)


def _attn_core_bwd(qkv, o, d_o, lse, D, H, hd, img_plan, txt_plan, S_txt, cos, sin, qk=None, key_bias=None, dw=None):
    """Returns d_qkv [B, S, 3D] given d_o.  `qk` = the (q, k) pair saved by the forward (spending 2 B S D bytes per block
    is cheaper than re-running the RMSNorm + RoPE pass in backward); recomputed when absent.  key_bias: the forward's.
    dw (full fine-tune): zeroed fp32 [4, hd] that receives the RMSNorm weight gradients (norm_q, norm_k, the text
    stream's norm_added_q, norm_added_k)."""
    B, S, _ = qkv.shape
    q, k = qk if qk is not None else _qk_fwd(qkv, D, H, hd, img_plan, txt_plan, S_txt, cos, sin)
    v = qkv[:, :, 2 * D:].unflatten(-1, (H, hd))
    d_qkv = torch.empty_like(qkv)
    dv = d_qkv[:, :, 2 * D:].unflatten(-1, (H, hd))
    if img_plan.norm_q is None and cos is None:
        ops.attn_bwd(q, k, v, o.view(B, S, H, hd), d_o.view(B, S, H, hd), lse,
                     dq=d_qkv[:, :, 0:D].unflatten(-1, (H, hd)), dk=d_qkv[:, :, D:2 * D].unflatten(-1, (H, hd)), dv=dv,
                     key_bias=key_bias)
        return d_qkv
    # The backward of RMSNorm + RoPE is a separate HBM-bound pass over the post-RoPE dq / dk.
    dq = torch.empty_like(q)
    dk = torch.empty_like(k)
    ops.attn_bwd(q, k, v, o.view(B, S, H, hd), d_o.view(B, S, H, hd), lse, dq=dq, dk=dk, dv=dv, key_bias=key_bias)
    del q, k
    tq = txt_plan.norm_q if txt_plan is not None else None
    tk = txt_plan.norm_k if txt_plan is not None else None
    ops.qk_rmsnorm_rope_bwd(dq, dk, qkv, D, H, hd, img_plan.norm_q, img_plan.norm_k, tq, tk, S_txt, cos, sin, EPS, dsrc=d_qkv,
                            dw=dw)
    return d_qkv


# ------------------------------------------------------------------------------------------------
# Double-stream (joint) block — Flux FluxTransformerBlock and SD3 JointTransformerBlock
# ------------------------------------------------------------------------------------------------
class DoubleBlockFn(torch.autograd.Function):
    """h_out = JointBlock(h_in) on the joint [B, S_txt + S_img, D] buffer (text rows first).

    Flux (reference flux/transformer.py:563-687) and SD3 (reference sd3/transformer.py:145-241; the joint
    attention is permutation-invariant without RoPE, so the [image, text] order of JointAttnProcessor2_0 is
    irrelevant).  `st` flags: `nan_to_num_txt` (Flux), `dual` (SD3.5 image-only attn2 fed by a second
    modulation of LayerNorm(h): mod_img then has 9 chunks), `context_pre_only` (SD3 last block: the text
    stream only feeds q/k/v; mod_txt = [scale | shift] as AdaLayerNormContinuous chunks it), `full` (full
    fine-tune, SD3: see below).

    inputs: h, mod_img [B, 6D|9D], mod_txt [B, 6D|2D] (adaLN vectors), cos, sin (or None), st, then the
    flat LoRA tensors (None where not adapted) in the order
      img : to_q.A, to_q.B, to_k.A, to_k.B, to_v.A, to_v.B, to_out.A, to_out.B            [0..7]
      txt : add_q.A, add_q.B, add_k.*, add_v.*, to_add_out.A, to_add_out.B               [8..15]
      attn2: to_q.A, to_q.B, to_k.*, to_v.*, to_out.A, to_out.B                          [16..23]
      mlp : ff.net.0.proj.A, .B, ff.net.2.A, .B, ff_context.net.0.proj.A, .B, ff_context.net.2.A, .B   [24..31]
    Full fine-tune: each (A, B) slot holds that Linear's (weight, bias) and gets its gradient from the group's dW
    (WgradPack); slots [32..37] hold the q / k RMSNorm weights (norm_q, norm_k, norm_added_q, norm_added_k, attn2's norm_q,
    norm_k), and mod_img / mod_txt get their gradients (shift / scale / gate column sums; the GATE_RES epilogues also write
    the pre-gate outputs for the gates).
    """

    @staticmethod
    def forward(ctx, h, mod_img, mod_txt, cos, sin, st, *lora):
        B, S, D = h.shape
        S_txt, H, hd = st["S_txt"], st["H"], st["hd"]
        plans: Dict[str, object] = st["plans"]
        scaling = st["lora_scaling"]
        pre_only = st.get("context_pre_only", False)
        dual = st.get("dual", False)
        nan_txt = st.get("nan_to_num_txt", True)
        dev = h.device
        drop: Optional[LoraDrop] = st.get("lora_drop")
        dr = (lambda off: drop.at(off)) if drop is not None else (lambda off: None)
        full = st.get("full", False)
        ls = st.get("lokr_scales")                   # per (A, B) pair of the flat list: LoKr scale, or None for LoRA
        assert not (full and (st.get("img_segs") or drop is not None or ls)), "full fine-tune: no segments, dropout or LoKr"
        n_lora_in = len(lora)
        lora = list(lora) + [None] * (32 - len(lora))
        segs = {"txt": _segments(mod_txt, None, S_txt), "img": _segments(mod_img, st.get("img_segs"), S - S_txt)}
        streams = (("txt", slice(0, S_txt), mod_txt, 8), ("img", slice(S_txt, S), mod_img, 0))
        mlp_base = {"img": 24, "txt": 28}
        lsc = (lambda i: ls[i // 2] if ls is not None and i // 2 < len(ls) else None)

        def lp(base, n_members, n_out, k_in):
            ps = []
            for m in range(n_members):
                a, b = lora[base + 2 * m], lora[base + 2 * m + 1]
                ps.append(None if a is None else (a, b))
            return make_pack(ps, n_out, k_in, scaling, dev, [lsc(base + 2 * m) for m in range(n_members)], full)

        def mod_shift_scale(name):      # chunk indices of (shift, scale)
            return (1, 0) if name == "txt" and pre_only else (0, 1)

        packs = {}
        qkv = torch.empty((B, S, 3 * D), device=dev, dtype=torch.bfloat16)
        small = {}
        keep_nh = any(x is not None for x in lora[0:6] + lora[8:14])     # only the adapters' weight gradients read it
        nh_joint = torch.empty_like(h) if keep_nh else None
        for name, sl, mod, base in streams:
            ap: AttnPlan = plans[name + "_attn"]
            packs[name + "_qkv"] = lp(base, 3, D, D)
            packs[name + "_out"] = lp(base + 6, 1, D, D) if ap.w_out is not None else None
            nh = _lnm_fwd(h[:, sl], segs[name], *mod_shift_scale(name), out=nh_joint[:, sl] if keep_nh else None)
            _, t = _linear_lora_fwd(nh, ap.w_qkv, ap.b_qkv, packs[name + "_qkv"], dr(base), out=qkv[:, sl])
            small[name + "_t_qkv"] = t
        ia: AttnPlan = plans["img_attn"]
        ta: AttnPlan = plans["txt_attn"]
        q, k = _qk_fwd(qkv, D, H, hd, ia, ta, S_txt, cos, sin)
        v = qkv[:, :, 2 * D:].unflatten(-1, (H, hd))
        o, lse = ops.attn_fwd(q, k, v, key_bias=st.get("key_bias"))
        keep_qk = q.data_ptr() != qkv.data_ptr()      # (views of qkv when the model has neither norm nor RoPE)
        if not keep_qk:
            del q, k
        o = o.view(B, S, D)
        h1 = torch.empty_like(h)
        h2 = torch.empty_like(h)
        y_attn = torch.empty_like(h) if full else None      # pre-gate outputs of the gated linears: the gate gradients
        y_mlp = torch.empty_like(h) if full else None
        y_at = (lambda y, sl: y[:, sl] if y is not None else None)
        for name, sl, mod, base in streams:
            ap = plans[name + "_attn"]
            if name == "txt" and pre_only:
                h1[:, sl].copy_(h[:, sl])
                h2[:, sl].copy_(h[:, sl])
                small[name + "_t_out"] = None
                continue
            small[name + "_t_out"] = _linear_lora_gate_res(o[:, sl], ap.w_out, ap.b_out, packs[name + "_out"], dr(base + 6),
                                                           segs[name], 2, res=h[:, sl], out=h1[:, sl], aux=y_at(y_attn, sl))
        qkv2 = o2 = lse2 = y_attn2 = None
        if dual:
            isl = slice(S_txt, S)
            a2: AttnPlan = plans["img_attn2"]
            packs["a2_qkv"] = lp(16, 3, D, D)
            packs["a2_out"] = lp(22, 1, D, D)
            nh2a = ops.ln_modulate_fwd(h[:, isl], mod_img[:, 6 * D:7 * D], mod_img[:, 7 * D:8 * D], EPS)
            qkv2, t = _linear_lora_fwd(nh2a, a2.w_qkv, a2.b_qkv, packs["a2_qkv"], dr(16))
            del nh2a
            small["a2_t_qkv"] = t
            q2, k2 = _qk_fwd(qkv2, D, H, hd, a2, None, 0, None, None)
            o2, lse2 = ops.attn_fwd(q2, k2, qkv2[:, :, 2 * D:].unflatten(-1, (H, hd)))
            del q2, k2
            o2 = o2.view(B, S - S_txt, D)
            y_attn2 = torch.empty_like(o2) if full else None
            # h1_img += gate_msa2 * to_out2(o2)   (in place: every element is read then written by one thread)
            _, t = _linear_lora_fwd(o2, a2.w_out, a2.b_out, packs["a2_out"], dr(22), out=h1[:, isl], epi=ops.EPI_GATE_RES,
                                    gate=mod_img[:, 8 * D:9 * D], res=h1[:, isl], aux=y_attn2)
            small["a2_t_out"] = t
        mlp_pre = {}
        for name, sl, mod, base in streams:
            if name == "txt" and pre_only:
                mlp_pre[name] = None
                continue
            mp: MlpPlan = plans[name + "_mlp"]
            nh2 = _lnm_fwd(h1[:, sl], segs[name], 3, 4)
            pre = torch.empty((B, sl.stop - sl.start, 4 * D), device=dev, dtype=torch.bfloat16)
            mb = mlp_base[name]
            pk1 = packs[name + "_fc1"] = _pack1(lora[mb], lora[mb + 1], 4 * D, D, scaling, dev, lsc(mb), full)
            pk2 = packs[name + "_fc2"] = _pack1(lora[mb + 2], lora[mb + 3], D, 4 * D, scaling, dev, lsc(mb + 2), full)
            act, t = _linear_lora_fwd(nh2, mp.w1, mp.b1, pk1, dr(base + 3), epi=ops.EPI_GELU, aux=pre)
            small[name + "_t_fc1"] = t
            del nh2
            small[name + "_t_fc2"] = _linear_lora_gate_res(act, mp.w2, mp.b2, pk2, dr(base + 4), segs[name], 5, res=h1[:, sl],
                                                           out=h2[:, sl], nan_to_num=(name == "txt" and nan_txt),
                                                           aux=y_at(y_mlp, sl))
            del act
            mlp_pre[name] = pre
        ctx.st = st
        ctx.packs = packs
        ctx.n_lora_in = n_lora_in
        ctx.lora_present = [x is not None for x in lora]
        E = h.new_empty(0)
        keep = lambda t: t if t is not None else E
        ctx.save_for_backward(h, mod_img, mod_txt, keep(cos), keep(sin), qkv, o, lse, h1, keep(mlp_pre["txt"]), mlp_pre["img"],
                              keep(small["txt_t_qkv"]), keep(small["img_t_qkv"]), keep(small["txt_t_out"]), keep(small["img_t_out"]),
                              keep(qkv2), keep(o2), keep(lse2), keep(small.get("a2_t_qkv")), keep(small.get("a2_t_out")),
                              q if keep_qk else E, k if keep_qk else E,
                              keep(small.get("txt_t_fc1")), keep(small.get("txt_t_fc2")), keep(small.get("img_t_fc1")),
                              keep(small.get("img_t_fc2")), keep(nh_joint), keep(y_attn), keep(y_mlp), keep(y_attn2))
        return h2

    @staticmethod
    def backward(ctx, dh2):
        (h, mod_img, mod_txt, cos, sin, qkv, o, lse, h1, pre_txt, pre_img, t_qkv_txt, t_qkv_img, t_out_txt, t_out_img,
         qkv2, o2, lse2, t_qkv_a2, t_out_a2, q_saved, k_saved, t_fc1_txt, t_fc2_txt, t_fc1_img, t_fc2_img, nh_saved,
         y_attn, y_mlp, y_attn2) = ctx.saved_tensors
        qk_saved = (q_saved, k_saved) if q_saved.numel() else None
        cos = cos if cos.numel() else None
        sin = sin if sin.numel() else None
        st = ctx.st
        packs = ctx.packs
        B, S, D = h.shape
        S_txt, H, hd = st["S_txt"], st["H"], st["hd"]
        plans = st["plans"]
        pre_only = st.get("context_pre_only", False)
        dual = st.get("dual", False)
        drop: Optional[LoraDrop] = st.get("lora_drop")
        dr = (lambda off: drop.at(off)) if drop is not None else (lambda off: None)
        full = st.get("full", False)
        dh2 = dh2.contiguous()
        segs = {"txt": _segments(mod_txt, None, S_txt), "img": _segments(mod_img, st.get("img_segs"), S - S_txt)}
        # d mod (full fine-tune): fp32 column sums, every chunk written
        dms = {"txt": torch.zeros_like(mod_txt, dtype=torch.float32), "img": torch.zeros_like(mod_img, dtype=torch.float32)} \
            if full else None
        streams = (("txt", slice(0, S_txt), mod_txt, 8, pre_txt, t_qkv_txt, t_out_txt),
                   ("img", slice(S_txt, S), mod_img, 0, pre_img, t_qkv_img, t_out_img))
        mlp_t = {"txt": (28, t_fc1_txt, t_fc2_txt), "img": (24, t_fc1_img, t_fc2_img)}
        grads: List[Optional[torch.Tensor]] = [None] * 38
        dh1 = torch.empty_like(h)
        d_o = torch.empty_like(o)
        for name, sl, mod, base, pre, t_qkv, t_out in streams:
            ap: AttnPlan = plans[name + "_attn"]
            if name == "txt" and pre_only:
                dh1[:, sl].copy_(dh2[:, sl])
                d_o[:, sl].zero_()
                continue
            mp: MlpPlan = plans[name + "_mlp"]
            # ---- MLP branch: h2 = h1 + gate_mlp * fc2(gelu(fc1(LNmod(h1))))
            if full:
                _dmod_gate(dms[name], dh2[:, sl], y_mlp[:, sl], 5)
            g2 = _gate_mul(dh2[:, sl], segs[name], 5)
            mb, t_fc1, t_fc2 = mlp_t[name]
            pk1, pk2 = packs.get(name + "_fc1"), packs.get(name + "_fc2")
            d_pre, t_up = _dgrad_through_gelu(g2, mp.w2_t, pk2, dr(base + 4), pre)
            if pk2 is not None:
                act = ops.gelu_tanh(pre)
                (grads[mb + 2], grads[mb + 3]), = _lora_grads(pk2, act, t_fc2, g2, t_up, dr(base + 4))
                del act
            del g2
            d_nh2, t_up = _linear_lora_dgrad(d_pre, mp.w1_t, pk1, dr(base + 3))
            if pk1 is not None:
                nh2 = _lnm_fwd(h1[:, sl], segs[name], 3, 4)
                (grads[mb], grads[mb + 1]), = _lora_grads(pk1, nh2, t_fc1, d_pre, t_up, dr(base + 3))
                del nh2
            del d_pre
            if full:
                _dmod_shift_scale(dms[name], d_nh2, h1[:, sl], 3, 4)
            _lnm_bwd(d_nh2, h1[:, sl], segs[name], 4, add=dh2[:, sl], out=dh1[:, sl])
            del d_nh2
            # ---- attention output projection: h1 = h + gate_msa * to_out(o)
            if full:
                _dmod_gate(dms[name], dh1[:, sl], y_attn[:, sl], 2)
            g1 = _gate_mul(dh1[:, sl], segs[name], 2)
            pk = packs[name + "_out"]
            _, t_up = _linear_lora_dgrad(g1, ap.w_out_t, pk, dr(base + 6), out=d_o[:, sl])
            if pk is not None:
                (da, db), = _lora_grads(pk, o[:, sl], t_out, g1, t_up, dr(base + 6))
                grads[base + 6], grads[base + 7] = da, db
            del g1
        # ---- image-only second attention (SD3.5 dual attention)
        d_nh2a = None
        if dual:
            isl = slice(S_txt, S)
            a2: AttnPlan = plans["img_attn2"]
            if full:
                _dmod_gate(dms["img"], dh1[:, isl], y_attn2, 8)
            g = ops.gate_mul(dh1[:, isl], mod_img[:, 8 * D:9 * D])
            pk = packs["a2_out"]
            d_o2, t_up = _linear_lora_dgrad(g, a2.w_out_t, pk, dr(22))
            if pk is not None:
                (da, db), = _lora_grads(pk, o2, t_out_a2, g, t_up, dr(22))
                grads[22], grads[23] = da, db
            del g
            dw2 = torch.zeros((4, hd), device=h.device, dtype=torch.float32) if full and a2.norm_q is not None else None
            d_qkv2 = _attn_core_bwd(qkv2, o2, d_o2, lse2, D, H, hd, a2, None, 0, None, None, dw=dw2)
            if dw2 is not None:
                grads[36], grads[37] = dw2.to(torch.bfloat16)[:2]
            del d_o2
            pk = packs["a2_qkv"]
            d_nh2a, t_up = _linear_lora_dgrad(d_qkv2, a2.w_qkv_t, pk, dr(16))
            if pk is not None:
                nh2a = ops.ln_modulate_fwd(h[:, isl], mod_img[:, 6 * D:7 * D], mod_img[:, 7 * D:8 * D], EPS)
                for m, (da, db) in enumerate(_lora_grads(pk, nh2a, t_qkv_a2, d_qkv2, t_up, dr(16))):
                    grads[16 + 2 * m], grads[16 + 2 * m + 1] = da, db
                del nh2a
            del d_qkv2
            if full:
                _dmod_shift_scale(dms["img"], d_nh2a, h[:, isl], 6, 7)
        # ---- joint attention core
        dw = torch.zeros((4, hd), device=h.device, dtype=torch.float32) if full and plans["img_attn"].norm_q is not None else None
        d_qkv = _attn_core_bwd(qkv, o, d_o, lse, D, H, hd, plans["img_attn"], plans["txt_attn"], S_txt, cos, sin, qk=qk_saved,
                               key_bias=st.get("key_bias"), dw=dw)
        if dw is not None:
            grads[32:36] = dw.to(torch.bfloat16)
        del qk_saved, q_saved, k_saved
        dh = torch.empty_like(h)
        for name, sl, mod, base, pre, t_qkv, t_out in streams:
            ap = plans[name + "_attn"]
            pk = packs[name + "_qkv"]
            ish, isc = (1, 0) if name == "txt" and pre_only else (0, 1)     # chunk indices of (shift, scale)
            d_nh, t_up = _linear_lora_dgrad(d_qkv[:, sl], ap.w_qkv_t, pk, dr(base))
            if pk is not None:
                for m, (da, db) in enumerate(_lora_grads(pk, nh_saved[:, sl], t_qkv, d_qkv[:, sl], t_up, dr(base))):
                    grads[base + 2 * m], grads[base + 2 * m + 1] = da, db
            if full:
                _dmod_shift_scale(dms[name], d_nh, h[:, sl], ish, isc)
            _lnm_bwd(d_nh, h[:, sl], segs[name], isc, add=dh1[:, sl], out=dh[:, sl])
            del d_nh
        if dual:
            isl = slice(S_txt, S)
            ops.ln_modulate_bwd(d_nh2a, h[:, isl], mod_img[:, 7 * D:8 * D], add=dh[:, isl], eps=EPS, out=dh[:, isl])
        out_grads = []
        for i in range(ctx.n_lora_in):
            out_grads.append(grads[i] if ctx.lora_present[i] else None)
        if full:
            return (dh, dms["img"].to(mod_img.dtype), dms["txt"].to(mod_txt.dtype), None, None, None, *out_grads)
        return (dh, None, None, None, None, None, *out_grads)


# ------------------------------------------------------------------------------------------------
# Single-stream block
# ------------------------------------------------------------------------------------------------
class SingleBlockFn(torch.autograd.Function):
    """h_out = FluxSingleTransformerBlock(h_in); LoRA order: to_q.A, to_q.B, to_k.A, to_k.B, to_v.A, to_v.B,
    proj_mlp.A, proj_mlp.B, proj_out.A, proj_out.B (the last four only for the "+ffs" / "tiny" / "nano" targets).
    Dropout mask streams: q, k, v = 0..2, proj_mlp = 3, proj_out = 4 (over the logical cat[attn, mlp] input)."""

    @staticmethod
    def forward(ctx, h, mod, cos, sin, st, *lora):
        B, S, D = h.shape
        H, hd = st["H"], st["hd"]
        plans = st["plans"]
        ap: AttnPlan = plans["attn"]
        mp: MlpPlan = plans["mlp"]
        dev = h.device
        n_lora_in = len(lora)
        lora = list(lora) + [None] * (10 - len(lora))
        scaling = st["lora_scaling"]
        ps = []
        for m in range(3):
            a, b = lora[2 * m], lora[2 * m + 1]
            ps.append(None if a is None else (a, b))
        ls = st.get("lokr_scales")
        lsc = (lambda i: ls[i // 2] if ls is not None and i // 2 < len(ls) else None)
        pk = make_pack(ps, D, D, scaling, dev, [lsc(0), lsc(2), lsc(4)])
        pk_mlp = _pack1(lora[6], lora[7], 4 * D, D, scaling, dev, lsc(6))
        pk_out = _pack1(lora[8], lora[9], D, 5 * D, scaling, dev, lsc(8))
        if isinstance(pk_out, WgradPack):
            raise NotImplementedError("LoKr on the single blocks' proj_out is not part of the LyCORIS presets supported here")
        drop: Optional[LoraDrop] = st.get("lora_drop")
        dr = (lambda off: drop.at(off)) if drop is not None else (lambda off: None)
        segs = _segments(mod, st.get("segs"), S)
        nh = _lnm_fwd(h, segs, 0, 1)
        qkv, t_qkv = _linear_lora_fwd(nh, ap.w_qkv, ap.b_qkv, pk, drop)
        q, k = ops.qk_rmsnorm_rope_fwd(qkv, D, H, hd, ap.norm_q, ap.norm_k, None, None, 0, cos, sin, EPS)
        v = qkv[:, :, 2 * D:].unflatten(-1, (H, hd))
        o, lse = ops.attn_fwd(q, k, v, key_bias=st.get("key_bias"))
        o = o.view(B, S, D)
        pre = torch.empty((B, S, 4 * D), device=dev, dtype=torch.bfloat16)
        act, t_mlp = _linear_lora_fwd(nh, mp.w1, mp.b1, pk_mlp, dr(3), epi=ops.EPI_GELU, aux=pre)
        nh_keep = nh if (pk is not None or pk_mlp is not None) else None
        del nh
        # proj_out(cat[attn, mlp]) as two K-segments of one GEMM; gate, residual, nan_to_num in the epilogue
        t_out = None
        if pk_out is None:
            h_out = _gemm_gate_res([o, act], [mp.w2[:, :D], mp.w2[:, D:]], mp.b2, segs, 2, res=h, nan_to_num=True)
        else:
            if drop is None:
                t_out = ops.gemm([o, act], [pk_out.a_stack[:, :D], pk_out.a_stack[:, D:]])
            else:                       # one mask over the logical [B, S, 5D] input of the adapted Linear
                t_out = _lora_down(torch.cat([o, act], 2), pk_out, dr(4))
            h_out = _gemm_gate_res([o, act, t_out], [mp.w2[:, :D], mp.w2[:, D:], pk_out.b_ext], mp.b2, segs, 2, res=h,
                                   nan_to_num=True)
        del act
        ctx.st = st
        ctx.packs = (pk, pk_mlp, pk_out)
        ctx.n_lora_in = n_lora_in
        ctx.lora_present = [x is not None for x in lora]
        E = h.new_empty(0)
        keep = lambda t: t if t is not None else E
        ctx.save_for_backward(h, mod, cos, sin, qkv, o, lse, pre, keep(t_qkv), q, k, keep(t_mlp), keep(t_out), keep(nh_keep))
        return h_out

    @staticmethod
    def backward(ctx, dh_out):
        h, mod, cos, sin, qkv, o, lse, pre, t_qkv, q, k, t_mlp, t_out, nh = ctx.saved_tensors
        st = ctx.st
        pk, pk_mlp, pk_out = ctx.packs
        B, S, D = h.shape
        H, hd = st["H"], st["hd"]
        ap: AttnPlan = st["plans"]["attn"]
        mp: MlpPlan = st["plans"]["mlp"]
        drop: Optional[LoraDrop] = st.get("lora_drop")
        dr = (lambda off: drop.at(off)) if drop is not None else (lambda off: None)
        dh_out = dh_out.contiguous()
        grads: List[Optional[torch.Tensor]] = [None] * 10
        segs = _segments(mod, st.get("segs"), S)
        g = _gate_mul(dh_out, segs, 2)
        if pk_out is None:
            d_o = ops.gemm([g], [mp.w2_t[:D]], None)
            d_pre = ops.gemm([g], [mp.w2_t[D:]], None, epi=ops.EPI_MUL_DGELU, aux=pre)
        else:
            t_up = ops.gemm([g], [pk_out.b_ext_t])
            act = ops.gelu_tanh(pre)
            if drop is None:
                d_o = ops.gemm([g, t_up], [mp.w2_t[:D], pk_out.a_stack_t[:D]], None)
                d_pre = ops.gemm([g, t_up], [mp.w2_t[D:], pk_out.a_stack_t[D:]], None, epi=ops.EPI_MUL_DGELU, aux=pre)
                (grads[8], grads[9]), = _lora_grads(pk_out, (o, act), t_out, g, t_up, None)
            else:
                d_cat = ops.gemm([g], [mp.w2_t], None)
                _lora_dgrad_dropout(d_cat, t_up, pk_out, dr(4))
                d_o = d_cat[:, :, :D].contiguous()
                d_pre = ops.mul_dgelu_tanh(d_cat[:, :, D:], pre)
                del d_cat
                (grads[8], grads[9]), = _lora_grads(pk_out, torch.cat([o, act], 2), t_out, g, t_up, dr(4))
            del act, t_up
        del g
        d_qkv = _attn_core_bwd(qkv, o, d_o, lse, D, H, hd, ap, None, 0, cos, sin, qk=(q, k), key_bias=st.get("key_bias"))
        del d_o, q, k
        # d_nh = d_pre W_mlp + d_qkv W_qkv (+ LoRA branches as one more K-segment)
        t_ups, a_ts = [], []
        t_up_qkv = t_up_mlp = None
        is_lora = lambda q: q is not None and not isinstance(q, WgradPack)
        if is_lora(pk):
            t_up_qkv = ops.gemm([d_qkv], [pk.b_ext_t])
            t_ups.append(t_up_qkv); a_ts.append(pk.a_stack_t)
        if is_lora(pk_mlp):
            t_up_mlp = ops.gemm([d_pre], [pk_mlp.b_ext_t])
            t_ups.append(t_up_mlp); a_ts.append(pk_mlp.a_stack_t)
        if not t_ups or drop is not None:
            d_nh = ops.gemm([d_pre, d_qkv], [mp.w1_t, ap.w_qkv_t], None)
            if is_lora(pk):
                _lora_dgrad_dropout(d_nh, t_up_qkv, pk, drop)
            if is_lora(pk_mlp):
                _lora_dgrad_dropout(d_nh, t_up_mlp, pk_mlp, dr(3))
        elif len(t_ups) == 1:
            d_nh = ops.gemm([d_pre, d_qkv, t_ups[0]], [mp.w1_t, ap.w_qkv_t, a_ts[0]], None)
        else:                           # the GEMM takes three K-segments: both rank blocks travel as one
            d_nh = ops.gemm([d_pre, d_qkv, torch.cat(t_ups, 2)], [mp.w1_t, ap.w_qkv_t, torch.cat(a_ts, 1)], None)
        if pk is not None:
            for m, (da, db) in enumerate(_lora_grads(pk, nh, t_qkv, d_qkv, t_up_qkv, drop)):
                grads[2 * m], grads[2 * m + 1] = da, db
        if pk_mlp is not None:
            (grads[6], grads[7]), = _lora_grads(pk_mlp, nh, t_mlp, d_pre, t_up_mlp, dr(3))
        del nh, d_pre, d_qkv
        dh = _lnm_bwd(d_nh, h, segs, 1, add=dh_out)
        out = [grads[i] if ctx.lora_present[i] else None for i in range(ctx.n_lora_in)]
        return (dh, None, None, None, None, *out)


# ------------------------------------------------------------------------------------------------
# Tail: AdaLayerNormContinuous + proj_out   (reference flux/transformer.py:1503-1506)
# ------------------------------------------------------------------------------------------------
class TailFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h, mod, st, *lora):
        """h [B, S, D] joint buffer; mod [B, 2D] = (scale | shift) (AdaLayerNormContinuous chunk order).  lora: the final
        proj_out's (A, B) — PEFT's suffix rule makes the "proj_out" target of "all+ffs" select it too — or, with
        st["full"], proj_out's (weight, bias), and d mod is returned too.  Rows [S_txt, S_end) are projected (S_end: the
        end of the Kontext scene tokens, default S)."""
        D = h.shape[2]
        S_txt, S_end = st["S_txt"], st.get("S_end") or h.shape[1]
        x = h[:, S_txt:S_end]
        nx = ops.ln_modulate_fwd(x, mod[:, D:2 * D], mod[:, 0:D], EPS)
        a, b = (lora[0], lora[1]) if len(lora) >= 2 else (None, None)
        pk = _pack1(a, b, st["w_proj"].shape[0], D, st.get("lora_scaling", 1.0), h.device, full=st.get("full", False))
        out, t = _linear_lora_fwd(nx, st["w_proj"], st["b_proj"], pk, st.get("lora_drop"))
        ctx.st, ctx.pack, ctx.n_lora_in = st, pk, len(lora)
        ctx.save_for_backward(h, mod, t if t is not None else h.new_empty(0))
        return out

    @staticmethod
    def backward(ctx, d_out):
        h, mod, t = ctx.saved_tensors
        st, pk = ctx.st, ctx.pack
        D = h.shape[2]
        S_txt, S_end = st["S_txt"], st.get("S_end") or h.shape[1]
        d_out = d_out.contiguous()
        d_nx, t_up = _linear_lora_dgrad(d_out, st["w_proj_t"], pk, st.get("lora_drop"))
        lg = [None] * ctx.n_lora_in
        if pk is not None:
            nx = ops.ln_modulate_fwd(h[:, S_txt:S_end], mod[:, D:2 * D], mod[:, 0:D], EPS)
            (lg[0], lg[1]), = _lora_grads(pk, nx, t, d_out, t_up, st.get("lora_drop"))
        dm = None
        if st.get("full", False):
            dm = torch.zeros_like(mod, dtype=torch.float32)
            _dmod_shift_scale(dm, d_nx, h[:, S_txt:S_end], 1, 0)
            dm = dm.to(mod.dtype)
        dh = torch.zeros_like(h) if S_txt > 0 or S_end < h.shape[1] else torch.empty_like(h)
        ops.ln_modulate_bwd(d_nx, h[:, S_txt:S_end], mod[:, 0:D], add=None, eps=EPS, out=dh[:, S_txt:S_end])
        return (dh, dm, None, *lg)


class FlowLossFn(torch.autograd.Function):
    """loss = mean_b mean_chw (unpack(pred) - (noise - latents))^2 ; backward = precomputed d loss/d pred."""

    @staticmethod
    def forward(ctx, pred_packed, latents, noise, layout=0, loss_type="l2", huber_c=None):
        loss, dpred = ops.flow_mse_loss(pred_packed.contiguous(), latents, noise, want_grad=True, layout=layout,
                                        loss_type=loss_type, huber_c=huber_c)
        ctx.save_for_backward(dpred)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (dpred,) = ctx.saved_tensors
        # g is the scalar upstream gradient (1.0 for loss.backward(), 1/accum under gradient accumulation); it stays on
        # the device and multiplies in fp32 — rounding g itself to bf16 (1/3 -> 0.33398) would bias every gradient
        return (dpred.float() * g.float()).to(dpred.dtype), None, None, None, None, None
