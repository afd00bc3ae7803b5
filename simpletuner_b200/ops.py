"""Tensor-level launchers for libstb200 (no autograd here — see functional.py).

Every function takes CUDA bf16 tensors (views with arbitrary batch/row strides are fine as long as
the last dimension is contiguous), launches on torch's *current* stream and returns torch tensors
that own their memory through torch's caching allocator.  PyTorch is plumbing only: all arithmetic
happens inside libstb200.so.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import QkPrep, AttnBwdArgs, AttnFwdArgs, GemmArgs, check

EPI_STORE, EPI_GELU, EPI_GATE_RES, EPI_MUL_DGELU, EPI_ADD_RES, EPI_MUL, EPI_QUICK_GELU = 0, 1, 2, 3, 4, 5, 6


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _as3d(t: torch.Tensor) -> torch.Tensor:
    """[M, K] -> [1, M, K]; [B, S, K] stays (views allowed)."""
    if t.dim() == 2:
        return t.unsqueeze(0)
    if t.dim() != 3:
        raise ValueError(f"expected a 2-D or 3-D tensor, got {tuple(t.shape)}")
    return t


def _chk(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise _lib.StbError(f"{name} must be a CUDA tensor (simpletuner_b200 has no CPU path)")
    if t.dtype != torch.bfloat16:
        raise TypeError(f"{name} must be bfloat16, got {t.dtype}")
    if t.stride(-1) != 1:
        raise ValueError(f"{name} must be contiguous in its last dimension")


class WT:
    """W^T without a copy: stands for the transpose of a forward weight `w` [N, K] wherever a dgrad GEMM wants W^T [K, N]
    in nn.Linear layout.  `gemm` hands `w` itself to the kernel as a [K_contract, N_out] operand (stb_gemm_seg.w_kn: the B
    tile is staged MN-major by TMA), so no transposed copy of the weights exists in HBM.  Row slices of the virtual W^T are
    column slices of w."""
    __slots__ = ("w",)

    def __init__(self, w: torch.Tensor):
        self.w = w

    def __getitem__(self, idx):
        if isinstance(idx, slice):
            return WT(self.w[:, idx])
        raise TypeError("WT supports row slices only")

    @property
    def shape(self):
        return (self.w.shape[1], self.w.shape[0])


def gemm(
    a_list: Sequence[torch.Tensor],
    w_list: Sequence[torch.Tensor],
    bias: Optional[torch.Tensor] = None,
    *,
    out: Optional[torch.Tensor] = None,
    epi: int = EPI_STORE,
    gate: Optional[torch.Tensor] = None,
    res: Optional[torch.Tensor] = None,
    aux: Optional[torch.Tensor] = None,
    nan_to_num: bool = False,
    tile: Tuple[int, int] = (0, 0),
    w_kn: Optional[Sequence[bool]] = None,
) -> torch.Tensor:
    """out[b, s, :] = epi( sum_i a_list[i][b, s, :] @ w_list[i].T + bias ).

    a_list[i]: [B, S, K_i] or [M, K_i];  w_list[i]: [N, K_i] (nn.Linear layout, row stride free) — or, where w_kn[i] is
    set, [K_i, N] (the contraction index is the row: `a @ w`, e.g. the dgrad of a Linear on its forward weight).
    gate: [B, N];  res / aux / out: same leading shape as a_list[0] with last dim N.
    tile = (mt, bn): bn 64, 128 or 256 forces the tile width (0 = automatic); mt 2 runs 128 x 128 tiles as 2-CTA
    clusters that share the W tile (the other widths run single CTAs), 1 single CTAs, 0 chooses (clusters for the
    GELU / dGELU epilogues with at least 16 m-tiles).  Both give the same bits.
    """
    nseg = len(a_list)
    assert 1 <= nseg <= 3 and len(w_list) == nseg
    if any(isinstance(w, WT) for w in w_list):
        w_kn = [isinstance(w, WT) or bool(w_kn[i] if w_kn is not None else False) for i, w in enumerate(w_list)]
        w_list = [w.w if isinstance(w, WT) else w for w in w_list]
    a0 = _as3d(a_list[0])
    B, S, _ = a0.shape
    kn = list(w_kn) if w_kn is not None else [False] * nseg
    N = w_list[0].shape[1] if kn[0] else w_list[0].shape[0]
    squeeze = a_list[0].dim() == 2
    if out is None:
        out = torch.empty((B, S, N), device=a0.device, dtype=torch.bfloat16)
    out3 = _as3d(out)
    _chk(out3, "out")
    args = GemmArgs()
    args.num_batches, args.rows_per_batch, args.N, args.nseg = B, S, N, nseg
    for i, (a, w) in enumerate(zip(a_list, w_list)):
        a3 = _as3d(a)
        _chk(a3, f"a[{i}]")
        _chk(w, f"w[{i}]")
        wn, wk = (w.shape[1], w.shape[0]) if kn[i] else (w.shape[0], w.shape[1])
        if a3.shape[0] != B or a3.shape[1] != S or wn != N or wk != a3.shape[2]:
            raise ValueError(f"segment {i}: shapes {tuple(a3.shape)} x {tuple(w.shape)} do not match")
        sg = args.seg[i]
        sg.a, sg.a_batch_stride, sg.a_row_stride = a3.data_ptr(), a3.stride(0), a3.stride(1)
        sg.w, sg.w_row_stride, sg.K, sg.w_kn = w.data_ptr(), w.stride(0), a3.shape[2], int(bool(kn[i]))
    args.d, args.d_batch_stride, args.d_row_stride = out3.data_ptr(), out3.stride(0), out3.stride(1)
    args.bias = _ptr(bias)
    args.epi = epi
    args.nan_to_num = int(nan_to_num)
    if gate is not None:
        _chk(gate, "gate")
        g2 = gate if gate.dim() == 2 else gate.reshape(B, N)
        args.gate, args.gate_batch_stride = g2.data_ptr(), g2.stride(0)
    if res is not None:
        r3 = _as3d(res)
        _chk(r3, "res")
        args.res, args.res_batch_stride, args.res_row_stride = r3.data_ptr(), r3.stride(0), r3.stride(1)
    if aux is not None:
        x3 = _as3d(aux)
        _chk(x3, "aux")
        args.aux, args.aux_batch_stride, args.aux_row_stride = x3.data_ptr(), x3.stride(0), x3.stride(1)
    args.tile_mt, args.tile_bn = tile
    check(_lib.lib().stb_gemm_bf16(C.byref(args), _stream()))
    return out.squeeze(0) if (squeeze and out.dim() == 3) else out


def _key_bias_stride(key_bias: torch.Tensor, B: int, Sk: int) -> int:
    """Batch stride of a per-key logit bias bf16 [B or 1, Sk] (keys contiguous); 0 when one row serves the batch."""
    _chk(key_bias, "key_bias")
    if key_bias.dim() != 2 or key_bias.shape[0] not in (1, B) or key_bias.shape[1] != Sk or key_bias.stride(1) != 1:
        raise ValueError(f"key_bias must be [B or 1, Sk] = [{B} or 1, {Sk}] with contiguous keys, got "
                         f"{tuple(key_bias.shape)} strides {key_bias.stride()}")
    return 0 if key_bias.shape[0] == 1 else key_bias.stride(0)


def attn_fwd(q, k, v, scale: Optional[float] = None, out: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
             key_bias: Optional[torch.Tensor] = None):
    """q/k/v: [B, S, H, HD] views (HD contiguous).  Returns (o [B,Sq,H,HD] bf16, lse [B,H,Sq] fp32).
    bias (forward only): bf16 [H or 1, Sq, Sk] additive logit bias / mask shared by the batch.
    key_bias: bf16 [B or 1, Sk] additive logit bias per sample and key (Flux masked training); attn_bwd takes it too."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _chk(t, n)
    B, Sq, H, HD = q.shape
    Sk = k.shape[1]
    if scale is None:
        scale = HD ** -0.5
    if out is None:
        out = torch.empty((B, Sq, H, HD), device=q.device, dtype=torch.bfloat16)
    lse = torch.empty((B, H, Sq), device=q.device, dtype=torch.float32)
    a = AttnFwdArgs()
    a.B, a.H, a.Sq, a.Sk, a.HD, a.scale = B, H, Sq, Sk, HD, float(scale)
    a.q, a.k, a.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    a.q_b, a.q_s, a.q_h = q.stride(0), q.stride(1), q.stride(2)
    a.k_b, a.k_s, a.k_h = k.stride(0), k.stride(1), k.stride(2)
    a.v_b, a.v_s, a.v_h = v.stride(0), v.stride(1), v.stride(2)
    a.o = out.data_ptr()
    a.o_b, a.o_s, a.o_h = out.stride(0), out.stride(1), out.stride(2)
    a.lse = lse.data_ptr()
    if bias is not None and key_bias is not None:
        raise ValueError("give either bias or key_bias, not both")
    if bias is not None:
        _chk(bias, "bias")
        assert bias.dim() == 3 and bias.shape[0] in (1, H) and bias.shape[1] == Sq and bias.shape[2] == Sk
        a.bias, a.bias_h, a.bias_q = bias.data_ptr(), (0 if bias.shape[0] == 1 else bias.stride(0)), bias.stride(1)
    if key_bias is not None:
        a.bias, a.bias_b, a.bias_h, a.bias_q = key_bias.data_ptr(), _key_bias_stride(key_bias, B, Sk), 0, 0
    check(_lib.lib().stb_attn_fwd(C.byref(a), _stream()))
    return out, lse


def attn_bwd(q, k, v, o, d_o, lse, scale: Optional[float] = None, dq=None, dk=None, dv=None, qk_prep: Optional[dict] = None,
             key_bias: Optional[torch.Tensor] = None):
    """Backward of attn_fwd.  Returns (dq, dk, dv) shaped like q, k, v ([B, S, H, HD], bf16).  key_bias: the forward's.

    qk_prep (self-attention only): dict(src=[B,S,C] pre-norm projection output, k_off, wq, wk, wq_added, wk_added,
    s_split, cos, sin, eps) — fuses the backward of qk_rmsnorm_rope_fwd into the epilogues, so dq / dk receive the
    gradient w.r.t. the projection outputs (what qk_rmsnorm_rope_bwd would write)."""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (o, "o"), (d_o, "d_o")):
        _chk(t, n)
    B, Sq, H, HD = q.shape
    Sk = k.shape[1]
    if scale is None:
        scale = HD ** -0.5
    dq = torch.empty((B, Sq, H, HD), device=q.device, dtype=torch.bfloat16) if dq is None else dq
    dk = torch.empty((B, Sk, H, HD), device=q.device, dtype=torch.bfloat16) if dk is None else dk
    dv = torch.empty((B, Sk, H, HD), device=q.device, dtype=torch.bfloat16) if dv is None else dv
    delta = torch.empty((B, H, Sq), device=q.device, dtype=torch.float32)
    a = AttnBwdArgs()
    a.B, a.H, a.Sq, a.Sk, a.HD, a.scale = B, H, Sq, Sk, HD, float(scale)
    a.q, a.k, a.v, a.o, a.d_o = q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), d_o.data_ptr()
    a.q_b, a.q_s, a.q_h = q.stride(0), q.stride(1), q.stride(2)
    a.k_b, a.k_s, a.k_h = k.stride(0), k.stride(1), k.stride(2)
    a.v_b, a.v_s, a.v_h = v.stride(0), v.stride(1), v.stride(2)
    a.o_b, a.o_s, a.o_h = o.stride(0), o.stride(1), o.stride(2)
    a.do_b, a.do_s, a.do_h = d_o.stride(0), d_o.stride(1), d_o.stride(2)
    a.lse, a.delta, a.dq_accum = lse.data_ptr(), delta.data_ptr(), None
    a.dq, a.dk, a.dv = dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
    a.dq_b, a.dq_s, a.dq_h = dq.stride(0), dq.stride(1), dq.stride(2)
    a.dk_b, a.dk_s, a.dk_h = dk.stride(0), dk.stride(1), dk.stride(2)
    a.dv_b, a.dv_s, a.dv_h = dv.stride(0), dv.stride(1), dv.stride(2)
    if qk_prep is not None:
        f = _lib.QkPrep()
        src = qk_prep["src"]
        _chk(src, "qk_prep.src")
        f.src, f.src_b, f.src_s, f.k_off = src.data_ptr(), src.stride(0), src.stride(1), int(qk_prep["k_off"])
        f.wq, f.wk = _ptr(qk_prep.get("wq")), _ptr(qk_prep.get("wk"))
        f.wq_added, f.wk_added = _ptr(qk_prep.get("wq_added")), _ptr(qk_prep.get("wk_added"))
        f.s_split = int(qk_prep.get("s_split", 0))
        cos, sin = qk_prep.get("cos"), qk_prep.get("sin")
        if cos is not None:
            assert cos.dtype == torch.float32 and cos.is_contiguous() and cos.shape == (Sq, HD) and sin.shape == (Sq, HD)
        f.cos_t, f.sin_t = _ptr(cos), _ptr(sin)
        f.eps = float(qk_prep.get("eps", 1e-6))
        a.qk_prep = C.pointer(f)
    if key_bias is not None:
        a.bias, a.bias_b = key_bias.data_ptr(), _key_bias_stride(key_bias, B, Sk)
    check(_lib.lib().stb_attn_bwd(C.byref(a), _stream()))
    return dq, dk, dv


def ln_modulate_fwd(x, shift, scale, eps: float = 1e-6, out=None):
    """out = LayerNorm(x) * (1 + scale[:, None]) + shift[:, None];  x [B,S,D], shift/scale [B,D] views
    that share one batch stride (slices of the same modulation tensor)."""
    _chk(x, "x"); _chk(shift, "shift"); _chk(scale, "scale")
    B, S, D = x.shape
    assert shift.shape == (B, D) and scale.shape == (B, D) and shift.stride(0) == scale.stride(0)
    if out is None:
        out = torch.empty((B, S, D), device=x.device, dtype=torch.bfloat16)
    check(_lib.lib().stb_ln_modulate_fwd(
        x.data_ptr(), x.stride(0), x.stride(1), shift.data_ptr(), scale.data_ptr(), shift.stride(0),
        out.data_ptr(), out.stride(0), out.stride(1), B, S, D, eps, _stream()))
    return out


def ln_modulate_bwd(dy, x, scale, add=None, eps: float = 1e-6, out=None):
    """dx of ln_modulate_fwd w.r.t. x (+ add, the residual-branch gradient)."""
    _chk(dy, "dy"); _chk(x, "x"); _chk(scale, "scale")
    B, S, D = x.shape
    if out is None:
        out = torch.empty((B, S, D), device=x.device, dtype=torch.bfloat16)
    ab, as_ = (add.stride(0), add.stride(1)) if add is not None else (0, 0)
    check(_lib.lib().stb_ln_modulate_bwd(
        dy.data_ptr(), dy.stride(0), dy.stride(1), x.data_ptr(), x.stride(0), x.stride(1),
        scale.data_ptr(), scale.stride(0), _ptr(add), ab, as_,
        out.data_ptr(), out.stride(0), out.stride(1), B, S, D, eps, _stream()))
    return out


def qk_rmsnorm_rope_fwd(src, k_off, H, HD, wq, wk, wq_added=None, wk_added=None, s_split=0,
                        cos=None, sin=None, eps: float = 1e-6, q_out=None, k_out=None):
    """src [B, S, C] projection output with q at column 0 and k at column k_off.
    Returns q, k as [B, S, H, HD]."""
    _chk(src, "src")
    B, S, _ = src.shape
    if q_out is None:
        q_out = torch.empty((B, S, H, HD), device=src.device, dtype=torch.bfloat16)
    if k_out is None:
        k_out = torch.empty((B, S, H, HD), device=src.device, dtype=torch.bfloat16)
    assert q_out.stride() == k_out.stride() and q_out.stride(2) == HD and q_out.stride(3) == 1
    if cos is not None:
        assert cos.dtype == torch.float32 and cos.is_contiguous() and cos.shape == (S, HD)
        assert sin.dtype == torch.float32 and sin.is_contiguous() and sin.shape == (S, HD)
    check(_lib.lib().stb_qk_rmsnorm_rope_fwd(
        src.data_ptr(), src.stride(0), src.stride(1), k_off, _ptr(wq), _ptr(wk), _ptr(wq_added), _ptr(wk_added),
        s_split, _ptr(cos), _ptr(sin), q_out.data_ptr(), k_out.data_ptr(), q_out.stride(0), q_out.stride(1),
        B, S, H, HD, eps, _stream()))
    return q_out, k_out


def qk_rmsnorm_rope_bwd(dq, dk, src, k_off, H, HD, wq, wk, wq_added=None, wk_added=None, s_split=0,
                        cos=None, sin=None, eps: float = 1e-6, dsrc=None, dw=None):
    """Writes the q / k column ranges of dsrc ([B, S, C], same layout as src).  dw (optional): zero-initialised fp32
    [4, HD] that receives the RMSNorm weight gradients (wq, wk, wq_added, wk_added) — full fine-tune."""
    B, S, _ = src.shape
    assert dq.stride() == dk.stride() and dq.stride(2) == HD
    if dsrc is None:
        dsrc = torch.empty_like(src)
    check(_lib.lib().stb_qk_rmsnorm_rope_bwd(
        dq.data_ptr(), dk.data_ptr(), dq.stride(0), dq.stride(1), src.data_ptr(), src.stride(0), src.stride(1),
        k_off, _ptr(wq), _ptr(wk), _ptr(wq_added), _ptr(wk_added), s_split, _ptr(cos), _ptr(sin),
        dsrc.data_ptr(), dsrc.stride(0), dsrc.stride(1), B, S, H, HD, eps, _ptr(dw), _stream()))
    return dsrc


def flow_prep_pack(latents, noise, sigmas, want_unpacked: bool = True, out=None):
    """Returns (noisy [B,C,H,W] or None, packed [B, H/2*W/2, 4C]).  out: a [B, H/2*W/2, 4C] view with dense tokens
    (e.g. a token range of a longer joint sequence) that receives the packed tokens.  noise = sigmas = None: plain
    pack_latents of `latents` (no noisy output)."""
    assert latents.is_contiguous()
    _chk(latents, "latents")
    if noise is not None:
        assert noise.is_contiguous() and sigmas.dtype == torch.float32
        _chk(noise, "noise")
    else:
        assert sigmas is None
        want_unpacked = False
    B, Cc, Hh, Ww = latents.shape
    noisy = torch.empty_like(latents) if want_unpacked else None
    shape = (B, (Hh // 2) * (Ww // 2), 4 * Cc)
    if out is None:
        out = torch.empty(shape, device=latents.device, dtype=torch.bfloat16)
    _chk(out, "out")
    if tuple(out.shape) != shape or out.stride(2) != 1 or out.stride(1) != 4 * Cc or out.dtype != torch.bfloat16:
        raise ValueError(f"flow_prep_pack: out must be a bf16 {shape} view with dense tokens")
    check(_lib.lib().stb_flow_prep_pack(latents.data_ptr(), _ptr(noise), _ptr(None if sigmas is None else sigmas.contiguous()),
                                        _ptr(noisy), out.data_ptr(), out.stride(0), B, Cc, Hh, Ww, _stream()))
    return noisy, out


LOSS_TYPES = {"l2": 0, "huber": 1, "smooth_l1": 2}


def _huber_arg(loss_type, huber_c, B, device):
    lt = LOSS_TYPES[loss_type] if isinstance(loss_type, str) else int(loss_type)
    if lt == 0:
        return lt, None
    if huber_c is None:
        raise ValueError("huber / smooth_l1 need huber_c")
    if not torch.is_tensor(huber_c):
        huber_c = torch.full((B,), float(huber_c), dtype=torch.float32)
    huber_c = huber_c.to(device=device, dtype=torch.float32).reshape(-1)
    if huber_c.numel() == 1:
        huber_c = huber_c.expand(B)
    assert huber_c.numel() == B
    return lt, huber_c.contiguous()


def flow_mse_loss(pred_packed, latents, noise, want_grad: bool = True, grad_scale: float = 1.0, layout: int = 0,
                  loss_type="l2", huber_c=None):
    """Returns (loss fp32 scalar tensor [1], dpred_packed or None).  loss_type: "l2" | "huber" | "smooth_l1"."""
    assert pred_packed.is_contiguous() and latents.is_contiguous() and noise.is_contiguous()
    B, Cc, Hh, Ww = latents.shape
    lt, hc = _huber_arg(loss_type, huber_c, B, latents.device)
    loss = torch.empty((1,), device=latents.device, dtype=torch.float32)
    dpred = torch.empty_like(pred_packed) if want_grad else None
    check(_lib.lib().stb_flow_mse_loss(pred_packed.data_ptr(), latents.data_ptr(), noise.data_ptr(),
                                       loss.data_ptr(), _ptr(dpred), grad_scale, B, Cc, Hh, Ww, layout, lt, _ptr(hc), _stream()))
    return loss, dpred


def ddpm_prep_pack(latents, noise, coef_a, coef_b, want_unpacked: bool = True, want_packed: bool = True):
    """noisy = (coef_a[b] * latents.float() + coef_b[b] * noise.float()).bf16 -> (noisy or None, packed (c,dy,dx) or None)."""
    assert latents.is_contiguous() and noise.is_contiguous() and coef_a.dtype == torch.float32 and coef_b.dtype == torch.float32
    _chk(latents, "latents"); _chk(noise, "noise")
    B, Cc, Hh, Ww = latents.shape
    noisy = torch.empty_like(latents) if want_unpacked else None
    packed = torch.empty((B, (Hh // 2) * (Ww // 2), 4 * Cc), device=latents.device, dtype=torch.bfloat16) if want_packed else None
    check(_lib.lib().stb_ddpm_prep_pack(latents.data_ptr(), noise.data_ptr(), coef_a.contiguous().data_ptr(),
                                        coef_b.contiguous().data_ptr(), _ptr(noisy), _ptr(packed), B, Cc, Hh, Ww, _stream()))
    return noisy, packed


def target_mse_loss(pred_packed, target, weights=None, want_grad: bool = True, grad_scale: float = 1.0, layout: int = 1,
                    loss_type="l2", huber_c=None):
    """mean_b[w_b * mean_chw (pred - target)^2]; pred packed [B, S, 4C], target [B,C,H,W] -> (loss [1] fp32, dpred or None)."""
    assert pred_packed.is_contiguous() and target.is_contiguous()
    _chk(pred_packed, "pred"); _chk(target, "target")
    B, Cc, Hh, Ww = target.shape
    assert pred_packed.shape == target.shape if layout == 2 else pred_packed.shape[-1] == 4 * Cc
    if weights is not None:
        assert weights.dtype == torch.float32 and weights.numel() == B and weights.is_cuda
        weights = weights.contiguous()
    lt, hc = _huber_arg(loss_type, huber_c, B, target.device)
    loss = torch.empty((1,), device=target.device, dtype=torch.float32)
    dpred = torch.empty_like(pred_packed) if want_grad else None
    check(_lib.lib().stb_target_mse_loss(pred_packed.data_ptr(), target.data_ptr(), _ptr(weights), loss.data_ptr(),
                                         _ptr(dpred), grad_scale, B, Cc, Hh, Ww, layout, lt, _ptr(hc), _stream()))
    return loss, dpred


def gate_mul(x, gate, out=None):
    """out[b, s, :] = gate[b, :] * x[b, s, :]."""
    _chk(x, "x"); _chk(gate, "gate")
    B, S, D = x.shape
    if out is None:
        out = torch.empty((B, S, D), device=x.device, dtype=torch.bfloat16)
    check(_lib.lib().stb_gate_mul(x.data_ptr(), x.stride(0), x.stride(1), gate.data_ptr(), gate.stride(0),
                                  out.data_ptr(), out.stride(0), out.stride(1), B, S, D, _stream()))
    return out


def lokr_rebuild(W, w1, w2, scale: float, out, out_t=None):
    """out = bf16(W + kron(w1, w2) * scale) (and its transpose into out_t): row-strided 2-D views (fused projection layouts)."""
    for t, nm in ((W, "W"), (w1, "w1"), (w2, "w2"), (out, "out")):
        _chk(t, nm)
    (a, c), (b, d) = w1.shape, w2.shape
    assert W.shape == (a * b, c * d) and out.shape == W.shape and w1.is_contiguous() and w2.is_contiguous()
    if out_t is not None:
        _chk(out_t, "out_t")
        assert out_t.shape == (c * d, a * b)
    check(_lib.lib().stb_lokr_rebuild(W.data_ptr(), W.stride(0), w1.data_ptr(), w2.data_ptr(), float(scale), out.data_ptr(),
                                      out.stride(0), _ptr(out_t), out_t.stride(0) if out_t is not None else 0, a, b, c, d, _stream()))
    return out


def lokr_factor_grads(dW, w1, w2, scale: float):
    """(dw1 [a, c], dw2 [b, d]) fp32 from the full weight gradient dW [a b, c d] (bf16 view with unit inner stride)."""
    for t, nm in ((dW, "dW"), (w1, "w1"), (w2, "w2")):
        _chk(t, nm)
    (a, c), (b, d) = w1.shape, w2.shape
    assert dW.shape == (a * b, c * d) and w1.is_contiguous() and w2.is_contiguous()
    dw1 = torch.empty((a, c), device=dW.device, dtype=torch.float32)
    dw2 = torch.empty((b, d), device=dW.device, dtype=torch.float32)
    check(_lib.lib().stb_lokr_factor_grads(dW.data_ptr(), dW.stride(0), w1.data_ptr(), w2.data_ptr(), float(scale),
                                           dw1.data_ptr(), dw2.data_ptr(), a, b, c, d, _stream()))
    return dw1, dw2


def rmsnorm_fwd(x, w, eps: float, out=None):
    """T5LayerNorm: out = w * bf16(x * rsqrt(mean(x^2) + eps)) for a [B, S, D] view."""
    _chk(x, "x"); _chk(w, "w")
    B, S, D = x.shape
    if out is None:
        out = torch.empty((B, S, D), device=x.device, dtype=torch.bfloat16)
    check(_lib.lib().stb_rmsnorm_fwd(x.data_ptr(), x.stride(0), x.stride(1), w.data_ptr(), out.data_ptr(), out.stride(0),
                                     out.stride(1), B, S, D, float(eps), _stream()))
    return out


def gelu_tanh(pre, out=None):
    """out = gelu_tanh(pre) for a [B, S, D] view — the activation EPI_GELU produced, re-created from the saved pre-activation."""
    _chk(pre, "pre")
    B, S, D = pre.shape
    if out is None:
        out = torch.empty((B, S, D), device=pre.device, dtype=torch.bfloat16)
    check(_lib.lib().stb_gelu_tanh(pre.data_ptr(), pre.stride(0), pre.stride(1), None, 0, 0, out.data_ptr(), out.stride(0),
                                   out.stride(1), B, S, D, 0, _stream()))
    return out


def mul_dgelu_tanh(g, pre, out=None):
    """out = g * gelu_tanh'(pre)  ([B, S, D] views; out may alias g)."""
    _chk(pre, "pre"); _chk(g, "g")
    B, S, D = pre.shape
    assert g.shape == pre.shape
    if out is None:
        out = torch.empty((B, S, D), device=pre.device, dtype=torch.bfloat16)
    check(_lib.lib().stb_gelu_tanh(pre.data_ptr(), pre.stride(0), pre.stride(1), g.data_ptr(), g.stride(0), g.stride(1),
                                   out.data_ptr(), out.stride(0), out.stride(1), B, S, D, 1, _stream()))
    return out


def dropout_expand(x, members: int, p: float, seed: int, stream0: int):
    """x [B, S, K] (view) -> [members, B, S, K]: x * keep_m / (1 - p) with an independent counter-based mask per member."""
    _chk(x, "x")
    B, S, K = x.shape
    out = torch.empty((members, B, S, K), device=x.device, dtype=torch.bfloat16)
    check(_lib.lib().stb_dropout_expand(x.data_ptr(), x.stride(0), x.stride(1), out.data_ptr(), members, B, S, K, float(p),
                                        int(seed) & 0xFFFFFFFF, int(stream0) & 0xFFFFFFFF, _stream()))
    return out


def dropout_accum_(dx, d, p: float, seed: int, stream0: int):
    """dx [B, S, K] (view, in place) += sum_m keep_m / (1 - p) * d[m]; d [members, B, S, K] contiguous."""
    _chk(dx, "dx"); _chk(d, "d")
    assert d.is_contiguous() and d.dim() == 4 and tuple(d.shape[1:]) == tuple(dx.shape)
    members, B, S, K = d.shape
    check(_lib.lib().stb_dropout_accum(d.data_ptr(), dx.data_ptr(), dx.stride(0), dx.stride(1), members, B, S, K, float(p),
                                       int(seed) & 0xFFFFFFFF, int(stream0) & 0xFFFFFFFF, _stream()))
    return dx


def wgrad_full(dy, x, out: Optional[torch.Tensor] = None, alpha: float = 1.0, accumulate: bool = False):
    """dW [N, K] bf16 = alpha * sum over tokens dy[..., n] * x[..., k] (+ out if accumulate).  dy [B,S,N] / x [B,S,K] views."""
    d3, x3 = _as3d(dy), _as3d(x)
    _chk(d3, "dy"); _chk(x3, "x")
    B, S, N = d3.shape
    K = x3.shape[2]
    assert x3.shape[0] == B and x3.shape[1] == S
    if out is None:
        assert not accumulate
        out = torch.empty((N, K), device=dy.device, dtype=torch.bfloat16)
    assert out.dtype == torch.bfloat16 and out.shape == (N, K) and out.stride(1) == 1
    check(_lib.lib().stb_wgrad_full(d3.data_ptr(), d3.stride(0), d3.stride(1), x3.data_ptr(), x3.stride(0), x3.stride(1),
                                    out.data_ptr(), out.stride(0), B, S, N, K, float(alpha), int(accumulate), _stream()))
    return out


def colsum2(dy, z=None, want_sum: bool = True):
    """(sum [B, D] or None, dot [B, D] or None) in fp32: sum_s dy, sum_s dy * z."""
    d3 = _as3d(dy)
    _chk(d3, "dy")
    B, S, D = d3.shape
    sm = torch.zeros((B, D), device=dy.device, dtype=torch.float32) if want_sum else None
    dt = None
    zb = zs = 0
    if z is not None:
        z3 = _as3d(z)
        _chk(z3, "z")
        assert z3.shape == d3.shape
        dt = torch.zeros((B, D), device=dy.device, dtype=torch.float32)
        zb, zs = z3.stride(0), z3.stride(1)
    check(_lib.lib().stb_colsum2(d3.data_ptr(), d3.stride(0), d3.stride(1), _ptr(z3) if z is not None else None, zb, zs,
                                 _ptr(sm), _ptr(dt), B, S, D, _stream()))
    return sm, dt


DETERMINISTIC = os.environ.get("STB_DETERMINISTIC", "1") != "0"
# per (device, stream) reduction workspace.  A buffer that is outgrown is kept alive, never freed: a CUDA graph captured
# while it was current still reads and writes it on replay, so its memory must not go back to an allocator pool.
_ws_cache: dict = {}
_ws_retired: list = []


def set_deterministic(on: bool) -> None:
    """LoRA weight gradients without floating-point atomics (slab partials + ordered reduction): bit-identical run to run.
    On by default; off (or STB_DETERMINISTIC=0) accumulates the row splits with fp32 atomics instead."""
    global DETERMINISTIC
    DETERMINISTIC = bool(on)


def skinny_tn(L, Rm, alpha: float = 1.0, out: Optional[torch.Tensor] = None):
    """out[r, n] += alpha * sum_m L[m, r] * Rm[m, n].  L [B,S,R] or [M,R]; Rm [B,S,N] or [M,N]; out fp32."""
    L3, R3 = _as3d(L), _as3d(Rm)
    _chk(L3, "L"); _chk(R3, "Rm")
    B, S, R = L3.shape
    N = R3.shape[2]
    if out is None:
        out = torch.zeros((R, N), device=L.device, dtype=torch.float32)
    assert out.dtype == torch.float32 and out.is_contiguous()
    if DETERMINISTIC and R % 8 == 0 and R <= 128 and N % 8 == 0:
        need = int(_lib.lib().stb_skinny_tn_workspace(B, S, R, N))
        key = (L.device.index, _stream())
        ws = _ws_cache.get(key)
        if ws is None or ws.numel() < need:
            if ws is not None:
                _ws_retired.append(ws)
            ws = _ws_cache[key] = torch.empty((need,), device=L.device, dtype=torch.float32)
        check(_lib.lib().stb_skinny_tn_ws(L3.data_ptr(), L3.stride(0), L3.stride(1), R3.data_ptr(), R3.stride(0), R3.stride(1),
                                          out.data_ptr(), B, S, R, N, alpha, ws.data_ptr(), ws.numel(), _stream()))
        return out
    check(_lib.lib().stb_skinny_tn(L3.data_ptr(), L3.stride(0), L3.stride(1), R3.data_ptr(), R3.stride(0),
                                   R3.stride(1), out.data_ptr(), B, S, R, N, alpha, _stream()))
    return out


_graph_launches = 0   # libstb200 kernels executed by CUDA-graph replays (the C counter only sees direct launches)


def launch_count() -> int:
    return int(_lib.lib().stb_launch_count()) + _graph_launches


def reset_launch_count() -> None:
    global _graph_launches
    _graph_launches = 0
    _lib.lib().stb_reset_launch_count()


def note_graph_replay(n_kernels: int) -> None:
    """training.step.GraphedTrainStep: a replay runs the `n_kernels` libstb200 launches recorded at capture time."""
    global _graph_launches
    _graph_launches += int(n_kernels)


# ---------------------------------------------------------------------------------------------- VAE encode
def conv3x3_nhwc(x, w9, bias=None, res=None, stride: int = 1, out=None):
    """x [B,H,W,Ci] NHWC contiguous; w9 [Co, 9*Ci] tap-major; returns [B,Ho,Wo,Co]."""
    _chk(x, "x"); _chk(w9, "w9")
    assert x.is_contiguous() and w9.is_contiguous()
    B, H, W, Ci = x.shape
    Co = w9.shape[0]
    assert w9.shape[1] == 9 * Ci
    Ho, Wo = (H, W) if stride == 1 else (H // 2, W // 2)
    if out is None:
        out = torch.empty((B, Ho, Wo, Co), device=x.device, dtype=torch.bfloat16)
    if res is not None:
        assert res.is_contiguous() and res.shape == out.shape
    check(_lib.lib().stb_conv3x3_nhwc(x.data_ptr(), w9.data_ptr(), _ptr(bias), _ptr(res), out.data_ptr(),
                                      B, H, W, Ci, Co, stride, _stream()))
    return out


def conv_in_3ch(pixels, w, bias):
    """pixels [B,3,H,W] NCHW bf16; w [C,3,3,3]; returns NHWC [B,H,W,C]."""
    _chk(pixels, "pixels")
    assert pixels.is_contiguous() and w.is_contiguous()
    B, _, H, W = pixels.shape
    C = w.shape[0]
    out = torch.empty((B, H, W, C), device=pixels.device, dtype=torch.bfloat16)
    check(_lib.lib().stb_conv_in_3ch(pixels.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), B, H, W, C, _stream()))
    return out


def groupnorm_nhwc(x, gamma, beta, groups: int = 32, eps: float = 1e-6, silu: bool = True, out=None):
    """x [B, ..., C] NHWC contiguous."""
    _chk(x, "x")
    assert x.is_contiguous()
    B, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * C)
    if out is None:
        out = torch.empty_like(x)
    stats = torch.empty((B * groups * 2,), device=x.device, dtype=torch.float32)
    check(_lib.lib().stb_groupnorm_nhwc(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(), stats.data_ptr(),
                                        B, HW, C, groups, eps, int(silu), _stream()))
    return out


def softmax_rows_(s, scale: float):
    """in-place softmax(scale * s) over the last dim of a contiguous [..., cols] bf16 tensor."""
    _chk(s, "s")
    assert s.is_contiguous()
    cols = s.shape[-1]
    check(_lib.lib().stb_softmax_rows(s.data_ptr(), cols, s.numel() // cols, cols, scale, _stream()))
    return s


def gaussian_sample_scale(moments_nhwc, eps_nchw, shift, scale):
    """moments [B, h, w, 2L] NHWC; eps [B, L, h, w]; returns scaled latents [B, L, h, w]."""
    B, h, w, L2 = moments_nhwc.shape
    L = L2 // 2
    assert moments_nhwc.is_contiguous() and eps_nchw.is_contiguous() and eps_nchw.shape == (B, L, h, w)
    out = torch.empty((B, L, h, w), device=moments_nhwc.device, dtype=torch.bfloat16)
    check(_lib.lib().stb_gaussian_sample_scale(moments_nhwc.data_ptr(), eps_nchw.data_ptr(), out.data_ptr(), B, L, h * w,
                                               float(shift or 0.0), float(scale), int(shift is not None), _stream()))
    return out
