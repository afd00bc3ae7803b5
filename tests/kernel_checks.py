"""Kernel-level parity checks of libstb200 against plain PyTorch math on the same GPU tensors (fp64 for attention).

Each check is a function returning a dict {"ok": bool, "max_err": ..., "tol": ..., ...}.  They are used
by the `-m gpu` pytest tests and by tools/run_gpu_checks.py (which runs every check in its own
subprocess so that a trapped kernel cannot poison the rest of the run).
"""
from __future__ import annotations

import math

import torch

from simpletuner_b200 import ops

DEV = "cuda"


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def _report(name, got, ref, atol, rtol, extra=None):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = err > tol
    nbad = int(bad.sum().item())
    out = {
        "name": name,
        "ok": nbad == 0 and bool(torch.isfinite(got).all().item()),
        "max_err": float(err.max().item()),
        "ref_absmax": float(ref.abs().max().item()),
        "n_bad": nbad,
        "numel": got.numel(),
    }
    if nbad:
        idx = torch.nonzero(bad)[:8].tolist()
        out["first_bad"] = idx
        # error structure along the last two dims in 16-wide blocks: reveals tile / descriptor mistakes
        e2 = err.reshape(-1, err.shape[-1])
        rows = e2.shape[0]
        rb = max(1, rows // 8)
        cb = max(1, e2.shape[1] // 8)
        out["row_block_maxerr"] = [round(float(e2[i * rb:(i + 1) * rb].max().item()), 4) for i in range(min(8, math.ceil(rows / rb)))]
        out["col_block_maxerr"] = [round(float(e2[:, j * cb:(j + 1) * cb].max().item()), 4) for j in range(min(8, math.ceil(e2.shape[1] / cb)))]
    if extra:
        out.update(extra)
    # share of the tolerance the worst element uses (1.0 = at the limit)
    use = torch.where(err == 0, torch.zeros_like(err), err / tol)
    out["tol_use"] = round(float(use.max().item()), 4) if use.numel() else 0.0
    return out


# --------------------------------------------------------------------------------------------- GEMM
def gelu_tanh(x):
    return torch.nn.functional.gelu(x, approximate="tanh")


def check_gemm(M=256, N=256, K=128, B=1, bias=False, epi=ops.EPI_STORE, tile=(0, 0), segs=None, strided=False,
               nan_to_num=False, name=None, w_kn=None):
    """segs: list of extra K sizes appended as additional segments.  w_kn[i]: hand segment i's weight over as [K, N]
    (the contraction index is the row — what a dgrad reads from the forward weight) instead of [N, K]."""
    Ks = [K] + list(segs or [])
    S = M
    a_list, w_list = [], []
    for i, k in enumerate(Ks):
        if strided:
            full = _rand(B, S + 3, k + 16, seed=10 + i)
            a_list.append(full[:, 1:S + 1, 8:8 + k])
            wfull = _rand(N, k + 8, scale=0.5, seed=20 + i)
            w_list.append(wfull[:, :k])
        else:
            a_list.append(_rand(B, S, k, seed=10 + i))
            w_list.append(_rand(N, k, scale=0.5, seed=20 + i))
    bias_t = _rand(N, seed=30) if bias else None
    acc = sum(a.float() @ w.float().t() for a, w in zip(a_list, w_list))
    if bias_t is not None:
        acc = acc + bias_t.float()
    gate = res = aux = None
    kw = {}
    if epi == ops.EPI_STORE:
        ref = acc
    elif epi == ops.EPI_GELU:
        aux = torch.zeros(B, S, N, dtype=torch.bfloat16, device=DEV)
        ref = gelu_tanh(acc.bfloat16().float())
    elif epi == ops.EPI_GATE_RES:
        gate = _rand(B, N, seed=31)
        res = _rand(B, S, N, seed=32)
        y = acc.bfloat16().float()
        ref = res.float() + (gate.float()[:, None, :] * y).bfloat16().float()
    elif epi == ops.EPI_MUL_DGELU:
        aux = _rand(B, S, N, seed=33)
        x = aux.float().requires_grad_(True)
        gelu_tanh(x).sum().backward()
        ref = acc * x.grad
    elif epi == ops.EPI_ADD_RES:
        res = _rand(B, S, N, seed=32)
        ref = acc + res.float()
    elif epi == ops.EPI_MUL:
        aux = _rand(B, S, N, seed=34)
        ref = acc.bfloat16().float() * aux.float()
    elif epi == ops.EPI_QUICK_GELU:
        y = acc.bfloat16().float()
        ref = y * torch.sigmoid(1.702 * y)
    else:
        raise ValueError(f"no reference for epilogue {epi}")
    out = None
    if strided:
        outfull = torch.zeros(B, S + 2, N + 8, dtype=torch.bfloat16, device=DEV)
        out = outfull[:, 1:S + 1, :N]
    w_pass = list(w_list)
    if w_kn is not None:
        for i, flag in enumerate(w_kn):
            if flag:                      # [K, N] storage; with `strided` a column range of a wider matrix (row stride > N)
                if strided:
                    wide = torch.zeros(w_list[i].shape[1], N + 24, dtype=torch.bfloat16, device=DEV)
                    wide[:, 8:8 + N] = w_list[i].t()
                    w_pass[i] = wide[:, 8:8 + N]
                else:
                    w_pass[i] = w_list[i].t().contiguous()
    got = ops.gemm(a_list, w_pass, bias_t, out=out, epi=epi, gate=gate, res=res, aux=aux, nan_to_num=nan_to_num, tile=tile, w_kn=w_kn)
    torch.cuda.synchronize()
    scale = float(ref.abs().max().item())
    r = _report(name or f"gemm_M{M}_N{N}_K{Ks}_B{B}_epi{epi}_tile{tile}", got, ref, atol=scale * 6e-3, rtol=1.6e-2)
    if epi == ops.EPI_GELU:
        r2 = _report("aux", aux, acc, atol=float(acc.abs().max()) * 6e-3, rtol=1.6e-2)
        r["aux_ok"] = r2["ok"]
        r["ok"] = r["ok"] and r2["ok"]
    if strided:
        # nothing outside the view may be touched
        mask = torch.ones_like(outfull, dtype=torch.bool)
        mask[:, 1:S + 1, :N] = False
        r["halo_clean"] = bool((outfull[mask] == 0).all().item())
        r["ok"] = r["ok"] and r["halo_clean"]
    return r


# --------------------------------------------------------------------------------------------- attention
def _attn_ref(q, k, v, scale, bias=None, key_bias=None, d_o=None, o=None):
    """fp64 attention on the kernel's own bf16 inputs, one (batch, head) at a time so that memory stays at a few S x S
    matrices.  q / k / v / d_o [B, S, H, HD]; bias [H or 1, Sq, Sk] shared by the batch, or key_bias [B or 1, Sk].
    Returns {"o", "lse"} and, with d_o, {"dq", "dk", "dv"} from the explicit formulas:
      P = softmax(scale Q K^T + bias),  dV = P^T dO,  dS = P o (dO V^T - rowsum(dO o O)),  dQ = scale dS K,  dK = scale dS^T Q
    o: the forward output the backward is given (bf16), used for O in rowsum(dO o O) as the backward uses it; the exact
    output when None.  With a peaked softmax dS is the small difference of two nearly equal terms and the forward's bf16
    rounding of O alone moves dq / dk by several times their tolerance; that error belongs to the forward's o, which
    the checks compare with the exact one."""
    B, Sq, H, _ = q.shape
    o_in = o
    f64 = lambda t: t.detach().to(torch.float64)
    ref = {"o": torch.empty(q.shape, dtype=torch.float64, device=q.device),
           "lse": torch.empty(B, H, Sq, dtype=torch.float64, device=q.device)}
    if d_o is not None:
        ref.update(dq=torch.empty_like(ref["o"]), dk=torch.empty(k.shape, dtype=torch.float64, device=q.device),
                   dv=torch.empty(v.shape, dtype=torch.float64, device=q.device))
    for b in range(B):
        for h in range(H):
            qh, kh, vh = f64(q[b, :, h]), f64(k[b, :, h]), f64(v[b, :, h])
            s = (qh @ kh.t()) * scale
            if bias is not None:
                s += f64(bias[h % bias.shape[0]])
            if key_bias is not None:
                s += f64(key_bias[b % key_bias.shape[0]])[None, :]
            lse = torch.logsumexp(s, -1)
            p = torch.exp(s - lse[:, None])
            o = p @ vh
            ref["o"][b, :, h], ref["lse"][b, h] = o, lse
            if d_o is not None:
                g = f64(d_o[b, :, h])
                ob = o if o_in is None else f64(o_in[b, :, h])
                ds = p * (g @ vh.t() - (g * ob).sum(-1, keepdim=True))
                ref["dq"][b, :, h] = scale * (ds @ kh)
                ref["dk"][b, :, h] = scale * (ds.t() @ qh)
                ref["dv"][b, :, h] = p.t() @ g
    return ref


# Per-element tolerance atol + rtol |ref| against the fp64 reference.  atol is in units of the RMS of the element's own
# reference row (one query or key of one head, over the head dim), not of max |ref|: for unit-variance inputs max |ref| is
# 4-5x the RMS, so a max-scaled atol let typical elements be off by 10 % of the RMS.  Per row rather than over the whole
# tensor because a per-key bias scales each key's dk / dv (and a peaked softmax each query's dq) by a factor of its own:
# with an N(0, 2^2) bias a few keys carry most of the tensor's RMS, and a global RMS would be 7x too small an atol for the
# rest (measured on H100 at the Flux shape, and reproduced by a model of the kernels' bf16 roundings).
#   o, dq, dk, dv: rtol 2^-7 because the bf16 store alone rounds by up to half an ulp = 2^-8 |x|, which would use all of
#                  an rtol of 2^-8 on a large element.  The atol covers P (forward) and P^T / dS (backward) rounded to
#                  bf16 before their MMAs: 2e-2 RMS for o (1e-2 was used up to 0.88 on H100) and 2.5e-2 for the
#                  gradients (2e-2 was used up to 0.56 with a 64-key tail), so that the unmodified kernels stay at or
#                  below half of every tolerance.
#   lse:           fp32 throughout.
# When every row has a single key (P = 1) the reference gradients dq / dk are 0, and the kernel's are the ~1e-6 residue of
# dP - Delta (two fp32 dot products of the same values, summed in different orders): hence the floor on the RMS.
ATTN_TOL = {"o": (2 ** -7, 2e-2), "dq": (2 ** -7, 2.5e-2), "dk": (2 ** -7, 2.5e-2), "dv": (2 ** -7, 2.5e-2)}
LSE_TOL = 2e-4


def _row_rms(ref, floor=1e-3):
    """RMS of each row of the last dim, floored: the atol scale of attn_compare."""
    return ref.double().pow(2).mean(-1, keepdim=True).sqrt().clamp_min(floor)


def attn_compare(name, got, ref):
    """got / ref: dicts holding some of o, lse, dq, dk, dv.  One result dict: ok, the worst share of the tolerance used
    (tol_use, overall and per tensor), max errors, and the element-wise detail of a failing tensor."""
    out = {"name": name, "ok": True}
    for nm in ("o", "lse", "dq", "dk", "dv"):
        if nm not in got:
            continue
        if nm == "lse":
            r = _report(nm, got[nm], ref[nm], atol=LSE_TOL, rtol=LSE_TOL)
        else:
            rtol, arms = ATTN_TOL[nm]
            r = _report(nm, got[nm], ref[nm], atol=arms * _row_rms(ref[nm]), rtol=rtol)
        out[f"{nm}_tol_use"], out[f"{nm}_max_err"] = r["tol_use"], r["max_err"]
        if not r["ok"]:
            out["ok"] = False
            out[f"{nm}_detail"] = r
    out["tol_use"] = max(v for n, v in out.items() if n.endswith("_tol_use"))
    return out


def _attn_bias(kind, H, Sq, Sk, keep=None):
    """Additive logit bias [H or 1, Sq, Sk] (bf16) for the general instantiation of attn_fwd (text encoders).  Every query
    row needs one finite key anywhere; a 128-key tile that is -inf for a row contributes nothing to it.
      head / shared: dense relative-position-like bias, per head or one for all heads
      causal:        0 on and below the diagonal, -inf above it
      keypad:        0 for the first `keep` keys, -inf for the rest (whole later key tiles masked)
      leftpad:       dense per head, with -inf in front of some rows (left-padded text): rows 3i over the whole first
                     128-key tile, rows 3i + 1 over every key but the last (in the partial tail tile), rows 3i + 2 over
                     their first i % 128 keys"""
    if kind in ("head", "shared"):
        return _rand(H if kind == "head" else 1, Sq, Sk, scale=2.0, seed=6)
    if kind == "leftpad":
        assert Sk > 128
        b = _rand(H, Sq, Sk, scale=2.0, seed=6).float().cpu()
        for r in range(Sq):
            b[:, r, :(128, Sk - 1, (r // 3) % 128)[r % 3]] = float("-inf")
        return b.to(torch.bfloat16).to(DEV)
    b = torch.zeros(1, Sq, Sk, dtype=torch.float32)
    if kind == "causal":
        b.masked_fill_(torch.ones(Sq, Sk, dtype=torch.bool).triu(1), float("-inf"))
    elif kind == "keypad":
        b[..., keep:] = float("-inf")
    else:
        raise ValueError(kind)
    return b.to(torch.bfloat16).to(DEV)


def _key_bias(kind, B, Sk, seed=0):
    """Per-key logit bias [B or 1, Sk] (bf16, Flux masked training), different for every sample unless stated:
      dense:          N(0, 2^2) per (sample, key): a bias taken from the wrong key, row, lane or sample moves every element
      01 / neg:       ones with one run of 0 / -10000 per sample (the 0/1 mask of the reference and its additive form)
      inf:            -inf over the first 128-key tile (all keys but the last when Sk <= 128) and over whole 64-key blocks
      inf_first_tile: dense, -inf over the whole first 128-key tile (Sk > 128)
      inf_straddle:   dense, -inf runs across the 64- and 128-key boundaries (the backward's and the forward's key tiles)
      last_key_only:  -inf on every key but Sk - 1 (dense), which lies in the partial tail tile
      mixed:          sample 0 all zeros, the others dense
      shared:         one dense [1, Sk] row for the whole batch (batch stride 0)"""
    g = torch.Generator().manual_seed(seed)
    bias = torch.randn(B, Sk, generator=g) * 2.0
    if kind in ("01", "neg", "inf"):
        bias.fill_(1.0)
        for b in range(B):
            n = int(torch.randint(0, Sk, (1,), generator=g)) if Sk > 1 else 0
            if kind == "inf":
                bias[b, :min(128, Sk - 1)] = -math.inf
                for k0 in range(192, Sk - 64, 128 * (b + 1)):
                    bias[b, k0:k0 + 64] = -math.inf
            else:
                bias[b, n:min(Sk, n + 1 + Sk // (b + 2))] = 0.0 if kind == "01" else -10000.0
    elif kind == "inf_first_tile":
        assert Sk > 128
        bias[:, :128] = -math.inf
    elif kind == "inf_straddle":
        for b in range(B):
            for edge in (64, 128, 192, 256, 320):
                bias[b, max(1, edge - 5 - 3 * b):min(Sk, edge + 7 + 2 * b)] = -math.inf
    elif kind == "last_key_only":
        bias[:, :-1] = -math.inf
    elif kind == "mixed":
        bias[0] = 0.0
    elif kind == "shared":
        bias = bias[:1]
    elif kind != "dense":
        raise ValueError(kind)
    return bias.to(torch.bfloat16).to(DEV)


def check_attn_fwd(B=1, H=2, Sq=256, Sk=None, HD=128, strided=False, name=None, qscale=1.0, bias=None, keep=None,
                   key_bias=None, seed=0):
    """bias: None or an _attn_bias kind; key_bias: None or a _key_bias kind.  o and lse against the fp64 reference."""
    Sk = Sk or Sq
    if strided:
        # q/k/v as slices of a fused [B, S, 3*H*HD] projection buffer (the layout the model uses)
        assert Sk == Sq
        qkv = _rand(B, Sq, 3 * H * HD, seed=1, scale=qscale)
        q = qkv[..., 0 * H * HD:1 * H * HD].unflatten(-1, (H, HD))
        k = qkv[..., 1 * H * HD:2 * H * HD].unflatten(-1, (H, HD))
        v = qkv[..., 2 * H * HD:3 * H * HD].unflatten(-1, (H, HD))
    else:
        q = _rand(B, Sq, H, HD, seed=1, scale=qscale)
        k = _rand(B, Sk, H, HD, seed=2, scale=qscale)
        v = _rand(B, Sk, H, HD, seed=3)
    scale = HD ** -0.5
    bias_t = _attn_bias(bias, H, Sq, Sk, keep) if bias else None
    kb = _key_bias(key_bias, B, Sk, seed) if key_bias else None
    o, lse = ops.attn_fwd(q, k, v, scale, bias=bias_t, key_bias=kb)
    torch.cuda.synchronize()
    ref = _attn_ref(q, k, v, scale, bias=bias_t, key_bias=kb)
    return attn_compare(name or f"attn_fwd_B{B}_H{H}_Sq{Sq}_Sk{Sk}_HD{HD}", {"o": o, "lse": lse}, ref)


def check_attn_bwd(B=1, H=2, Sq=256, Sk=None, HD=128, name=None, strided=False, qscale=1.0, key_bias=None, seed=0):
    """Forward then backward; o, lse, dq, dk, dv against the fp64 reference.  key_bias: None or a _key_bias kind; keys it
    masks with -inf must get dk = dv = 0 exactly.
    strided: q / k / v are views of a fused [B, S, 3 H HD] projection and dq / dk / dv are written through views of a
    zero-filled fused gradient buffer with a halo of extra rows and columns, which must stay zero."""
    Sk = Sk or Sq
    D = H * HD
    if strided:
        assert Sk == Sq
        qkv = _rand(B, Sq, 3 * D, seed=1)
        q, k, v = (qkv[..., i * D:(i + 1) * D].unflatten(-1, (H, HD)) for i in range(3))
        if qscale != 1.0:
            qkv[..., :2 * D] *= qscale
        gfull = torch.zeros(B, Sq + 2, 3 * D + 24, dtype=torch.bfloat16, device=DEV)
        g = gfull[:, 1:Sq + 1, 8:8 + 3 * D]
        dq_o, dk_o, dv_o = (g[..., i * D:(i + 1) * D].unflatten(-1, (H, HD)) for i in range(3))
    else:
        q = _rand(B, Sq, H, HD, seed=1, scale=qscale)
        k = _rand(B, Sk, H, HD, seed=2, scale=qscale)
        v = _rand(B, Sk, H, HD, seed=3)
        dq_o = dk_o = dv_o = None
    d_o = _rand(B, Sq, H, HD, seed=4)
    scale = HD ** -0.5
    kb = _key_bias(key_bias, B, Sk, seed) if key_bias else None
    o, lse = ops.attn_fwd(q, k, v, scale, key_bias=kb)
    dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse, scale, dq=dq_o, dk=dk_o, dv=dv_o, key_bias=kb)
    torch.cuda.synchronize()
    ref = _attn_ref(q, k, v, scale, key_bias=kb, d_o=d_o, o=o)
    out = attn_compare(name or f"attn_bwd_B{B}_H{H}_Sq{Sq}_Sk{Sk}_HD{HD}" + (f"_kb_{key_bias}" if key_bias else ""),
                       {"o": o, "lse": lse, "dq": dq, "dk": dk, "dv": dv}, ref)
    if kb is not None and bool(torch.isinf(kb.float()).any()):
        dead = torch.isinf(kb.float())[:, :, None, None].expand(B, Sk, H, HD)
        out["masked_keys_zero"] = bool((dk[dead] == 0).all()) and bool((dv[dead] == 0).all())
        out["ok"] = out["ok"] and out["masked_keys_zero"]
    if strided:
        mask = torch.ones_like(gfull, dtype=torch.bool)
        mask[:, 1:Sq + 1, 8:8 + 3 * D] = False
        out["halo_clean"] = bool((gfull[mask] == 0).all().item())
        out["ok"] = out["ok"] and out["halo_clean"]
    return out


def check_attn_bwd_repeatable(B=1, H=2, S=4608, HD=128):
    """Both backward kernels are free of atomics: dq, dk, dv are bit-identical from run to run."""
    q, k, v, d_o = (_rand(B, S, H, HD, seed=i) for i in (1, 2, 3, 4))
    o, lse = ops.attn_fwd(q, k, v)
    first = ops.attn_bwd(q, k, v, o, d_o, lse)
    second = ops.attn_bwd(q, k, v, o, d_o, lse)
    torch.cuda.synchronize()
    same = {nm: bool(torch.equal(a, b)) for nm, a, b in zip(("dq", "dk", "dv"), first, second)}
    finite = all(bool(torch.isfinite(t).all().item()) for t in first)
    return {"name": f"attn_bwd_repeatable_S{S}_H{H}_HD{HD}", "ok": all(same.values()) and finite, **same}


# --------------------------------------------------------------------------------------------- elementwise
def check_ln_modulate(B=2, S=64, D=3072):
    x = _rand(B, S, D, seed=1)
    mod = _rand(B, 6 * D, seed=2, scale=0.3)
    shift, scale = mod[:, :D], mod[:, D:2 * D]
    out = ops.ln_modulate_fwd(x, shift, scale)
    ln = torch.nn.functional.layer_norm(x.float(), (D,), eps=1e-6)
    ref = ln * (1 + scale.float()[:, None]) + shift.float()[:, None]
    r = _report(f"ln_modulate_fwd_D{D}", out, ref, atol=3e-2, rtol=2e-2)
    # backward
    dy = _rand(B, S, D, seed=3)
    add = _rand(B, S, D, seed=4)
    dx = ops.ln_modulate_bwd(dy, x, scale, add=add)
    xf = x.float().requires_grad_(True)
    lnf = torch.nn.functional.layer_norm(xf, (D,), eps=1e-6)
    (lnf * (1 + scale.float().bfloat16().float()[:, None])).backward(dy.float())
    ref_dx = xf.grad + add.float()
    r2 = _report("ln_modulate_bwd", dx, ref_dx, atol=3e-2 * float(ref_dx.abs().max()), rtol=2e-2)
    r["bwd_ok"] = r2["ok"]
    r["bwd_max_err"] = r2["max_err"]
    r["ok"] = r["ok"] and r2["ok"]
    return r


def _rope_tables(S, HD, seed=5):
    g = torch.Generator().manual_seed(seed)
    ang = torch.rand(S, HD // 2, generator=g) * 6.28
    cos = ang.cos().repeat_interleave(2, dim=-1).float().to(DEV).contiguous()
    sin = ang.sin().repeat_interleave(2, dim=-1).float().to(DEV).contiguous()
    return cos, sin


def _rmsnorm_rope_ref(x, w, cos, sin, eps=1e-6):
    # x [B,S,H,HD] fp32
    var = x.pow(2).mean(-1, keepdim=True)
    y = x * torch.rsqrt(var + eps) * w
    xr, xi = y.reshape(*y.shape[:-1], -1, 2).unbind(-1)
    rot = torch.stack([-xi, xr], dim=-1).flatten(3)
    return y * cos[None, :, None, :] + rot * sin[None, :, None, :]


def check_qk_rmsnorm_rope(B=2, S=96, H=4, HD=128, s_split=32):
    Cc = 3 * H * HD
    src = _rand(B, S, Cc, seed=1)
    wq, wk, wq1, wk1 = (_rand(HD, seed=10 + i, scale=0.2) + 1 for i in range(4))
    cos, sin = _rope_tables(S, HD)
    q, k = ops.qk_rmsnorm_rope_fwd(src, H * HD, H, HD, wq, wk, wq1, wk1, s_split, cos, sin)
    torch.cuda.synchronize()

    def ref_of(xf):
        xq = xf[..., :H * HD].unflatten(-1, (H, HD))
        xk = xf[..., H * HD:2 * H * HD].unflatten(-1, (H, HD))
        outq = torch.cat([_rmsnorm_rope_ref(xq[:, :s_split], wq1.float(), cos[:s_split], sin[:s_split]),
                          _rmsnorm_rope_ref(xq[:, s_split:], wq.float(), cos[s_split:], sin[s_split:])], 1)
        outk = torch.cat([_rmsnorm_rope_ref(xk[:, :s_split], wk1.float(), cos[:s_split], sin[:s_split]),
                          _rmsnorm_rope_ref(xk[:, s_split:], wk.float(), cos[s_split:], sin[s_split:])], 1)
        return outq, outk

    xf = src.float().requires_grad_(True)
    rq, rk = ref_of(xf)
    r = _report(f"qk_rmsnorm_rope_fwd_HD{HD}", torch.cat([q, k], -1), torch.cat([rq, rk], -1), atol=4e-2, rtol=2e-2)
    dq = _rand(B, S, H, HD, seed=20)
    dk = _rand(B, S, H, HD, seed=21)
    dsrc = torch.zeros_like(src)
    ops.qk_rmsnorm_rope_bwd(dq, dk, src, H * HD, H, HD, wq, wk, wq1, wk1, s_split, cos, sin, dsrc=dsrc)
    torch.cuda.synchronize()
    (rq * dq.float()).sum().backward(retain_graph=True)
    (rk * dk.float()).sum().backward()
    ref = xf.grad[..., :2 * H * HD]
    r2 = _report("qk_rmsnorm_rope_bwd", dsrc[..., :2 * H * HD], ref, atol=3e-2 * float(ref.abs().max()), rtol=3e-2)
    r["bwd_ok"] = r2["ok"]
    r["bwd_max_err"] = r2["max_err"]
    r["v_untouched"] = bool((dsrc[..., 2 * H * HD:] == 0).all().item())
    r["ok"] = r["ok"] and r2["ok"] and r["v_untouched"]
    return r


def check_qk_rmsnorm_dw(B=2, S=1255, H=24, HD=128, s_split=77, rope=True):
    """The RMSNorm weight gradients of qk_rmsnorm_rope_bwd (full fine-tune): dw [4, HD] = d/d(wq, wk, wq_added, wk_added),
    summed over B * S * H head rows by per-block shared-memory atomics and one global atomic per block.  Reference:
    fp64 autograd of the same forward on the same bf16 inputs."""
    Cc = 3 * H * HD
    src = _rand(B, S, Cc, seed=1)
    ws = [_rand(HD, seed=10 + i, scale=0.2) + 1 for i in range(4)]   # wq, wk, wq_added, wk_added
    cos, sin = _rope_tables(S, HD) if rope else (None, None)
    dq = _rand(B, S, H, HD, seed=20)
    dk = _rand(B, S, H, HD, seed=21)
    dw = torch.zeros(4, HD, dtype=torch.float32, device=DEV)
    ops.qk_rmsnorm_rope_bwd(dq, dk, src, H * HD, H, HD, *ws, s_split, cos, sin, dsrc=torch.zeros_like(src), dw=dw)
    torch.cuda.synchronize()
    wd = [w.double().requires_grad_(True) for w in ws]
    c64 = cos.double() if rope else torch.ones(S, HD, dtype=torch.float64, device=DEV)
    s64 = sin.double() if rope else torch.zeros(S, HD, dtype=torch.float64, device=DEV)
    x = src.double()
    total = 0.0
    for off, g, w_img, w_txt in ((0, dq, wd[0], wd[2]), (H * HD, dk, wd[1], wd[3])):
        xs = x[..., off:off + H * HD].unflatten(-1, (H, HD))
        y = torch.cat([_rmsnorm_rope_ref(xs[:, :s_split], w_txt, c64[:s_split], s64[:s_split]),
                       _rmsnorm_rope_ref(xs[:, s_split:], w_img, c64[s_split:], s64[s_split:])], 1)
        total = total + (y * g.double()).sum()
    total.backward()
    ref = torch.stack([w.grad for w in wd])
    r = _report(f"qk_rmsnorm_dw_B{B}_S{S}_H{H}_HD{HD}_rope{int(rope)}", dw, ref, atol=1e-3 * float(ref.abs().max()), rtol=1e-3)
    r["dw_rows_absmax"] = [round(float(v), 3) for v in ref.abs().amax(1)]
    return r


def check_flow(B=2, Cc=16, Hh=32, Ww=48):
    lat = _rand(B, Cc, Hh, Ww, seed=1)
    noise = _rand(B, Cc, Hh, Ww, seed=2)
    sig = torch.tensor([0.25, 0.8125][:B] + [0.5] * max(0, B - 2), dtype=torch.float32, device=DEV)
    noisy, packed = ops.flow_prep_pack(lat, noise, sig)
    torch.cuda.synchronize()
    # eager bf16 chain exactly as the reference writes it (common.py:4953-4960, 4989-4991)
    grid = sig.view(B, 1, 1, 1).to(torch.bfloat16)
    ref_noisy = (1.0 - grid) * lat + grid * noise
    ref_packed = ref_noisy.view(B, Cc, Hh // 2, 2, Ww // 2, 2).permute(0, 2, 4, 1, 3, 5).reshape(B, (Hh // 2) * (Ww // 2), Cc * 4)
    bit_noisy = bool(torch.equal(noisy, ref_noisy))
    bit_packed = bool(torch.equal(packed, ref_packed))
    pred = _rand(B, (Hh // 2) * (Ww // 2), Cc * 4, seed=3)
    loss, dpred = ops.flow_mse_loss(pred, lat, noise)
    torch.cuda.synchronize()
    pf = pred.float().requires_grad_(True)
    unp = pf.view(B, Hh // 2, Ww // 2, Cc, 2, 2).permute(0, 3, 1, 4, 2, 5).reshape(B, Cc, Hh, Ww)
    tgt = (noise - lat).float()
    ref_loss = torch.nn.functional.mse_loss(unp, tgt, reduction="none").mean(dim=(1, 2, 3)).mean()
    ref_loss.backward()
    lerr = abs(float(loss.item()) - float(ref_loss.item()))
    r = _report("flow_loss_grad", dpred, pf.grad, atol=1e-2 * float(pf.grad.abs().max()), rtol=1e-2)
    r.update({"name": "flow_prep_loss", "bit_exact_noisy": bit_noisy, "bit_exact_packed": bit_packed,
              "loss": float(loss.item()), "loss_ref": float(ref_loss.item()), "loss_err": lerr})
    r["ok"] = r["ok"] and bit_noisy and bit_packed and lerr <= 1e-5 * max(1.0, abs(float(ref_loss.item())))
    return r


class _deterministic:
    """Select the skinny_tn reduction for a block: True = slab workspace + ordered reduce, False = fp32 atomics,
    None = leave the process setting alone.  The previous setting is restored on exit."""

    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.prev = ops.DETERMINISTIC
        if self.on is not None:
            ops.set_deterministic(self.on)

    def __exit__(self, *exc):
        ops.set_deterministic(self.prev)


def check_skinny(B=2, S=300, R=16, N=3072, deterministic=None):
    L = _rand(B, S, R, seed=1)
    Rm = _rand(B, S, N, seed=2)
    with _deterministic(deterministic):
        out = ops.skinny_tn(L, Rm, alpha=0.5)
        torch.cuda.synchronize()
    ref = 0.5 * (L.float().reshape(-1, R).t() @ Rm.float().reshape(-1, N))
    return _report(f"skinny_tn_B{B}_S{S}_R{R}_N{N}_det{deterministic}", out, ref, atol=1e-3 * float(ref.abs().max()), rtol=1e-3)


def check_skinny_repeatable(B=4, S=4608, R=48, N=9216):
    """The slab-workspace LoRA weight gradient is bit-identical from run to run."""
    L = _rand(B, S, R, seed=1)
    Rm = _rand(B, S, N, seed=2)
    with _deterministic(True):
        a = ops.skinny_tn(L, Rm, alpha=0.5)
        b = ops.skinny_tn(L, Rm, alpha=0.5)
        torch.cuda.synchronize()
    same = bool(torch.equal(a, b))
    return {"name": f"skinny_tn_repeatable_B{B}_S{S}_R{R}_N{N}", "ok": same and bool(torch.isfinite(a).all().item()),
            "max_diff": float((a - b).abs().max().item())}


def check_gate_mul(B=3, S=333, D=3072, chunk=2):
    """y = gate[:, None] * x with x a row / column window of a wider buffer and gate column chunk `chunk` of a [B, 9 D]
    modulation tensor; the kernel rounds the fp32 product once, exactly like the eager bf16 multiply."""
    xfull = _rand(B, S + 3, D + 16, seed=1)
    x = xfull[:, 2:S + 2, 8:8 + D]
    mod = _rand(B, 9 * D, seed=2)
    gate = mod[:, chunk * D:(chunk + 1) * D]
    yfull = torch.zeros(B, S + 2, D + 24, dtype=torch.bfloat16, device=DEV)
    y = ops.gate_mul(x, gate, out=yfull[:, 1:S + 1, 16:16 + D])
    torch.cuda.synchronize()
    ref = gate[:, None, :] * x
    r = _report(f"gate_mul_B{B}_S{S}_D{D}", y, ref, atol=0.0, rtol=0.0)
    r["bit_exact"] = bool(torch.equal(y, ref))
    mask = torch.ones_like(yfull, dtype=torch.bool)
    mask[:, 1:S + 1, 16:16 + D] = False
    r["halo_clean"] = bool((yfull[mask] == 0).all().item())
    r["ok"] = r["ok"] and r["bit_exact"] and r["halo_clean"]
    return r


# --------------------------------------------------------------------------------------------- registry
E = ops
CHECKS = {
    # GEMM: descriptor / pipeline basics first
    "gemm_basic": lambda: check_gemm(256, 256, 128),
    "gemm_k64": lambda: check_gemm(128, 256, 64),
    "gemm_deepk": lambda: check_gemm(256, 512, 1024),
    "gemm_tails": lambda: check_gemm(200, 328, 200, B=2),
    "gemm_bn128": lambda: check_gemm(256, 384, 256, tile=(1, 128)),
    "gemm_bn64": lambda: check_gemm(256, 64, 256, tile=(1, 64)),
    "gemm_mt2": lambda: check_gemm(512, 512, 256, tile=(2, 256)),
    "gemm_mt2_bn128": lambda: check_gemm(384, 256, 256, tile=(2, 128)),
    "gemm_persistent": lambda: check_gemm(4096, 3072, 512),
    "gemm_seg2": lambda: check_gemm(256, 256, 192, segs=[64]),
    "gemm_seg3_lora": lambda: check_gemm(256, 512, 256, segs=[128, 16], bias=True),
    "gemm_strided": lambda: check_gemm(200, 256, 136, B=2, strided=True, bias=True),
    "gemm_bias": lambda: check_gemm(256, 256, 128, bias=True),
    "gemm_gelu": lambda: check_gemm(256, 512, 128, bias=True, epi=E.EPI_GELU),
    "gemm_gate_res": lambda: check_gemm(256, 256, 128, B=2, bias=True, epi=E.EPI_GATE_RES, nan_to_num=True),
    "gemm_mul_dgelu": lambda: check_gemm(256, 256, 128, epi=E.EPI_MUL_DGELU),
    "gemm_add_res": lambda: check_gemm(256, 256, 128, epi=E.EPI_ADD_RES),
    "gemm_flux_shape": lambda: check_gemm(4096, 3072, 3072, B=1, bias=True),
    # attention
    "attn_fwd_256": lambda: check_attn_fwd(1, 2, 256),
    "attn_fwd_128": lambda: check_attn_fwd(1, 1, 128),
    "attn_fwd_512": lambda: check_attn_fwd(2, 3, 512),
    "attn_fwd_ragged": lambda: check_attn_fwd(1, 2, 333, 417),
    "attn_fwd_strided": lambda: check_attn_fwd(2, 4, 384, strided=True),
    "attn_fwd_hd64": lambda: check_attn_fwd(1, 2, 320, HD=64),
    "attn_fwd_long": lambda: check_attn_fwd(1, 2, 4608),
    "attn_fwd_bigscore": lambda: check_attn_fwd(1, 2, 512, qscale=4.0),
    "attn_bwd_256": lambda: check_attn_bwd(1, 2, 256),
    "attn_bwd_128": lambda: check_attn_bwd(1, 1, 128),
    "attn_bwd_ragged": lambda: check_attn_bwd(1, 2, 333, 417),
    "attn_bwd_hd64": lambda: check_attn_bwd(1, 2, 320, HD=64),
    "attn_bwd_long": lambda: check_attn_bwd(1, 2, 2304),
    # elementwise
    "ln_modulate": lambda: check_ln_modulate(),
    "ln_modulate_d1536": lambda: check_ln_modulate(D=1536),
    "qk_rmsnorm_rope": lambda: check_qk_rmsnorm_rope(),
    "qk_rmsnorm_rope_hd64": lambda: check_qk_rmsnorm_rope(HD=64),
    "flow": lambda: check_flow(),
    "skinny": lambda: check_skinny(),
    "skinny_r48": lambda: check_skinny(R=48, N=4096),
    "skinny_flux": lambda: check_skinny(B=4, S=4608, R=48, N=9216),
    "skinny_ragged": lambda: check_skinny(B=3, S=333, R=16, N=200),
    "skinny_cuda_core_path": lambda: check_skinny(B=2, S=100, R=16, N=250),
}
# BASELINE-geometry kernel shapes (VERDICT r1 weak #1): the deepest K of the Flux step (fc2 / single-block proj_out, K = 12288 and
# the 2-segment 3072 + 12288 `cat([attn, mlp]) @ W_out`), and the attention backward at the full joint sequence
CHECKS["gemm_k12288"] = lambda: check_gemm(4608, 3072, 12288, B=1, bias=True)
CHECKS["gemm_seg2_3072_12288_gate_res"] = lambda: check_gemm(4608, 3072, 3072, B=1, segs=[12288], bias=True, epi=E.EPI_GATE_RES,
                                                              nan_to_num=True)
CHECKS["gemm_seg3_dgrad_12288_9216_48"] = lambda: check_gemm(4608, 3072, 12288, B=1, segs=[9216, 48])
CHECKS["attn_bwd_s4608"] = lambda: check_attn_bwd(1, 2, 4608)
CHECKS["attn_bwd_s4608_ragged_cross"] = lambda: check_attn_bwd(1, 2, 4096, 4608 - 77)
CHECKS["attn_fwd_hd64_long"] = lambda: check_attn_fwd(2, 3, 1255, HD=64)
CHECKS["attn_bwd_hd64_long"] = lambda: check_attn_bwd(2, 3, 1255, HD=64)
CHECKS["skinny_r96"] = lambda: check_skinny(B=2, S=700, R=96, N=1536)
CHECKS["skinny_r24"] = lambda: check_skinny(B=1, S=300, R=24, N=512)


# --------------------------------------------------------------------------------------------- VAE encode kernels
def check_conv3x3(B=2, H=24, W=40, Ci=64, Co=128, stride=1, bias=True, res=False):
    import torch.nn.functional as F
    x = _rand(B, H, W, Ci, seed=1)
    w = _rand(Co, Ci, 3, 3, scale=(9 * Ci) ** -0.5, seed=2)
    bv = _rand(Co, scale=0.1, seed=3) if bias else None
    Ho, Wo = (H, W) if stride == 1 else (H // 2, W // 2)
    rv = _rand(B, Ho, Wo, Co, seed=4) if res else None
    w9 = w.permute(0, 2, 3, 1).reshape(Co, -1).contiguous()
    out = ops.conv3x3_nhwc(x, w9, bv, rv, stride)
    torch.cuda.synchronize()
    xn = x.float().permute(0, 3, 1, 2)
    if stride == 1:
        ref = F.conv2d(xn, w.float(), bv.float() if bias else None, padding=1)
    else:
        ref = F.conv2d(F.pad(xn, (0, 1, 0, 1)), w.float(), bv.float() if bias else None, stride=2)
    ref = ref.permute(0, 2, 3, 1)
    if res:
        ref = ref + rv.float()
    return _report(f"conv3x3_s{stride}_{Ci}to{Co}_{H}x{W}", out, ref, atol=2e-2, rtol=1e-2)


def check_conv_in(B=2, H=20, W=36, C=128):
    import torch.nn.functional as F
    x = _rand(B, 3, H, W, seed=1)
    w = _rand(C, 3, 3, 3, scale=27 ** -0.5, seed=2)
    bv = _rand(C, scale=0.1, seed=3)
    out = ops.conv_in_3ch(x, w, bv)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), w.float(), bv.float(), padding=1).permute(0, 2, 3, 1)
    return _report("conv_in_3ch", out, ref, atol=1e-2, rtol=1e-2)


def check_groupnorm(B=2, H=16, W=24, C=128, G=32, silu=True, mean=0.0):
    import torch.nn.functional as F
    x = (_rand(B, H, W, C, seed=1).float() + mean).bfloat16()
    gm = (1.0 + 0.1 * _rand(C, seed=2).float()).bfloat16()
    bt = _rand(C, scale=0.1, seed=3)
    out = ops.groupnorm_nhwc(x, gm, bt, G, 1e-6, silu)
    torch.cuda.synchronize()
    ref = F.group_norm(x.float().permute(0, 3, 1, 2), G, gm.float(), bt.float(), 1e-6)
    if silu:
        ref = F.silu(ref)
    return _report(f"groupnorm_C{C}_silu{int(silu)}_mean{mean}", out, ref.permute(0, 2, 3, 1), atol=2e-2, rtol=1e-2)


def check_softmax_rows(rows=300, cols=1024, scale=0.0442):
    s = _rand(rows, cols, scale=20.0, seed=1)
    ref = torch.softmax(s.float() * scale, dim=-1)
    ops.softmax_rows_(s, scale)
    torch.cuda.synchronize()
    return _report("softmax_rows", s, ref, atol=2e-3, rtol=1e-2)


def check_gaussian_sample(B=2, L=16, h=12, w=20, shift=0.1159):
    m = _rand(B, h, w, 2 * L, seed=1)
    eps = _rand(B, L, h, w, seed=2)
    out = ops.gaussian_sample_scale(m, eps, shift, 0.3611)
    torch.cuda.synchronize()
    mn = m.permute(0, 3, 1, 2)
    mean, logvar = mn[:, :L], mn[:, L:]
    z = mean + torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0)) * eps          # bf16 tensor ops, like diffusers
    ref = (z - shift) * 0.3611 if shift is not None else z * 0.3611
    r = _report("gaussian_sample_scale", out, ref, atol=0.0, rtol=0.0)
    if not r["ok"]:  # exp() ulp differences may move a bf16 rounding; never more than 1 bf16 ulp
        r2 = _report("gaussian_sample_scale", out, ref, atol=1e-3, rtol=2 ** -7)
        r2["bit_exact"] = False
        return r2
    r["bit_exact"] = True
    return r


CHECKS.update({
    "conv3x3_s1": lambda: check_conv3x3(),
    "conv3x3_s1_res": lambda: check_conv3x3(Ci=128, Co=256, res=True),
    "conv3x3_s1_wide": lambda: check_conv3x3(B=1, H=8, W=300, Ci=128, Co=128),
    "conv3x3_s1_512": lambda: check_conv3x3(B=1, H=16, W=16, Ci=512, Co=512, res=True),
    "conv3x3_out32": lambda: check_conv3x3(B=2, H=16, W=16, Ci=512, Co=32),
    "conv3x3_s2": lambda: check_conv3x3(stride=2, Ci=128, Co=128),
    "conv3x3_s2_wide": lambda: check_conv3x3(B=1, H=6, W=600, stride=2, Ci=64, Co=64),
    "conv_in_3ch": lambda: check_conv_in(),
    "groupnorm_silu": lambda: check_groupnorm(),
    "groupnorm_plain_512": lambda: check_groupnorm(C=512, silu=False),
    "groupnorm_256_offset": lambda: check_groupnorm(C=256, mean=3.0),
    "groupnorm_c64": lambda: check_groupnorm(C=64),
    "softmax_rows": lambda: check_softmax_rows(),
    "gaussian_sample": lambda: check_gaussian_sample(),
    "gaussian_sample_noshift": lambda: check_gaussian_sample(shift=None),
})


# --------------------------------------------------------------------------------------------- epsilon-family step kernels
def check_ddpm_prep(B=3, C=4, Hh=16, Ww=24):
    lat, noise = _rand(B, C, Hh, Ww, seed=1), _rand(B, C, Hh, Ww, seed=2)
    ac = torch.cumprod(1 - torch.linspace(1e-4, 0.02, 1000), 0).to(DEV)
    t = torch.tensor([3, 500, 999], device=DEV)[:B]
    ca, cb = (ac[t] ** 0.5).contiguous(), ((1 - ac[t]) ** 0.5).contiguous()
    noisy, packed = ops.ddpm_prep_pack(lat, noise, ca, cb)
    torch.cuda.synchronize()
    ref = (ca.view(-1, 1, 1, 1) * lat.float() + cb.view(-1, 1, 1, 1) * noise.float()).bfloat16()   # eager fp32 chain
    refp = ref.view(B, C, Hh // 2, 2, Ww // 2, 2).permute(0, 2, 4, 1, 3, 5).reshape(B, -1, C * 4)
    r = _report("ddpm_prep_pack", noisy, ref, atol=0.0, rtol=0.0)
    r["packed_exact"] = bool(torch.equal(packed, refp))
    r["ok"] = r["ok"] and r["packed_exact"]
    return r


def check_target_mse(B=3, C=4, Hh=16, Ww=24, weighted=True):
    S = (Hh // 2) * (Ww // 2)
    pred = _rand(B, S, 4 * C, seed=1).requires_grad_(False)
    tgt = _rand(B, C, Hh, Ww, seed=2)
    w = torch.tensor([0.5, 1.0, 2.5], device=DEV)[:B] if weighted else None
    loss, dpred = ops.target_mse_loss(pred, tgt, w, layout=1)
    torch.cuda.synchronize()
    p32 = pred.float().requires_grad_(True)
    un = torch.einsum("nhwpqc->nchpwq", p32.reshape(B, Hh // 2, Ww // 2, 2, 2, C)).reshape(B, C, Hh, Ww)
    l = (un - tgt.float()) ** 2
    if weighted:
        l = l * w.view(-1, 1, 1, 1)
    lref = l.mean(dim=[1, 2, 3]).mean()
    lref.backward()
    r = _report("target_mse_dpred", dpred, p32.grad, atol=1e-6, rtol=1e-2)
    r["loss"], r["loss_ref"] = float(loss.item()), float(lref.item())
    r["ok"] = r["ok"] and abs(r["loss"] - r["loss_ref"]) <= 1e-5 * abs(r["loss_ref"])
    return r


def check_loss_full_size(kind="flow", B=4, Cc=16, Hh=128, Ww=128):
    """flow_mse_loss / target_mse_loss at a Flux 1024^2 latent: the 8-CTA cluster reduction gives the same loss and dpred
    bit for bit on a second run, and the loss matches an fp64 reference to 1e-6 relative."""
    S = (Hh // 2) * (Ww // 2)
    pred = _rand(B, S, 4 * Cc, seed=3)
    if kind == "flow":
        lat, noise = _rand(B, Cc, Hh, Ww, seed=1), _rand(B, Cc, Hh, Ww, seed=2)
        run = lambda: ops.flow_mse_loss(pred, lat, noise)
        tgt = (noise - lat).double()                       # the target is formed in bf16, as the training step does
        unpack = lambda p: p.view(B, Hh // 2, Ww // 2, Cc, 2, 2).permute(0, 3, 1, 4, 2, 5).reshape(B, Cc, Hh, Ww)
        w = None
    else:
        tgt_bf = _rand(B, Cc, Hh, Ww, seed=2)
        w = torch.tensor([0.5, 1.0, 2.5, 0.75][:B], device=DEV)
        run = lambda: ops.target_mse_loss(pred, tgt_bf, w, layout=1)
        tgt = tgt_bf.double()
        unpack = lambda p: torch.einsum("nhwpqc->nchpwq", p.reshape(B, Hh // 2, Ww // 2, 2, 2, Cc)).reshape(B, Cc, Hh, Ww)
    loss1, dpred1 = run()
    loss2, dpred2 = run()
    torch.cuda.synchronize()
    p64 = pred.double().requires_grad_(True)
    l = (unpack(p64) - tgt) ** 2
    if w is not None:
        l = l * w.double().view(-1, 1, 1, 1)
    lref = l.mean(dim=(1, 2, 3)).mean()
    lref.backward()
    r = _report(f"{kind}_loss_dpred_B{B}_{Cc}x{Hh}x{Ww}", dpred1, p64.grad, atol=1e-2 * float(p64.grad.abs().max()), rtol=1e-2)
    r["loss"], r["loss_ref"] = float(loss1.item()), float(lref.item())
    r["loss_rel_err"] = abs(r["loss"] - r["loss_ref"]) / abs(r["loss_ref"])
    r["repeatable"] = bool(torch.equal(loss1, loss2)) and bool(torch.equal(dpred1, dpred2))
    r["ok"] = r["ok"] and r["loss_rel_err"] <= 1e-6 and r["repeatable"]
    return r


CHECKS.update({
    "ddpm_prep_pack": lambda: check_ddpm_prep(),
    "target_mse_weighted": lambda: check_target_mse(),
    "target_mse_plain": lambda: check_target_mse(weighted=False),
    "attn_fwd_cross_300": lambda: check_attn_fwd(2, 4, 1024, 300),
    "attn_bwd_cross_300": lambda: check_attn_bwd(2, 4, 1024, 300),
})


# --------------------------------------------------------------------------------------------- GEMM with BN = 256 forced
# (the auto choice drops to 128 when 256-wide tiles would leave SMs idle, so small problems need the width forced).
# The "pair" in the names is historical: these shapes once exercised a two-CTA tile; on sm_90a every tile is one CTA of
# 128 rows, and what the checks pin is the 256-wide tile with its 4-stage ring.
CHECKS.update({
    "gemm_pair_basic": lambda: check_gemm(512, 512, 256, tile=(0, 256)),
    "gemm_pair_one_tile": lambda: check_gemm(256, 256, 64, tile=(0, 256)),
    "gemm_pair_tails": lambda: check_gemm(200, 328, 200, B=2, tile=(0, 256)),
    "gemm_pair_half_empty": lambda: check_gemm(100, 256, 128, B=3, tile=(0, 256)),
    "gemm_pair_seg3_lora": lambda: check_gemm(512, 512, 256, segs=[128, 16], bias=True, tile=(0, 256)),
    "gemm_pair_gate_res": lambda: check_gemm(512, 256, 128, B=2, bias=True, epi=E.EPI_GATE_RES, nan_to_num=True, tile=(0, 256)),
    "gemm_pair_gelu": lambda: check_gemm(256, 512, 128, bias=True, epi=E.EPI_GELU, tile=(0, 256)),
    "gemm_pair_persistent": lambda: check_gemm(4096, 3072, 512, tile=(0, 256)),
    "gemm_pair_flux_shape": lambda: check_gemm(4608, 3072, 3072, B=2, bias=True, tile=(0, 256)),
})


# --------------------------------------------------------------------------------------------- fused q/k-prep backward epilogue
def check_attn_bwd_fused_prep(B=2, S=333, H=3, HD=128, s_split=77, rope=True, norm_w=True, key_bias=None):
    """attn_bwd(qk_prep=...) == attn_bwd -> qk_rmsnorm_rope_bwd (the two-kernel path) on the same inputs; dv, which the
    prep does not touch, bit for bit.  key_bias: None or a _key_bias kind."""
    D = H * HD
    qkv = _rand(B, S, 3 * D, seed=1)
    d_o = _rand(B, S, H, HD, seed=2)
    mk = lambda sd: (1.0 + 0.1 * _rand(HD, seed=sd).float()).bfloat16() if norm_w else None
    wq, wk, wqa, wka = mk(3), mk(4), mk(5), mk(6)
    cos, sin = _rope_tables(S, HD) if rope else (None, None)
    kb = _key_bias(key_bias, B, S, seed=9) if key_bias else None
    q, k = ops.qk_rmsnorm_rope_fwd(qkv, D, H, HD, wq, wk, wqa, wka, s_split, cos, sin, 1e-6)
    v = qkv[:, :, 2 * D:].unflatten(-1, (H, HD))
    o, lse = ops.attn_fwd(q, k, v, key_bias=kb)
    # reference: two kernels
    dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=kb)
    ref = torch.zeros_like(qkv)
    ops.qk_rmsnorm_rope_bwd(dq, dk, qkv, D, H, HD, wq, wk, wqa, wka, s_split, cos, sin, 1e-6, dsrc=ref)
    ref[:, :, 2 * D:] = dv.reshape(B, S, D)
    got = torch.zeros_like(qkv)
    ops.attn_bwd(q, k, v, o, d_o, lse, dq=got[:, :, 0:D].unflatten(-1, (H, HD)), dk=got[:, :, D:2 * D].unflatten(-1, (H, HD)),
                 dv=got[:, :, 2 * D:].unflatten(-1, (H, HD)), key_bias=kb,
                 qk_prep=dict(src=qkv, k_off=D, wq=wq, wk=wk, wq_added=wqa, wk_added=wka, s_split=s_split, cos=cos, sin=sin, eps=1e-6))
    torch.cuda.synchronize()
    # Both sides are bf16 and the two-kernel path rounds dq / dk to bf16 before the norm backward, the fused one does not:
    # the two results may land on neighbouring bf16 values, one ulp = up to 2^-7 |x| apart, hence rtol 2^-6.
    rows = lambda t: t.unflatten(-1, (3 * H, HD))   # one row per token and head, as attn_compare scales its atol
    r = _report(f"attn_bwd_fused_prep_S{S}_HD{HD}_rope{int(rope)}_w{int(norm_w)}" + (f"_kb_{key_bias}" if key_bias else ""),
                rows(got), rows(ref), atol=2e-2 * _row_rms(rows(ref)), rtol=2 ** -6)
    r["dv_exact"] = bool(torch.equal(got[:, :, 2 * D:], ref[:, :, 2 * D:]))
    r["ok"] = r["ok"] and r["dv_exact"]
    return r


CHECKS.update({
    "attn_bwd_fused_prep": lambda: check_attn_bwd_fused_prep(),
    "attn_bwd_fused_prep_hd64_norope": lambda: check_attn_bwd_fused_prep(B=1, S=320, H=4, HD=64, s_split=0, rope=False),
    "attn_bwd_fused_prep_now": lambda: check_attn_bwd_fused_prep(B=1, S=256, H=2, HD=128, s_split=0, rope=True, norm_w=False),
    "attn_bwd_fused_prep_key_bias": lambda: check_attn_bwd_fused_prep(key_bias="dense"),
})


# --------------------------------------------------------------------------------------------- implicit-GEMM conv at VAE sizes
# (many persistent tiles per CTA; output rows that are not a multiple of the 128-pixel tile).  "pair" in the names is
# historical: these are the larger conv shapes, run by the same one-CTA wgmma kernel as the small ones.
CHECKS.update({
    "conv3x3_pair_rows2": lambda: check_conv3x3(B=2, H=96, W=128, Ci=128, Co=128),
    "conv3x3_pair_oddrows": lambda: check_conv3x3(B=1, H=149, W=120, Ci=128, Co=128, res=True),
    "conv3x3_pair_wide": lambda: check_conv3x3(B=1, H=80, W=300, Ci=64, Co=256, res=True),
    "conv3x3_pair_512": lambda: check_conv3x3(B=2, H=64, W=128, Ci=512, Co=512),
    "conv3x3_pair_s2": lambda: check_conv3x3(B=2, H=160, W=256, stride=2, Ci=128, Co=128),
    "conv3x3_pair_s2_wide": lambda: check_conv3x3(B=1, H=160, W=600, stride=2, Ci=64, Co=256),
})

CHECKS.update({
    "conv_in_3ch_wide": lambda: check_conv_in(B=2, H=9, W=300, C=128),     # tile tail (300 = 2 * 128 + 44), tensor-core path
    "conv_in_3ch_c64": lambda: check_conv_in(B=1, H=33, W=130, C=64),
    "conv_in_3ch_c8_cuda_core": lambda: check_conv_in(B=1, H=12, W=20, C=8),  # C % 16 != 0 -> CUDA-core fallback kernel
})


# --------------------------------------------------------------------------------------------- full-rank weight gradient
def check_wgrad_full(B=2, S=300, N=256, K=320, strided=False, accumulate=False, alpha=1.0):
    if strided:   # row ranges / column ranges of larger buffers, like the joint hidden buffer and the fused qkv gradient
        dyf = _rand(B, S + 5, N + 64, seed=41)
        xf = _rand(B, S + 9, K + 32, seed=42)
        dy, x = dyf[:, 3:S + 3, 32:32 + N], xf[:, 4:S + 4, 8:8 + K]
    else:
        dy, x = _rand(B, S, N, seed=41), _rand(B, S, K, seed=42)
    ref = alpha * torch.einsum("bsn,bsk->nk", dy.float(), x.float())
    out = None
    if accumulate:
        out = _rand(N, K, seed=43)
        ref = ref + out.float()
    got = ops.wgrad_full(dy, x, out=out, alpha=alpha, accumulate=accumulate)
    torch.cuda.synchronize()
    return _report(f"wgrad_full_B{B}_S{S}_N{N}_K{K}", got, ref, atol=float(ref.abs().max()) * 6e-3, rtol=1.6e-2)


def check_colsum2(B=3, S=333, D=1536):
    dyf, zf = _rand(B, S + 3, D + 16, seed=51), _rand(B, S, D, seed=52)
    dy = dyf[:, 1:S + 1, 8:8 + D]
    sm, dt = ops.colsum2(dy, zf)
    torch.cuda.synchronize()
    r1 = _report("colsum", sm, dy.float().sum(1), atol=0.05, rtol=1e-3)
    r2 = _report("coldot", dt, (dy.float() * zf.float()).sum(1), atol=0.05, rtol=1e-3)
    only = ops.colsum2(dy, None)[0]
    return {"name": f"colsum2_B{B}_S{S}_D{D}", "ok": r1["ok"] and r2["ok"] and bool(torch.allclose(only, sm, atol=1e-3)),
            "max_err": max(r1["max_err"], r2["max_err"])}


CHECKS.update({
    "wgrad_full_basic": lambda: check_wgrad_full(),
    "wgrad_full_strided_accum": lambda: check_wgrad_full(B=3, S=231, N=384, K=200, strided=True, accumulate=True, alpha=0.5),
    "wgrad_full_sd3_qkv": lambda: check_wgrad_full(B=2, S=1255, N=4608, K=1536),
    "wgrad_full_narrow": lambda: check_wgrad_full(B=1, S=1000, N=128, K=64),
    "wgrad_full_flux_mlp": lambda: check_wgrad_full(B=1, S=4608, N=3072, K=12288),
    "colsum2": lambda: check_colsum2(),
    "colsum2_small": lambda: check_colsum2(B=1, S=7, D=64),
})


# --------------------------------------------------------------------------------------------- LyCORIS LoKr + stand-alone GELU
def check_lokr_rebuild(a=8, b=48, c=4, d=40, scale=0.5, fused=True):
    """out = bf16(W + kron(w1, w2) * scale) and its transpose, written into slices of larger (fused q|k|v style) buffers."""
    N, K = a * b, c * d
    W, w1, w2 = _rand(N, K, seed=61) * 0.05, _rand(a, c, seed=62), _rand(b, d, seed=63) * 0.05
    ref = (W.float() + torch.kron(w1.float(), w2.float()) * scale).bfloat16()
    if fused:
        big, big_t = torch.zeros(3 * N, K, device="cuda", dtype=torch.bfloat16), torch.zeros(K, 3 * N, device="cuda", dtype=torch.bfloat16)
        out, out_t = big[N:2 * N], big_t[:, N:2 * N]
    else:
        out, out_t = torch.empty(N, K, device="cuda", dtype=torch.bfloat16), None
    ops.lokr_rebuild(W, w1, w2, scale, out, out_t)
    torch.cuda.synchronize()
    # fp32 association differs (scale * w1 first), so a rare bf16 rounding tie may land on the neighbouring value
    close = lambda x, y: float((x != y).float().mean()) < 2e-3 and bool(torch.allclose(x.float(), y.float(), rtol=2 ** -7, atol=1e-6))
    ok = close(out, ref)
    if fused:
        ok = ok and bool(torch.equal(out_t, out.t())) and float(big[:N].abs().sum() + big[2 * N:].abs().sum() + big_t[:, :N].abs().sum()) == 0.0
    return {"name": f"lokr_rebuild_{a}x{b}_{c}x{d}", "ok": ok, "max_err": float((out.float() - ref.float()).abs().max())}


def check_lokr_factor_grads(a=8, b=48, c=4, d=40, scale=0.5, strided=True):
    N, K = a * b, c * d
    w1, w2 = _rand(a, c, seed=64), _rand(b, d, seed=65)
    g_full = _rand(N + 8, K + 16, seed=66)
    dW = g_full[4:4 + N, 8:8 + K] if strided else g_full[:N, :K].contiguous()
    g4 = dW.float().view(a, b, c, d) if not strided else dW.float().reshape(a, b, c, d)
    r1 = torch.einsum("ajcl,jl->ac", g4, w2.float()) * scale
    r2 = torch.einsum("ajcl,ac->jl", g4, w1.float()) * scale
    d1, d2 = ops.lokr_factor_grads(dW, w1, w2, scale)
    torch.cuda.synchronize()
    x1 = _report("lokr_dw1", d1, r1, atol=float(r1.abs().max()) * 1e-4, rtol=1e-4)
    x2 = _report("lokr_dw2", d2, r2, atol=float(r2.abs().max()) * 1e-4, rtol=1e-4)
    return {"name": f"lokr_factor_grads_{a}x{b}_{c}x{d}", "ok": x1["ok"] and x2["ok"], "max_err": max(x1["max_err"], x2["max_err"])}


def check_gelu_tanh(B=2, S=77, D=640):
    import torch.nn.functional as F
    pf, gf = _rand(B, S + 2, D + 8, seed=71), _rand(B, S, D, seed=72)
    pre = pf[:, 1:S + 1, :D]
    act = ops.gelu_tanh(pre)
    ref = F.gelu(pre.float(), approximate="tanh")
    r1 = _report("gelu", act, ref, atol=2e-2, rtol=1.6e-2)
    x = pre.float().requires_grad_(True)
    (F.gelu(x, approximate="tanh") * gf.float()).sum().backward()
    out = ops.mul_dgelu_tanh(gf, pre)
    r2 = _report("dgelu", out, x.grad, atol=3e-2, rtol=1.6e-2)
    inplace = gf.clone()
    ops.mul_dgelu_tanh(inplace, pre, out=inplace)
    torch.cuda.synchronize()
    return {"name": f"gelu_tanh_B{B}_S{S}_D{D}", "ok": r1["ok"] and r2["ok"] and bool(torch.equal(inplace, out)), "max_err": max(r1["max_err"], r2["max_err"])}


def check_gelu_matches_gemm_epilogue(B=1, S=256, N=512, K=128):
    """ops.gelu_tanh(pre) must be BIT-identical to the activation EPI_GELU wrote next to `pre` (the LoRA-on-fc2 weight gradient
    re-creates the activation from the saved pre-activation)."""
    x, w, bias = _rand(B, S, K, seed=73), _rand(N, K, seed=74) * 0.2, _rand(N, seed=75)
    pre = torch.empty(B, S, N, device="cuda", dtype=torch.bfloat16)
    act = ops.gemm([x], [w], bias, epi=E.EPI_GELU, aux=pre)
    again = ops.gelu_tanh(pre)
    torch.cuda.synchronize()
    return {"name": "gelu_matches_gemm_epilogue", "ok": bool(torch.equal(act, again)), "max_err": float((act.float() - again.float()).abs().max())}


CHECKS.update({
    "lokr_rebuild_fused_slices": lambda: check_lokr_rebuild(),
    "lokr_rebuild_plain_ragged": lambda: check_lokr_rebuild(a=3, b=37, c=5, d=13, scale=1.0, fused=False),
    "lokr_rebuild_flux_attn": lambda: check_lokr_rebuild(a=8, b=384, c=8, d=384, scale=1.0),
    "lokr_factor_grads": lambda: check_lokr_factor_grads(),
    "lokr_factor_grads_flux_ff": lambda: check_lokr_factor_grads(a=4, b=3072, c=4, d=768, scale=1.0, strided=False),
    "lokr_factor_grads_tiny": lambda: check_lokr_factor_grads(a=2, b=3, c=2, d=8, strided=False),
    "gelu_tanh": lambda: check_gelu_tanh(),
    "gelu_matches_gemm_epilogue": lambda: check_gelu_matches_gemm_epilogue(),
})


# --------------------------------------------------------------------------------------------- [K, N] weight segments (dgrad on W itself)
# (gemm_wkn_pair*: BN = 256 forced, the name is historical as above)
CHECKS.update({
    "gemm_wkn_basic": lambda: check_gemm(256, 256, 128, w_kn=[True]),
    "gemm_wkn_bn64_tails": lambda: check_gemm(200, 72, 200, B=2, w_kn=[True], tile=(1, 64)),
    "gemm_wkn_bn128_ktail": lambda: check_gemm(300, 136, 72, w_kn=[True], tile=(1, 128)),
    "gemm_wkn_strided_bias": lambda: check_gemm(333, 320, 192, B=2, bias=True, strided=True, w_kn=[True]),
    "gemm_wkn_pair": lambda: check_gemm(4096, 3072, 512, w_kn=[True], tile=(0, 256)),
    "gemm_wkn_pair_tails": lambda: check_gemm(700, 328, 456, B=2, w_kn=[True], tile=(0, 256)),
    "gemm_wkn_mixed_segments": lambda: check_gemm(512, 384, 256, B=2, segs=[48, 128], w_kn=[True, False, True], tile=(0, 256)),
    "gemm_wkn_dgelu_epilogue": lambda: check_gemm(256, 512, 128, epi=E.EPI_MUL_DGELU, w_kn=[True]),
    "gemm_wkn_flux_dgrad": lambda: check_gemm(4608, 3072, 9216, w_kn=[True], tile=(0, 256)),
})


# --------------------------------------------------------------------------------------------- Hopper tile structure
# GemmCfg<BN> gives a ring of 4 stages at BN = 256, 6 at 128 and 8 at 64, and stage / phase carry from one persistent tile
# to the next inside a CTA.  The checks below pin the width (tile=(0, BN)) instead of relying on the run-time choice.
_EPIS = {"store": (E.EPI_STORE, False), "gelu": (E.EPI_GELU, False), "gate_res": (E.EPI_GATE_RES, False),
         "gate_res_nan": (E.EPI_GATE_RES, True), "mul_dgelu": (E.EPI_MUL_DGELU, False), "add_res": (E.EPI_ADD_RES, False),
         "mul": (E.EPI_MUL, False), "quick_gelu": (E.EPI_QUICK_GELU, False)}
_BNS = (64, 128, 256)


def _case(fn, *args, **kw):
    return lambda: fn(*args, **kw)


# every epilogue at every tile width, [N, K] and [K, N] weights, on one shape with row, column and K tails
for _en, (_epi, _nan) in _EPIS.items():
    for _bn in _BNS:
        for _kn in (False, True):
            CHECKS[f"gemm_epi_{_en}_bn{_bn}" + ("_wkn" if _kn else "")] = _case(
                check_gemm, 200, 328, 200, B=2, bias=True, epi=_epi, nan_to_num=_nan, tile=(0, _bn), w_kn=[True] if _kn else None)

# ring phase out of step at every tile boundary: segments of 200 + 72 + 16 = 4 + 2 + 1 = 7 k-blocks per tile (not a
# multiple of 4, 6 or 8) and several tiles per CTA
for _bn in _BNS:
    CHECKS[f"gemm_ring7_bn{_bn}"] = _case(check_gemm, 4608, 3072, 200, B=1, segs=[72, 16], bias=True, tile=(0, _bn))
CHECKS["gemm_ring7_bn128_wkn_mixed"] = _case(check_gemm, 4608, 3072, 200, B=1, segs=[72, 16], w_kn=[True, False, True],
                                             tile=(0, 128))
CHECKS["gemm_ring7_bn64_wkn"] = _case(check_gemm, 4608, 3072, 200, B=1, segs=[72, 16], w_kn=[True, True, True], tile=(0, 64))
# 6 m-tiles per batch x 3 batches = 18 m-tiles: the 8-tile rasterisation bands straddle batch boundaries
CHECKS["gemm_ring7_band_straddle_b3"] = _case(check_gemm, 700, 3072, 200, B=3, segs=[72, 16], bias=True, epi=E.EPI_ADD_RES,
                                              tile=(0, 128))
CHECKS["gemm_ring7_band_straddle_b3_bn256"] = _case(check_gemm, 700, 3072, 200, B=3, segs=[72, 16], bias=True, tile=(0, 256))

# skinny M (conditioning / modulation GEMMs run M = batch rows) and 128-row tiles whose second 64-row warpgroup is empty
# or holds a single row; N = 6 * 3072 is the Flux modulation width
for _m in (1, 2, 4, 64, 65, 129):
    for _b in (1, 4):
        CHECKS[f"gemm_skinny_m{_m}_b{_b}"] = _case(check_gemm, _m, 18432, 3072, B=_b, bias=True)
        CHECKS[f"gemm_skinny_m{_m}_b{_b}_bn64"] = _case(check_gemm, _m, 18432, 3072, B=_b, bias=True, tile=(0, 64))

# writes through row- and column-strided views of a wider output: the halo must stay zero
for _bn in _BNS:
    CHECKS[f"gemm_strided_gate_res_bn{_bn}"] = _case(check_gemm, 200, 328, 136, B=2, bias=True, strided=True,
                                                     epi=E.EPI_GATE_RES, nan_to_num=True, tile=(0, _bn))
    CHECKS[f"gemm_strided_mul_dgelu_bn{_bn}_wkn"] = _case(check_gemm, 200, 328, 136, B=2, strided=True,
                                                          epi=E.EPI_MUL_DGELU, tile=(0, _bn), w_kn=[True])


# --------------------------------------------------------------------------------------------- attention edges
# one valid key, keys inside one 128-key tile, a last tile with a single valid key, query tiles below 64 rows
for _sq, _sk in ((256, 1), (256, 8), (256, 64), (256, 129), (7, 300), (33, 33), (129, 129)):
    for _hd in (64, 128):
        CHECKS[f"attn_fwd_sq{_sq}_sk{_sk}_hd{_hd}"] = _case(check_attn_fwd, 2, 2, _sq, _sk, HD=_hd)
        CHECKS[f"attn_bwd_sq{_sq}_sk{_sk}_hd{_hd}"] = _case(check_attn_bwd, 2, 2, _sq, _sk, HD=_hd)
for _hd in (64, 128):
    # the model's layout: q / k / v read from, and dq / dk / dv written into, fused [B, S, 3 H HD] buffers
    CHECKS[f"attn_bwd_strided_hd{_hd}"] = _case(check_attn_bwd, 2, 3, 333, HD=_hd, strided=True)
    # peaked softmax: logits 16x larger than with unit-variance q / k
    CHECKS[f"attn_bwd_bigscore_hd{_hd}"] = _case(check_attn_bwd, 1, 2, 512, HD=_hd, qscale=4.0)
    # additive bias / mask (text encoders)
    CHECKS[f"attn_fwd_bias_head_hd{_hd}"] = _case(check_attn_fwd, 2, 3, 256, HD=_hd, bias="head")
    CHECKS[f"attn_fwd_bias_shared_hd{_hd}"] = _case(check_attn_fwd, 2, 3, 200, 256, HD=_hd, bias="shared")
    CHECKS[f"attn_fwd_bias_causal_hd{_hd}"] = _case(check_attn_fwd, 2, 2, 333, HD=_hd, bias="causal")
    CHECKS[f"attn_fwd_bias_keypad_hd{_hd}"] = _case(check_attn_fwd, 2, 2, 512, HD=_hd, bias="keypad", keep=77)
    CHECKS[f"attn_fwd_bias_ragged_hd{_hd}"] = _case(check_attn_fwd, 1, 2, 150, 333, HD=_hd, bias="head")
CHECKS["attn_bwd_strided_bigscore"] = lambda: check_attn_bwd(1, 2, 1024, strided=True, qscale=4.0)
CHECKS["attn_bwd_bigscore_long"] = lambda: check_attn_bwd(1, 2, 4608, qscale=4.0)
for _hd in (64, 128):
    # general bias after the all--inf-tile fix: rows -inf over their whole first 128-key tile, or over every key but the
    # last one; with Sk = 150 every finite key of those rows lies in the partial second tile
    CHECKS[f"attn_fwd_bias_leftpad_hd{_hd}"] = _case(check_attn_fwd, 2, 3, 200, 333, HD=_hd, bias="leftpad")
    CHECKS[f"attn_fwd_bias_leftpad_tail_hd{_hd}"] = _case(check_attn_fwd, 1, 2, 129, 150, HD=_hd, bias="leftpad")


# --------------------------------------------------------------------------------------------- per-key bias (masked training)
# Every _key_bias kind meets every key-count tail class: one key, one short of a 64-key tile, whole tiles, one past a
# tile, ragged.  Sq (1, 7, 65, 129, 333), HD and B in {1, 3} rotate along the grid.  The backward checks also check the
# forward's o and lse, which the backward reads.
_KB_KINDS = ("dense", "01", "neg", "inf", "inf_first_tile", "inf_straddle", "last_key_only", "mixed", "shared")
_KB_SK = ((1,), (63, 127, 191), (64, 128), (65, 129), (333,))
_KB_SQ = (1, 7, 65, 129, 333)
for _ki, _kind in enumerate(_KB_KINDS):
    for _ci, _sks in enumerate(_KB_SK):
        _sks = [s for s in _sks if _kind != "inf_first_tile" or s > 128]
        if not _sks:
            continue
        _sk, _sq, _hd = _sks[_ki % len(_sks)], _KB_SQ[(_ki + _ci) % 5], (64, 128)[(_ki + _ci) % 2]
        _b = 1 if (2 * _ci + _ki) % 3 == 0 and _kind not in ("mixed", "shared") else 3
        CHECKS[f"attn_bwd_kb_{_kind}_sq{_sq}_sk{_sk}_hd{_hd}_b{_b}"] = _case(check_attn_bwd, _b, 2, _sq, _sk, HD=_hd,
                                                                             key_bias=_kind, seed=_ki + _ci)
for _hd in (64, 128):
    for _s in (1, 17, 64, 77, 128, 129):
        for _kind in ("01", "neg"):
            CHECKS[f"attn_bwd_kb_{_kind}_self_s{_s}_hd{_hd}"] = _case(check_attn_bwd, 1 + _s % 3, 2, _s, HD=_hd, key_bias=_kind,
                                                                     seed=_s)
    for _sq, _sk, _kind in ((100, 300, "01"), (300, 77, "01"), (129, 520, "01"), (100, 300, "inf"), (129, 520, "inf")):
        CHECKS[f"attn_bwd_kb_{_kind}_cross_sq{_sq}_sk{_sk}_hd{_hd}"] = _case(check_attn_bwd, 3, 3, _sq, _sk, HD=_hd,
                                                                             key_bias=_kind, seed=_sq + _sk)
    # the model's layout (fused [B, S, 3 H HD] buffers, halo must stay zero) and a peaked softmax
    CHECKS[f"attn_bwd_kb_strided_hd{_hd}"] = _case(check_attn_bwd, 2, 3, 333, HD=_hd, strided=True, key_bias="dense")
    CHECKS[f"attn_bwd_kb_strided_straddle_hd{_hd}"] = _case(check_attn_bwd, 3, 2, 200, HD=_hd, strided=True,
                                                            key_bias="inf_straddle")
    CHECKS[f"attn_bwd_kb_bigscore_hd{_hd}"] = _case(check_attn_bwd, 2, 2, 512, HD=_hd, qscale=4.0, key_bias="dense")
    CHECKS[f"attn_fwd_kb_strided_hd{_hd}"] = _case(check_attn_fwd, 2, 4, 384, HD=_hd, strided=True, key_bias="dense")
    CHECKS[f"attn_fwd_kb_ragged_hd{_hd}"] = _case(check_attn_fwd, 3, 2, 333, 417, HD=_hd, key_bias="inf_straddle")
# Flux.1: 24 heads of 128, 512 text + 4096 image tokens; and the HD 64 long shape
for _kind in ("dense", "01", "inf"):
    CHECKS[f"attn_bwd_kb_flux_{_kind}"] = _case(check_attn_bwd, 1, 24, 4608, HD=128, key_bias=_kind, seed=7)
CHECKS["attn_bwd_kb_hd64_long_dense"] = _case(check_attn_bwd, 2, 3, 1255, HD=64, key_bias="dense")


# --------------------------------------------------------------------------------------------- entry points without another check
CHECKS.update({
    "gate_mul": lambda: check_gate_mul(),
    "gate_mul_small": lambda: check_gate_mul(B=1, S=7, D=64, chunk=8),
    "qk_rmsnorm_dw_hd128": lambda: check_qk_rmsnorm_dw(HD=128),
    "qk_rmsnorm_dw_hd128_norope": lambda: check_qk_rmsnorm_dw(HD=128, rope=False),
    "qk_rmsnorm_dw_hd64": lambda: check_qk_rmsnorm_dw(HD=64),
    "qk_rmsnorm_dw_hd64_norope": lambda: check_qk_rmsnorm_dw(HD=64, rope=False),
})
# skinny_tn tensor-core path on both reductions (slab workspace / fp32 atomics) and both kernels (rank block 64 / 128)
for _r in (8, 64, 72, 128):
    for _det in (True, False):
        CHECKS[f"skinny_r{_r}_" + ("ws" if _det else "atomic")] = _case(check_skinny, B=2, S=700, R=_r, N=1536,
                                                                         deterministic=_det)
for _det in (True, False):   # several batches, S not a multiple of the row split
    CHECKS["skinny_b3_split_tail_" + ("ws" if _det else "atomic")] = _case(check_skinny, B=3, S=1000, R=48, N=1024,
                                                                          deterministic=_det)


# --------------------------------------------------------------------------------------------- run-to-run determinism
CHECKS.update({
    "attn_bwd_repeatable_hd128": lambda: check_attn_bwd_repeatable(HD=128),
    "attn_bwd_repeatable_hd64": lambda: check_attn_bwd_repeatable(HD=64),
    "skinny_repeatable_flux_lora": lambda: check_skinny_repeatable(),
    "flow_loss_full_size": lambda: check_loss_full_size("flow"),
    "target_loss_full_size": lambda: check_loss_full_size("target"),
})
