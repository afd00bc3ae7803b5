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
    dt = torch.float64 if ref.dtype == torch.float64 else torch.float32   # an fp64 reference is compared in fp64
    got = got.to(dt)
    ref = ref.to(dt)
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


# --------------------------------------------------------------------------------------------- GEMM-family reference model
# The GEMM-family checks (gemm, wgrad_full, skinny_tn, conv3x3_nhwc, conv_in_3ch, colsum2) compare the kernel with an fp64
# reference computed on the kernel's own bf16 inputs, element by element, in one of two input modes.
#
# Realistic inputs (exact=False): N(0, s^2) operands.  Per-element tolerance
#     tol = rtol |ref| + GEMM_C 2^-24 sqrt(K) (|A| |W|^T)_ij
# with K the whole contraction length (all segments of a gemm, the tokens of wgrad_full / skinny_tn / colsum2, 9 C_in of a
# conv).  The second term is the usual scale of an fp32 dot product's rounding error; |A| |W|^T is one more fp64 product,
# of the absolute values.  rtol is 2^-7 for bf16 outputs, not 2^-8: the bf16 store alone rounds by up to half an ulp =
# 2^-8 |x|, which would use all of an rtol of 2^-8 (ATTN_TOL has the same reason).  fp32 outputs (skinny_tn, colsum2) have
# rtol 2^-23, one fp32 ulp.  Epilogues that write the pre-activation (EPI_GELU / EPI_GATE_RES aux) have it checked with
# this tolerance and the output checked as a function of it: GATE_RES bit for bit, GELU as one of the two bf16 neighbours
# of fp64 gelu_tanh(aux).  The others propagate the tolerance: |derivative| x atol plus one bf16 ulp (2^-7 |x|) for each
# rounding.  Each result reports tol_use (the worst element's share of its tolerance) and, where the accumulation term
# applies directly, c_half: the smallest GEMM_C at which that check's tol_use would be 0.5.
#   GEMM_C = 0.5, measured on H100 80GB HBM3 (SXM, 700 W limit): the largest c_half of any unmodified kernel was 0.143
#   (gemm_pair_flux_shape; wgrad 0.104, conv 0.142, colsum2 0.108, skinny_tn 0.073; the largest tol_use 0.498), so every error of the wgmma
#   accumulation stayed below 0.07 x 2^-24 sqrt(K) sum |a w| where it can be seen through an fp32 output.  This is a
#   measured value, not a model of the tensor core's rounding.
#
# Exact inputs (exact=True): A / dy / L / pixel operands are integers in [-2, 2], W / x operands integers in [-6, 6] times
# 2^-4 (_gen).  exact_bound_ok asserts on the host, from the drawn values, that every product is a multiple of 2^-4 and
# sum_k |a_k w_k| < 2^19, so every partial sum in any order is a multiple of 2^-4 below 2^19: 23 significant bits, exact
# in fp32 (and still exact if the tensor core aligned its addends to fewer bits than fp32, down to 2^-4; unmeasured).  The
# fp64 accumulation then equals the kernel's fp32 accumulator whatever the tile, split or atomic order, and the epilogue
# is replayed with fp32 torch ops: the output must be bit-identical.  Bias, gate, res and aux stay ordinary bf16 values.
# GELU, QuickGELU and dGELU use tanhf / __expf: their output must be one of the two bf16 neighbours of the fp64 value.
# alpha * acc + old (wgrad_full accumulate, the skinny_tn slab reduce) may be contracted into an FMA: power-of-two alphas
# are bit-exact either way; a non-power-of-two case accepts either rounding.
GEMM_C = 0.5
GEMM_RTOL_BF16 = 2 ** -7
GEMM_RTOL_F32 = 2 ** -23
EXACT_BOUND = 2 ** 19
_U = 2 ** -7          # one bf16 ulp relative to |x| (an upper bound)


def gelu_tanh(x):
    return torch.nn.functional.gelu(x, approximate="tanh")


def gelu64(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def dgelu64(x):
    k0, k1 = math.sqrt(2.0 / math.pi), 0.044715
    t = torch.tanh(k0 * (x + k1 * x ** 3))
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * k0 * (1.0 + 3.0 * k1 * x * x)


def quick_gelu64(y):
    return y * torch.sigmoid(1.702 * y)


def dquick_gelu64(y):
    s = torch.sigmoid(1.702 * y)
    return s + 1.702 * y * s * (1.0 - s)


def _gen(*shape, seed=0, scale=1.0, exact=None):
    """A bf16 operand on the GPU.  exact None: N(0, scale^2) (_rand); "int": integers in [-2, 2] (A, dy, L, pixels);
    "frac": integers in [-6, 6] x 2^-4 (W, x)."""
    if exact is None:
        return _rand(*shape, scale=scale, seed=seed)
    g = torch.Generator(device="cpu").manual_seed(seed)
    hi = 2 if exact == "int" else 6
    v = torch.randint(-hi, hi + 1, shape, generator=g).float()
    return (v if exact == "int" else v / 16).to(torch.bfloat16).to(DEV)


def exact_bound_ok(ints, fracs, mag):
    """The exact-input bound from the drawn values: `ints` hold integers, `fracs` multiples of 2^-4, and every
    mag = sum_k |a_k w_k| (fp64) is below 2^19, which bounds every partial sum of the dot product in any order."""
    is_int = lambda t: bool((t.double() == t.double().round()).all())
    return all(is_int(t) for t in ints) and all(is_int(t.double() * 16) for t in fracs) and float(mag.max()) < EXACT_BOUND


def _is_pow2(x):
    return x != 0 and math.frexp(abs(x))[0] == 0.5


def _f32(x):
    """x rounded to fp32, as a Python float (what a float kernel argument holds)."""
    return float(torch.tensor(x, dtype=torch.float32))


def gate_res_replay(y, gate, res, nan_to_num=False):
    """EPI_GATE_RES output from the bf16 linear output y [B, S, N]: res + bf16(gate * y) in fp32, rounded once; with
    nan_to_num the rounded value maps NaN -> 0 and +-inf -> +-65504 (which is 65536 in bf16)."""
    out = (res.float() + (gate.float()[:, None, :] * y.float()).bfloat16().float()).bfloat16()
    if nan_to_num:
        out = torch.nan_to_num(out, nan=0.0, posinf=65504.0, neginf=-65504.0)
    return out


def replay_epilogue(epi, acc, bias=None, gate=None, res=None, aux=None, nan_to_num=False):
    """The fp32 epilogue of gemm.cuh on an exact fp32 accumulator acc [B, S, N].  Returns (out, pre), bf16, with
    pre = bf16(acc + bias) (the aux output of EPI_GELU / EPI_GATE_RES) and out the bits the kernel writes for EPI_STORE,
    EPI_ADD_RES, EPI_GATE_RES and EPI_MUL; None for the transcendental epilogues, which have no bit-exact replay."""
    f = acc.float() if bias is None else acc.float() + bias.float()
    pre = f.bfloat16()
    out = None
    if epi == ops.EPI_STORE:
        out = pre
    elif epi == ops.EPI_ADD_RES:
        out = (f + res.float()).bfloat16()
    elif epi == ops.EPI_GATE_RES:
        out = gate_res_replay(pre, gate, res, nan_to_num)
    elif epi == ops.EPI_MUL:
        out = (pre.float() * aux.float()).bfloat16()
    return out, pre


def _bf16_steps(g):
    """(next bf16 value below g, next above g) in fp64, for finite bf16 g."""
    m = g.float().abs().contiguous().view(torch.int32)
    up_mag = (m + (1 << 16)).view(torch.float32).double()
    dn_mag = (m - (1 << 16)).clamp_min(0).view(torch.float32).double()
    gf = g.float()
    return torch.where(gf > 0, dn_mag, -up_mag), torch.where(gf < 0, -dn_mag, up_mag)


def _first(mask, got, ref, out):
    idx = torch.nonzero(mask)[:8]
    out["first_bad"] = idx.tolist()
    out["got"] = [float(got[tuple(i)]) for i in idx.tolist()]
    out["want"] = [float(ref[tuple(i)]) for i in idx.tolist()]


def _bits(name, got, ref):
    """got and ref (both bf16 or both fp32) hold the same bits, NaN at the same places (payloads not compared)."""
    iv = torch.int16 if got.dtype == torch.bfloat16 else torch.int32
    both_nan = torch.isnan(got) & torch.isnan(ref)
    diff = (got.contiguous().view(iv) != ref.contiguous().view(iv)) & ~both_nan
    n = int(diff.sum().item())
    out = {"name": name, "ok": n == 0, "n_diff": n, "numel": got.numel()}
    if n:
        _first(diff, got, ref, out)
    return out


def _neighbour(name, got, ref, atol=None):
    """got (bf16) is one of the two bf16 neighbours of the fp64 ref: no bf16 value lies strictly between them.  atol: an
    absolute error also accepted (the fp32 formula's own cancellation, see _gelu_atol)."""
    dn, up = _bf16_steps(got)
    near = (dn <= ref) & (ref <= up)
    if atol is not None:
        near = near | ((got.double() - ref).abs() <= atol)
    bad = ~(near & torch.isfinite(got))
    n = int(bad.sum().item())
    out = {"name": name, "ok": n == 0, "n_bad": n, "numel": got.numel()}
    if n:
        _first(bad, got, ref, out)
    return out


def _gelu_atol(x):
    """For x << 0 the fp32 formulas 0.5 x (1 + tanh u) and its derivative cancel: 1 + tanh u carries the rounding of tanh
    near -1, about 2^-24, so gelu is off by ~2^-24 |x| absolutely (torch's own fp32 / bf16 GELU too) while its value is
    tiny.  Allowed: 2^-22 |x| for gelu, 2^-21 (1 + |x| u') for its derivative."""
    du = math.sqrt(2.0 / math.pi) * (1.0 + 3 * 0.044715 * x * x)
    return 2.0 ** -22 * x.abs(), 2.0 ** -21 * (1.0 + x.abs() * du)


def _slope(deriv, x):
    """|deriv| over the interval the bf16 rounding of x can move it (x (1 +- 2^-8)): the derivative that propagates the
    pre-activation's rounding, which a value at x alone understates where the curvature is large."""
    return torch.maximum(deriv(x).abs(), torch.maximum(deriv(x * (1 + 2 ** -8)).abs(), deriv(x * (1 - 2 ** -8)).abs()))


def _acc_unit(mag, K):
    return 2.0 ** -24 * math.sqrt(K) * mag


def _report_acc(name, got, ref, mag, K, rtol, c=GEMM_C):
    """_report with the accumulation tolerance rtol |ref| + c 2^-24 sqrt(K) mag, plus c_half."""
    unit = _acc_unit(mag, K)
    r = _report(name, got, ref, atol=c * unit, rtol=rtol)
    err = (got.double() - ref).abs()
    need = torch.where(unit > 0, (2 * err - rtol * ref.abs()) / unit.clamp_min(1e-300), torch.zeros_like(err))
    r["c_half"] = round(float(need.max().clamp_min(0).item()), 3) if need.numel() else 0.0
    return r


def _combine(name, parts, **extra):
    """One result from the parts of a check: ok if every part is, the largest tol_use / c_half, failing parts in full."""
    out = {"name": name, "ok": all(p["ok"] for p in parts) and all(v for v in extra.values() if isinstance(v, bool))}
    for key in ("tol_use", "c_half"):
        vals = [p[key] for p in parts if key in p]
        if vals:
            out[key] = max(vals)
    for p in parts:
        out[f"{p['name']}_ok"] = p["ok"]
        if not p["ok"]:
            out[f"{p['name']}_detail"] = p
    out.update(extra)
    return out


def _pad8(n):
    return (n + 7) // 8 * 8


def check_gemm(M=256, N=256, K=128, B=1, bias=False, epi=ops.EPI_STORE, tile=(0, 0), segs=None, strided=False,
               nan_to_num=False, name=None, w_kn=None, exact=False, aux_out=None, res_special=False):
    """segs: list of extra K sizes appended as additional segments.  w_kn[i]: hand segment i's weight over as [K, N]
    (the contraction index is the row — what a dgrad reads from the forward weight) instead of [N, K].
    exact: the exact-input mode (bit for bit).  aux_out: give EPI_GELU / EPI_GATE_RES an aux output (default: GELU yes,
    GATE_RES no).  res_special (GATE_RES, with aux): res holds +inf, -inf and NaN, and +-bf16 max in columns whose gate
    (2^120) pushes res + gate y past it; out must match the replay from the kernel's aux bit for bit.
    strided, or odd N: out is a view of a wider zero-filled buffer whose halo must stay zero; with odd N gate / res / aux
    are views of wider buffers too (row strides must be multiples of 8 elements)."""
    Ks = [K] + list(segs or [])
    S = M
    ea, ew = ("int", "frac") if exact else (None, None)
    NP = _pad8(N) + 8                      # row length of the padded buffers
    if aux_out is None:
        aux_out = epi == ops.EPI_GELU
    assert not res_special or (epi == ops.EPI_GATE_RES and aux_out)
    a_list, w_list = [], []
    for i, k in enumerate(Ks):
        if strided:
            a_list.append(_gen(B, S + 3, k + 16, seed=10 + i, exact=ea)[:, 1:S + 1, 8:8 + k])
            w_list.append(_gen(N, k + 8, scale=0.5, seed=20 + i, exact=ew)[:, :k])
        else:
            a_list.append(_gen(B, S, k, seed=10 + i, exact=ea))
            w_list.append(_gen(N, k, scale=0.5, seed=20 + i, exact=ew))
    bias_t = _rand(N, seed=30) if bias else None

    def rows(seed=None):
        """[B, S, N] bf16 (zeros without a seed); a view of a [B, S, NP] buffer when N is odd."""
        t = _rand(B, S, N, seed=seed) if seed is not None else torch.zeros(B, S, N, dtype=torch.bfloat16, device=DEV)
        if N % 2 == 0:
            return t
        full = torch.zeros(B, S, NP, dtype=torch.bfloat16, device=DEV)
        full[..., :N] = t
        return full[..., :N]

    gate = res = aux = None
    if epi == ops.EPI_GATE_RES:
        gfull = torch.zeros(B, NP, dtype=torch.bfloat16, device=DEV)
        gfull[:, :N] = _rand(B, N, seed=31)
        gate = gfull[:, :N] if N % 2 else gfull[:, :N].contiguous()
        res = rows(32)
    elif epi == ops.EPI_ADD_RES:
        res = rows(32)
    elif epi == ops.EPI_MUL_DGELU:
        aux = rows(33)
    elif epi == ops.EPI_MUL:
        aux = rows(34)
    if aux_out:
        aux = rows()
    if res_special:
        big = torch.finfo(torch.bfloat16).max
        res[..., 0::8] = float("inf")
        res[..., 1::8] = float("-inf")
        res[..., 2::8] = float("nan")
        res[:, 0::2, 3::8] = big
        res[:, 1::2, 3::8] = -big
        gate[:, 3::8] = 2.0 ** 120
    out = None
    padded = strided or N % 2 == 1
    if padded:
        outfull = torch.zeros(B, S + 2, NP, dtype=torch.bfloat16, device=DEV)
        out = outfull[:, 1:S + 1, :N]
    w_pass = list(w_list)
    if w_kn is not None:
        for i, flag in enumerate(w_kn):
            if flag:                      # [K, N] storage; with `strided` a column range of a wider matrix (row stride > N)
                if strided:
                    wide = torch.zeros(w_list[i].shape[1], _pad8(N) + 24, dtype=torch.bfloat16, device=DEV)
                    wide[:, 8:8 + N] = w_list[i].t()
                    w_pass[i] = wide[:, 8:8 + N]
                else:
                    w_pass[i] = w_list[i].t().contiguous()
    got = ops.gemm(a_list, w_pass, bias_t, out=out, epi=epi, gate=gate, res=res, aux=aux, nan_to_num=nan_to_num, tile=tile,
                   w_kn=w_kn)
    torch.cuda.synchronize()

    acc64 = sum(a.double() @ w.double().t() for a, w in zip(a_list, w_list))
    mag = sum(a.double().abs() @ w.double().abs().t() for a, w in zip(a_list, w_list))
    Kt = sum(Ks)
    parts, extra = [], {}
    if exact:
        extra["exact_bound"] = exact_bound_ok(a_list, w_list, mag)
        want, pre = replay_epilogue(epi, acc64.float(), bias_t, gate, res, aux, nan_to_num)
        if aux_out:
            parts.append(_bits("aux", aux, pre))
        if want is not None:
            parts.append(_bits("out", got, want))
        elif epi == ops.EPI_GELU:
            parts.append(_neighbour("out", got, gelu64(pre.double()), _gelu_atol(pre.double())[0]))
        elif epi == ops.EPI_QUICK_GELU:
            parts.append(_neighbour("out", got, quick_gelu64(pre.double())))
        elif epi == ops.EPI_MUL_DGELU:
            f = acc64.float() if bias_t is None else acc64.float() + bias_t.float()
            parts.append(_neighbour("out", got, f.double() * dgelu64(aux.double()),
                                    f.double().abs() * _gelu_atol(aux.double())[1]))
    else:
        f64 = acc64 if bias_t is None else acc64 + bias_t.double()
        atol = GEMM_C * _acc_unit(mag, Kt)
        if aux_out:
            parts.append(_report_acc("aux", aux, f64, mag, Kt, GEMM_RTOL_BF16))
        if epi == ops.EPI_STORE:
            parts.append(_report_acc("out", got, f64, mag, Kt, GEMM_RTOL_BF16))
        elif epi == ops.EPI_ADD_RES:
            parts.append(_report_acc("out", got, f64 + res.double(), mag, Kt, GEMM_RTOL_BF16))
        elif epi == ops.EPI_GATE_RES and aux_out:
            parts.append(_bits("out", got, gate_res_replay(aux, gate, res, nan_to_num)))
        elif epi == ops.EPI_GATE_RES:
            g = gate.double()[:, None, :]
            ref = res.double() + g * f64
            parts.append(_report("out", got, ref, atol=g.abs() * atol + 2 * _U * (g * f64).abs(), rtol=_U))
        elif epi == ops.EPI_GELU and aux_out:
            parts.append(_neighbour("out", got, gelu64(aux.double()), _gelu_atol(aux.double())[0]))
        elif epi == ops.EPI_GELU:
            parts.append(_report("out", got, gelu64(f64), atol=_slope(dgelu64, f64) * (atol + _U * f64.abs()) + _gelu_atol(f64)[0],
                                 rtol=_U))
        elif epi == ops.EPI_MUL:
            x = aux.double()
            parts.append(_report("out", got, f64 * x, atol=x.abs() * (atol + _U * f64.abs()), rtol=_U))
        elif epi == ops.EPI_QUICK_GELU:
            parts.append(_report("out", got, quick_gelu64(f64), atol=_slope(dquick_gelu64, f64) * (atol + _U * f64.abs()),
                                 rtol=_U))
        elif epi == ops.EPI_MUL_DGELU:
            d = dgelu64(aux.double())
            parts.append(_report("out", got, f64 * d, atol=d.abs() * atol + f64.abs() * _gelu_atol(aux.double())[1], rtol=_U))
        else:
            raise ValueError(f"no reference for epilogue {epi}")
    if padded:
        # nothing outside the view may be touched
        mask = torch.ones_like(outfull, dtype=torch.bool)
        mask[:, 1:S + 1, :N] = False
        extra["halo_clean"] = bool((outfull[mask] == 0).all().item())
    mode = "_exact" if exact else ""
    return _combine(name or f"gemm_M{M}_N{N}_K{Ks}_B{B}_epi{epi}_tile{tile}{mode}", parts, **extra)


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


# --------------------------------------------------------------------------------------------- row-wise reference model
# The row-wise kernels of elementwise.cuh (ln_modulate, qk_rmsnorm_rope, rmsnorm, gelu_tanh, the losses) are compared with
# fp64 references computed on the kernels' own bf16 inputs, element by element, in one of three ways.
#
# Forward kernels with bf16 intermediates (ln_modulate_fwd, rmsnorm_fwd, qk_rmsnorm_rope_fwd): interval replay.  The
# normalised value n = (x - mean) rstd (LayerNorm) or x rstd (RMSNorm) is computed in fp64 and widened by a bound on the
# kernel's fp32 error (ln_interval / rms_range derive it).  The kernel rounds its fp32 n to bf16, and rounding is
# monotone, so its bf16 n lies in [bf16(n - err), bf16(n + err)]: one value unless n lies within err of a rounding
# midpoint.  The rest of the chain is replayed on both ends with the bf16 roundings of the eager module chain:
#   ln_modulate: bf16(bf16(n * bf16(1 + scale)) + shift)    rmsnorm / RMSNorm weight: bf16(n * w)
# Both are monotone in n for a fixed factor, so the output must lie between the two replays; where the interval holds one
# value this is bit for bit.  The RoPE rotation o = y cos + rot(y) sin is linear in the pair (y_2j, y_2j+1): its ends are
# taken over the four corners of the pair's interval, and at each corner the kernel may round y c and rot(y) s and their
# sum separately (the eager order) or contract one product into an FMA.  n_fma / n_eager count the bit-exact elements
# that only the FMA / only the eager order explains.
# A mutant that drops or adds a rounding moves the output by up to an output ulp on every element where the two orders
# round differently: for random inputs that is a fixed share of elements (over 1 % for ln_modulate's dropped rounding,
# test_rowwise_reference_cpu.py) and the accepted set is a single value on almost all of them.
#
# Backward kernels (ln_modulate_bwd, qk_rmsnorm_rope_bwd and its dw): fp64 autograd of the forward on the same bf16
# inputs (the modulation factor the forward applies, bf16(1 + scale)), and the per-element tolerance of _report_acc:
#   tol = rtol |ref| + c 2^-24 sqrt(K) M_ij,   K = D (HD) for dx, the number of token rows for dw
# with M_ij the magnitude of the terms of the element's own formula: LayerNorm rstd (|g_i| + mean|g| + |xhat_i| mean|g xhat|)
# with g = dy bf16(1 + scale); RMSNorm rstd (|g_i| + |xhat_i| mean|g xhat|) with g = w R^T dout taken in magnitudes;
# dw the sum over rows of |R^T dout|_i |xhat_i|.  rtol is one ulp of the output (2^-7 bf16, as GEMM_RTOL_BF16: the store
# alone rounds by up to 2^-8 |x|; 2^-23 fp32 dw).  ROW_C holds c per kernel, chosen on H100 80GB HBM3 (SXM, 700 W limit)
# at more than twice the largest c_half (the c at which a check's tol_use would be 0.5) measured over the registry:
#   ln_modulate_bwd 0.028, qk_rmsnorm_rope_bwd 0.101 (flat and warp-per-token kernels, the Flux shape), dw 0.008;
# the largest tol_use was 0.498, the store's own half ulp.
#
# Loss kernels: dpred is replayed bit for bit in fp32 in the kernel's operation order; the huber / smooth_l1 root
# sqrt(d d + c c) is contracted into an FMA in the H100 build (SASS: FFMA d, d, c c), so either rounding is accepted and
# counted (n_fma / n_twice: on the registered inputs the two never round to different bf16 values).  The loss scalar
# is held against fp64 with the summation bound of loss_bound.
ROW_C = {"ln_modulate_bwd": 0.25, "qk_rmsnorm_rope_bwd": 0.25, "qk_rmsnorm_dw": 0.25}


def _bf16_range(n64, err):
    """[bf16(n64 - err), bf16(n64 + err)]: every fp32 value within err of n64 rounds to bf16 inside it (fp64 -> fp32 ->
    bf16 rounding is monotone).  err is widened by 2^-20 of itself for the fp64 arithmetic of the bound."""
    err = err * (1 + 2 ** -20)
    return (n64 - err).float().bfloat16(), (n64 + err).float().bfloat16()


def _in_range(name, got, lo, hi):
    """got lies in [lo, hi] element by element and is finite; frac_exact: share of elements whose range is one value."""
    g, lo, hi = got.float(), lo.float(), hi.float()
    bad = ~((lo <= g) & (g <= hi) & torch.isfinite(g))
    n = int(bad.sum().item())
    out = {"name": name, "ok": n == 0, "n_bad": n, "numel": got.numel(),
           "frac_exact": round(float((lo == hi).double().mean().item()), 4) if got.numel() else 1.0}
    if n:
        _first(bad, g, (lo + hi) / 2, out)
    return out


def ln_vpt(D, fwd=True):
    """The VPT instantiation stb_ln_modulate_fwd / _bwd launch for D (8 x VPT elements per thread)."""
    v = (D + 1023) // 1024
    return v if v <= 4 else (8 if fwd else 4)


def ln_interval(x, eps, vpt):
    """bf16 range of the kernel's LayerNorm output bf16((x - mean) rstd) per element of x [.., D] (bf16).

    The kernel sums x in fp32: each thread adds its 8 VPT elements in order, then 5 shuffle levels and 3 adds of the
    warp sums, so no element passes more than L = 8 VPT + 8 additions and |mean32 - mean| <= 2^-24 (L + 1) mean|x|
    (+1: the division by D), with mean|x| <= |mean| + sigma.  The sum of (x - mean32)^2, all terms positive, has a
    relative error below 2^-24 (L + 2); / D, + eps and rsqrtf (2 ulp = 2^-22) add 2^-24 (2 + 4), so rstd is within
    2^-24 (L / 2 + 6) of its value; x - mean32 and the product with rstd round once each.  In all:
        |n32 - n| <= 2^-24 [(L / 2 + 8) |n| + (L + 1)(|mean| + sigma) rstd]
    (the D (mean32 - mean)^2 the variance gains is second order and is inside the 2^-24 |n| margin).  A row of zeros
    has n = 0 and err = 0: the output must be exactly bf16(0 * factor) + shift."""
    x64 = x.double()
    m = x64.mean(-1, keepdim=True)
    sig = (x64 - m).pow(2).mean(-1, keepdim=True).sqrt()
    r = (sig * sig + _f32(eps)).rsqrt()
    n = (x64 - m) * r
    L = 8 * vpt + 8
    return _bf16_range(n, 2 ** -24 * ((L / 2 + 8) * n.abs() + (L + 1) * (m.abs() + sig) * r))


def ln_modulate_replay(n, scale, shift):
    """diffusers `norm(x) * (1 + scale[:, None]) + shift[:, None]` on the bf16 LayerNorm output n [B, S, D]: three bf16
    tensor ops, each rounded."""
    t1 = (1 + scale.float()).bfloat16()
    return ((n.float() * t1.float()[:, None]).bfloat16().float() + shift.float()[:, None]).bfloat16()


def rms_weight_replay(n, w):
    """diffusers RMSNorm / T5LayerNorm after the cast to the weight dtype: bf16(n * w); n itself without a weight."""
    return n if w is None else (n.float() * w.float()).bfloat16()


def rms_range(x, w, eps, L):
    """bf16 range of bf16(bf16(x rstd) w) (w None: bf16(x rstd)) per element of x [.., D] (bf16), rstd from the fp32
    sum of squares.  All its L partial additions add positive terms (L: the longest chain of additions an element goes
    through), so the sum is within 2^-24 L relative; / D, + eps and rsqrtf add 2^-24 (2 + 4) and the product with x one
    rounding: |n32 - n| <= 2^-24 (L / 2 + 8) |n|.  Zero rows give n = 0 exactly."""
    x64 = x.double()
    n = x64 * (x64.pow(2).mean(-1, keepdim=True) + _f32(eps)).rsqrt()
    lo, hi = _bf16_range(n, 2 ** -24 * (L / 2 + 8) * n.abs())
    a, b = rms_weight_replay(lo, w), rms_weight_replay(hi, w)
    return torch.minimum(a, b), torch.maximum(a, b)


def _rot(y):
    """The rotated partner of each element: (-y_2j+1, y_2j) (diffusers _apply_rotary_emb_anyshape, use_real_unbind_dim -1)."""
    return torch.stack([-y[..., 1::2], y[..., 0::2]], -1).flatten(-2)


def _swap(t):
    """Exchange the two members of each pair: (t_2j+1, t_2j)."""
    return torch.stack([t[..., 1::2], t[..., 0::2]], -1).flatten(-2)


def rope_modes(y, yr, cos, sin):
    """y cos + yr sin in fp32, rounded to bf16, the three ways the kernel may evaluate it: eager (both products and the sum
    rounded, as `(x.float() * cos + x_rotated.float() * sin).to(x.dtype)`), and with either product contracted into an
    FMA.  y, yr bf16; cos, sin fp32 (broadcast).  The bf16 x fp32 product is exact in fp64."""
    a, b = y.float() * cos, yr.float() * sin
    eager = (a + b).bfloat16()
    fma_c = (y.double() * cos.double() + b.double()).float().bfloat16()
    fma_s = (yr.double() * sin.double() + a.double()).float().bfloat16()
    return eager, fma_c, fma_s


def rope_range(ylo, yhi, cos, sin):
    """[lo, hi] (fp32) of the rotation over the four corners of each pair's y interval and the three evaluation orders."""
    lo = hi = None
    for ys in (ylo, yhi):
        for yp in (ylo, yhi):
            for v in rope_modes(ys, _rot(yp), cos, sin):
                v = v.float()
                lo = v if lo is None else torch.minimum(lo, v)
                hi = v if hi is None else torch.maximum(hi, v)
    return lo, hi


def _rope_fma_counts(got, ylo, yhi, cos, sin):
    """On elements whose pair interval is one point: (n_fma, n_eager), the elements that only an FMA / only the eager order
    explains."""
    point = (ylo == yhi) & (_rot(ylo) == _rot(yhi))
    eager, fc, fs = rope_modes(ylo, _rot(ylo), cos, sin)
    is_fma = (got == fc) | (got == fs)
    n_fma = int((point & is_fma & (got != eager)).sum().item())
    n_eager = int((point & (got == eager) & ~is_fma).sum().item())
    return n_fma, n_eager


# --------------------------------------------------------------------------------------------- elementwise
def _ln_edge_rows(x, eps):
    """Rows 0-3 of every sample: all zero (padded text tokens), constant 0.3, mean 256 with sigma ~1, sigma ~sqrt(eps)."""
    B, S, D = x.shape
    g = torch.Generator().manual_seed(77)
    x[:, 0] = 0
    x[:, 1] = 0.3
    x[:, 2] = (256 + torch.randn(B, D, generator=g)).to(torch.bfloat16).to(x.device)
    x[:, 3] = (math.sqrt(eps) * torch.randn(B, D, generator=g)).to(torch.bfloat16).to(x.device)


def check_ln_modulate(B=2, S=64, D=3072, eps=1e-6, window=False, chunks=6, chunk=0, add="add"):
    """out = LayerNorm(x) * (1 + scale) + shift by interval replay, and dx (+ add) against fp64 autograd.
    Rows 0-3 of every sample are _ln_edge_rows: zero rows must give shift bit for bit.
    window: x, dy, add and out are row / column windows of joint [B, 77 + S + 2, D + 16] buffers (text rows first), the
    halo of out must stay zero.  shift / scale: chunks `chunk`, `chunk + 1` of a [B, chunks D] modulation tensor.
    add: "add" (a separate residual gradient), None, or "alias" (add is the output buffer, as the dual-attention backward of
    flux/blocks.py::DoubleBlockFn does).
    D > 4096 (the VPT = 8 forward) has no backward."""
    def rows(seed, zero=False):
        if not window:
            return torch.zeros(B, S, D, dtype=torch.bfloat16, device=DEV) if zero else _rand(B, S, D, seed=seed)
        full = torch.zeros(B, 77 + S + 2, D + 16, dtype=torch.bfloat16, device=DEV) if zero else \
            _rand(B, 77 + S + 2, D + 16, seed=seed)
        return full, full[:, 77:77 + S, 8:8 + D]

    xv = rows(1)
    x = xv[1] if window else xv
    _ln_edge_rows(x, eps)
    mod = _rand(B, chunks * D, seed=2, scale=0.3)
    shift, scale = mod[:, chunk * D:(chunk + 1) * D], mod[:, (chunk + 1) * D:(chunk + 2) * D]
    ov = rows(0, zero=True)
    out = ops.ln_modulate_fwd(x, shift, scale, eps=eps, out=ov[1] if window else None)
    torch.cuda.synchronize()
    n_lo, n_hi = ln_interval(x, eps, ln_vpt(D))
    a, b = ln_modulate_replay(n_lo, scale, shift), ln_modulate_replay(n_hi, scale, shift)
    parts = [_in_range("fwd", out, torch.minimum(a, b), torch.maximum(a, b)), _bits("fwd_zero_rows", out[:, 0], shift)]
    extra = {}
    if window:
        mask = torch.ones_like(ov[0], dtype=torch.bool)
        mask[:, 77:77 + S, 8:8 + D] = False
        extra["halo_clean"] = bool((ov[0][mask] == 0).all().item())
    name = f"ln_modulate_D{D}_eps{eps:g}" + ("_window" if window else "") + f"_mod{chunks}" + f"_add{add}"
    if D > 4096:
        return _combine(name, parts, **extra)

    dyv = rows(3)
    dy = dyv[1] if window else dyv
    addt = None
    if add is not None:
        addv = rows(4)
        addt = addv[1] if window else addv
    add64 = addt.double() if addt is not None else 0.0
    dx = ops.ln_modulate_bwd(dy, x, scale, add=addt, eps=eps, out=addt if add == "alias" else None)
    torch.cuda.synchronize()
    xd = x.double().requires_grad_(True)
    t = (1 + scale.float()).bfloat16().double()[:, None]
    (torch.nn.functional.layer_norm(xd, (D,), eps=_f32(eps)) * t).backward(dy.double())
    x64 = x.double()
    m = x64.mean(-1, keepdim=True)
    r = ((x64 - m).pow(2).mean(-1, keepdim=True) + _f32(eps)).rsqrt()
    xh = (x64 - m) * r
    g = (dy.double() * t).abs()
    mag = r * (g + g.mean(-1, keepdim=True) + xh.abs() * (g * xh.abs()).mean(-1, keepdim=True))
    parts.append(_report_acc("bwd", dx, xd.grad + add64, mag, D, GEMM_RTOL_BF16, c=ROW_C["ln_modulate_bwd"]))
    return _combine(name, parts, **extra)


def _rope_tables(S, HD, seed=5, paired=True):
    """fp32 cos / sin [S, HD].  paired: one angle per pair, both members of a pair hold it (the model's tables); else
    every element its own angles, so that a table entry taken from the wrong member of a pair changes the result."""
    g = torch.Generator().manual_seed(seed)
    if paired:
        ang = torch.rand(S, HD // 2, generator=g) * 6.28
        cos = ang.cos().repeat_interleave(2, dim=-1)
        sin = ang.sin().repeat_interleave(2, dim=-1)
    else:
        cos = (torch.rand(S, HD, generator=g) * 6.28).cos()
        sin = (torch.rand(S, HD, generator=g) * 6.28).sin()
    return cos.float().to(DEV).contiguous(), sin.float().to(DEV).contiguous()


def _rmsnorm_rope_ref(x, w, cos, sin, eps=1e-6):
    """RMSNorm (* w unless None), then y cos + rot(y) sin with [S, HD] tables (None: no rotation), in x's dtype;
    x [B, S, H, HD]."""
    y = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)
    if w is not None:
        y = y * w
    if cos is None:
        return y
    return y * cos[None, :, None, :] + _rot(y) * sin[None, :, None, :]


def _qk_rope_mag(x, go, w, cos, sin, eps):
    """(M of the dx tolerance, |R^T dout| |xhat| summed per element for dw) of one q or k part [B, S, H, HD]."""
    x64 = x.double()
    r = (x64.pow(2).mean(-1, keepdim=True) + _f32(eps)).rsqrt()
    xh = (x64 * r).abs()
    ga = go.double().abs()
    dya = ga if cos is None else ga * cos.double().abs()[None, :, None, :] + _swap(ga * sin.double().abs()[None, :, None, :])
    g = dya if w is None else dya * w.double().abs()
    return r * (g + xh * (g * xh).mean(-1, keepdim=True)), dya * xh


def check_qk_rmsnorm_rope(B=2, S=96, H=4, HD=128, s_split=32, tables="free", weights=True, strided_out=False,
                          loop_bwd=False, zero_rows=False, eps=1e-6):
    """Forward by interval replay, backward (dsrc) against fp64 autograd, on a fused [B, S, 3 H HD] source whose v
    columns the backward must leave untouched.
    tables: "free" (every element its own cos / sin), "paired" (the model's tables) or None (no rotation).
    weights: False passes no RMSNorm weights.  strided_out: q / k written into [B, S + 2, H + 1, HD] buffers whose halo
    must stay zero.  loop_bwd: k at column H HD + 4 of a source padded to 3 H HD + 8 columns (8-byte aligned, not 16), which
    the flat HD-128 backward cannot read, so the warp-per-token kernel runs.  zero_rows: token 3 and the q of token S - 1
    are all zero."""
    D = H * HD
    k_off, C = (D + 4, 3 * D + 8) if loop_bwd else (D, 3 * D)
    src = _rand(B, S, C, seed=1)
    if zero_rows:
        src[:, min(3, S - 1)] = 0
        src[:, S - 1, :D] = 0
    wq, wk, wq1, wk1 = (_rand(HD, seed=10 + i, scale=0.2) + 1 for i in range(4)) if weights else (None,) * 4
    cos, sin = _rope_tables(S, HD, paired=tables == "paired") if tables else (None, None)
    q_out = k_out = None
    if strided_out:
        qfull, kfull = (torch.zeros(B, S + 2, H + 1, HD, dtype=torch.bfloat16, device=DEV) for _ in range(2))
        q_out, k_out = qfull[:, 1:S + 1, :H], kfull[:, 1:S + 1, :H]
    q, k = ops.qk_rmsnorm_rope_fwd(src, k_off, H, HD, wq, wk, wq1, wk1, s_split, cos, sin, eps, q_out=q_out, k_out=k_out)
    torch.cuda.synchronize()
    parts, n_fma, n_eager = [], 0, 0
    one, zero = torch.ones(1, device=DEV), torch.zeros(1, device=DEV)
    for nm, off, got, w_img, w_txt in (("q", 0, q, wq, wq1), ("k", k_off, k, wk, wk1)):
        xs = src[..., off:off + D].unflatten(-1, (H, HD))
        for part, sl, w in (("txt", slice(0, s_split), w_txt), ("img", slice(s_split, S), w_img)):
            if sl.start == sl.stop:
                continue
            ylo, yhi = rms_range(xs[:, sl], w, eps, HD // 32 + 5)
            c = cos[sl][None, :, None, :] if cos is not None else one
            s = sin[sl][None, :, None, :] if cos is not None else zero
            lo, hi = rope_range(ylo, yhi, c, s)
            parts.append(_in_range(f"fwd_{nm}_{part}", got[:, sl], lo, hi))
            nf, ne = _rope_fma_counts(got[:, sl], ylo, yhi, c, s)
            n_fma, n_eager = n_fma + nf, n_eager + ne
    extra = {"n_fma": n_fma, "n_eager": n_eager}
    if strided_out:
        halo = lambda f: bool((f[:, 0] == 0).all() and (f[:, S + 1] == 0).all() and (f[:, :, H] == 0).all())
        extra["halo_clean"] = halo(qfull) and halo(kfull)

    dq, dk = _rand(B, S, H, HD, seed=20), _rand(B, S, H, HD, seed=21)
    dsrc = torch.zeros_like(src)
    ops.qk_rmsnorm_rope_bwd(dq, dk, src, k_off, H, HD, wq, wk, wq1, wk1, s_split, cos, sin, eps, dsrc=dsrc)
    torch.cuda.synchronize()
    x64 = src.double().requires_grad_(True)
    c64, s64 = (cos.double(), sin.double()) if cos is not None else (None, None)
    total = 0.0
    mags = []
    for off, go, w_img, w_txt in ((0, dq, wq, wq1), (k_off, dk, wk, wk1)):
        xs = x64[..., off:off + D].unflatten(-1, (H, HD))
        ys, ms = [], []
        for sl, w in ((slice(0, s_split), w_txt), (slice(s_split, S), w_img)):
            w64 = w.double() if w is not None else None
            cs_ = (c64[sl], s64[sl]) if cos is not None else (None, None)
            ys.append(_rmsnorm_rope_ref(xs[:, sl], w64, *cs_, eps=_f32(eps)))
            ms.append(_qk_rope_mag(src[:, sl, off:off + D].unflatten(-1, (H, HD)), go[:, sl], w,
                                   *((cos[sl], sin[sl]) if cos is not None else (None, None)), eps)[0])
        total = total + (torch.cat(ys, 1) * go.double()).sum()
        mags.append(torch.cat(ms, 1).flatten(-2))
    total.backward()
    for nm, off, mag in (("q", 0, mags[0]), ("k", k_off, mags[1])):
        parts.append(_report_acc(f"bwd_{nm}", dsrc[..., off:off + D], x64.grad[..., off:off + D], mag, HD, GEMM_RTOL_BF16,
                                 c=ROW_C["qk_rmsnorm_rope_bwd"]))
    rest = torch.ones(C, dtype=torch.bool, device=DEV)
    rest[:D] = False
    rest[k_off:k_off + D] = False
    extra["v_untouched"] = bool((dsrc[..., rest] == 0).all().item())
    name = f"qk_rmsnorm_rope_B{B}_S{S}_H{H}_HD{HD}_split{s_split}_{tables}_w{int(weights)}" + \
        ("_strided" if strided_out else "") + ("_loop" if loop_bwd else "") + ("_zero" if zero_rows else "")
    return _combine(name, parts, **extra)


def check_qk_rmsnorm_dw(B=2, S=1255, H=24, HD=128, s_split=77, rope=True, eps=1e-6):
    """The RMSNorm weight gradients of qk_rmsnorm_rope_bwd (full fine-tune): dw [4, HD] = d/d(wq, wk, wq_added, wk_added),
    summed over B * S * H head rows by per-block shared-memory atomics and one global atomic per block.  Reference:
    fp64 autograd of the same forward on the same bf16 inputs; tolerance per element with K = the rows of that weight.
    rope: element-wise (not paired) tables, or none."""
    Cc = 3 * H * HD
    src = _rand(B, S, Cc, seed=1)
    ws = [_rand(HD, seed=10 + i, scale=0.2) + 1 for i in range(4)]   # wq, wk, wq_added, wk_added
    cos, sin = _rope_tables(S, HD, paired=False) if rope else (None, None)
    dq = _rand(B, S, H, HD, seed=20)
    dk = _rand(B, S, H, HD, seed=21)
    dw = torch.zeros(4, HD, dtype=torch.float32, device=DEV)
    ops.qk_rmsnorm_rope_bwd(dq, dk, src, H * HD, H, HD, *ws, s_split, cos, sin, eps, dsrc=torch.zeros_like(src), dw=dw)
    torch.cuda.synchronize()
    wd = [w.double().requires_grad_(True) for w in ws]
    c64, s64 = (cos.double(), sin.double()) if rope else (None, None)
    x = src.double()
    total = 0.0
    mag = torch.zeros(4, HD, dtype=torch.float64, device=DEV)
    for j, (off, g, w_img, w_txt) in enumerate(((0, dq, wd[0], wd[2]), (H * HD, dk, wd[1], wd[3]))):
        xs = x[..., off:off + H * HD].unflatten(-1, (H, HD))
        ys = []
        for i, sl, w in ((2 + j, slice(0, s_split), w_txt), (j, slice(s_split, S), w_img)):
            tab = (c64[sl], s64[sl]) if rope else (None, None)
            ys.append(_rmsnorm_rope_ref(xs[:, sl], w, *tab, eps=_f32(eps)))
            mag[i] = _qk_rope_mag(src[:, sl, off:off + H * HD].unflatten(-1, (H, HD)), g[:, sl], ws[i],
                                  *((cos[sl], sin[sl]) if rope else (None, None)), eps)[1].sum((0, 1, 2))
        total = total + (torch.cat(ys, 1) * g.double()).sum()
    total.backward()
    ref = torch.stack([w.grad for w in wd])
    rows = [B * (S - s_split) * H, B * (S - s_split) * H, B * s_split * H, B * s_split * H]
    parts = [_report_acc(f"dw{i}", dw[i], ref[i], mag[i], rows[i], GEMM_RTOL_F32, c=ROW_C["qk_rmsnorm_dw"])
             for i in range(4) if rows[i]]
    return _combine(f"qk_rmsnorm_dw_B{B}_S{S}_H{H}_HD{HD}_rope{int(rope)}", parts,
                    dw_rows_absmax=[round(float(v), 3) for v in ref.abs().amax(1)])


def check_rmsnorm(B=2, S=77, D=4096, eps=1e-6, strided=False, wscale=1.0):
    """T5LayerNorm out = bf16(w bf16(x rstd)) by interval replay.  Token 0 of every sample is all zero and must give 0.
    wscale: the weights are wscale (1 + 0.1 N(0, 1)).  strided: x and out are row / column windows of wider buffers,
    the halo of out must stay zero."""
    if strided:
        x = _rand(B, S + 3, D + 16, seed=1)[:, 2:S + 2, 8:8 + D]
        ofull = torch.zeros(B, S + 2, D + 24, dtype=torch.bfloat16, device=DEV)
        out = ofull[:, 1:S + 1, 16:16 + D]
    else:
        x, out = _rand(B, S, D, seed=1), None
    x[:, 0] = 0
    w = (wscale * (1 + 0.1 * _rand(D, seed=2).float())).bfloat16()
    got = ops.rmsnorm_fwd(x, w, eps, out=out)
    torch.cuda.synchronize()
    lo, hi = rms_range(x, w, eps, 8 * ((D + 255) // 256) + 5)
    parts = [_in_range("out", got, lo, hi), _bits("zero_rows", got[:, 0], torch.zeros_like(got[:, 0]))]
    extra = {}
    if strided:
        mask = torch.ones_like(ofull, dtype=torch.bool)
        mask[:, 1:S + 1, 16:16 + D] = False
        extra["halo_clean"] = bool((ofull[mask] == 0).all().item())
    return _combine(f"rmsnorm_B{B}_S{S}_D{D}_w{wscale:g}" + ("_strided" if strided else ""), parts, **extra)


# --------------------------------------------------------------------------------------------- loss kernels
HUBER_C = (0.05, 0.5, 2.0, 0.25)   # per-sample huber_c (a scheduled c differs per timestep)
MIN_SNR_W = (0.5, 1.0, 2.5, 0.75)


def unpack_nchw(p, layout, B, C, Hh, Ww):
    """The loss kernels' pred / dpred layout -> [B, C, Hh, Ww]: 0 Flux pack_latents (c, dy, dx) features, 1 SD3
    unpatchify (dy, dx, c), 2 NCHW."""
    if layout == 2:
        return p
    if layout == 0:
        return p.reshape(B, Hh // 2, Ww // 2, C, 2, 2).permute(0, 3, 1, 4, 2, 5).reshape(B, C, Hh, Ww)
    return p.reshape(B, Hh // 2, Ww // 2, 2, 2, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, Hh, Ww)


def _f32_inv(n, B):
    """The kernels' 1.f / float(n) / float(B)."""
    return torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(n)) / torch.tensor(float(B))


def loss_grad_replay(d, loss_type, c, w, inv, grad_scale):
    """dpred of pointwise_loss in fp32, in the kernel's order, rounded to bf16: bf16(((grad w) inv) grad_scale) with
    grad 2 d (l2) or k d / sqrt(d d + c c), k = 2 c (huber) or 2 (smooth_l1).  d, c, w fp32 on the CPU ([B, ...], [B]).
    Returns the candidates: one for l2; for the root, the sum rounded twice and d d + c c contracted either way."""
    if loss_type == "l2":
        grads = [2 * d]
    else:
        cb = c.view(-1, *([1] * (d.dim() - 1)))
        k = 2 * cb if loss_type == "huber" else torch.tensor(2.0)
        dd, cc = d * d, cb * cb
        sums = [dd + cc, (d.double() * d.double() + cc.double()).float(), (cb.double() * cb.double() + dd.double()).float()]
        grads = [(k * d) / torch.sqrt(s) for s in sums]
    gs = torch.tensor(grad_scale, dtype=torch.float32)
    if w is not None:
        grads = [g * w.view(-1, *([1] * (d.dim() - 1))) for g in grads]
    return [(g * inv * gs).bfloat16() for g in grads]


def loss_value64(d64, loss_type, c64):
    """fp64 pointwise loss of the reference conditional_loss."""
    if loss_type == "l2":
        return d64 * d64
    cb = c64.view(-1, *([1] * (d64.dim() - 1)))
    k = 2 * cb if loss_type == "huber" else 2.0
    return k * ((d64 * d64 + cb * cb).sqrt() - cb)


def loss_bound(d64, loss_type, c64, w64, n_per_thread):
    """Bound on |loss32 - loss64| of the loss kernels.  Each element's fp32 value is off by at most 3 u d^2 (l2: d, the
    square, the weight) or 5 u k r (root: c c, the FMA, sqrt, r - c, k (r - c), the weight), u = 2^-24.  The sum runs
    n_per_thread sequential adds per thread, 5 shuffle levels in the warp, 5 over the warp sums and 7 over the 8 CTAs:
    L = n_per_thread + 17 additions, each within u of its partial sum, which is at most sum |w l|; and two roundings of
    the final scale.  Hence inv (sum e + u L sum |w l|) + 2 u |loss|."""
    u = 2.0 ** -24
    B = d64.shape[0]
    wa = w64.abs().view(-1, *([1] * (d64.dim() - 1))) if w64 is not None else 1.0
    lv = loss_value64(d64, loss_type, c64) * (w64.view(-1, *([1] * (d64.dim() - 1))) if w64 is not None else 1.0)
    if loss_type == "l2":
        e = 3 * u * d64 * d64 * wa
    else:
        cb = c64.view(-1, *([1] * (d64.dim() - 1)))
        k = 2 * cb if loss_type == "huber" else 2.0
        e = 5 * u * k * (d64 * d64 + cb * cb).sqrt() * wa
    inv = 1.0 / d64[0].numel() / B
    loss = float(lv.sum() * inv)
    return inv * (float(e.sum()) + u * (n_per_thread + 17) * float(lv.abs().sum())) + 2 * u * abs(loss), loss


def _check_loss(name, loss, dpred, pred, tgt, layout, loss_type, huber_c, w, grad_scale, extra=None):
    """dpred bit for bit against loss_grad_replay and the loss against fp64 within loss_bound.  tgt: the target as the
    kernel forms it (bf16, NCHW)."""
    B, C, Hh, Ww = tgt.shape
    d = (unpack_nchw(pred, layout, B, C, Hh, Ww).float() - tgt.float()).cpu()
    cands = loss_grad_replay(d, loss_type, huber_c.cpu() if huber_c is not None else None,
                             w.cpu() if w is not None else None, _f32_inv(C * Hh * Ww, B), grad_scale)
    got = unpack_nchw(dpred, layout, B, C, Hh, Ww).cpu()
    parts, out = [], dict(extra or {})
    if len(cands) == 1:
        parts.append(_bits("dpred", got, cands[0]))
    else:
        hit = [got.view(torch.int16) == cd.view(torch.int16) for cd in cands]
        any_hit = hit[0] | hit[1] | hit[2]
        out["dpred_fma_or_two_roundings"] = bool(any_hit.all())
        out["n_fma"] = int(((hit[1] | hit[2]) & ~hit[0]).sum())
        out["n_twice"] = int((hit[0] & ~hit[1] & ~hit[2]).sum())
    d64 = (unpack_nchw(pred, layout, B, C, Hh, Ww).double() - tgt.double())
    n_per_thread = -(-d64.numel() // (8 * 1024))
    bound, ref = loss_bound(d64, loss_type, huber_c.double() if huber_c is not None else None,
                            w.double() if w is not None else None, n_per_thread)
    err = abs(float(loss.item()) - ref)
    out.update(loss=float(loss.item()), loss_ref=ref, loss_err=err, loss_tol_use=round(err / bound, 4))
    parts.append({"name": "loss", "ok": err <= bound, "tol_use": round(err / bound, 4)})
    return _combine(name, parts, **out)


def _huber(loss_type, B):
    return None if loss_type == "l2" else torch.tensor(HUBER_C[:B] + (0.5,) * max(0, B - 4), dtype=torch.float32, device=DEV)


def check_flow(B=2, Cc=16, Hh=32, Ww=48, layout=0, loss_type="l2", grad_scale=1.0):
    """flow_prep_pack bit for bit against the eager bf16 chain, then flow_mse_loss: dpred bit for bit, loss against fp64."""
    lat = _rand(B, Cc, Hh, Ww, seed=1)
    noise = _rand(B, Cc, Hh, Ww, seed=2)
    sig = torch.tensor([0.25, 0.8125][:B] + [0.5] * max(0, B - 2), dtype=torch.float32, device=DEV)
    noisy, packed = ops.flow_prep_pack(lat, noise, sig)
    torch.cuda.synchronize()
    # eager bf16 chain exactly as the reference writes it (common.py:4953-4960, 4989-4991)
    grid = sig.view(B, 1, 1, 1).to(torch.bfloat16)
    ref_noisy = (1.0 - grid) * lat + grid * noise
    ref_packed = ref_noisy.view(B, Cc, Hh // 2, 2, Ww // 2, 2).permute(0, 2, 4, 1, 3, 5).reshape(B, (Hh // 2) * (Ww // 2), Cc * 4)
    extra = {"bit_exact_noisy": bool(torch.equal(noisy, ref_noisy)), "bit_exact_packed": bool(torch.equal(packed, ref_packed))}
    pred = _rand(B, Cc, Hh, Ww, seed=3) if layout == 2 else _rand(B, (Hh // 2) * (Ww // 2), Cc * 4, seed=3)
    hc = _huber(loss_type, B)
    loss, dpred = ops.flow_mse_loss(pred, lat, noise, grad_scale=grad_scale, layout=layout, loss_type=loss_type, huber_c=hc)
    torch.cuda.synchronize()
    return _check_loss(f"flow_prep_loss_{loss_type}_layout{layout}_gs{grad_scale:g}", loss, dpred, pred, noise - lat, layout,
                       loss_type, hc, None, grad_scale, extra)


def check_skinny(B=2, S=300, R=16, N=3072, exact=False, accumulate=False, alpha=0.5, view=False):
    """out[r, n] += alpha sum_m L[m, r] Rm[m, n] (fp32), per-split slabs added in index order.  accumulate: out starts
    non-zero (N(0, 1), or integers x 2^-4 with exact inputs, so that every partial sum stays exact).  A non-power-of-two
    alpha (with exact inputs) accepts alpha acc + out rounded once (FMA) or twice.  view: L and Rm are token and column
    windows of wider buffers, as _lora_grads passes one member's rank slice of a fused rank block and its column range of
    the fused output; the values around the windows must not reach out."""
    if view:
        L = _gen(B, S + 3, R + 24, seed=1, exact="int" if exact else None)[:, 2:S + 2, 8:8 + R]
        Rm = _gen(B, S + 5, N + 40, seed=2, exact="frac" if exact else None)[:, 3:S + 3, 16:16 + N]
    else:
        L = _gen(B, S, R, seed=1, exact="int" if exact else None)
        Rm = _gen(B, S, N, seed=2, exact="frac" if exact else None)
    out0 = None
    if accumulate:
        g = torch.Generator(device="cpu").manual_seed(3)
        out0 = (torch.randint(-64, 65, (R, N), generator=g).float() / 16 if exact else torch.randn(R, N, generator=g)).to(DEV)
    out = ops.skinny_tn(L, Rm, alpha=alpha, out=out0.clone() if accumulate else None)
    torch.cuda.synchronize()
    L2, R2 = L.double().reshape(-1, R), Rm.double().reshape(-1, N)
    acc64, mag = L2.t() @ R2, L2.abs().t() @ R2.abs()
    a32 = _f32(alpha)
    base = out0.double() if accumulate else torch.zeros_like(acc64)
    name = f"skinny_tn_B{B}_S{S}_R{R}_N{N}" + ("_view" if view else "") + ("_accum" if accumulate else "") + ("_exact" if exact else "")
    if not exact:
        r = _report_acc("out", out, base + a32 * acc64, abs(a32) * mag + base.abs(), B * S, GEMM_RTOL_F32)
        return _combine(name, [r])
    bound = exact_bound_ok([L], [Rm], mag)
    if _is_pow2(a32):
        return _combine(name, [_bits("out", out, (base + a32 * acc64).float())], exact_bound=bound)
    once, twice = (base + a32 * acc64).float(), base.float() + a32 * acc64.float()
    either = ((out == once) | (out == twice)).all().item()
    return _combine(name, [], exact_bound=bound, fma_or_two_roundings=bool(either),
                    n_fma=int((out == once).sum().item()), n_twice=int((out == twice).sum().item()))


def check_skinny_repeatable(B=4, S=4608, R=48, N=9216):
    """The LoRA weight gradient is bit-identical from run to run."""
    L = _rand(B, S, R, seed=1)
    Rm = _rand(B, S, N, seed=2)
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
def check_conv3x3(B=2, H=24, W=40, Ci=64, Co=128, stride=1, bias=True, res=False, exact=False):
    """Implicit-GEMM 3x3 conv (K = 9 Ci): the fp64 conv of the same bf16 inputs; exact: bf16((acc + bias) + res)."""
    import torch.nn.functional as F
    x = _gen(B, H, W, Ci, seed=1, exact="int" if exact else None)
    w = _gen(Co, Ci, 3, 3, scale=(9 * Ci) ** -0.5, seed=2, exact="frac" if exact else None)
    bv = _rand(Co, scale=0.1, seed=3) if bias else None
    Ho, Wo = (H, W) if stride == 1 else (H // 2, W // 2)
    rv = _rand(B, Ho, Wo, Co, seed=4) if res else None
    w9 = w.permute(0, 2, 3, 1).reshape(Co, -1).contiguous()
    out = ops.conv3x3_nhwc(x, w9, bv, rv, stride)
    torch.cuda.synchronize()

    def conv(xt, wt):
        xn = xt.double().permute(0, 3, 1, 2)
        if stride == 1:
            return F.conv2d(xn, wt.double(), padding=1).permute(0, 2, 3, 1)
        return F.conv2d(F.pad(xn, (0, 1, 0, 1)), wt.double(), stride=2).permute(0, 2, 3, 1)

    acc64, mag = conv(x, w), conv(x.abs(), w.abs())
    name = f"conv3x3_s{stride}_{Ci}to{Co}_{H}x{W}" + ("_exact" if exact else "")
    if exact:
        f = acc64.float() + (bv.float() if bias else 0.0)
        want = (f + rv.float() if res else f).bfloat16()
        return _combine(name, [_bits("out", out, want)], exact_bound=exact_bound_ok([x], [w], mag))
    ref = acc64 + (bv.double() if bias else 0.0) + (rv.double() if res else 0.0)
    return _combine(name, [_report_acc("out", out, ref, mag, 9 * Ci, GEMM_RTOL_BF16)])


def check_conv_in(B=2, H=20, W=36, C=128, exact=False):
    """RGB stem conv (K = 27).  C = 64 / 128 / 256: the tensor-core kernel, bf16(acc + bias); other C: the CUDA-core
    kernel, which starts from the bias and adds the 27 taps in (channel, dy, dx) order, replayed as such when exact."""
    import torch.nn.functional as F
    x = _gen(B, 3, H, W, seed=1, exact="int" if exact else None)
    w = _gen(C, 3, 3, 3, scale=27 ** -0.5, seed=2, exact="frac" if exact else None)
    bv = _rand(C, scale=0.1, seed=3)
    out = ops.conv_in_3ch(x, w, bv)
    torch.cuda.synchronize()
    acc64 = F.conv2d(x.double(), w.double(), padding=1).permute(0, 2, 3, 1)
    mag = F.conv2d(x.double().abs(), w.double().abs(), padding=1).permute(0, 2, 3, 1)
    name = f"conv_in_3ch_C{C}_{H}x{W}" + ("_exact" if exact else "")
    if not exact:
        return _combine(name, [_report_acc("out", out, acc64 + bv.double(), mag, 27, GEMM_RTOL_BF16)])
    if C in (64, 128, 256):
        want = (acc64.float() + bv.float()).bfloat16()
    else:
        xp = F.pad(x.float(), (1, 1, 1, 1))
        acc = bv.float().expand(B, H, W, C).clone()
        for c in range(3):
            for dy in range(3):
                for dx in range(3):
                    acc = acc + xp[:, c, dy:dy + H, dx:dx + W, None] * w.float()[:, c, dy, dx]
        want = acc.bfloat16()
    return _combine(name, [_bits("out", out, want)], exact_bound=exact_bound_ok([x], [w], mag))


# --------------------------------------------------------------------------------------------- VAE-encode reference model
# GroupNorm, the mid-block row softmax and the latent sampling are compared with fp64 references on the kernels' own bf16
# inputs, element by element, with every bound derived below.  u = 2^-24 (half an fp32 ulp, relative).
#
# GroupNorm (stb_groupnorm_nhwc): interval replay.  The stats kernel sums t = x - p and t^2 around a pivot p per (image,
# group), the group's first channel at pixel 0 (gn_pivot).  Every term passes through at most L fp32 additions
# (gn_chains: the thread's own pixels, the 8-lane vector sum when cpg >= 8, the CTA's shared atomics, the image's global
# atomics, from the chunking of api.cu), so with d = mean - p, E2 = mean t^2 = var + d^2 and A1 = mean |t|:
#     |d32 - d| <= e_d = (L + 1) u A1 + 2 u |d|                   (+1: t itself rounds when x and p are far apart)
#     |var32 - var| <= e_v = (L + 7) u E2 + 2 |d| e_d + e_d^2     (t^2, / n, d d, the subtraction)
# rstd = rsqrtf(var32 + eps) (2 ulp = 4 u, + u for the sum) lies in [rsqrt(var + eps + e_v), rsqrt(var - e_v + eps)]
# widened by 5 u: rel_r; a = rstd gamma adds u.  mean32 = p + d32 is within e_d + u |mean|, and the output
# y = x a + (beta - mean32 a) is one FMA after one rounding of b, so
#     |y32 - y| <= |x - mean| |a| rel_a + (e_d + u |mean|) |a| (1 + rel_a) + u (|beta| + |mean a|) + u |y|
# and bf16(y32) lies in [bf16(y - err), bf16(y + err)] (_bf16_range): one value almost everywhere.  The bound has no
# (mean / sigma)^2 term: E2 holds (mean - p)^2, a few sigma^2 for a group whose first element is a typical member.
# Without SiLU that range is the check.  With SiLU the kernel rounds y to bf16 (the GroupNorm module's output) and
# evaluates __fdividef(v, 1 + __expf(-v)): the output must be a bf16 neighbour of fp64 silu(v) for v one of the two
# ends of the range.  One deliberate absolute floor: once 1 + __expf(-v) passes 2^126 (v < about -87) __fdividef
# returns 0, which is accepted only where |silu(v)| < 2^-120.  A constant group (sigma = 0) has t = 0 exactly, so
# var = 0 and rstd = 1 / sqrt(eps); its output is beta up to the u |mean a| of the FMA form.  tol_use: the worst |got - y| / (err + half a bf16 ulp of y).
#
# Row softmax (stb_softmax_rows): out_i = __expf((s_i - m) scale) / sum.  z = (s - m) scale rounds twice (2 u |z|
# absolute in the exponent), and __expf is within 2 + floor(1.173 |z|) fp32 ulps (CUDA programming guide), so every term
# is within delta_i = 2^-23 (2 + 2.173 |z_i|) relative; the sum adds L u (8 terms per 2048-column sweep, 5 shuffle levels,
# 7 adds over the warps) plus the terms' own errors, weighted; 1 / sum and the product add 2 u.  The output must lie in
# the bf16 range of p_i (1 +- rel_i).  ex2.approx.ftz flushes terms below 2^-126, so where p_i < 2^-126 any output in
# [0, 2^-126] is accepted.  A uniform row must give bf16(fp32(1 / cols)) bit for bit.
#
# Latent sampling (stb_gaussian_sample_scale): std = bf16(__expf(0.5 clamp(logvar, -30, 20))) lies in the bf16 range of
# exp(x) (1 +- (2 + floor(1.173 |x|)) 2^-23): one value almost everywhere, two near a rounding midpoint.  The eager
# bf16 chain of diffusers' DiagonalGaussianDistribution.sample and the latent scaling, bf16(mean + bf16(std eps)) then
# bf16(bf16(z - shift) scale) (no shift: bf16(z scale)), is replayed on each candidate; the output must equal one.
U24 = 2.0 ** -24


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if DEV == "cuda" else 132


def gn_chains(B, HW, C, G, sms=132):
    """Longest chain of fp32 additions a term of one group's sums passes through in stb_groupnorm_nhwc's stats kernel,
    from the chunking of api.cu: the thread's pixels, the 8-lane vector sum (cpg >= 8), the CTA's shared-memory atomics
    into the group and the global atomics of the image's CTAs."""
    chunks = max(1, min((HW + 255) // 256, (sms * 4 + B - 1) // B))
    ppc = -(-HW // chunks)
    ctas = -(-HW // ppc)
    rows_par = 256 // (C // 8)
    cpg = C // G
    shared = rows_par * (cpg if cpg < 8 else cpg // 8)
    return -(-ppc // rows_par) + (7 if cpg >= 8 else 0) + shared + ctas


def gn_pivot(x, G):
    """The kernel's pivot per (image, group) of x [B, HW, C]: the group's first channel at pixel 0; [B, G] fp64."""
    return x[:, 0, ::x.shape[-1] // G].double()


def gn_reference(x, gamma, beta, G, eps, L=None, pivot=None):
    """(y, err) [B, HW, C] fp64: the GroupNorm value and the bound on the kernel's fp32 error (see above) for x
    [B, HW, C] bf16.  L: the addition chain length (gn_chains); pivot: [B, G] (gn_pivot)."""
    B, HW, C = x.shape
    cpg = C // G
    u = U24
    if L is None:
        L = gn_chains(B, HW, C, G, _sms())
    x64 = x.double().view(B, HW, G, cpg)
    p = (gn_pivot(x, G) if pivot is None else pivot.double())[:, None, :, None]
    t = x64 - p
    d = t.mean((1, 3), keepdim=True)
    E2 = t.pow(2).mean((1, 3), keepdim=True)
    A1 = t.abs().mean((1, 3), keepdim=True)
    xc = t - d                                            # x - mean
    var = xc.pow(2).mean((1, 3), keepdim=True)            # two-pass
    e_d = (L + 1) * u * A1 + 2 * u * d.abs()
    e_v = (L + 7) * u * E2 + 2 * d.abs() * e_d + e_d * e_d
    e32 = _f32(eps)
    r = (var + e32).rsqrt()
    r_lo = (var + e32 + e_v).rsqrt() * (1 - 5 * u)
    r_hi = ((var - e_v).clamp_min(0) + e32).rsqrt() * (1 + 5 * u)
    rel_a = torch.maximum(1 - r_lo / r, r_hi / r - 1) + u
    a = r * gamma.double().view(1, 1, G, cpg)
    b64 = beta.double().view(1, 1, G, cpg)
    y = xc * a + b64
    mean = (p + d).abs()
    err = (xc.abs() * a.abs() * rel_a + (e_d + u * mean) * a.abs() * (1 + rel_a) + u * (b64.abs() + (mean * a).abs())
           + u * y.abs())
    return y.view(B, HW, C), err.view(B, HW, C)


def _half_ulp(y):
    """Half a bf16 ulp at |y| (fp64)."""
    e = torch.frexp(y.abs())[1]
    return torch.where(y == 0, torch.zeros_like(y), torch.ldexp(torch.ones_like(y), e - 9))


def _range_use(got, y, err, where=None):
    """The largest share of the fp32 error bound err an element needs: (|got - y| - half a bf16 ulp of y)+ / err; above
    1 the element lies outside its range (up to the ulp at a power of two)."""
    use = ((got.double() - y).abs() - _half_ulp(y)).clamp_min(0) / (err + 1e-300)
    if where is not None:
        use = use[where]
    return round(float(use.max().item()), 4) if use.numel() else 0.0


def silu64(v):
    return v * torch.sigmoid(v)


SILU_ARGMIN = -1.2784645427610738      # silu is decreasing below, increasing above


def silu_check(name, got, lo, hi):
    """got (bf16) is a bf16 neighbour of fp64 silu(v) for some v in [lo, hi] (the GroupNorm output's range; near 0 it
    holds several bf16 values): its two neighbours bracket a point of silu([lo, hi]).  Or 0 where |silu(v)| < 2^-120
    (the __fdividef floor)."""
    dn, up = _bf16_steps(got)
    sl, sh = silu64(lo.double()), silu64(hi.double())
    smin = torch.where((lo.double() <= SILU_ARGMIN) & (SILU_ARGMIN <= hi.double()),
                       torch.full_like(sl, silu64(torch.tensor(SILU_ARGMIN, dtype=torch.float64)).item()), torch.minimum(sl, sh))
    smax = torch.maximum(sl, sh)
    ok = (dn <= smax) & (up >= smin)
    ok |= (got == 0) & (torch.minimum(sl.abs(), sh.abs()) < 2.0 ** -120)
    bad = ~(ok & torch.isfinite(got))
    n = int(bad.sum().item())
    out = {"name": name, "ok": n == 0, "n_bad": n, "numel": got.numel()}
    if n:
        _first(bad, got.float(), silu64(lo.double()), out)
    return out


def _gn_input(B, HW, C, G, ratio, const=False, seed=1):
    """x [B, HW, C] bf16.  Group (b, g), k = b G + g, is N(mu, s^2) with its own s = 2^(k % 5 - 2) and
    mu = (-1)^k ratio s (1 + (7 k % 16) / 64): mean / sigma between ratio and 1.23 ratio, different for every group
    and image, so a wrong group index or image offset moves the statistics.  const: every third group is the constant
    0.3 (1 + k / 8), sigma = 0."""
    cpg = C // G
    gen = torch.Generator().manual_seed(seed)
    k = torch.arange(B * G, dtype=torch.float64).view(B, G)
    s = torch.pow(2.0, (k % 5) - 2)
    mu = torch.where(k % 2 == 0, 1.0, -1.0) * ratio * s * (1 + ((7 * k) % 16) / 64)
    x = torch.randn(B, HW, G, cpg, generator=gen, dtype=torch.float32) * s[:, None, :, None].float() + \
        mu[:, None, :, None].float()
    if const:
        cm = (k % 3 == 0)[:, None, :, None].expand_as(x)
        x = torch.where(cm, (0.3 * (1 + k / 8))[:, None, :, None].float().expand_as(x), x)
    return x.reshape(B, HW, C).to(torch.bfloat16).to(DEV)


def check_groupnorm(B=2, H=16, W=24, C=128, G=32, silu=True, ratio=0.0, const=False, beta0=False, control=False):
    """stb_groupnorm_nhwc by interval replay (above).  ratio: mean / sigma of the groups (_gn_input); const: every
    third group constant; beta0: beta = 0.
    control: also run torch's F.group_norm on the same bf16 input on the device and report its tol_use under the same
    bound (information: torch is not held to this kernel's bound)."""
    import torch.nn.functional as F
    HW = H * W
    x = _gn_input(B, HW, C, G, ratio, const).view(B, H, W, C)
    gm = (1.0 + 0.1 * _rand(C, seed=2).float()).bfloat16()
    bt = torch.zeros(C, dtype=torch.bfloat16, device=DEV) if beta0 else _rand(C, scale=0.1, seed=3)
    out = ops.groupnorm_nhwc(x, gm, bt, G, 1e-6, silu)
    torch.cuda.synchronize()
    x3 = x.view(B, HW, C)
    y, err = gn_reference(x3, gm, bt, G, 1e-6)
    lo, hi = _bf16_range(y, err)
    got = out.view(B, HW, C)
    extra = {"gn_frac_exact": round(float((lo == hi).double().mean().item()), 4), "chain_L": gn_chains(B, HW, C, G, _sms())}
    if silu:
        parts = [silu_check("out", got, lo, hi)]
    else:
        parts = [_in_range("out", got, lo, hi)]
        parts[0]["tol_use"] = _range_use(got, y, err)
    if control:
        ref = F.group_norm(x.permute(0, 3, 1, 2), G, gm, bt, 1e-6).permute(0, 2, 3, 1).reshape(B, HW, C)
        extra["torch_tol_use"] = _range_use(ref, y, err)
        if not silu:
            extra["kernel_tol_use"] = parts[0]["tol_use"]
    name = f"groupnorm_B{B}_HW{HW}_C{C}_G{G}_silu{int(silu)}_r{ratio:g}" + ("_const" if const else "") + \
        ("_beta0" if beta0 else "")
    return _combine(name, parts, **extra)


def softmax_range(s, scale):
    """(lo, hi) bf16 range of softmax(f32(scale) s) per element of s [rows, cols] (bf16) under the kernel's error bound,
    with the flush-to-zero floor: where p < 2^-126, lo = 0 and hi >= 2^-126."""
    rows, cols = s.shape
    s64 = s.double()
    z = (s64 - s64.amax(-1, keepdim=True)) * _f32(scale)
    e = z.exp()
    p = e / e.sum(-1, keepdim=True)
    delta = 2.0 ** -23 * (2 + 2.173 * z.abs())
    L = 8 * -(-cols // 2048) + 5 + 7
    rel = delta + L * U24 + (e * delta).sum(-1, keepdim=True) / e.sum(-1, keepdim=True) + 3 * U24
    lo, hi = _bf16_range(p, rel * p)
    tiny = p < 2.0 ** -126
    lo = torch.where(tiny, torch.zeros_like(lo), lo)
    hi = torch.where(tiny, torch.maximum(hi, torch.full_like(hi, 2.0 ** -126)), hi)
    return lo, hi, p, rel * p


def _softmax_rows_input(rows, cols, scale, sigma, seed=1):
    """bf16 scores [rows, cols] (unscaled).  Row 0 uniform (3.0), row 1 peaked (one logit, at column 2 cols / 3, 40
    above N(0, 1) scaled logits), row 2 wide (N(0, 25^2) scaled logits, some flushed to zero), row 3 a ramp of scaled
    logits from -120 up to 0 at the last column (the row max lies far from the first columns); the rest N(0, sigma^2)."""
    gen = torch.Generator().manual_seed(seed)
    s = torch.randn(rows, cols, generator=gen) * sigma
    if rows >= 4:
        s[0] = 3.0
        s[1] = torch.randn(cols, generator=gen) / scale
        s[1, (2 * cols) // 3] = (float(s[1].max()) * scale + 40.0) / scale
        s[2] = torch.randn(cols, generator=gen) * 25.0 / scale
        s[3] = torch.linspace(-120.0, 0.0, cols) / scale
    return s.to(torch.bfloat16).to(DEV)


def check_softmax_rows(rows=300, cols=1024, scale=0.0442, sigma=20.0):
    """In-place row softmax against fp64 softmax(f32(scale) s) by the bound above; row 0 (uniform) bit for bit."""
    s = _softmax_rows_input(rows, cols, scale, sigma)
    s0 = s.clone()
    ops.softmax_rows_(s, scale)
    torch.cuda.synchronize()
    lo, hi, p, err = softmax_range(s0, scale)
    parts = [_in_range("out", s, lo, hi)]
    parts[0]["tol_use"] = _range_use(s, p, err, where=p >= 2.0 ** -126)
    if rows >= 4:
        parts.append(_bits("uniform_row", s[0], torch.full_like(s[0], 1.0 / cols, dtype=torch.float32).bfloat16()))
    return _combine(f"softmax_rows_{rows}x{cols}_scale{scale:g}", parts, flushed=int((p < 2.0 ** -126).sum().item()))


LOGVAR_EDGES = (-40.0, -30.0, -29.875, 19.875, 20.0, 25.0)


def gaussian_std_range(logvar):
    """bf16 range of the kernel's std = bf16(__expf(0.5 clamp(logvar, -30, 20))) (logvar bf16)."""
    x = 0.5 * logvar.double().clamp(-30.0, 20.0)
    e = x.exp()
    return _bf16_range(e, e * 2.0 ** -23 * (2 + torch.floor(1.173 * x.abs())))


def gaussian_replay(mean, std, eps, shift, scale):
    """The eager bf16 chain on a bf16 std: bf16(mean + bf16(std eps)), then bf16(bf16(z - shift) scale) (no shift:
    bf16(z scale)), fp32 arithmetic rounded after every op as torch's bf16 tensor ops do."""
    z = (mean.float() + (std.float() * eps.float()).bfloat16().float()).bfloat16()
    if shift is None:
        return (z.float() * _f32(scale)).bfloat16()
    return ((z.float() - _f32(shift)).bfloat16().float() * _f32(scale)).bfloat16()


def _gaussian_input(B, L, h, w, seed=1):
    """moments NHWC [B, h, w, 2L], eps NCHW [B, L, h, w]: logvar N(0, 1) with LOGVAR_EDGES at (pixel + channel) % 8 < 6,
    so the clamp is reached from both sides and at its ends."""
    m = _rand(B, h, w, 2 * L, seed=seed)
    pix = torch.arange(h * w, device=DEV).view(h, w, 1)
    sel = (pix + torch.arange(L, device=DEV).view(1, 1, L)) % 8
    lv = m[..., L:]
    for i, v in enumerate(LOGVAR_EDGES):
        lv[:, sel == i] = v
    return m, _rand(B, L, h, w, seed=seed + 1)


def check_gaussian_sample(B=2, L=16, h=12, w=20, shift=0.1159, scale=0.3611):
    """Interval replay of the latent sample (above); shift None: no shift (SDXL, sample())."""
    m, eps = _gaussian_input(B, L, h, w)
    out = ops.gaussian_sample_scale(m, eps, shift, scale)
    torch.cuda.synchronize()
    mn = m.permute(0, 3, 1, 2)
    mean, logvar = mn[:, :L], mn[:, L:]
    s_lo, s_hi = gaussian_std_range(logvar)
    r_lo, r_hi = gaussian_replay(mean, s_lo, eps, shift, scale), gaussian_replay(mean, s_hi, eps, shift, scale)
    iv = torch.int16
    hit = (out.view(iv) == r_lo.view(iv)) | (out.view(iv) == r_hi.view(iv))
    n = int((~hit).sum().item())
    part = {"name": "out", "ok": n == 0, "n_bad": n, "numel": out.numel()}
    if n:
        _first(~hit, out.float(), r_lo.float(), part)
    return _combine(f"gaussian_sample_B{B}_L{L}_{h}x{w}_shift{shift}_scale{scale:g}", [part],
                    n_two_std=int((s_lo != s_hi).sum().item()), n_two_out=int((r_lo != r_hi).sum().item()))


# --------------------------------------------------------------------------------------------- LoKr and LoRA dropout reference model
# LoKr rebuild: out = bf16(fmaf(f32(scale w1[i, k']), w2[j, l], W)).  f32(scale w1) has 24 significant bits and w2 8,
# so the product is exact in fp64; adding the bf16 W rounds at most once in fp64, and lokr_single_rounding asserts from
# the drawn values that the fp32 rounding of that sum is the exact sum's (the fp64 sum is exact, or it is not an fp32
# rounding midpoint): fp64 -> fp32 -> bf16 then reproduces the kernel's single fp32 rounding and the bf16 store bit for
# bit.  out_t must be out transposed, bit for bit.  n_vs_eager counts the elements
# where this differs from lycoris's own fp32 chain bf16(W + kron(w1, w2) scale) (information).
# LoKr factor gradients: d w1 = scale sum_{j,l} dW w2 (K = b d terms) and d w2 = scale sum_{i,k'} dW w1 (K = a c terms)
# against fp64 with tol = 2^-23 |ref| + LOKR_C 2^-24 sqrt(K) M_ij, M the magnitude sum.  d w2 is one sequential fp32
# FMA chain per element, whose error is typically about 0.5 u M; d w1 a tree of 8-term FMA chains, shuffles and atomics.
# LOKR_C = 1: on an H100 80GB HBM3 (700 W limit) the largest c_half was 0.91 (d w1 at the Flux ff shape, K = 2.4M) and
# the largest tol_use 0.47.  Exact inputs (dW integers in [-2, 2], w1 / w2 integers in [-6, 6] x 2^-4, a power-of-two scale): every
# partial sum is a multiple of 2^-8 below 2^19, so both outputs match fp64 bit for bit in any atomic order.
# LoRA dropout: the mask is replayed in numpy uint32 (dropout_keep_np: mix32 / dropout_keep of elementwise.cuh and the
# llround(p 2^24) threshold of api.cu); expand must be bf16(x f32(1 / (1 - p))) where kept, 0 elsewhere, bit for bit;
# accum is replayed in member order in fp32, each kept term added with an FMA or rounded twice: either is accepted per
# element and counted.
LOKR_C = 1.0


def lokr_single_rounding(prod, W):
    """fp64 prod + W, rounded to fp32, is the exact sum rounded once: the fp64 sum is exact (its TwoSum error is 0) or
    it is not an fp32 rounding midpoint (only there could rounding twice differ)."""
    s = prod + W
    bb = s - prod
    err = (prod - (s - bb)) + (W - bb)
    f = s.float()
    g = torch.nextafter(f, torch.where(s > f.double(), torch.full_like(f, math.inf), torch.full_like(f, -math.inf)))
    mid = (f.double() + g.double()) * 0.5 == s
    return bool(((err == 0) | ~mid).all().item())


def lokr_rebuild_replay(W, w1, w2, scale):
    """(bf16 out, single): the kernel's fmaf(f32(scale w1), w2, W) rounded to fp32 then bf16, from the fp64 sum."""
    s1 = (w1.float() * _f32(scale)).double()
    prod = torch.kron(s1, w2.double())
    return (prod + W.double()).float().bfloat16(), lokr_single_rounding(prod, W.double())


def lokr_eager(W, w1, w2, scale):
    """lycoris.py's host chain: bf16(W + kron(w1, w2) scale) in fp32."""
    return (W.float() + torch.kron(w1.float(), w2.float()) * scale).bfloat16()


def check_lokr_rebuild(a=8, b=48, c=4, d=40, scale=0.5, fused=True, pad=0):
    """stb_lokr_rebuild bit for bit (above).  fused: out / out_t are the middle slices of [3 N, K] / [K, 3 N] buffers
    whose other slices must stay zero.  pad: W, out and out_t rows are padded by `pad` elements (row strides that are
    not multiples of 8 take the scalar paths); the padding must stay zero."""
    N, K = a * b, c * d
    W = (_rand(N, K + pad, seed=61) * 0.05)[:, :K]
    w1, w2 = _rand(a, c, seed=62), _rand(b, d, seed=63) * 0.05
    big = torch.zeros(3 * N if fused else N, K + pad, device=DEV, dtype=torch.bfloat16)
    big_t = torch.zeros(K, 3 * N + pad if fused else N + pad, device=DEV, dtype=torch.bfloat16)
    n0 = N if fused else 0
    out, out_t = big[n0:n0 + N, :K], big_t[:, n0:n0 + N]
    ops.lokr_rebuild(W, w1, w2, scale, out, out_t)
    torch.cuda.synchronize()
    want, fits = lokr_rebuild_replay(W, w1, w2, scale)
    parts = [_bits("out", out, want), _bits("out_t", out_t, want.t())]
    mask, mask_t = torch.ones_like(big, dtype=torch.bool), torch.ones_like(big_t, dtype=torch.bool)
    mask[n0:n0 + N, :K] = False
    mask_t[:, n0:n0 + N] = False
    clean = bool((big[mask] == 0).all().item()) and bool((big_t[mask_t] == 0).all().item())
    n_eager = int((want.view(torch.int16) != lokr_eager(W, w1, w2, scale).view(torch.int16)).sum().item())
    return _combine(f"lokr_rebuild_{a}x{b}_{c}x{d}_s{scale:.4g}" + (f"_pad{pad}" if pad else ""), parts, single_rounding=fits,
                    halo_clean=clean, n_vs_eager=n_eager)


def check_lokr_factor_grads(a=8, b=48, c=4, d=40, scale=0.5, strided=True, exact=False):
    """stb_lokr_factor_grads against fp64 (tolerance above) or, exact, bit for bit; d w2 (no atomics) must be
    bit-identical on a second run.  strided: dW is a window of a wider buffer."""
    N, K = a * b, c * d
    ea, ew = ("int", "frac") if exact else (None, None)
    w1, w2 = _gen(a, c, seed=64, exact=ew), _gen(b, d, seed=65, exact=ew)
    g_full = _gen(N + 8, K + 16, seed=66, exact=ea)
    dW = g_full[4:4 + N, 8:8 + K] if strided else g_full[:N, :K].contiguous()
    g4 = dW.double().reshape(a, b, c, d)
    r1, m1 = torch.einsum("ajcl,jl->ac", g4, w2.double()), torch.einsum("ajcl,jl->ac", g4.abs(), w2.double().abs())
    r2, m2 = torch.einsum("ajcl,ac->jl", g4, w1.double()), torch.einsum("ajcl,ac->jl", g4.abs(), w1.double().abs())
    d1, d2 = ops.lokr_factor_grads(dW, w1, w2, scale)
    d2_again = ops.lokr_factor_grads(dW, w1, w2, scale)[1]
    torch.cuda.synchronize()
    s = _f32(scale)
    extra = {"dw2_repeatable": bool(torch.equal(d2, d2_again))}
    if exact:
        assert _is_pow2(s)
        extra["exact_bound"] = exact_bound_ok([dW], [w1, w2], torch.cat([m1.flatten(), m2.flatten()]))
        parts = [_bits("dw1", d1, (s * r1).float()), _bits("dw2", d2, (s * r2).float())]
    else:
        parts = [_report_acc("dw1", d1, s * r1, abs(s) * m1, b * d, GEMM_RTOL_F32, c=LOKR_C),
                 _report_acc("dw2", d2, s * r2, abs(s) * m2, a * c, GEMM_RTOL_F32, c=LOKR_C)]
    return _combine(f"lokr_factor_grads_{a}x{b}_{c}x{d}_s{scale:g}" + ("_strided" if strided else "") +
                    ("_exact" if exact else ""), parts, **extra)


def mix32_np(h):
    """elementwise.cuh mix32 (murmur3 finaliser) on a numpy uint32 array."""
    import numpy as np
    h = h ^ (h >> np.uint32(16))
    h = h * np.uint32(0x85EBCA6B)
    h = h ^ (h >> np.uint32(13))
    h = h * np.uint32(0xC2B2AE35)
    return h ^ (h >> np.uint32(16))


def dropout_thresh(p):
    """api.cu's llround(double(float(p)) * 2^24)."""
    return int(math.floor(_f32(p) * 16777216.0 + 0.5))


def dropout_keep_np(seed, stream, idx, p):
    """dropout_keep(seed, stream, idx, thresh) for a numpy uint64 array of logical element indices."""
    import numpy as np
    lo, hi = (idx & np.uint64(0xFFFFFFFF)).astype(np.uint32), (idx >> np.uint64(32)).astype(np.uint32)
    inner = mix32_np(hi + np.uint32((stream * 0x85EBCA77 + seed) & 0xFFFFFFFF))
    h = mix32_np(lo * np.uint32(0x9E3779B1) + inner)
    return (h >> np.uint32(8)) >= np.uint32(dropout_thresh(p))


def dropout_masks(members, B, S, K, p, seed, stream0):
    """Bool [members, B, S, K] on DEV: the keep mask of member m is stream stream0 + m over the logical [B, S, K] index."""
    import numpy as np
    idx = np.arange(B * S * K, dtype=np.uint64)
    return torch.from_numpy(np.stack([dropout_keep_np(seed, (stream0 + m) & 0xFFFFFFFF, idx, p)
                                      for m in range(members)])).view(members, B, S, K).to(DEV)


def dropout_inv_keep(p):
    """api.cu's 1.f / (1.f - p) in fp32."""
    one = torch.tensor(1.0, dtype=torch.float32)
    return one / (one - torch.tensor(p, dtype=torch.float32))


def dropout_accum_replay(dx0, d, keep, inv):
    """(fma, twice): dx0 + sum_m keep_m d_m inv in member order in fp32, each kept term added by one FMA (the bf16 x fp32
    product is exact in fp64) or rounded twice; bf16."""
    fma, twice = dx0.float(), dx0.float()
    inv64 = inv.double().to(d.device)
    for m in range(d.shape[0]):
        fma = torch.where(keep[m], (d[m].double() * inv64 + fma.double()).float(), fma)
        twice = torch.where(keep[m], twice + d[m].float() * inv.to(d.device), twice)
    return fma.bfloat16(), twice.bfloat16()


def check_dropout(members=3, B=2, S=77, K=200, p=0.1, window=False, seed=1234, stream0=7):
    """dropout_expand and dropout_accum_ bit for bit against the numpy mask (above).  window: x and dx are row / column
    windows of wider buffers whose halo must stay unchanged."""
    if window:
        xfull = _rand(B, S + 3, K + 16, seed=81)
        x = xfull[:, 1:S + 1, 8:8 + K]
        dxfull = _rand(B, S + 3, K + 16, seed=82)
        dx = dxfull[:, 2:S + 2, 8:8 + K]
        halo0 = dxfull.clone()
    else:
        x, dx = _rand(B, S, K, seed=81), _rand(B, S, K, seed=82)
    dx0 = dx.clone()
    d = _rand(members, B, S, K, seed=83)
    xm = ops.dropout_expand(x, members, p, seed, stream0)
    ops.dropout_accum_(dx, d, p, seed, stream0)
    torch.cuda.synchronize()
    keep = dropout_masks(members, B, S, K, p, seed, stream0)
    inv = dropout_inv_keep(p)
    want = torch.where(keep, (x.float() * inv.to(DEV)).bfloat16(), torch.zeros_like(x))
    parts = [_bits("expand", xm, want)]
    fma, twice = dropout_accum_replay(dx0, d, keep, inv)
    iv = torch.int16
    hit_f, hit_t = dx.view(iv) == fma.view(iv), dx.view(iv) == twice.view(iv)
    extra = {"accum_fma_or_two_roundings": bool((hit_f | hit_t).all().item()), "n_fma": int((hit_f & ~hit_t).sum().item()),
             "n_twice": int((hit_t & ~hit_f).sum().item()), "keep_rate": round(float(keep.float().mean().item()), 4)}
    if window:
        m = torch.ones_like(dxfull, dtype=torch.bool)
        m[:, 2:S + 2, 8:8 + K] = False
        extra["halo_clean"] = bool(torch.equal(dxfull[m], halo0[m]))
    return _combine(f"dropout_m{members}_B{B}_S{S}_K{K}_p{p:g}" + ("_window" if window else ""), parts, **extra)


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
    "groupnorm_256_offset": lambda: check_groupnorm(C=256, ratio=4.0),
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


def check_target_mse(B=3, C=4, Hh=16, Ww=24, weighted=True, layout=1, loss_type="l2", grad_scale=1.0):
    """target_mse_loss with min-SNR weights (or none): dpred bit for bit, loss against fp64."""
    S = (Hh // 2) * (Ww // 2)
    pred = _rand(B, C, Hh, Ww, seed=1) if layout == 2 else _rand(B, S, 4 * C, seed=1)
    tgt = _rand(B, C, Hh, Ww, seed=2)
    w = torch.tensor(MIN_SNR_W[:B], device=DEV) if weighted else None
    hc = _huber(loss_type, B)
    loss, dpred = ops.target_mse_loss(pred, tgt, w, grad_scale=grad_scale, layout=layout, loss_type=loss_type, huber_c=hc)
    torch.cuda.synchronize()
    return _check_loss(f"target_mse_{loss_type}_layout{layout}_w{int(weighted)}_gs{grad_scale:g}", loss, dpred, pred, tgt,
                       layout, loss_type, hc, w, grad_scale)


def check_loss_full_size(kind="flow", B=4, Cc=16, Hh=128, Ww=128, loss_type="l2"):
    """flow_mse_loss / target_mse_loss at a Flux 1024^2 latent: the 8-CTA cluster reduction gives the same loss and dpred
    bit for bit on a second run; dpred bit for bit against the replay, the loss against fp64 within loss_bound and, for
    l2, within 1e-6 relative."""
    S = (Hh // 2) * (Ww // 2)
    pred = _rand(B, S, 4 * Cc, seed=3)
    hc = _huber(loss_type, B)
    if kind == "flow":
        lat, noise = _rand(B, Cc, Hh, Ww, seed=1), _rand(B, Cc, Hh, Ww, seed=2)
        run = lambda: ops.flow_mse_loss(pred, lat, noise, loss_type=loss_type, huber_c=hc)
        tgt, w, layout = noise - lat, None, 0             # the target is formed in bf16, as the training step does
    else:
        tgt = _rand(B, Cc, Hh, Ww, seed=2)
        w = torch.tensor(MIN_SNR_W[:B], device=DEV)
        run = lambda: ops.target_mse_loss(pred, tgt, w, layout=1, loss_type=loss_type, huber_c=hc)
        layout = 1
    loss1, dpred1 = run()
    loss2, dpred2 = run()
    torch.cuda.synchronize()
    r = _check_loss(f"{kind}_loss_dpred_B{B}_{Cc}x{Hh}x{Ww}_{loss_type}", loss1, dpred1, pred, tgt, layout, loss_type, hc, w,
                    1.0, {"repeatable": bool(torch.equal(loss1, loss2)) and bool(torch.equal(dpred1, dpred2))})
    r["loss_rel_err"] = r["loss_err"] / abs(r["loss_ref"])
    if loss_type == "l2":
        r["ok"] = r["ok"] and r["loss_rel_err"] <= 1e-6
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
def wgrad_tile_width(N, K, sms=132):
    """The tile width stb_wgrad_full picks: 256 unless that leaves more than half of the SMs idle, and always for K <= 128."""
    return 256 if ((N + 127) // 128) * ((K + 255) // 256) >= sms // 2 or K <= 128 else 128


def check_wgrad_full(B=2, S=300, N=256, K=320, strided=False, accumulate=False, alpha=1.0, exact=False):
    """dW [N, K] = alpha sum_tokens dy[:, n] x[:, k] (+ dW): contraction over the B S tokens.  exact: bf16(alpha acc + old)
    bit for bit; a non-power-of-two alpha with accumulate accepts the FMA or the two-rounding result per element."""
    ed, ex = ("int", "frac") if exact else (None, None)
    if strided:   # row ranges / column ranges of larger buffers, like the joint hidden buffer and the fused qkv gradient
        dyf = _gen(B, S + 5, N + 64, seed=41, exact=ed)
        xf = _gen(B, S + 9, K + 32, seed=42, exact=ex)
        dy, x = dyf[:, 3:S + 3, 32:32 + N], xf[:, 4:S + 4, 8:8 + K]
    else:
        dy, x = _gen(B, S, N, seed=41, exact=ed), _gen(B, S, K, seed=42, exact=ex)
    out = old = None
    if accumulate:
        out = _rand(N, K, seed=43)
        old = out.clone()
    got = ops.wgrad_full(dy, x, out=out, alpha=alpha, accumulate=accumulate)
    torch.cuda.synchronize()
    acc64 = torch.einsum("bsn,bsk->nk", dy.double(), x.double())
    mag = torch.einsum("bsn,bsk->nk", dy.double().abs(), x.double().abs())
    a32 = _f32(alpha)
    name = f"wgrad_full_B{B}_S{S}_N{N}_K{K}_bn{wgrad_tile_width(N, K)}" + ("_accum" if accumulate else "") + \
        ("_exact" if exact else "")
    base = old.double() if accumulate else torch.zeros_like(acc64)
    if not exact:
        return _combine(name, [_report_acc("dw", got, base + a32 * acc64, abs(a32) * mag, B * S, GEMM_RTOL_BF16)])
    bound = exact_bound_ok([dy], [x], mag)
    twice = ((a32 * acc64.float() + old.float()) if accumulate else a32 * acc64.float()).bfloat16()
    if _is_pow2(a32) or not accumulate:
        return _combine(name, [_bits("dw", got, twice)], exact_bound=bound)
    once = (base + a32 * acc64).float().bfloat16()
    either = ((got.view(torch.int16) == once.view(torch.int16)) | (got.view(torch.int16) == twice.view(torch.int16))).all()
    return _combine(name, [], exact_bound=bound, fma_or_two_roundings=bool(either.item()),
                    n_fma=int((got == once).sum().item()), n_twice=int((got == twice).sum().item()))


def check_colsum2(B=3, S=333, D=1536, exact=False):
    """sum_s dy and sum_s dy z (fp32, atomics over row chunks) against fp64; exact: bit for bit."""
    dyf = _gen(B, S + 3, D + 16, seed=51, exact="int" if exact else None)
    zf = _gen(B, S, D, seed=52, exact="frac" if exact else None)
    dy = dyf[:, 1:S + 1, 8:8 + D]
    sm, dt = ops.colsum2(dy, zf)
    only = ops.colsum2(dy, None)[0]
    torch.cuda.synchronize()
    d64, z64 = dy.double(), zf.double()
    s_ref, s_mag = d64.sum(1), d64.abs().sum(1)
    p_ref, p_mag = (d64 * z64).sum(1), (d64 * z64).abs().sum(1)
    name = f"colsum2_B{B}_S{S}_D{D}" + ("_exact" if exact else "")
    if exact:
        parts = [_bits("colsum", sm, s_ref.float()), _bits("coldot", dt, p_ref.float()), _bits("colsum_only", only, s_ref.float())]
        return _combine(name, parts, exact_bound=exact_bound_ok([dy], [zf], p_mag) and float(s_mag.max()) < EXACT_BOUND)
    parts = [_report_acc("colsum", sm, s_ref, s_mag, S, GEMM_RTOL_F32), _report_acc("coldot", dt, p_ref, p_mag, S, GEMM_RTOL_F32),
             _report_acc("colsum_only", only, s_ref, s_mag, S, GEMM_RTOL_F32)]
    return _combine(name, parts)


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
def check_gelu_tanh(B=2, S=77, D=640, scale=1.0):
    """gelu_tanh(pre) is a bf16 neighbour of fp64 gelu_tanh(pre), and mul_dgelu_tanh(g, pre) one of g gelu'(pre) with the
    fp32 formulas' cancellation allowance (_gelu_atol), as the GEMM's exact-mode EPI_GELU / EPI_MUL_DGELU; in place equals
    out of place.  pre (N(0, scale^2)) is a row / column window of a wider buffer."""
    pf, gf = _rand(B, S + 2, D + 8, seed=71, scale=scale), _rand(B, S, D, seed=72)
    pre = pf[:, 1:S + 1, :D]
    act = ops.gelu_tanh(pre)
    out = ops.mul_dgelu_tanh(gf, pre)
    inplace = gf.clone()
    ops.mul_dgelu_tanh(inplace, pre, out=inplace)
    torch.cuda.synchronize()
    p64, g64 = pre.double(), gf.double()
    atol = _gelu_atol(p64)
    parts = [_neighbour("gelu", act, gelu64(p64), atol[0]), _neighbour("dgelu", out, g64 * dgelu64(p64), g64.abs() * atol[1])]
    return _combine(f"gelu_tanh_B{B}_S{S}_D{D}_x{scale:g}", parts, inplace=bool(torch.equal(inplace, out)))


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
# skinny_tn on both kernels (rank block 64 / 128, the last padded rank below each edge), several batches whose S is not
# a multiple of the row split (b3_split_tail), one token, a sequence shorter than one 64-token chunk, N below one 128-row
# tile, 16 short text-length batches, the widest Flux projection, and strided windows of wider buffers; each into a zero
# and a non-zero out, against fp64 and with exact inputs
for _n, _kw in (("r8", dict(B=2, S=700, R=8, N=1536)), ("r56", dict(B=2, S=700, R=56, N=1536)),
                ("r64", dict(B=2, S=700, R=64, N=1536)), ("r72", dict(B=2, S=700, R=72, N=1536)),
                ("r120", dict(B=2, S=700, R=120, N=1536)), ("r128", dict(B=2, S=700, R=128, N=1536)),
                ("b3_split_tail", dict(B=3, S=1000, R=48, N=1024)), ("s1", dict(B=3, S=1, R=16, N=512)),
                ("s63", dict(B=2, S=63, R=8, N=1024)), ("n72", dict(B=2, S=300, R=16, N=72)),
                ("b16_s77", dict(B=16, S=77, R=32, N=3072)), ("n12288", dict(B=1, S=4608, R=16, N=12288)),
                ("view_r16", dict(B=2, S=300, R=16, N=3072, view=True)),
                ("view_b3_r48", dict(B=3, S=333, R=48, N=1024, view=True)),
                ("view_r128", dict(B=2, S=700, R=128, N=1536, view=True))):
    for _acc in (False, True):
        for _x in (False, True):
            CHECKS[f"skinny_{_n}_ws" + ("_accum" if _acc else "") + ("_exact" if _x else "")] = _case(
                check_skinny, **_kw, accumulate=_acc, exact=_x)


# --------------------------------------------------------------------------------------------- run-to-run determinism
CHECKS.update({
    "attn_bwd_repeatable_hd128": lambda: check_attn_bwd_repeatable(HD=128),
    "attn_bwd_repeatable_hd64": lambda: check_attn_bwd_repeatable(HD=64),
    "skinny_repeatable_flux_lora": lambda: check_skinny_repeatable(),
    "flow_loss_full_size": lambda: check_loss_full_size("flow"),
    "target_loss_full_size": lambda: check_loss_full_size("target"),
})


# --------------------------------------------------------------------------------------------- GEMM family, exact inputs
# The exact-input mode over the grid above: every epilogue at every tile width and weight layout, 2-CTA clusters with an
# odd m-tile count, ring-7 segments, skinny M and the Flux shapes (K = 12288; segments 3072 + 12288 and 12288 + 9216 + 48).
for _en, (_epi, _nan) in _EPIS.items():
    for _bn in _BNS:
        for _kn in (False, True):
            CHECKS[f"gemm_epi_{_en}_bn{_bn}" + ("_wkn" if _kn else "") + "_exact"] = _case(
                check_gemm, 200, 328, 200, B=2, bias=True, epi=_epi, nan_to_num=_nan, tile=(0, _bn),
                w_kn=[True] if _kn else None, exact=True)
for _en in ("store", "gelu", "gate_res_nan", "mul_dgelu", "mul", "quick_gelu"):
    _epi, _nan = _EPIS[_en]
    CHECKS[f"gemm_cluster_odd_mtiles_{_en}_exact"] = _case(check_gemm, 300, 328, 200, B=3, segs=[72, 16], bias=True, epi=_epi,
                                                           nan_to_num=_nan, tile=(2, 128), exact=True)
for _bn in _BNS:
    CHECKS[f"gemm_ring7_bn{_bn}_exact"] = _case(check_gemm, 4608, 3072, 200, B=1, segs=[72, 16], bias=True, tile=(0, _bn),
                                                exact=True)
CHECKS["gemm_ring7_bn128_wkn_mixed_exact"] = _case(check_gemm, 4608, 3072, 200, B=1, segs=[72, 16], w_kn=[True, False, True],
                                                   tile=(0, 128), exact=True)
for _m in (1, 2, 65, 129):
    for _b in (1, 4):
        CHECKS[f"gemm_skinny_m{_m}_b{_b}_exact"] = _case(check_gemm, _m, 18432, 3072, B=_b, bias=True, exact=True)
CHECKS["gemm_k12288_exact"] = _case(check_gemm, 4608, 3072, 12288, B=1, bias=True, exact=True)
CHECKS["gemm_seg2_3072_12288_gate_res_exact"] = _case(check_gemm, 4608, 3072, 3072, B=1, segs=[12288], bias=True,
                                                      epi=E.EPI_GATE_RES, nan_to_num=True, exact=True)
CHECKS["gemm_seg3_dgrad_12288_9216_48_exact"] = _case(check_gemm, 4608, 3072, 12288, B=1, segs=[9216, 48], exact=True)
CHECKS["gemm_wkn_flux_dgrad_exact"] = _case(check_gemm, 4608, 3072, 9216, w_kn=[True], tile=(0, 256), exact=True)

# --------------------------------------------------------------------------------------------- GEMM paths without a reference before
for _x in (False, True):
    _s = "_exact" if _x else ""
    for _bn in _BNS:
        # the bf16 linear output full fine-tune keeps for the gate gradient
        CHECKS[f"gemm_gate_res_aux_bn{_bn}{_s}"] = _case(check_gemm, 200, 328, 200, B=2, bias=True, epi=E.EPI_GATE_RES,
                                                         nan_to_num=True, aux_out=True, tile=(0, _bn), exact=_x)
        # nan_to_num on +-inf / NaN in res and on res + gate y pushed past the bf16 maximum; without it they pass through
        for _nan in (True, False):
            CHECKS[f"gemm_gate_res_nonfinite_nan{int(_nan)}_bn{_bn}{_s}"] = _case(
                check_gemm, 200, 328, 200, B=2, bias=True, epi=E.EPI_GATE_RES, nan_to_num=_nan, aux_out=True,
                res_special=True, tile=(0, _bn), exact=_x)
        CHECKS[f"gemm_gelu_noaux_bn{_bn}{_s}"] = _case(check_gemm, 200, 328, 200, B=2, bias=True, epi=E.EPI_GELU,
                                                       aux_out=False, tile=(0, _bn), exact=_x)
    CHECKS[f"gemm_gelu_noaux_cluster{_s}"] = _case(check_gemm, 300, 328, 200, B=3, bias=True, epi=E.EPI_GELU, aux_out=False,
                                                   tile=(2, 128), exact=_x)
    # odd N: the lone last column of every row (bias, gate, res / aux words and the store of one element)
    for _n in (1, 3, 65, 327):
        for _en, _kw in (("store", dict(epi=E.EPI_STORE)), ("gate_res_aux", dict(epi=E.EPI_GATE_RES, nan_to_num=True, aux_out=True)),
                         ("mul", dict(epi=E.EPI_MUL)), ("gelu", dict(epi=E.EPI_GELU)), ("add_res", dict(epi=E.EPI_ADD_RES))):
            CHECKS[f"gemm_odd_n{_n}_{_en}{_s}"] = _case(check_gemm, 200, _n, 200, B=2, bias=True, **_kw, exact=_x)
    CHECKS[f"gemm_odd_n327_gelu_cluster{_s}"] = _case(check_gemm, 300, 327, 200, B=3, bias=True, epi=E.EPI_GELU,
                                                      tile=(2, 128), exact=_x)
    CHECKS[f"gemm_odd_n65_bn256{_s}"] = _case(check_gemm, 200, 65, 200, B=2, bias=True, tile=(0, 256), exact=_x)

    # skinny_tn into a non-zero out
    CHECKS[f"skinny_ws_accum{_s}"] = _case(check_skinny, B=2, S=700, R=48, N=1536, accumulate=True, exact=_x)
    # wgrad_full with N % 128 != 0 at both tile widths (K <= 128 forces 256; 520 gives 128 on 132 SMs)
    for _n in (200, 136):
        for _k in (120, 520):
            CHECKS[f"wgrad_full_n{_n}_k{_k}{_s}"] = _case(check_wgrad_full, B=2, S=300, N=_n, K=_k, exact=_x)
    CHECKS[f"wgrad_full_n200_accum{_s}"] = _case(check_wgrad_full, B=2, S=300, N=200, K=520, accumulate=True, alpha=0.25, exact=_x)
    # conv3x3 with C_out not a multiple of the tile width (72 at 128, 136 and 200 at 256)
    for _co in (72, 136, 200):
        CHECKS[f"conv3x3_co{_co}{_s}"] = _case(check_conv3x3, B=2, H=24, W=40, Ci=64, Co=_co, res=_co == 136, exact=_x)
    CHECKS[f"conv3x3_s2_co200{_s}"] = _case(check_conv3x3, B=1, H=32, W=48, Ci=128, Co=200, stride=2, exact=_x)

# exact mode of the existing weight-gradient, LoRA-gradient, reduction and conv checks
CHECKS.update({
    "skinny_exact": lambda: check_skinny(exact=True),
    "skinny_flux_exact": lambda: check_skinny(B=4, S=4608, R=48, N=9216, exact=True),
    "skinny_ragged_exact": lambda: check_skinny(B=3, S=333, R=16, N=200, exact=True),
    "skinny_ws_accum_alpha0.3_exact": lambda: check_skinny(B=2, S=700, R=48, N=1536, accumulate=True, alpha=0.3, exact=True),
    "wgrad_full_basic_exact": lambda: check_wgrad_full(exact=True),
    "wgrad_full_strided_accum_exact": lambda: check_wgrad_full(B=3, S=231, N=384, K=200, strided=True, accumulate=True,
                                                               alpha=0.5, exact=True),
    "wgrad_full_accum_alpha0.3_exact": lambda: check_wgrad_full(B=3, S=231, N=384, K=200, accumulate=True, alpha=0.3,
                                                                exact=True),
    "wgrad_full_sd3_qkv_exact": lambda: check_wgrad_full(B=2, S=1255, N=4608, K=1536, exact=True),
    "wgrad_full_narrow_exact": lambda: check_wgrad_full(B=1, S=1000, N=128, K=64, exact=True),
    "wgrad_full_flux_mlp_exact": lambda: check_wgrad_full(B=1, S=4608, N=3072, K=12288, exact=True),
    "colsum2_exact": lambda: check_colsum2(exact=True),
    "colsum2_small_exact": lambda: check_colsum2(B=1, S=7, D=64, exact=True),
    "conv3x3_s1_res_exact": lambda: check_conv3x3(Ci=128, Co=256, res=True, exact=True),
    "conv3x3_out32_exact": lambda: check_conv3x3(B=2, H=16, W=16, Ci=512, Co=32, exact=True),
    "conv3x3_pair_oddrows_exact": lambda: check_conv3x3(B=1, H=149, W=120, Ci=128, Co=128, res=True, exact=True),
    "conv3x3_pair_s2_wide_exact": lambda: check_conv3x3(B=1, H=160, W=600, stride=2, Ci=64, Co=256, exact=True),
    "conv3x3_s1_512_exact": lambda: check_conv3x3(B=1, H=16, W=16, Ci=512, Co=512, res=True, exact=True),
    "conv_in_3ch_exact": lambda: check_conv_in(exact=True),
    "conv_in_3ch_wide_exact": lambda: check_conv_in(B=2, H=9, W=300, C=128, exact=True),
    "conv_in_3ch_c8_cuda_core_exact": lambda: check_conv_in(B=1, H=12, W=20, C=8, exact=True),
})


# --------------------------------------------------------------------------------------------- row-wise kernels
# LayerNorm-modulate at every model width (CLIP-L / CLIP-G with eps 1e-5), the VPT = 8 forward (D > 4096), the joint
# [text + image] windows and modulation chunks of Flux (6 D) and SD3 (9 D), and the three ways of adding the residual
# gradient; every ln_modulate check includes zero, constant, offset and tiny-variance rows
for _d in (8, 72, 768, 1000, 1152, 1280, 4096, 4104, 8192):
    CHECKS[f"ln_modulate_d{_d}"] = _case(check_ln_modulate, D=_d, eps=1e-5 if _d in (768, 1280) else 1e-6)
CHECKS["ln_modulate_d3072_eps1e-5"] = _case(check_ln_modulate, D=3072, eps=1e-5)
CHECKS["ln_modulate_window_d3072"] = _case(check_ln_modulate, B=2, S=300, D=3072, window=True, chunks=6, chunk=3)
CHECKS["ln_modulate_window_d1536_mod9"] = _case(check_ln_modulate, B=2, S=128, D=1536, window=True, chunks=9, chunk=6)
CHECKS["ln_modulate_bwd_noadd_d1536"] = _case(check_ln_modulate, D=1536, add=None)
CHECKS["ln_modulate_bwd_alias_d1536"] = _case(check_ln_modulate, D=1536, add="alias")
CHECKS["ln_modulate_bwd_alias_window_d3072"] = _case(check_ln_modulate, D=3072, window=True, add="alias")

# q/k RMSNorm + RoPE: element-wise, paired and no tables, with and without norm weights, a text split inside a block of 8
# tokens, no text rows and only text rows, strided outputs, zero rows, the warp-per-token backward at HD 128 (a source
# layout the flat kernel cannot read), and the Flux shape
for _hd in (64, 128):
    for _tab in ("free", "paired", None):
        for _w in (True, False):
            CHECKS[f"qk_rmsnorm_rope_hd{_hd}_{_tab or 'none'}_w{int(_w)}"] = _case(
                check_qk_rmsnorm_rope, B=2, S=45, H=3, HD=_hd, s_split=13, tables=_tab, weights=_w)
    for _sp in (0, 45):
        CHECKS[f"qk_rmsnorm_rope_hd{_hd}_split{_sp}"] = _case(check_qk_rmsnorm_rope, B=2, S=45, H=3, HD=_hd, s_split=_sp)
    CHECKS[f"qk_rmsnorm_rope_hd{_hd}_strided_zero"] = _case(check_qk_rmsnorm_rope, B=2, S=45, H=3, HD=_hd, s_split=13,
                                                             strided_out=True, zero_rows=True)
    CHECKS[f"qk_rmsnorm_rope_hd{_hd}_loop_layout"] = _case(check_qk_rmsnorm_rope, B=2, S=96, H=4, HD=_hd, s_split=13,
                                                            loop_bwd=True)
CHECKS["qk_rmsnorm_rope_hd128_loop_layout_paired_w0_zero"] = _case(check_qk_rmsnorm_rope, B=2, S=45, H=3, HD=128,
                                                                   s_split=13, tables="paired", weights=False,
                                                                   loop_bwd=True, zero_rows=True)
CHECKS["qk_rmsnorm_rope_flux"] = _case(check_qk_rmsnorm_rope, B=1, S=4608, H=24, HD=128, s_split=512, tables="paired")

# T5LayerNorm / Qwen-Image txt_norm
for _d in (8, 264, 3584, 4096):
    CHECKS[f"rmsnorm_d{_d}"] = _case(check_rmsnorm, D=_d)
CHECKS["rmsnorm_d4096_strided"] = _case(check_rmsnorm, D=4096, strided=True)
CHECKS["rmsnorm_d3584_wbig"] = _case(check_rmsnorm, D=3584, wscale=64.0)
CHECKS["rmsnorm_d264_strided_wbig"] = _case(check_rmsnorm, B=3, S=300, D=264, strided=True, wscale=64.0)

CHECKS["gelu_tanh_wide_x3"] = _case(check_gelu_tanh, B=1, S=300, D=3072, scale=3.0)

# loss kernels: every loss type x pred layout, per-sample huber_c, min-SNR weights, grad_scale != 1
for _lt in ("l2", "huber", "smooth_l1"):
    for _lay in (0, 1, 2):
        CHECKS[f"flow_{_lt}_layout{_lay}"] = _case(check_flow, layout=_lay, loss_type=_lt, grad_scale=0.75)
        CHECKS[f"target_mse_{_lt}_layout{_lay}"] = _case(check_target_mse, layout=_lay, loss_type=_lt, grad_scale=1.5)
for _lt in ("huber", "smooth_l1"):
    CHECKS[f"flow_loss_full_size_{_lt}"] = _case(check_loss_full_size, "flow", loss_type=_lt)
    CHECKS[f"target_loss_full_size_{_lt}"] = _case(check_loss_full_size, "target", loss_type=_lt)


# --------------------------------------------------------------------------------------------- VAE encode, LoKr, LoRA dropout
# GroupNorm: cpg 4 / 8 / 16 at G = 32, cpg 1 / 2 at G = 64, C = 384 at G = 48 (16 idle threads per CTA), C = 8; HW 1,
# 7, 1000;
# B = 3; the Flux VAE stage sizes; offset groups at mean / sigma 0, 4, 16, 64 and 256 with torch's GroupNorm as a control;
# constant groups with beta = 0 and beta != 0 at a pixel count that is not a power of two.
for _c, _g in ((128, 32), (256, 32), (512, 32), (64, 64), (128, 64), (384, 48), (8, 8), (8, 4)):
    for _silu in (True, False):
        CHECKS[f"groupnorm_c{_c}_g{_g}_silu{int(_silu)}"] = _case(check_groupnorm, B=2, H=20, W=36, C=_c, G=_g, silu=_silu)
for _h, _w in ((1, 1), (1, 7), (25, 40)):
    for _c, _g in ((128, 32), (64, 64), (512, 32)):
        CHECKS[f"groupnorm_hw{_h * _w}_c{_c}_g{_g}"] = _case(check_groupnorm, B=2, H=_h, W=_w, C=_c, G=_g, silu=_h == 1)
CHECKS["groupnorm_b3"] = _case(check_groupnorm, B=3, H=33, W=17, C=256, G=32, ratio=4.0)
CHECKS["groupnorm_flux_512px_c128"] = _case(check_groupnorm, B=1, H=512, W=512, C=128, G=32)
CHECKS["groupnorm_flux_128px_c512"] = _case(check_groupnorm, B=1, H=128, W=128, C=512, G=32)
CHECKS["groupnorm_flux_1024px_c128"] = _case(check_groupnorm, B=1, H=1024, W=1024, C=128, G=32)
for _r in (0, 4, 16, 64, 256):
    for _c, _g in ((128, 32), (512, 32), (128, 64)):
        CHECKS[f"groupnorm_offset_r{_r}_c{_c}_g{_g}"] = _case(check_groupnorm, B=2, H=32, W=48, C=_c, G=_g, silu=False,
                                                             ratio=float(_r), control=True)
    CHECKS[f"groupnorm_offset_r{_r}_silu"] = _case(check_groupnorm, B=2, H=32, W=48, C=256, G=32, ratio=float(_r))
for _silu in (True, False):
    for _b0 in (True, False):
        CHECKS[f"groupnorm_const_silu{int(_silu)}_beta{'0' if _b0 else 'x'}"] = _case(
            check_groupnorm, B=2, H=7, W=11, C=128, G=32, silu=_silu, const=True, beta0=_b0)

# row softmax: short rows, a partial second 2048-column sweep, the mid-block S at 512 px and 1024 px, scale 512^-0.5
for _cols in (8, 24, 1024, 2056, 4096, 16384):
    CHECKS[f"softmax_rows_c{_cols}"] = _case(check_softmax_rows, rows=64 if _cols >= 4096 else 300, cols=_cols)
CHECKS["softmax_rows_c4096_midblock_scale"] = _case(check_softmax_rows, rows=128, cols=4096, scale=512 ** -0.5, sigma=30.0)

# latent sampling: the Flux, SD3, SDXL and sample() scalings, L = 4 / 16, odd h x w, B = 3
for _nm, _sh, _sc in (("flux", 0.1159, 0.3611), ("sd3", 0.0609, 1.5305), ("sdxl", None, 0.13025), ("sample", None, 1.0)):
    for _l in (4, 16):
        CHECKS[f"gaussian_sample_{_nm}_l{_l}"] = _case(check_gaussian_sample, B=2, L=_l, h=13, w=21, shift=_sh, scale=_sc)
CHECKS["gaussian_sample_b3_flux_64px"] = _case(check_gaussian_sample, B=3, L=16, h=64, w=64, shift=0.1159, scale=0.3611)

# LoKr rebuild: N and K not multiples of 8 (both scalar paths and the scalar transpose), row strides that are not
# multiples of 8, scale 0.75 and 1/3, and lycoris.factorization of Flux's 3072 / 12288 widths at factor -1 and 16
CHECKS["lokr_rebuild_ragged_transposed"] = _case(check_lokr_rebuild, a=3, b=37, c=5, d=13, scale=0.75, fused=False)
CHECKS["lokr_rebuild_odd_strides"] = _case(check_lokr_rebuild, a=4, b=40, c=6, d=32, scale=1 / 3, pad=3)
CHECKS["lokr_rebuild_ragged_odd_strides"] = _case(check_lokr_rebuild, a=3, b=37, c=5, d=13, scale=1 / 3, fused=False, pad=5)
_FLUX_LOKR = {(3072, -1): (48, 64), (3072, 16): (16, 192), (12288, -1): (96, 128), (12288, 16): (16, 768)}
for _n, _k in ((3072, 3072), (12288, 3072), (3072, 12288)):
    for _f in (-1, 16):
        (_a, _b), (_cc, _d) = _FLUX_LOKR[(_n, _f)], _FLUX_LOKR[(_k, _f)]
        CHECKS[f"lokr_rebuild_flux_{_n}x{_k}_f{_f}"] = _case(check_lokr_rebuild, a=_a, b=_b, c=_cc, d=_d, scale=0.75,
                                                             fused=_n == _k)
        CHECKS[f"lokr_factor_grads_flux_{_n}x{_k}_f{_f}"] = _case(check_lokr_factor_grads, a=_a, b=_b, c=_cc, d=_d,
                                                                  scale=0.75, strided=False)
# factor gradients: b d not a multiple of 2048 (dead threads in the last CTA), b d < 2048, a c near the 12288 limit of
# the partial-sum buffer, a strided dW; each also with exact inputs (bit for bit)
for _nm, _kw in (("bd4800", dict(a=6, b=300, c=3, d=16)), ("bd1920", dict(a=8, b=48, c=4, d=40)),
                 ("ac12192", dict(a=96, b=16, c=127, d=8)), ("tiny", dict(a=2, b=3, c=2, d=8))):
    for _x in (False, True):
        CHECKS[f"lokr_factor_grads_{_nm}_strided" + ("_exact" if _x else "")] = _case(
            check_lokr_factor_grads, **_kw, scale=0.5, strided=True, exact=_x)
CHECKS["lokr_factor_grads_flux_3072x3072_f-1_exact"] = _case(check_lokr_factor_grads, a=48, b=64, c=48, d=64, scale=0.25,
                                                             strided=False, exact=True)

# LoRA dropout: 1 / 3 / 8 members, p 0 / 0.1 / 0.5, K 8 / 200, row and column windows of x and dx
for _m in (1, 3, 8):
    for _p in (0.0, 0.1, 0.5):
        CHECKS[f"dropout_m{_m}_p{_p:g}"] = _case(check_dropout, members=_m, B=2, S=77, K=200 if _m != 8 else 8, p=_p,
                                                 window=_p == 0.1)
CHECKS["dropout_m3_k8_window"] = _case(check_dropout, members=3, B=3, S=33, K=8, p=0.5, window=True, seed=99, stream0=0xFFFFFFFE)
CHECKS["dropout_m3_flux_3072"] = _case(check_dropout, members=3, B=1, S=4608, K=3072, p=0.1, seed=5, stream0=3)


# --------------------------------------------------------------------------------------------- AdamW-bf16 reference model
# stb_adamw_bf16_multi runs through AdamWBF16.step, its production path, and is compared bit for bit with the reference's
# own eager op chain on copies of the same CUDA tensors: clip_grad_value_ when a clamp is set, the oracle's
# adamw_bf16_step with scalar_semantics="cpu" (the op sequence of the reference's `_make_step`, pinned to it by
# tests/golden/adamw_bf16_golden.pt; on CUDA tensors it runs torch's CUDA kernels, so it rounds as the reference does on
# a GPU), then EMAModel.step.  The stochastic-rounding integers of the production path are replayed in numpy
# (adamw_rnd_np: the two hash_u32 keys per tensor, the Weyl counter with its high-32-bit term, the two mix32 and the
# halving into r0..r3) from the launch seed, restated here (adamw_seed) rather than imported, so a change to the
# generator or to the seed formula fails.  p, exp_avg, exp_avg_sq, shift and the EMA shadows must hold the same bits;
# any NaN matches any NaN (__float2bfloat16 and torch's cast give different payloads).  Each tensor lives in one flat
# buffer per role, at a 16-byte boundary or, where the case asks, 2 bytes past it (the kernel's scalar path); the rest of
# every buffer must stay unchanged.  Every case starts from random, non-zero exp_avg / exp_avg_sq / shift.
# A NaN reaching a stochastic rounding becomes -0.0: fp32 arithmetic gives the NaN 0x7FFFFFFF, adding a nonzero 16-bit
# integer wraps it to 0x8000xxxx and the mask leaves 0x80000000 (only r = 0 keeps the NaN).  The reference's
# copy_stochastic_ does the same integer arithmetic, so it is matched, not changed; n_nan_neg0 counts the exp_avg
# elements of a NaN gradient that came out -0.
_M64 = 0xFFFFFFFFFFFFFFFF
ADAMW_ROLES = ("p", "g", "m", "v", "s", "e")       # param, grad, exp_avg, exp_avg_sq, shift, EMA shadow
BF16_MAX = 3.3895313892515355e38


def adamw_seed(seed, step, salt=0, group=0):
    """training/optim.py launch_seed, restated: the 64-bit seed of the launch of `group` / chunk `salt` at `step`."""
    return (seed * 0x9E3779B1 + int(step) * 0x85EBCA77 + salt * 0xC2B2AE3D27D4EB4F + group * 0xD6E8FEB86659FD93) & _M64


def hash_u32_py(x):
    """optim.cuh hash_u32 (splitmix64 finaliser, upper 32 bits) on a Python int."""
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return (x ^ (x >> 31)) >> 32


def adamw_keys(seed64, t):
    """(key0, key1) of launch tensor t."""
    t = t & 0xFFFFFFFF
    return hash_u32_py(seed64 ^ ((t << 40) & _M64)), hash_u32_py(((seed64 + 0x632BE59BD9B4E019) & _M64) ^ (t << 17))


def adamw_rnd_np(seed64, t, n, first=0):
    """The integers optim.cuh draws for elements first .. first + n - 1 of launch tensor t: int32 [4, n] (r0..r3)."""
    import numpy as np
    k0, k1 = adamw_keys(seed64, t)
    i = np.arange(first, first + n, dtype=np.uint64)
    lo, hi = (i & np.uint64(0xFFFFFFFF)).astype(np.uint32), (i >> np.uint64(32)).astype(np.uint32)
    c = lo * np.uint32(0x9E3779B1) + hi * np.uint32(0x7FEB352D)
    h0, h1 = mix32_np(c ^ np.uint32(k0)), mix32_np(c + np.uint32(k1))
    low, sh = np.uint32(0xFFFF), np.uint32(16)
    return np.stack([h0 & low, h0 >> sh, h1 & low, h1 >> sh]).astype(np.int32)


def _adamw_edges(n, seed):
    """Gradient / state overrides by element class i % 16 (sign alternating every 16 elements): zero and -0 gradients
    with zero moments (0 / 0 at eps 0), |g| = 2^-60 / 2^-65 (alpha2 g^2 a subnormal), 2^-70 / 2^-100 (underflow), 2^64 /
    2^100 (exp_avg_sq overflows), +-inf, NaN, +-0.36 / +-0.38 (inside / outside a 0.37 clamp), p at +bf16 max and near
    -bf16 max with a shift that can round it to inf, and subnormal moments."""
    i = torch.arange(n)
    cls, sgn = i % 16, torch.where((i // 16) % 2 == 0, 1.0, -1.0)
    g = torch.full((n,), math.nan)
    for c, val in ((2, 2.0 ** -60), (3, 2.0 ** -65), (4, 2.0 ** -70), (5, 2.0 ** -100), (6, 2.0 ** 64), (7, 2.0 ** 100),
                   (11, 0.36), (12, 0.38), (15, 2.0 ** -65)):
        g = torch.where(cls == c, sgn * val, g)
    g = torch.where(cls == 0, 0.0, torch.where(cls == 1, -0.0, g))
    g = torch.where(cls == 8, math.inf, torch.where(cls == 9, -math.inf, g))
    rest = (cls == 13) | (cls == 14)
    g = torch.where(rest, torch.randn(n, generator=torch.Generator().manual_seed(seed)) * 0.02, g)
    near_max = -torch.tensor([0x7F7D], dtype=torch.int16).view(torch.bfloat16).float()
    p = {13: BF16_MAX, 14: float(near_max)}
    s = {13: 2.0 ** 119, 14: -(2.0 ** 120)}
    return cls, g, p, s


def _adamw_values(kind, sizes, steps, seed):
    """CPU bf16 starting values {role: [tensor per size]} and gradients init["g"][step][tensor]."""
    gen = torch.Generator().manual_seed(seed)
    rn = lambda n, s: torch.randn(n, generator=gen) * s
    init = {r: [] for r in ADAMW_ROLES if r != "g"}
    init["g"] = [[] for _ in range(steps)]
    for t, n in enumerate(sizes):
        p, m, v, s = rn(n, 0.05), rn(n, 0.01), rn(n, 0.02) ** 2 * 0.05, rn(n, 1e-4)
        e = p + rn(n, 1e-3)
        gs = [rn(n, 0.02) for _ in range(steps)]
        if kind == "edges":
            cls, g_e, p_e, s_e = _adamw_edges(n, seed + t)
            gs = [torch.where(torch.isnan(g_e) & ~((cls == 10)), g, g_e) for g in gs]
            zero = (cls == 0) | (cls == 1)
            m, v = torch.where(zero, 0.0, m), torch.where(zero, 0.0, v)
            m, v = torch.where(cls == 15, 2.0 ** -130, m), torch.where(cls == 15, 2.0 ** -130, v)
            for c in p_e:
                p, s, e = torch.where(cls == c, p_e[c], p), torch.where(cls == c, s_e[c], s), torch.where(cls == c, p_e[c], e)
        for r, x in zip("pmvse", (p, m, v, s, e)):
            init[r].append(x.bfloat16())
        for k in range(steps):
            init["g"][k].append(gs[k].bfloat16())
    return init


def _adamw_place(vals, shifted, seed):
    """One flat CUDA bf16 buffer holding vals[u] at a 16-byte boundary, or 2 bytes past it where shifted[u], with 8 spare
    elements after each.  Returns (views, buffer, mask of the spare elements); the spare elements hold random values."""
    starts, pos = [], 0
    for x, sh in zip(vals, shifted):
        pos = _pad8(pos) + (1 if sh else 0)
        starts.append(pos)
        pos += x.numel() + 8
    buf = _rand(pos, seed=seed)
    halo = torch.ones(pos, dtype=torch.bool, device=DEV)
    views = []
    for x, a in zip(vals, starts):
        halo[a:a + x.numel()] = False
        views.append(buf[a:a + x.numel()])
        views[-1].copy_(x.to(DEV))
    return views, buf, halo


def _cat_bits(xs):
    return torch.cat([x.detach().reshape(-1) for x in xs])


def check_adamw(name, sizes, *, steps=2, step0=0, beta1=0.9, beta2=0.999, eps=1e-8, lr=1e-4, clamp=None, ema=None,
                shifted=(), mixed=False, values="normal", decays=None, wd_lr=2e-3, chunks=1, groups=1, golden=False,
                repeat=False, seed=11):
    """AdamWBF16.step against the reference chain, bit for bit (above).
    sizes: the tensors of one param group.  groups=2: a second group holding identical copies (same values, same
    gradients): each group must match its own replay, and after the first step the number of exp_avg elements that
    differ between the groups must be within 6 sigma of what independent streams give (sum of 2 q (1 - q), q the
    rounding-up probability of each element's fp32 value), which is far from 0.  chunks: each step is `chunks` calls
    with `only=` a contiguous slice of the tensors and salt 0, 1, ...  decays: per tensor, whether accumulated_decay is
    preset so that the tensor's delayed weight decay fires on the first step (weight_decay * lr = wd_lr, 2e-3 by default:
    the others fire later; above 5e-3 every tensor decays on every step).  ema: 1 - decay of a fused EMA update (shadows in their own buffer).  shifted: roles placed 2 bytes past a
    16-byte boundary (mixed: odd tensors only).  golden: p0, gradients and random integers of the CPU golden, through
    `_rnd`.  repeat: the production path runs twice and must give the same bits."""
    import numpy as np
    from oracle import adamw_bf16_oracle as A
    from simpletuner_b200.training.ema import EMAModel
    from simpletuner_b200.training.optim import AdamWBF16

    T = len(sizes)
    init = _adamw_values(values, sizes, steps, seed)
    golden_rnd = None
    if golden:
        from pathlib import Path
        G = torch.load(Path(__file__).parent / "golden" / "adamw_bf16_golden.pt")
        assert sum(sizes) == G["p0"].numel() and groups == 1 and chunks == 1
        cuts = [0] + list(np.cumsum(sizes))
        flat = G["p0"].flatten()
        init["p"] = [flat[a:b].clone() for a, b in zip(cuts[:-1], cuts[1:])]
        steps = len(G["decays"])
        init["g"] = [[G[f"step{k}.grad"].flatten()[a:b].clone() for a, b in zip(cuts[:-1], cuts[1:])] for k in range(steps)]
        golden_rnd = [G[f"step{k}.rnd"].reshape(4, -1).to(DEV).contiguous() for k in range(steps)]
        hp = G["hp"]
        beta1, beta2, eps, lr = hp["beta1"], hp["beta2"], hp["eps"], hp["lr"]
    U = groups * T
    vals = {r: [init[r][u % T] for u in range(U)] for r in "pmvse"}
    grads = [[init["g"][k][u % T] for u in range(U)] for k in range(steps)]
    wd = 0.0 if decays is None else wd_lr / lr
    acc0 = [4e-3 if decays is not None and decays[u % T] else 0.0 for u in range(U)]
    chunk_ts = [list(c) for c in np.array_split(np.arange(T), chunks)]
    moved = lambda role, u: role in shifted and (not mixed or u % 2 == 1)

    def production():
        views, bufs = {}, {}
        for k, r in enumerate(ADAMW_ROLES):
            src = vals[r] if r != "g" else grads[0]
            views[r], buf, halo = _adamw_place(src, [moved(r, u) for u in range(U)], seed=900 + k)
            bufs[r] = (buf, halo, buf[halo].clone())
        params = [torch.nn.Parameter(x) for x in views["p"]]
        opt = AdamWBF16([{"params": params[gi * T:(gi + 1) * T]} for gi in range(groups)], lr=lr, betas=(beta1, beta2),
                        eps=eps, weight_decay=wd, seed=seed)
        for u, p_ in enumerate(params):
            opt.state[p_].update(step=float(step0), exp_avg=views["m"][u], exp_avg_sq=views["v"][u], shift=views["s"][u],
                                 accumulated_decay=acc0[u])
            p_.grad = views["g"][u]
        em = None
        if ema is not None:
            em = EMAModel(params, decay=1.0 - ema, warmup_steps=1)
            em.shadow_params = list(views["e"])
        return {"views": views, "bufs": bufs, "params": params, "opt": opt, "ema": em}

    def prod_step(run, k):
        for u in range(U):
            run["views"]["g"][u].copy_(grads[k][u].to(DEV))
        for c, ts in enumerate(chunk_ts):
            only = None if chunks == 1 else [run["params"][gi * T + t] for gi in range(groups) for t in ts]
            run["opt"].step(_rnd=golden_rnd[k] if golden else None, grad_clamp=clamp, ema=run["ema"], only=only, salt=c)

    runs = [production() for _ in range(2 if repeat else 1)]
    rp = [torch.nn.Parameter(x.to(DEV, copy=True)) for x in vals["p"]]
    rs, rm, rv = ([x.to(DEV, copy=True) for x in vals[r]] for r in "smv")
    r_ema = EMAModel(rp, decay=1.0 - ema, warmup_steps=1) if ema is not None else None
    if r_ema is not None:
        r_ema.shadow_params = [x.to(DEV, copy=True) for x in vals["e"]]
    acc = list(acc0)
    offs = [0] + list(np.cumsum(sizes))
    parts, counts = [], {"n_scalar": 0, "n_nan_neg0": 0, "n_decayed": 0, "n_inf": 0}
    extra = {}
    for k in range(steps):
        for run in runs:
            prod_step(run, k)
        stepk = step0 + k + 1
        with torch.no_grad():
            for u in range(U):
                rp[u].grad = grads[k][u].to(DEV, copy=True)
            if clamp is not None:
                torch.nn.utils.clip_grad_value_(rp, clamp)
            for gi in range(groups):
                for c, ts in enumerate(chunk_ts):
                    seed64 = adamw_seed(seed, stepk, c, gi)
                    for j, t in enumerate(ts):
                        u, n = gi * T + t, sizes[t]
                        dec, acc[u] = A.decay_schedule(acc[u], wd, lr)
                        if golden:
                            rnd = golden_rnd[k][:, offs[t]:offs[t] + n]
                        else:
                            rnd = torch.from_numpy(adamw_rnd_np(seed64, j, n)).to(DEV)
                        if k == 0 and groups == 2 and gi == 1 and c == 0 and j == 0:
                            extra.update(_adamw_group_stats(rp, rm, T, beta1, chunk_ts))
                        A.adamw_bf16_step(rp[u], rp[u].grad, rs[u], rm[u], rv[u], beta1=beta1, beta2=beta2, step=float(stepk),
                                          lr=lr, eps=eps, decay_this_iteration=dec, rnd=list(rnd), scalar_semantics="cpu")
                        counts["n_scalar"] += n if any(moved(r, u) for r in ADAMW_ROLES if r != "e" or ema is not None) \
                            else n % 8
                        counts["n_decayed"] += n if dec > 0 else 0
                        counts["n_nan_neg0"] += int((torch.isnan(rp[u].grad) & (rm[u].view(torch.int16) == -32768)).sum())
            if r_ema is not None:
                r_ema.step(rp)
        torch.cuda.synchronize()
        counts["n_inf"] += sum(int(torch.isinf(x).sum()) for xs in (rp, rm, rv, rs) for x in xs)
        run = runs[0]
        want = {"p": rp, "m": rm, "v": rv, "s": rs, "e": r_ema.shadow_params if r_ema is not None else None}
        for r in "pmvse":
            if want[r] is not None:
                parts.append(_bits(f"{r}_step{k}", _cat_bits(run["views"][r]), _cat_bits(want[r])))
        if repeat:
            extra["repeatable"] = extra.get("repeatable", True) and all(
                torch.equal(_cat_bits(runs[0]["views"][r]).view(torch.int16), _cat_bits(runs[1]["views"][r]).view(torch.int16))
                for r in "pmvse")
        if k == 0 and groups == 2:
            mg = _cat_bits(run["views"]["m"]).view(torch.int16)
            half = mg.numel() // 2
            extra["groups_n_diff"] = int((mg[:half] != mg[half:]).sum())
            lo, hi = extra["groups_expect"] - 6 * extra["groups_sigma"], extra["groups_expect"] + 6 * extra["groups_sigma"]
            extra["groups_independent"] = bool(lo <= extra["groups_n_diff"] <= hi and extra["groups_expect"] > 100)
    for run in runs:
        extra["halo_clean"] = extra.get("halo_clean", True) and all(torch.equal(b[halo], b0) for b, halo, b0 in run["bufs"].values())
        if run["ema"] is not None:
            extra["ema_decay_used"] = run["ema"].cur_decay_value
    return _combine(name, parts, **extra, **counts, numel=groups * sum(sizes))


def _adamw_group_stats(rp, rm, T, beta1, chunk_ts):
    """Expected number (and sigma) of group 0 / group 1 exp_avg elements that differ after the first step if the two
    groups' streams are independent: the fp32 value before the exp_avg rounding is grad + (1 - beta1) bf16(beta1 m),
    the same in both groups (identical copies, group 0 not yet stepped in rm for group 1's tensors); it rounds up with
    probability q = low 16 bits / 2^16, and two independent draws differ with probability 2 q (1 - q)."""
    q = []
    for t in range(T):
        u = T + t
        res = rp[u].grad.float().add_(rm[u].mul(beta1), alpha=1 - beta1)
        low = (res.view(torch.int32) & 0xFFFF).double() / 65536.0
        q.append(torch.where(torch.isfinite(res), low, torch.zeros_like(low)))
    q = torch.cat(q)
    pd = 2 * q * (1 - q)
    return {"groups_expect": float(pd.sum()), "groups_sigma": float((pd * (1 - pd)).sum().sqrt())}


# AdamW-bf16: the CPU golden's integers through `_rnd`; sizes around the vector width and the 2048-element block (one
# launch), and a Flux-LoRA-sized launch (532 tensors, 26M elements) at beta2 0.95 where most tensors decay; every role
# 2 bytes off a 16-byte boundary in turn, all at once and mixed with aligned tensors; edge values with and without the
# clamp, at eps 0 and at beta1 = beta2 = 0; beta1 x beta2 x eps x step x lr; per-tensor decay; the fused EMA at
# 1 - decay of 0, 0.03 and 1; three `only=` chunks; two identical param groups; the same seed twice
_ADAMW_SIZES = [2049, 8, 333, 4096 + 5]
CHECKS["adamw_golden_rnd"] = _case(check_adamw, "adamw_golden_rnd", [1000, 1, 3999, 3481], golden=True,
                                   decays=[True, False, True, False])
CHECKS["adamw_sizes"] = _case(check_adamw, "adamw_sizes", [1, 7, 8, 9, 2047, 2048, 2049, 8 * 2048 + 3],
                              decays=[t % 2 == 1 for t in range(8)])
CHECKS["adamw_flux_lora_532"] = _case(check_adamw, "adamw_flux_lora_532", [3072 * 16 + t % 3 for t in range(532)],
                                      beta2=0.95, decays=[t % 5 != 0 for t in range(532)], seed=3)
for _r in ADAMW_ROLES:
    CHECKS[f"adamw_offset_{_r}"] = _case(check_adamw, f"adamw_offset_{_r}", _ADAMW_SIZES, shifted=(_r,), ema=0.03)
CHECKS["adamw_offset_all"] = _case(check_adamw, "adamw_offset_all", _ADAMW_SIZES, shifted=ADAMW_ROLES, ema=0.03)
CHECKS["adamw_offset_mixed"] = _case(check_adamw, "adamw_offset_mixed", _ADAMW_SIZES * 2, shifted=ADAMW_ROLES, mixed=True,
                                     ema=0.03, decays=[t % 3 == 0 for t in range(8)])
_EDGE_SIZES = [16 * 130, 16 * 7 + 5, 4096]
for _nm, _kw in (("plain", {}), ("clamp", dict(clamp=0.37)), ("eps0", dict(eps=0.0)),
                 ("clamp_eps0_offset", dict(clamp=0.37, eps=0.0, shifted=ADAMW_ROLES)), ("beta0", dict(beta1=0.0, beta2=0.0)),
                 ("lr1_step1e6", dict(lr=1.0, step0=10 ** 6 - 1)), ("offset_ema", dict(shifted=ADAMW_ROLES, ema=0.03))):
    CHECKS[f"adamw_edges_{_nm}"] = _case(check_adamw, f"adamw_edges_{_nm}", _EDGE_SIZES, values="edges", steps=3, **_kw)
for _i, (_b2, _st) in enumerate((_b2, _st) for _b2 in (0.0, 0.95, 0.999, 0.9999) for _st in (1, 2, 1000, 10 ** 6)):
    _b1, _eps, _lr = (0.0, 0.9)[_i % 2], (0.0, 1e-8, 1e-6)[_i % 3], (1e-4, 1.0)[(_i // 2) % 2]
    _nm = f"adamw_hp_b1_{_b1:g}_b2_{_b2:g}_eps{_eps:g}_step{_st}_lr{_lr:g}"
    CHECKS[_nm] = _case(check_adamw, _nm, _ADAMW_SIZES, beta1=_b1, beta2=_b2, eps=_eps, lr=_lr, step0=_st - 1,
                        decays=[True, False, False, True])
CHECKS["adamw_decay_per_tensor"] = _case(check_adamw, "adamw_decay_per_tensor", [3000, 2048, 7, 5000, 64],
                                         decays=[False, True, True, False, True], steps=3, lr=1e-3)
# every tensor decays on every step, by about 1/3 (a decay far above the default 5e-3 threshold's)
CHECKS["adamw_decay_third_every_step"] = _case(check_adamw, "adamw_decay_third_every_step", [(1 << 20) + 3, 4099],
                                               decays=[True, False], wd_lr=1 / 3, steps=3, lr=1e-3)
for _a in (0.0, 0.03, 1.0):
    CHECKS[f"adamw_ema_{_a:g}"] = _case(check_adamw, f"adamw_ema_{_a:g}", _ADAMW_SIZES, ema=_a, shifted=("e",), mixed=True)
CHECKS["adamw_chunks3_clamp"] = _case(check_adamw, "adamw_chunks3_clamp", [2049, 8, 333, 4101, 1, 9000, 64], chunks=3,
                                      clamp=0.03, decays=[t % 2 == 0 for t in range(7)])
CHECKS["adamw_two_groups"] = _case(check_adamw, "adamw_two_groups", [4096, 2049, 20000, 7], groups=2, steps=1)
CHECKS["adamw_two_groups_chunks3"] = _case(check_adamw, "adamw_two_groups_chunks3", [4096, 2049, 20000, 7, 333], groups=2,
                                           chunks=3, steps=1)
CHECKS["adamw_repeat_offset_mixed"] = _case(check_adamw, "adamw_repeat_offset_mixed", _ADAMW_SIZES * 3, shifted=ADAMW_ROLES,
                                            mixed=True, repeat=True, ema=0.03, steps=3)
