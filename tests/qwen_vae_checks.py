"""GPU checks of the Qwen-Image VAE encode path: 3x3 convs with C_in % 64 != 0, per-channel latent normalisation and
the whole encoder against the fp64 oracle (oracle/qwen_vae_oracle.py).  Used by tests/test_qwen_vae_gpu.py."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import qwen_vae_oracle as O
from simpletuner_b200 import ops
from tests import kernel_checks as K

DEV = "cuda"
# whole-encoder tolerance, per element: |got - ref| <= MODEL_ATOL rms(ref) + MODEL_RTOL |ref| (bf16 activations through
# about 30 convs, RMS norms and one attention, against fp64)
MODEL_ATOL, MODEL_RTOL = 0.08, 0.04


# Wan 2.1 channel RMS norm (ops.rmsnorm_fwd(normalize=True), stb_channel_rmsnorm_nhwc): interval replay.  The kernel's
# fp32 sum of squares of a row lies within (C + 4) u of the fp64 one in any order (positive terms, plus the squares' own
# rounding), and bf16(sqrtf(.)) is monotone in it, so the norm is one of the two bf16 values replayed from
# ss64 (1 -+ (C + 4) u) through fp32 (inf past the fp32 range, as the kernel's and torch's fp32 sums overflow) and
# sqrtf, clamped at bf16(eps).  The rest of the chain (csrc/vae.cuh) is replayed on each with fp32 torch ops, rounded to
# bf16 after every op: without SiLU the output must equal one replay bit for bit; with SiLU it must be a bf16 neighbour
# of fp64 silu(v) for v between the two replays' y.  tol_use: the worst |got - y64| over 2^-8 (4 |g64| + |y64|) (five
# roundings of up to half a bf16 ulp each; with SiLU its slope and one more rounding), y64 the fp64 value without
# roundings, over the rows whose fp32 sum of squares cannot overflow.
def channel_rmsnorm_input(R, C, seed=1):
    """x [R, C] bf16: row 0 zeros, 1 negative zeros, 2 constant 0.75, 3 N(0, 1) 2^60, 4 N(0, 1) 2^-60, 5 constant 2^60
    (its fp32 sum of squares overflows from C = 256 on), 6 N(0, 1) 2^-75 (below an eps of 1e-12 for small C); the others
    N(0, 1) 2^(r % 9 - 4)."""
    g = torch.Generator().manual_seed(seed)
    r = torch.arange(R, dtype=torch.float64).view(R, 1)
    x = torch.randn(R, C, generator=g, dtype=torch.float64) * torch.pow(2.0, r % 9 - 4)
    edges = [torch.zeros(C), torch.full((C,), -0.0), torch.full((C,), 0.75), torch.randn(C, generator=g) * 2.0 ** 60,
             torch.randn(C, generator=g) * 2.0 ** -60, torch.full((C,), 2.0 ** 60), torch.randn(C, generator=g) * 2.0 ** -75]
    for i, e in enumerate(edges[:R]):
        x[i] = e.double()
    return x.to(torch.bfloat16).to(DEV)


def channel_rmsnorm_replay(x, gamma, bias, n):
    """The eager chain after the norm, in fp32 torch ops rounded to bf16 after each: x [R, C] bf16, n [R, 1] fp32 (a
    bf16 norm, clamped).  Returns y (bf16, before SiLU)."""
    C = x.shape[-1]
    q = (x.float() / n).bfloat16().float()
    s = (q * K._f32(C ** 0.5)).bfloat16().float()
    g = (s * gamma.float()).bfloat16().float()
    return (g + (bias.float() if bias is not None else 0.0)).bfloat16()


def channel_rmsnorm_norms(x, eps=1e-12):
    """(n_lo, n_hi) [R, 1] fp32: the two bf16 norms the kernel may form, clamped at bf16(eps) as F.normalize's
    clamp_min does on a bf16 tensor."""
    C = x.shape[-1]
    ss = x.double().pow(2).sum(-1, keepdim=True)
    rel = (C + 4) * K.U24
    n_min = torch.tensor(eps).bfloat16().float().item()
    return [(ss * f).float().sqrt().bfloat16().float().clamp_min(n_min) for f in (1 - rel, 1 + rel)]


def check_channel_rmsnorm(R=300, C=96, silu=True, bias=False, eps=1e-12, seed=1):
    """Interval replay of ops.rmsnorm_fwd(normalize=True) (above) on channel_rmsnorm_input; also counts the elements
    where torch's eager chain on the device differs (n_vs_eager, information: its norm sums in another order)."""
    x = channel_rmsnorm_input(R, C, seed)
    gm = (1.0 + 0.1 * K._rand(C, seed=seed + 1).float()).bfloat16()
    bv = K._rand(C, scale=0.1, seed=seed + 2) if bias else None
    out = ops.rmsnorm_fwd(x.view(1, R, C), gm, eps, normalize=True, bias=bv, silu=silu).view(R, C)
    torch.cuda.synchronize()
    n_lo, n_hi = channel_rmsnorm_norms(x, eps)
    y_lo, y_hi = channel_rmsnorm_replay(x, gm, bv, n_lo), channel_rmsnorm_replay(x, gm, bv, n_hi)
    x64 = x.double()
    nrm = x64.pow(2).sum(-1, keepdim=True).sqrt().clamp_min(float(torch.tensor(eps).bfloat16()))
    g64 = x64 / nrm * C ** 0.5 * gm.double()
    y64 = g64 + (bv.double() if bias else 0.0)
    finite_rows = (x64.pow(2).sum(-1, keepdim=True) * (1 + (C + 4) * K.U24) < 2.0 ** 127).expand_as(x64)
    if silu:
        part = K.silu_check("out", out, torch.minimum(y_lo.float(), y_hi.float()), torch.maximum(y_lo.float(), y_hi.float()))
        v64 = K.silu64(y64)
        tol = 2.0 ** -8 * (4 * g64.abs() + y64.abs()) * (1 + 1.0 / (1 + (-y64).exp())) + 2.0 ** -8 * v64.abs()
        err = (out.double() - v64).abs()
    else:
        iv = torch.int16
        hit = (out.view(iv) == y_lo.view(iv)) | (out.view(iv) == y_hi.view(iv))
        n = int((~hit).sum().item())
        part = {"name": "out", "ok": n == 0, "n_bad": n, "numel": out.numel()}
        if n:
            K._first(~hit, out.float(), y_lo.float(), part)
        tol = 2.0 ** -8 * (4 * g64.abs() + y64.abs())
        err = (out.double() - y64).abs()
    use = torch.where((err > 0) & finite_rows, err / tol.clamp_min(1e-300), torch.zeros_like(err))
    part["tol_use"] = round(float(use.max().item()), 4)
    eager = F.normalize(x, dim=-1, eps=eps) * C ** 0.5 * gm + (bv if bias else 0.0)
    eager = F.silu(eager) if silu else eager
    return K._combine(f"channel_rmsnorm_R{R}_C{C}_silu{int(silu)}_bias{int(bias)}_eps{eps:g}", [part],
                      n_two_norms=int((n_lo != n_hi).sum().item()),
                      n_vs_eager=int((eager.view(torch.int16) != out.view(torch.int16)).sum().item()))


def check_conv_padded(B=2, H=13, W=21, Ci=96, Co=64, stride=1, res=False, exact=False):
    """ops.conv3x3_nhwc with a C_in that is not a multiple of 64 (weights from ops.conv_w9) against the fp64 conv of the
    same bf16 inputs; exact inputs bit for bit."""
    x = K._gen(B, H, W, Ci, seed=1, exact="int" if exact else None)
    w = K._gen(Co, Ci, 3, 3, scale=(9 * Ci) ** -0.5, seed=2, exact="frac" if exact else None)
    bv = K._rand(Co, scale=0.1, seed=3)
    Ho, Wo = (H, W) if stride == 1 else (H // 2, W // 2)
    rv = K._rand(B, Ho, Wo, Co, seed=4) if res else None
    out = ops.conv3x3_nhwc(x, ops.conv_w9(w), bv, rv, stride)
    torch.cuda.synchronize()

    def conv(xt, wt):
        xn = xt.double().permute(0, 3, 1, 2)
        if stride == 1:
            return F.conv2d(xn, wt.double(), padding=1).permute(0, 2, 3, 1)
        return F.conv2d(F.pad(xn, (0, 1, 0, 1)), wt.double(), stride=2).permute(0, 2, 3, 1)

    acc64, mag = conv(x, w), conv(x.abs(), w.abs())
    name = f"conv3x3_s{stride}_{Ci}to{Co}_{H}x{W}" + ("_exact" if exact else "")
    if exact:
        f = acc64.float() + bv.float()
        want = (f + rv.float() if res else f).bfloat16()
        return K._combine(name, [K._bits("out", out, want)], exact_bound=K.exact_bound_ok([x], [w], mag))
    ref = acc64 + bv.double() + (rv.double() if res else 0.0)
    return K._combine(name, [K._report_acc("out", out, ref, mag, 9 * Ci, K.GEMM_RTOL_BF16)])


def check_gaussian_channel_norm(B=2, L=16, h=12, w=20):
    """ops.gaussian_sample_scale with [L] shift / inv_std vectors: bit for bit against the eager chain of
    DiagonalGaussianDistribution.sample + post_vae_encode_transform_sample replayed on the same eps, for either of
    the two bf16 std values the kernel's __expf may give (kernel_checks.gaussian_std_range)."""
    m, eps = K._gaussian_input(B, L, h, w)
    cfg = O.QwenVaeConfig(z_dim=L, latents_mean=(O.QWEN_LATENTS_MEAN * 2)[:L], latents_std=(O.QWEN_LATENTS_STD * 2)[:L])
    mean_c = torch.tensor(cfg.latents_mean).to(DEV, torch.bfloat16)
    inv_c = 1.0 / torch.tensor(cfg.latents_std).to(DEV, torch.bfloat16)
    out = ops.gaussian_sample_scale(m, eps, mean_c, inv_c)
    torch.cuda.synchronize()
    mn = m.permute(0, 3, 1, 2)
    mean, logvar = mn[:, :L], mn[:, L:]
    s_lo, s_hi = K.gaussian_std_range(logvar)
    mc, ic = mean_c.view(1, L, 1, 1).float(), inv_c.view(1, L, 1, 1).float()

    def replay(std):
        z = (mean.float() + (std.float() * eps.float()).bfloat16().float()).bfloat16()
        return ((z.float() - mc).bfloat16().float() * ic).bfloat16()

    r_lo, r_hi = replay(s_lo), replay(s_hi)
    iv = torch.int16
    hit = (out.view(iv) == r_lo.view(iv)) | (out.view(iv) == r_hi.view(iv))
    n = int((~hit).sum().item())
    part = {"name": "out", "ok": n == 0, "n_bad": n, "numel": out.numel()}
    if n:
        K._first(~hit, out.float(), r_lo.float(), part)
    # the eager torch chain on the device, as the reference runs it (information: torch's expf is not __expf)
    std = torch.exp(0.5 * logvar.clamp(-30.0, 20.0))
    eager = ((mean + std * eps) - mean_c.view(1, L, 1, 1)) * inv_c.view(1, L, 1, 1)
    return K._combine(f"gaussian_channel_norm_B{B}_L{L}_{h}x{w}", [part], n_two_out=int((r_lo != r_hi).sum().item()),
                      n_vs_eager=int((eager.view(iv) != out.view(iv)).sum().item()))


def build_vae(cfg, P, device=DEV):
    from simpletuner_b200.vae.qwen_image import QwenImageVAE
    m = QwenImageVAE(**cfg.as_dict())
    m.load_state_dict({k: v.bfloat16() for k, v in P.items()}, strict=True)
    return m.to(device)


def model_parity(cfg, B=1, H=64, W=64, seed=0):
    """Moments and normalised latents of QwenImageVAE against the fp64 3-D oracle on the device; per-element
    tolerance MODEL_ATOL rms(ref) + MODEL_RTOL |ref|, worst tol_use reported."""
    P = O.init_params(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    px = (torch.rand(B, 3, 1, H, W, generator=g) * 2 - 1).bfloat16()
    eps = torch.randn(B, cfg.z_dim, 1, H // 8, W // 8, generator=g).bfloat16()
    vae = build_vae(cfg, P)
    dist = vae.encode(px.to(DEV)).latent_dist
    mom = dist.parameters
    lat = vae.encode_scaled(px.to(DEV), eps.to(DEV))
    torch.cuda.synchronize()
    P64 = {k: v.double().to(DEV) for k, v in P.items()}
    with torch.no_grad():
        m64 = O.encode3d(px.double().to(DEV), P64, cfg)
        l64 = O.sample_normalized(m64, eps.double().to(DEV), cfg)[:, :, 0]
    out = {"shape_moments": tuple(mom.shape), "shape_latents": tuple(lat.shape)}
    ok = mom.shape == m64.shape and lat.shape == l64.shape
    for nm, got, ref in (("moments", mom, m64), ("latents", lat, l64)):
        err = (got.double() - ref).abs()
        tol = MODEL_ATOL * ref.pow(2).mean().sqrt() + MODEL_RTOL * ref.abs()
        use = float((err / tol).max())
        out[f"{nm}_tol_use"] = round(use, 4)
        out[f"{nm}_max_err"] = float(err.max())
        out[f"{nm}_rel_rms"] = float((err.pow(2).mean() / ref.pow(2).mean()).sqrt())
        ok = ok and use <= 1.0 and bool(torch.isfinite(got).all())
    out["ok"] = ok
    out["tol_use"] = max(out["moments_tol_use"], out["latents_tol_use"])
    return out
