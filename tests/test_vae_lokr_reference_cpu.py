"""CPU: the reference model of the VAE-encode, LoKr and LoRA-dropout kernel checks in tests/kernel_checks.py.

Each host replay is held against the chain it stands for: the GroupNorm interval against fp32 emulations of the
statistics (pivoted, as the kernel sums, and unpivoted, which it must exclude at mean / sigma = 64), the SiLU criterion
against the eager module chain, the softmax range against torch's softmax, the latent-sample replay against the eager
bf16 chain of the reference, the LoKr rebuild's single rounding against lycoris's fp32 chain, and the numpy dropout mask
against an independent torch implementation."""
import math

import numpy as np
import pytest
import torch

import tests.kernel_checks as KC

F = torch.nn.functional


@pytest.fixture(autouse=True)
def _on_cpu(monkeypatch):
    monkeypatch.setattr(KC, "DEV", "cpu")


def _eq(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def _inside(got, lo, hi):
    return (lo.float() <= got.float()) & (got.float() <= hi.float())


def _gn_emulate(x, gamma, beta, G, eps, pivoted):
    """GroupNorm with fp32 statistics: numpy's pairwise fp32 sums of x - p and (x - p)^2 around the kernel's pivot
    (pivoted) or of x and x^2 (p = 0), d = S1 / n, var = S2 / n - d^2, rstd in fp32, and the output x a + b,
    b = beta - (p + d) a, as one rounding (an FMA).  Returns (y fp32 [B, HW, C], chain length of the sums)."""
    B, HW, C = x.shape
    cpg = C // G
    xf = x.float().numpy().reshape(B, HW, G, cpg)
    piv = KC.gn_pivot(x, G).float().numpy() if pivoted else np.zeros((B, G), np.float32)
    y = np.empty_like(xf)
    n = HW * cpg
    inv = np.float32(1) / np.float32(n)
    g32, b32 = gamma.float().numpy().reshape(G, cpg), beta.float().numpy().reshape(G, cpg)
    for b in range(B):
        for g in range(G):
            t = (xf[b, :, g, :] - piv[b, g]).astype(np.float32)
            tt = np.ascontiguousarray(t).ravel()
            s1, s2 = np.sum(tt, dtype=np.float32), np.sum(tt * tt, dtype=np.float32)
            d = np.float32(s1 * inv)
            var = max(np.float32(np.float32(s2 * inv) - np.float32(d * d)), np.float32(0))
            r = np.float32(1) / np.sqrt(np.float32(var + np.float32(eps)), dtype=np.float32)
            a = (r * g32[g]).astype(np.float32)
            sh = (b32[g] - np.float32(piv[b, g] + d) * a).astype(np.float32)
            y[b, :, g, :] = (xf[b, :, g, :].astype(np.float64) * a + sh).astype(np.float32)
    return torch.from_numpy(y.reshape(B, HW, C)), 32 + math.ceil(math.log2(n))


def _gn_case(ratio, C=128, G=32, B=2, HW=24 * 32, const=False, beta0=False):
    x = KC._gn_input(B, HW, C, G, ratio, const)
    gm = (1.0 + 0.1 * KC._rand(C, seed=2).float()).bfloat16()
    bt = torch.zeros(C, dtype=torch.bfloat16) if beta0 else KC._rand(C, scale=0.1, seed=3)
    return x, gm, bt


@pytest.mark.parametrize("ratio", [0.0, 4.0, 16.0, 64.0, 256.0])
@pytest.mark.parametrize("C,G", [(128, 32), (512, 32), (128, 64)])
def test_groupnorm_interval_holds_pivoted_fp32_statistics(ratio, C, G):
    x, gm, bt = _gn_case(ratio, C, G)
    y32, L = _gn_emulate(x, gm, bt, G, 1e-6, pivoted=True)
    y, err = KC.gn_reference(x, gm, bt, G, 1e-6, L=L)
    lo, hi = KC._bf16_range(y, err)
    assert bool(_inside(y32.bfloat16(), lo, hi).all())
    # one candidate almost everywhere; at large offsets the FMA form's u |mean a| widens the range of small outputs
    assert float((lo == hi).double().mean()) > (0.9 if ratio <= 16 else 0.7)


def test_groupnorm_interval_excludes_the_unpivoted_variance():
    # E[x^2] - mean^2 in fp32 loses ~ (mean / sigma)^2 of its precision: at mean / sigma = 64 its outputs leave the range
    # on a measurable share of elements, while at 0 they stay inside
    x, gm, bt = _gn_case(64.0)
    y, err = KC.gn_reference(x, gm, bt, 32, 1e-6, L=32 + math.ceil(math.log2(24 * 32 * 4)))
    lo, hi = KC._bf16_range(y, err)
    flat, _ = _gn_emulate(x, gm, bt, 32, 1e-6, pivoted=False)
    assert float((~_inside(flat.bfloat16(), lo, hi)).double().mean()) > 0.02
    x0, gm0, bt0 = _gn_case(0.0)
    y0, err0 = KC.gn_reference(x0, gm0, bt0, 32, 1e-6, L=32 + math.ceil(math.log2(24 * 32 * 4)))
    assert bool(_inside(_gn_emulate(x0, gm0, bt0, 32, 1e-6, pivoted=False)[0].bfloat16(), *KC._bf16_range(y0, err0)).all())


def test_groupnorm_chains_follow_the_chunking():
    # 512 x 512 at C = 128, B = 1 on 132 SMs: 528 CTAs of 497 pixels, 16 threads per vector column, cpg 4
    assert KC.gn_chains(1, 512 * 512, 128, 32) == 32 + 0 + 16 * 4 + 528
    assert KC.gn_chains(2, 7, 512, 32) == 2 + 7 + 4 * 2 + 1                   # 4 rows over 7 pixels; cpg 16: 2 vectors


@pytest.mark.parametrize("beta0", [True, False])
def test_groupnorm_constant_groups_stay_at_beta(beta0):
    # sigma = 0: rstd = 1 / sqrt(eps), and the output is beta up to the rounding of b = beta - mean a
    x, gm, bt = _gn_case(0.0, B=2, HW=77, const=True, beta0=beta0)
    y32, L = _gn_emulate(x, gm, bt, 32, 1e-6, pivoted=True)
    y, err = KC.gn_reference(x, gm, bt, 32, 1e-6, L=L)
    grp = (torch.arange(2 * 32).view(2, 32) % 3 == 0)[:, None, :, None].expand(2, 77, 32, 4).reshape(2, 77, 128)
    assert _eq(y[grp].float().bfloat16(), bt.expand(2, 77, 128)[grp])
    assert bool(_inside(y32.bfloat16(), *KC._bf16_range(y, err)).all())


def test_silu_criterion_accepts_the_eager_module_chain_and_rejects_a_dropped_rounding():
    # nn.GroupNorm's bf16 output, then nn.SiLU (fp32 inside, rounded once)
    x, gm, bt = _gn_case(4.0, C=256, HW=1536)
    y32, L = _gn_emulate(x, gm, bt, 32, 1e-6, pivoted=True)
    v = y32.bfloat16()
    assert KC.silu_check("eager", F.silu(v), v, v)["ok"]
    y, err = KC.gn_reference(x, gm, bt, 32, 1e-6, L=L)
    lo, hi = KC._bf16_range(y, err)
    assert KC.silu_check("eager_range", F.silu(v), lo, hi)["ok"]
    # SiLU of the unrounded fp32 value lands outside on a fraction of the elements
    assert KC.silu_check("unrounded", F.silu(y32).bfloat16(), lo, hi)["n_bad"] > 0


@pytest.mark.parametrize("cols", [8, 24, 1024, 2056, 4096])
def test_softmax_range_holds_torch_softmax(cols):
    scale = 0.0442
    s = KC._softmax_rows_input(16, cols, scale, 20.0)
    lo, hi, p, _ = KC.softmax_range(s, scale)
    ref = torch.softmax(s.float() * KC._f32(scale), -1).bfloat16()
    assert bool(_inside(ref, lo, hi).all())
    assert _eq(lo[0], torch.full((cols,), 1.0 / cols, dtype=torch.float32).bfloat16()) and _eq(hi[0], lo[0])
    assert float((lo == hi)[4:].double().mean()) > 0.9


def test_softmax_ramp_row_needs_the_whole_row_max():
    # with the max of the first 256 columns only, the ramp row's largest scaled logits are ~90 above it: exp overflows
    scale, cols = 0.0442, 1024
    s = KC._softmax_rows_input(4, cols, scale, 20.0).float()
    z = (s[3] - s[3, :256].max()) * scale
    assert not bool(torch.isfinite(torch.exp(z).sum()))


def test_gaussian_replay_holds_the_eager_chain():
    # diffusers DiagonalGaussianDistribution.sample on bf16 tensors, then (z - shift) * scale
    B, L, h, w = 3, 16, 13, 21
    m, eps = KC._gaussian_input(B, L, h, w)
    mn = m.permute(0, 3, 1, 2)
    mean, logvar = mn[:, :L], mn[:, L:]
    std = torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0))
    assert bool((logvar == -40).any() and (logvar == 25).any() and (logvar == -29.875).any())
    lo, hi = KC.gaussian_std_range(logvar)
    assert bool(_inside(std, lo, hi).all()) and int((lo != hi).sum()) < 0.01 * lo.numel()
    # the tensor part of the chain; the scaling's Python scalars are fp32 in torch's CUDA ops, as in the kernel (torch's
    # CPU bf16 ops round them to bf16 first, so they are not compared here)
    z = mean + std * eps
    r_lo, r_hi = KC.gaussian_replay(mean, lo, eps, None, 1.0), KC.gaussian_replay(mean, hi, eps, None, 1.0)
    assert bool(((z == r_lo) | (z == r_hi)).all())
    # the replay keeps the rounding of std * eps: fusing it changes some outputs
    fused = (mean.float() + std.float() * eps.float()).bfloat16()
    assert not bool(((fused == r_lo) | (fused == r_hi)).all())
    # and the shift is subtracted, not added
    r = KC.gaussian_replay(mean, lo, eps, 0.1159, 0.3611)
    assert not bool((r == KC.gaussian_replay(mean, lo, eps, -0.1159, 0.3611)).all())


@pytest.mark.parametrize("a,b,c,d,scale", [(3, 37, 5, 13, 0.75), (4, 40, 6, 32, 1 / 3), (48, 64, 48, 64, 0.75),
                                           (16, 192, 16, 768, 0.75)])
def test_lokr_rebuild_replay_is_one_exact_rounding(a, b, c, d, scale):
    N, K = a * b, c * d
    W = KC._rand(N, K, seed=61) * 0.05
    w1, w2 = KC._rand(a, c, seed=62), KC._rand(b, d, seed=63) * 0.05
    want, single = KC.lokr_rebuild_replay(W, w1, w2, scale)
    assert single
    # an fp32 FMA emulated per element: the fp32 product scale * w1, then one rounding of s1 w2 + W
    s1 = (w1.float() * KC._f32(scale)).double()
    i = torch.arange(N)[:, None]
    k = torch.arange(K)[None, :]
    fma = (s1[i // b, k // d] * w2.double()[i % b, k % d] + W.double()).float().bfloat16()
    assert _eq(want, fma)
    n_diff = int((want.view(torch.int16) != KC.lokr_eager(W, w1, w2, scale).view(torch.int16)).sum())
    print(f"lokr {a}x{b} {c}x{d} scale {scale:.4g}: {n_diff} of {N * K} elements differ from lycoris's fp32 chain")
    assert n_diff < 0.01 * N * K


def test_lokr_exact_inputs_are_order_free():
    # integers x 2^-4: every fp32 partial sum is exact, so fp32 sums in two different orders equal fp64
    a, b, c, d = 6, 300, 3, 16
    w1, w2 = KC._gen(a, c, seed=64, exact="frac"), KC._gen(b, d, seed=65, exact="frac")
    dW = KC._gen(a * b, c * d, seed=66, exact="int")
    g4 = dW.reshape(a, b, c, d)
    r1 = torch.einsum("ajcl,jl->ac", g4.double(), w2.double())
    m1 = torch.einsum("ajcl,jl->ac", g4.double().abs(), w2.double().abs())
    assert KC.exact_bound_ok([dW], [w1, w2], m1)
    prods = (g4.float() * w2.float()[None, :, None, :]).permute(0, 2, 1, 3).reshape(a, c, -1)
    fwd = torch.zeros(a, c)
    for t in range(prods.shape[-1]):
        fwd = fwd + prods[..., t]
    assert torch.equal(fwd.double(), r1) and torch.equal(prods.flip(-1).sum(-1, dtype=torch.float32).double(), r1)


def _mix32_torch(h):
    M = 0xFFFFFFFF
    h = h ^ (h >> 16)
    h = (h * 0x85EBCA6B) & M
    h = h ^ (h >> 13)
    h = (h * 0xC2B2AE35) & M
    return h ^ (h >> 16)


def _keep_torch(seed, stream, idx, p):
    M = 0xFFFFFFFF
    lo, hi = idx & M, idx >> 32
    inner = _mix32_torch((hi + stream * 0x85EBCA77 + seed) & M)
    h = _mix32_torch((lo * 0x9E3779B1 + inner) & M)
    return (h >> 8) >= round(float(np.float32(p)) * 2 ** 24)


@pytest.mark.parametrize("p", [0.0, 0.1, 0.5])
def test_dropout_mask_matches_an_independent_implementation(p):
    idx = torch.cat([torch.arange(20000, dtype=torch.int64), torch.arange(2 ** 32 - 50, 2 ** 32 + 50, dtype=torch.int64)])
    for seed, stream in ((1234, 7), (0, 0), (2 ** 32 - 1, 2 ** 32 - 2)):
        keep = KC.dropout_keep_np(seed, stream, idx.numpy().astype(np.uint64), p)
        assert np.array_equal(keep, _keep_torch(seed, stream, idx, p).numpy())
    rate = float(KC.dropout_keep_np(1234, 7, np.arange(200000, dtype=np.uint64), p).mean())
    assert abs(rate - (1 - p)) < 5e-3


def test_dropout_masks_are_stream_addressed_and_independent():
    m = KC.dropout_masks(3, 2, 77, 200, 0.1, 1234, 7)
    assert torch.equal(m[1], KC.dropout_masks(1, 2, 77, 200, 0.1, 1234, 8)[0])
    assert abs(float((m[0] & m[1]).double().mean()) - 0.81) < 0.01
    wrap = KC.dropout_masks(3, 1, 5, 8, 0.5, 1, 0xFFFFFFFE)
    assert torch.equal(wrap[2], KC.dropout_masks(1, 1, 5, 8, 0.5, 1, 0)[0])
    assert KC.dropout_thresh(0.1) == 1677722 and KC.dropout_thresh(0.0) == 0
    assert float(KC.dropout_inv_keep(0.1)) == float(np.float32(1) / (np.float32(1) - np.float32(0.1)))


def test_dropout_accum_replay_brackets_the_eager_chain():
    # eager: dx + d_m * keep_m * inv, one member at a time in fp32; the two-rounding replay is exactly that
    keep = KC.dropout_masks(3, 2, 10, 16, 0.5, 5, 0)
    d, dx0 = KC._rand(3, 2, 10, 16, seed=1), KC._rand(2, 10, 16, seed=2)
    inv = KC.dropout_inv_keep(0.5)
    acc = dx0.float()
    for m in range(3):
        acc = acc + torch.where(keep[m], d[m].float() * inv, torch.zeros(()))
    fma, twice = KC.dropout_accum_replay(dx0, d, keep, inv)
    assert _eq(twice, acc.bfloat16()) and _eq(fma, twice)                 # inv = 2: both orders are exact
