"""CPU: the reference model of the row-wise kernel checks in tests/kernel_checks.py.

The checks replay the eager bf16 module chains (diffusers adaLN modulation, RMSNorm + _apply_rotary_emb_anyshape, the
T5LayerNorm, the gradients of conditional_loss) from an interval around the fp64 normalised value; here each replay is
held bit for bit against the chain written as the modules write it, and each interval against the eager result."""
import math

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
    return bool(((lo.float() <= got.float()) & (got.float() <= hi.float())).all())


def _rows(B, S, D, eps, seed=0):
    x = KC._rand(B, S, D, seed=seed)
    KC._ln_edge_rows(x, eps)
    return x


@pytest.mark.parametrize("D,eps", [(72, 1e-6), (1000, 1e-6), (768, 1e-5), (3072, 1e-6), (8192, 1e-6)])
def test_ln_modulate_replay_is_the_eager_chain(D, eps):
    B, S = 2, 12
    x = _rows(B, S, D, eps)
    mod = KC._rand(B, 6 * D, seed=1, scale=0.3)
    shift, scale = mod[:, :D], mod[:, D:2 * D]
    n = torch.nn.LayerNorm(D, elementwise_affine=False, eps=eps)(x)          # bf16 module, fp32 inside
    eager = n * (1 + scale[:, None]) + shift[:, None]
    assert _eq(KC.ln_modulate_replay(n, scale, shift), eager)
    lo, hi = KC.ln_interval(x, eps, KC.ln_vpt(D))
    assert _inside(n, lo, hi)                                                 # random, zero, constant, offset, tiny rows
    assert _eq(n[:, 0], torch.zeros_like(n[:, 0])) and _eq(eager[:, 0], shift)
    assert float((lo == hi)[:, 4:].float().mean()) > 0.9                      # one candidate on almost every random row


def test_ln_interval_rejects_a_dropped_rounding():
    # the fused variant bf16(n t1 + shift) (one rounding instead of two) leaves the replay on a measurable share
    B, S, D = 2, 64, 3072
    x = _rows(B, S, D, 1e-6)
    mod = KC._rand(B, 6 * D, seed=1, scale=0.3)
    shift, scale = mod[:, :D], mod[:, D:2 * D]
    n = F.layer_norm(x.float(), (D,), eps=1e-6).bfloat16()
    lo, hi = KC.ln_interval(x, 1e-6, KC.ln_vpt(D))
    a, b = KC.ln_modulate_replay(lo, scale, shift), KC.ln_modulate_replay(hi, scale, shift)
    t1 = (1 + scale.float()).bfloat16().float()[:, None]
    fused = (n.float() * t1 + shift.float()[:, None]).bfloat16()
    outside = ~((torch.minimum(a, b).float() <= fused.float()) & (fused.float() <= torch.maximum(a, b).float()))
    assert float(outside.float().mean()) > 0.01


def _diffusers_rmsnorm(x, w, eps):
    h = x.float()
    h = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + eps)
    return h.to(torch.bfloat16) if w is None else h.to(w.dtype) * w


def _eager_rope(y, cos, sin):
    # _apply_rotary_emb_anyshape, use_real_unbind_dim = -1: (x.float() * cos + x_rotated.float() * sin).to(x.dtype)
    x_real, x_imag = y.reshape(*y.shape[:-1], -1, 2).unbind(-1)
    x_rot = torch.stack([-x_imag, x_real], dim=-1).flatten(3)
    return (y.float() * cos + x_rot.float() * sin).to(y.dtype)


@pytest.mark.parametrize("HD,paired,weights", [(128, True, True), (128, False, True), (64, False, False), (64, True, True)])
def test_rmsnorm_rope_replay_is_the_eager_chain(HD, paired, weights):
    B, S, H, eps = 2, 40, 3, 1e-6
    x = KC._rand(B, S, H, HD, seed=2)
    x[:, 5] = 0
    w = (KC._rand(HD, seed=3, scale=0.2) + 1) if weights else None
    cos, sin = KC._rope_tables(S, HD, paired=paired)
    y = _diffusers_rmsnorm(x, w, eps)
    lo, hi = KC.rms_range(x, w, eps, HD // 32 + 5)
    assert _inside(y, lo, hi) and _eq(KC.rms_weight_replay(_diffusers_rmsnorm(x, None, eps), w), y)
    c, s = cos[None, :, None, :], sin[None, :, None, :]
    eager = _eager_rope(y, c, s)
    modes = KC.rope_modes(y, KC._rot(y), c, s)
    assert _eq(modes[0], eager)
    assert bool((eager[:, 5] == 0).all())
    rlo, rhi = KC.rope_range(lo, hi, c, s)
    assert all(_inside(m, rlo, rhi) for m in modes)


def test_rope_range_rejects_a_swapped_sine():
    # o_2j = y_2j c_2j - y_2j+1 s_2j: with tables whose pair members differ, s_2j+1 in its place leaves the range
    B, S, H, HD = 1, 40, 2, 128
    x = KC._rand(B, S, H, HD, seed=4)
    cos, sin = KC._rope_tables(S, HD, paired=False)
    lo, hi = KC.rms_range(x, None, 1e-6, HD // 32 + 5)
    c, s = cos[None, :, None, :], sin[None, :, None, :]
    rlo, rhi = KC.rope_range(lo, hi, c, s)
    y = lo
    s_swapped = KC._swap(s.expand(B, S, H, HD))
    wrong = _eager_rope(y, c, torch.where(torch.arange(HD) % 2 == 0, s_swapped, s))
    assert not _inside(wrong, rlo, rhi)


@pytest.mark.parametrize("D", [8, 264, 4096])
def test_t5_layernorm_chain(D):
    # transformers T5LayerNorm: bf16 x * rsqrt(fp32 variance + eps) (fp32), cast to the weight dtype, * weight
    x = KC._rand(2, 20, D, seed=5)
    x[:, 0] = 0
    w = (1 + 0.1 * KC._rand(D, seed=6).float()).bfloat16()
    var = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
    t5 = w * (x * torch.rsqrt(var + 1e-6)).to(w.dtype)
    lo, hi = KC.rms_range(x, w, 1e-6, 8 * ((D + 255) // 256) + 5)
    assert _inside(t5, lo, hi) and bool((t5[:, 0] == 0).all()) and bool(torch.isfinite(t5).all())
    assert float((lo == hi).float().mean()) > 0.9


def _flux_pack(x):
    B, C, Hh, Ww = x.shape
    return x.view(B, C, Hh // 2, 2, Ww // 2, 2).permute(0, 2, 4, 1, 3, 5).reshape(B, (Hh // 2) * (Ww // 2), 4 * C)


def _sd3_patchify(x):
    B, C, Hh, Ww = x.shape
    return x.reshape(B, C, Hh // 2, 2, Ww // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, (Hh // 2) * (Ww // 2), 4 * C)


def test_unpack_inverts_the_model_layouts():
    x = KC._rand(2, 4, 6, 8, seed=7)
    assert _eq(KC.unpack_nchw(_flux_pack(x), 0, 2, 4, 6, 8), x)
    assert _eq(KC.unpack_nchw(_sd3_patchify(x), 1, 2, 4, 6, 8), x)
    # and the SD3 unpatchify of the reference, "nhwpqc->nchpwq"
    p = _sd3_patchify(x)
    ref = torch.einsum("nhwpqc->nchpwq", p.reshape(2, 3, 4, 2, 2, 4)).reshape(2, 4, 6, 8)
    assert _eq(KC.unpack_nchw(p, 1, 2, 4, 6, 8), ref)


def _conditional_loss_grad(pred, tgt, loss_type, c, w):
    """fp32 autograd of conditional_loss: the pointwise loss of pred.float() - target.float(), mean over (C, H, W),
    * min-SNR weights, mean over the batch."""
    p = pred.float().requires_grad_(True)
    if loss_type == "l2":
        l = F.mse_loss(p, tgt.float(), reduction="none")
    else:
        cb = c.view(-1, 1, 1, 1)
        k = 2 * cb if loss_type == "huber" else 2.0
        l = k * (torch.sqrt((p - tgt.float()) ** 2 + cb ** 2) - cb)
    l = l.mean(dim=[1, 2, 3])
    if w is not None:
        l = l * w
    l.mean().backward()
    return p.grad


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
def test_l2_grad_replay_is_autograd(weighted, grad_scale):
    # power-of-two B and C H W: every scaling of both orders is exact, so the kernel's order and autograd's agree bit for bit
    B, C, Hh, Ww = 4, 4, 16, 32
    pred, tgt = KC._rand(B, C, Hh, Ww, seed=8), KC._rand(B, C, Hh, Ww, seed=9)
    w = torch.tensor(KC.MIN_SNR_W[:B]) if weighted else None
    d = pred.float() - tgt.float()
    rep = KC.loss_grad_replay(d, "l2", None, w, KC._f32_inv(C * Hh * Ww, B), grad_scale)
    assert len(rep) == 1
    assert _eq(rep[0], (_conditional_loss_grad(pred, tgt, "l2", None, w) * grad_scale).bfloat16())


@pytest.mark.parametrize("loss_type", ["huber", "smooth_l1"])
def test_root_grad_replay_is_autograd_to_one_ulp(loss_type):
    # autograd differentiates sqrt and the square separately: the same value to a few fp32 ulps, so after the bf16 cast
    # one of the replay's candidates almost everywhere and a bf16 neighbour everywhere
    B, C, Hh, Ww = 4, 4, 16, 32
    pred, tgt = KC._rand(B, C, Hh, Ww, seed=10), KC._rand(B, C, Hh, Ww, seed=11)
    c = torch.tensor(KC.HUBER_C[:B])
    d = pred.float() - tgt.float()
    rep = KC.loss_grad_replay(d, loss_type, c, None, KC._f32_inv(C * Hh * Ww, B), 1.0)
    auto = _conditional_loss_grad(pred, tgt, loss_type, c, None).bfloat16()
    hit = (auto == rep[0]) | (auto == rep[1]) | (auto == rep[2])
    assert float(hit.float().mean()) > 0.99
    lo, hi = KC._bf16_steps(rep[0])
    assert bool(((lo <= auto.double()) & (auto.double() <= hi)).all())


@pytest.mark.parametrize("loss_type", ["l2", "huber", "smooth_l1"])
def test_loss_bound_covers_fp32_sums(loss_type):
    # a sequential fp32 sum, the worst order for the bound's L, stays inside loss_bound for L = n
    B, C, Hh, Ww = 2, 4, 16, 16
    pred, tgt = KC._rand(B, C, Hh, Ww, seed=12), KC._rand(B, C, Hh, Ww, seed=13)
    c = torch.tensor(KC.HUBER_C[:B]) if loss_type != "l2" else None
    d64 = pred.double() - tgt.double()
    lv = KC.loss_value64(d64, loss_type, c.double() if c is not None else None).float().flatten()
    acc = torch.zeros((), dtype=torch.float32)
    for v in lv:
        acc = acc + v
    loss32 = float(acc * KC._f32_inv(C * Hh * Ww, B))
    bound, ref = KC.loss_bound(d64, loss_type, c.double() if c is not None else None, None, lv.numel())
    assert abs(loss32 - ref) <= bound and math.isfinite(bound)
