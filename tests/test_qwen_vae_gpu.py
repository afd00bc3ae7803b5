"""GPU: the Qwen-Image VAE encode path — 3x3 convs with C_in % 64 != 0, the per-channel latent normalisation, argument
refusals of the new entry points, and the whole encoder against the fp64 3-D oracle (tests/qwen_vae_checks.py)."""
import pytest
import torch

from tests import kernel_checks as K

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("C", [8, 16, 24, 32, 40, 96, 192, 256, 384, 512])
@pytest.mark.parametrize("silu,bias", [(True, False), (False, True), (False, False), (True, True)])
def test_channel_rmsnorm_interval_replay(C, silu, bias):
    from tests.qwen_vae_checks import check_channel_rmsnorm
    r = check_channel_rmsnorm(C=C, silu=silu, bias=bias)
    print(r)
    assert r["ok"], r


@pytest.mark.parametrize("R,C,eps", [(20001, 40, 1e-12), (300, 16, 0.5), (300, 384, 1e-3)])
def test_channel_rmsnorm_rows_and_eps(R, C, eps):
    from tests.qwen_vae_checks import check_channel_rmsnorm
    r = check_channel_rmsnorm(R=R, C=C, silu=False, eps=eps)
    print(r)
    assert r["ok"], r


def test_t5_rmsnorm_form_refuses_the_normalize_options():
    from simpletuner_b200 import ops
    x = torch.zeros(1, 4, 64, dtype=torch.bfloat16, device="cuda")
    w = torch.ones(64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError):
        ops.rmsnorm_fwd(x, w, 1e-6, silu=True)
    with pytest.raises(ValueError):
        ops.rmsnorm_fwd(x[:, ::2], w, 1e-12, normalize=True)


@pytest.mark.parametrize("ci,co,stride,H,W,res", [
    (32, 64, 1, 13, 21, False), (96, 96, 1, 17, 31, True), (96, 192, 1, 9, 140, False), (160, 128, 1, 11, 19, True),
    (40, 256, 1, 7, 9, False), (32, 32, 2, 16, 24, False), (96, 96, 2, 32, 200, False), (160, 64, 2, 12, 18, True)])
@pytest.mark.parametrize("exact", [False, True])
def test_conv3x3_channel_tail(ci, co, stride, H, W, res, exact):
    from tests.qwen_vae_checks import check_conv_padded
    r = check_conv_padded(B=2, H=H, W=W, Ci=ci, Co=co, stride=stride, res=res, exact=exact)
    print(r)
    assert r["ok"], r


@pytest.mark.parametrize("B,L,h,w", [(2, 16, 12, 20), (1, 16, 128, 128), (3, 8, 5, 7)])
def test_gaussian_sample_channel_norm_bits(B, L, h, w):
    from tests.qwen_vae_checks import check_gaussian_channel_norm
    r = check_gaussian_channel_norm(B, L, h, w)
    print(r)
    assert r["ok"], r


def test_new_entry_points_refuse_bad_arguments():
    from simpletuner_b200 import _lib
    lib = _lib.lib()
    x = torch.zeros(4096, dtype=torch.bfloat16, device="cuda")
    p = x.data_ptr()
    mis = p + 2
    rms = lambda xp, gp, bp, op, rows, C, eps=1e-12: lib.stb_channel_rmsnorm_nhwc(xp, gp, bp, op, rows, C, eps, 1, None)
    for args in [(p, p, None, p, 4, 4), (p, p, None, p, 4, 12), (p, p, None, p, 4, 520), (p, p, None, p, 0, 64),
                 (None, p, None, p, 4, 64), (p, None, None, p, 4, 64), (p, p, None, None, 4, 64),
                 (mis, p, None, p, 4, 64), (p, mis, None, p, 4, 64), (p, p, mis, p, 4, 64), (p, p, None, mis, 4, 64),
                 (p, p, None, p, 4, 64, -1.0), (p, p, None, p, 4, 64, float("inf")), (p, p, None, p, 4, 64, float("nan"))]:
        assert rms(*args) != 0, args
    smp = lambda mp, ep, op, B, L, hw, sp, ip: lib.stb_gaussian_sample_channel_norm(mp, ep, op, B, L, hw, sp, ip, None)
    for args in [(p, p, p, 1, 16, 4, None, p), (p, p, p, 1, 16, 4, p, None), (p, p, p, 0, 16, 4, p, p),
                 (p, p, p, 1, 0, 4, p, p), (p, p, p, 1, 16, 0, p, p), (None, p, p, 1, 16, 4, p, p), (p, p, None, 1, 16, 4, p, p)]:
        assert smp(*args) != 0, args
    conv = lambda ci, co: lib.stb_conv3x3_nhwc(p, p, None, None, p, 1, 4, 4, ci, co, 1, None)
    for ci, co in [(4, 64), (12, 64), (0, 64), (96, 4), (96, 12)]:
        assert conv(ci, co) != 0, (ci, co)
    torch.cuda.synchronize()


def test_qwen_vae_reduced_width_against_fp64_oracle():
    from oracle import qwen_vae_oracle as O
    from tests.qwen_vae_checks import model_parity
    r = model_parity(O.QwenVaeConfig(base_dim=32), B=2, H=64, W=96)
    print(r)
    assert r["ok"], r


@pytest.mark.parametrize("H", [256, 1024])
def test_qwen_vae_real_geometry_against_fp64_oracle(H):
    from oracle import qwen_vae_oracle as O
    from tests.qwen_vae_checks import model_parity
    r = model_parity(O.QwenVaeConfig(), B=1, H=H, W=H)
    print(r)
    assert r["ok"], r


def test_qwen_vae_is_reproducible_and_batch_independent():
    from oracle import qwen_vae_oracle as O
    from tests.qwen_vae_checks import build_vae
    cfg = O.QwenVaeConfig()
    vae = build_vae(cfg, O.init_params(cfg, 0))
    g = torch.Generator().manual_seed(5)
    px = (torch.rand(3, 3, 1, 128, 160, generator=g) * 2 - 1).bfloat16().cuda()
    a = vae.encode(px).latent_dist.parameters
    b = vae.encode(px).latent_dist.parameters
    assert torch.equal(a, b)
    one = torch.cat([vae.encode(px[i:i + 1]).latent_dist.parameters for i in range(3)])
    assert torch.equal(a, one)
