"""GPU: the shipped shims driven the way the reference drives them (tests/shim_stub.py reproduces `load_model`'s hook
order and `Trainer.model_predict` / `_compute_model_prediction_loss`): the reference-shaped call chain must give the same
loss and gradients as the direct B200 step, `model_prediction` must be the un-packed [B, C, H, W] tensor of seam B9, and the
attention-only seams (B3 / B4) must agree with torch SDPA in forward and backward."""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _family(seed=0, **over):
    from simpletuner_b200.shim import make_b200_family
    from tests.test_shim_cpu import RefFlux, _cfg

    fam = make_b200_family(RefFlux, "flux")(_cfg(**over), "cuda")
    fam.load_model()
    fam.add_lora_adapter()
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for lin in fam.model.lora_linears().values():
            lin.lora_B["default"].weight.normal_(0, 0.02, generator=g)
    return fam


def _batch(B=2, hw=16, s_txt=32, seed=3):
    g = torch.Generator().manual_seed(seed)
    return {"latent_batch": torch.randn(B, 16, hw, hw, generator=g).bfloat16(),
            "prompt_embeds": torch.randn(B, s_txt, 64, generator=g).bfloat16(),
            "add_text_embeds": torch.randn(B, 32, generator=g).bfloat16()}


def test_reference_shaped_step_matches_direct_b200_step():
    from tests.shim_stub import StubTrainer

    fam = _family()
    assert fam._b200 is not None, fam._b200_fallback_reason
    trainer = StubTrainer(fam, noise_scheduler=SimpleNamespace(config=SimpleNamespace(prediction_type="flow_matching")))
    torch.manual_seed(7); torch.cuda.manual_seed(7)
    prepared = fam.prepare_batch({k: v.clone() for k, v in _batch().items()}, {"global_step": 0})
    loss, logs, out = trainer.compute_model_prediction_loss(prepared)
    # seam B9 dict contract (trainer.py:6085-6087, flux/model.py:855-864)
    assert set(("model_prediction", "hidden_states_buffer", "crepa_hidden_states")) <= set(out)
    assert out["model_prediction"].shape == prepared["latents"].shape and out["hidden_states_buffer"] is None
    from simpletuner_b200.flux.functional import unpack_latents
    assert torch.equal(out["model_prediction"], unpack_latents(out["_packed_prediction"], 16 * 8, 16 * 8, 16))
    loss.backward()
    grads = {n: p.grad.clone() for n, p in fam.model.named_parameters() if p.grad is not None}
    assert len(grads) == 22
    # the same step through the B200 wrapper directly
    direct = fam._b200
    for p in fam.model.parameters():
        p.grad = None
    torch.manual_seed(7); torch.cuda.manual_seed(7)
    prep2 = direct.prepare_batch({k: v.clone() for k, v in _batch().items()}, {"global_step": 0})
    out2 = direct.model_predict(prep2)
    loss2 = direct.loss(prep2, out2)
    loss2.backward()
    assert torch.equal(prepared["noisy_latents"], prep2["noisy_latents"])
    assert torch.equal(out["model_prediction"], out2["model_prediction"])
    assert abs(float(loss) - float(loss2)) <= 1e-6 * abs(float(loss2))
    for n, p in fam.model.named_parameters():
        if p.grad is not None:   # the same step through the same kernels
            assert torch.equal(p.grad, grads[n]), n
    # a loss computed by the CALLER from the un-packed prediction (what reference code downstream of B9 may do) agrees
    target = (prep2["noise"].float() - prep2["latents"].float())
    ref_loss = F.mse_loss(out2["model_prediction"].float(), target, reduction="none").mean(dim=(1, 2, 3)).mean()
    assert abs(float(ref_loss) - float(loss2)) <= 2e-5 * abs(float(loss2))


def test_x_prediction_fixup_through_the_stub_trainer():
    from tests.shim_stub import StubTrainer

    fam = _family()
    trainer = StubTrainer(fam, noise_scheduler=SimpleNamespace(config=SimpleNamespace(prediction_type="sample")))
    torch.manual_seed(7); torch.cuda.manual_seed(7)
    prepared = fam.prepare_batch({k: v.clone() for k, v in _batch().items()}, {"global_step": 0})
    with torch.no_grad():
        raw = fam.model_predict(prepared_batch=dict(prepared))["model_prediction"]
    # (model_predict rescales `timesteps` in the dict it is given — the shallow copy above keeps `prepared` untouched)
    loss, _, out = trainer.compute_model_prediction_loss(prepared)
    assert torch.equal(out["model_prediction"], raw - prepared["noise"])
    target = prepared["noise"].float() - prepared["latents"].float()
    expect = F.mse_loss((raw - prepared["noise"]).float(), target, reduction="none").mean(dim=(1, 2, 3)).mean()
    assert abs(float(loss) - float(expect)) <= 2e-5 * abs(float(expect))


@pytest.mark.parametrize("B,S,H,HD", [(2, 300, 4, 128), (1, 257, 3, 64)])
def test_packed_attention_backend_matches_sdpa_forward_and_backward(B, S, H, HD):
    from simpletuner_b200.shim import attention_backend as AB

    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B, S, 3, H, HD, device="cuda", generator=g).bfloat16().requires_grad_(True)
    do = torch.randn(B, S, H, HD, device="cuda", generator=g).bfloat16()
    out = AB.flash_attn_qkvpacked_func(qkv, 0.0, None, False)
    assert out.shape == (B, S, H, HD)
    out.backward(do)
    q32 = qkv.detach().float().requires_grad_(True)
    q, k, v = (t.transpose(1, 2) for t in q32.unbind(2))
    ref = F.scaled_dot_product_attention(q, k, v).transpose(1, 2)
    ref.backward(do.float())
    cos = lambda a, b: float(F.cosine_similarity(a.flatten().float(), b.flatten().float(), dim=0))
    assert cos(out, ref) >= 0.9999 and float((out.float() - ref).abs().max()) <= 2e-2
    assert cos(qkv.grad, q32.grad) >= 0.9995
    with pytest.raises(NotImplementedError):
        AB.flash_attn_qkvpacked_func(qkv, 0.1, None, False)
    with pytest.raises(NotImplementedError):
        AB.flash_attn_qkvpacked_func(qkv, 0.0, None, True)
    assert not hasattr(AB, "flash_attn_varlen_func")


def test_sdpa_override_installs_falls_back_and_restores():
    from simpletuner_b200.shim import attention_backend as AB

    stock = F.scaled_dot_product_attention
    try:
        AB.install_sdpa_override()
        assert getattr(F.scaled_dot_product_attention, "_b200", False) and F.scaled_dot_product_attention_sdpa is stock
        g = torch.Generator(device="cuda").manual_seed(1)
        q, k, v = (torch.randn(2, 4, 200, 128, device="cuda", generator=g).bfloat16() for _ in range(3))
        from simpletuner_b200 import ops
        ops.reset_launch_count()
        out = F.scaled_dot_product_attention(q, k, v)
        assert ops.launch_count() >= 1                      # ran on libstb200
        ref = stock(q.float(), k.float(), v.float())
        assert float((out.float() - ref).abs().max()) <= 2e-2
        # unsupported arguments follow the reference's convention: fall back to the stock kernel, no exception
        n0 = ops.launch_count()
        mask = torch.zeros(200, 200, device="cuda", dtype=torch.bfloat16)
        out_m = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        assert ops.launch_count() == n0 and out_m.shape == out.shape
        out_f = F.scaled_dot_product_attention(q.float(), k.float(), v.float())
        assert out_f.dtype == torch.float32 and ops.launch_count() == n0
    finally:
        AB.restore_sdpa()
    assert F.scaled_dot_product_attention is stock


def test_vae_shim_swaps_encode_with_vae():
    from oracle import vae_oracle as O
    from simpletuner_b200.shim import B200VAEMixin
    from tests import vae_parity as VP

    cfg = VP.small_config()
    P = {k: v.bfloat16().float() for k, v in O.init_vae_params(cfg, seed=0).items()}
    ref_vae = VP.build_cuda_vae(cfg, P)                      # stands in for the diffusers AutoencoderKL (same names / config)
    ref_vae.state_dict_full = None

    class RefFamily:
        def __init__(self):
            self.vae = ref_vae
            self.accelerator = SimpleNamespace(device=torch.device("cuda"))
            self.calls = []

        def post_vae_load_setup(self):
            self.calls.append("ref.post_vae_load_setup")

        def encode_with_vae(self, vae, samples):
            self.calls.append("ref.encode_with_vae")
            return vae.encode(samples)

    fam = type("FamB200", (B200VAEMixin, RefFamily), {})()
    fam.post_vae_load_setup()                                # common.py:2747 — called at the end of load_vae
    assert fam.calls == ["ref.post_vae_load_setup"] and fam._b200_vae is not None
    g = torch.Generator().manual_seed(5)
    px = (torch.rand(1, 3, 64, 64, generator=g) * 2 - 1).bfloat16().cuda()
    out = fam.encode_with_vae(fam.vae, px)                   # caching/vae.py:1331-1343 reads .latent_dist.sample()
    assert "ref.encode_with_vae" not in fam.calls
    z = out.latent_dist.sample()
    assert z.shape == (1, 16, 8, 8) and torch.isfinite(z.float()).all()
    # same weights, same kernels: equal up to the fp32-atomics summation order of the GroupNorm statistics
    a, b = out.latent_dist.parameters.float().flatten(), ref_vae.encode(px).latent_dist.parameters.float().flatten()
    assert float(torch.nn.functional.cosine_similarity(a, b, dim=0)) >= 0.9999
    other = SimpleNamespace(encode=lambda s_: "reference-encode")
    assert fam.encode_with_vae(other, px) == "reference-encode" and fam.calls[-1] == "ref.encode_with_vae"   # a VAE that is not self.vae
