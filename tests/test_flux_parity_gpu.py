"""GPU (-m gpu): the libstb200 Flux training step (prepare_batch -> model_predict -> loss -> backward)
against the fp32 CPU oracle on identical weights, batch, noise and sigmas."""
import pytest
import torch

from tests import flux_parity as FP

pytestmark = pytest.mark.gpu


def _assert(res):
    import inspect
    FP.record(inspect.stack()[1].function, res)
    assert res["noisy_bit_exact"], res
    assert res["loss_rel_err"] <= FP.LOSS_RTOL, res
    assert res["pred_cos"] >= FP.PRED_COS, res
    assert res["grad_cos_min"] >= FP.GRAD_COS, res


def test_flux_step_parity_small():
    _assert(FP.run_parity())


def test_flux_step_parity_ragged_sequence():
    # S_img = 10*14 = 140 and S_txt = 77: nothing is a multiple of the 128-row tiles
    _assert(FP.run_parity(B=3, Hh=20, Ww=28, S_txt=77, seed=3))


def test_flux_step_parity_hd64():
    _assert(FP.run_parity(cfg=FP.small_config(layers=1, single=1, heads=4, hd=64), seed=5))


def test_flow_prep_matches_reference_golden(golden):
    """The reference's own _prepare_flow_noisy_latents output (bf16), reproduced bit-exactly by the kernel."""
    from simpletuner_b200 import ops

    lat = golden["noisy.bf16.latents"].cuda()
    eps = golden["noisy.bf16.noise"].cuda()
    sg = golden["noisy.bf16.sigmas"].cuda()
    noisy, packed = ops.flow_prep_pack(lat, eps, sg)
    assert torch.equal(noisy.cpu(), golden["noisy.bf16.out"])
    from simpletuner_b200.flux.functional import pack_latents
    assert torch.equal(packed.cpu(), pack_latents(golden["noisy.bf16.out"], 3, 16, 6, 10))


def test_lora_disabled_equals_base_model():
    cfg = FP.small_config(layers=1, single=1)
    from oracle import flux_oracle as O
    P = {k: v.bfloat16().float() for k, v in O.init_flux_params(cfg, seed=0).items()}
    L = {k: v.bfloat16().float() for k, v in O.init_lora_params(cfg, 16, seed=1, b_std=0.05).items()}
    w = FP.build_cuda_model(cfg, P, L, 16)
    batch = FP.make_batch(2, 16, 16, 64, cfg)
    torch.manual_seed(0)
    with torch.no_grad():
        prep = w.prepare_batch({k: v.clone() for k, v in batch.items()}, {})
        a = w.model_predict(dict(prep))["model_prediction"].clone()
        w._denoiser().disable_lora()
        prep2 = dict(prep)
        prep2["timesteps"] = prep["timesteps"] * 1000  # model_predict rescales in place (reference side effect)
        b = w.model_predict(prep2)["model_prediction"].clone()
        w._denoiser().enable_lora()
    assert not torch.equal(a, b)
    w0 = FP.build_cuda_model(cfg, P, None, 16)
    with torch.no_grad():
        prep3 = dict(prep)
        prep3["timesteps"] = prep["timesteps"] * 1000
        c = w0.model_predict(prep3)["model_prediction"]
    assert torch.equal(b, c)


@pytest.mark.parametrize("rank", [4, 32, 64, 128])
def test_flux_step_parity_other_ranks(rank):
    # rank 4 is zero-padded to 8 inside the packed LoRA stacks; rank 32 -> a 96-wide fused q|k|v rank block
    _assert(FP.run_parity(cfg=FP.small_config(layers=1, single=1), rank=rank, seed=7))


def test_flux_gradient_checkpointing_matches():
    """enable_gradient_checkpointing(): blocks are re-run in backward (torch.utils.checkpoint around the block Functions);
    the step result must stay inside the same tolerances, for every block and with an interval."""
    from tests import flux_parity as FP
    for kw in ({"checkpoint": True}, {"checkpoint": True, "interval": 2}):
        res = FP.run_parity(**kw)
        assert res["noisy_bit_exact"] and res["loss_rel_err"] <= FP.LOSS_RTOL and res["pred_cos"] >= FP.PRED_COS \
            and res["grad_cos_min"] >= FP.GRAD_COS, (kw, res)


@pytest.mark.parametrize("target,rank", [("all+ffs", 16), ("all+ffs+embedder", 8), ("context+ffs", 16), ("context", 16), ("all+ffs", 64)])
def test_flux_step_parity_lora_targets(target, rank):
    """flux_lora_target presets beyond "all" (reference flux/model.py:1263-1376): adapters on the feed-forward projections,
    the single blocks' proj_mlp / proj_out (input = cat[attn, mlp]), the final proj_out (PEFT suffix rule) and x_embedder."""
    res = FP.run_parity(cfg=FP.small_config(layers=2, single=2), rank=rank, seed=11, target=target, B=2, Hh=20, Ww=12, S_txt=40)
    if target == "all+ffs":
        assert res["n_lora_tensors"] == 2 * (2 * 12 + 2 * 5 + 1)
    _assert(res)


def test_flux_tiny_target_adapts_only_the_named_single_blocks():
    from oracle import flux_oracle as O
    from simpletuner_b200.flux.transformer import FLUX_LORA_TARGETS
    cfg = FP.small_config(layers=1, single=9)
    assert O.lora_target_names(cfg, tuple(FLUX_LORA_TARGETS["tiny"])) == ["single_transformer_blocks.7.proj_out"]   # 20 does not exist here
    res = FP.run_parity(cfg=cfg, rank=16, seed=13, target="tiny")
    assert res["n_lora_tensors"] == 2
    _assert(res)


def test_unsupported_lora_targets_raise():
    from simpletuner_b200.flux.model import Flux, default_config
    with pytest.raises(NotImplementedError):
        Flux.validate_config(default_config(flux_lora_target="ai-toolkit"))
    w = FP.build_cuda_model(FP.small_config(layers=1, single=1), {k: v for k, v in __import__("oracle.flux_oracle", fromlist=["x"]).init_flux_params(FP.small_config(layers=1, single=1)).items()}, None, 8)
    with pytest.raises(NotImplementedError):
        w._denoiser().add_adapter(rank=8, target_modules=["norm1.linear"])


def test_two_runs_give_bit_identical_lora_gradients():
    """The LoRA weight-gradient kernel writes per-split slabs and a second kernel adds them in index order, so two runs of
    the same step agree bit for bit, and stay within the parity tolerances."""

    def grads():
        from oracle import flux_oracle as O
        cfg = FP.small_config(layers=1, single=1)
        P = {k: v.bfloat16().float() for k, v in O.init_flux_params(cfg, seed=0).items()}
        L = {k: v.bfloat16().float() for k, v in O.init_lora_params(cfg, 16, seed=1, b_std=0.02).items()}
        w = FP.build_cuda_model(cfg, P, L, 16)
        batch = FP.make_batch(3, 24, 40, 77, cfg, seed=2)
        torch.manual_seed(7); torch.cuda.manual_seed(7)
        prep = w.prepare_batch({k: v.clone() for k, v in batch.items()}, {"global_step": 0})
        w.loss(prep, w.model_predict(prep)).backward()
        torch.cuda.synchronize()
        return {n: p.grad.clone() for n, p in w._denoiser().named_parameters() if p.grad is not None}

    a, b = grads(), grads()
    assert len(a) == 22 and all(torch.equal(a[k], b[k]) for k in a)
    _assert(FP.run_parity(cfg=FP.small_config(layers=1, single=1), seed=21))
