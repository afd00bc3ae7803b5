"""GPU: the Flux LoRA step with `flux_attention_masked_training` (default processor, SURVEY.md quirk Q2) against the masked
fp32 oracle (tests/flux_mask_oracle.py), within the tolerances of tests/flux_parity.py."""
import pytest
import torch

from tests import flux_mask_oracle as MO
from tests import flux_parity as FP

pytestmark = pytest.mark.gpu

LENGTHS = (5, 77, 40)


def _check(res):
    FP.record("flux_mask", res)
    assert MO.within_tolerance(res), res


def test_masked_step_matches_the_oracle():
    _check(MO.run_masked_parity(MO.length_mask(LENGTHS, 77), B=3, S_txt=77))


def test_masked_step_head_dim_64():
    _check(MO.run_masked_parity(MO.length_mask(LENGTHS, 77), cfg=FP.small_config(layers=1, single=1, heads=4, hd=64), B=3,
                                S_txt=77, seed=5))


def test_masked_step_with_gradient_checkpointing_interval():
    _check(MO.run_masked_parity(MO.length_mask(LENGTHS, 77), cfg=FP.small_config(layers=3, single=3), B=3, S_txt=77,
                                checkpoint=True, interval=2))


def test_masked_step_trains_the_text_stream_adapters():
    res = MO.run_masked_parity(MO.length_mask(LENGTHS, 77), B=3, S_txt=77, target="all+ffs")
    _check(res)
    assert res["text_stream_grads_nonzero"] > 0


def test_mask_with_zeros_changes_the_loss_and_all_ones_does_not():
    plain = MO.run_masked_parity(None, B=3, S_txt=77)
    zeros = MO.run_masked_parity(MO.length_mask(LENGTHS, 77), B=3, S_txt=77)
    ones = MO.run_masked_parity(torch.ones(3, 77), B=3, S_txt=77)
    _check(ones)
    _check(zeros)
    # the padded keys change what the step computes, in the oracle as on the GPU
    assert zeros["loss"] != plain["loss"] and zeros["loss_ref"] != plain["loss_ref"], (zeros, plain)
    # an all-ones mask adds the same +1 to every logit: both runs sit within the parity tolerance of one oracle value
    assert abs(ones["loss_ref"] - plain["loss_ref"]) <= 1e-5 * abs(plain["loss_ref"]), (ones, plain)
    assert abs(ones["loss"] - plain["loss"]) <= 2 * FP.LOSS_RTOL * abs(plain["loss"]), (ones, plain)


def test_graph_replay_with_different_masks_equals_the_eager_step():
    """GraphedTrainStep builds the key bias inside the captured step: replays with other masks give the eager bits."""
    from oracle import flux_oracle as O
    from simpletuner_b200.training.step import GraphedTrainStep, TrainStep

    cfg = FP.small_config()
    P = {k: v.bfloat16().float() for k, v in O.init_flux_params(cfg, seed=0).items()}
    L = {k: v.bfloat16().float() for k, v in O.init_lora_params(cfg, 16, seed=1, b_std=0.02).items()}

    def make():
        w = MO.masked_config(FP.build_cuda_model(cfg, P, L, 16))
        params = [p for p in w._denoiser().parameters() if p.requires_grad]
        return w, TrainStep(w, torch.optim.SGD(params, lr=0.1), max_grad_norm=0.0)

    wa, eager = make()
    wb, step_b = make()
    graphed = GraphedTrainStep(step_b, capture_prepare=False)
    base = FP.make_batch(2, 16, 16, 64, cfg, seed=3)
    masks = [MO.length_mask((10, 64), 64), MO.length_mask((33, 1), 64), MO.length_mask((64, 20), 64)]
    for i, m in enumerate(masks):
        batch = {**{k: v.clone() for k, v in base.items()}, "encoder_attention_mask": m.cuda()}
        torch.manual_seed(100 + i)
        torch.cuda.manual_seed(100 + i)
        le = eager(dict(batch))
        batch = {**{k: v.clone() for k, v in base.items()}, "encoder_attention_mask": m.cuda()}
        torch.manual_seed(100 + i)
        torch.cuda.manual_seed(100 + i)
        lg = graphed(dict(batch))
        torch.cuda.synchronize()
        assert torch.equal(le, lg), (i, float(le), float(lg))
    assert len(graphed._graphs) == 1
    pa = [p for p in wa._denoiser().parameters() if p.requires_grad]
    pb = [p for p in wb._denoiser().parameters() if p.requires_grad]
    assert all(torch.equal(x, y) for x, y in zip(pa, pb))
