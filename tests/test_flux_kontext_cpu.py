"""CPU: Flux Kontext (model_flavour "kontext") — the host id builder and the fp32 oracle pieces against the reference's own
functions (tests/golden/flux_kontext_golden.pt, tools/make_golden_flux_kontext.py), the load-time rules, shim routing, the
batch conditions of both sampling modes, the 2-D timesteps `model_predict` leaves in the batch, and the guards that keep
conditioning inputs out of the plain Flux step."""
from pathlib import Path

import pytest
import torch

from simpletuner_b200.flux.model import Flux, default_config, kontext_ids
from simpletuner_b200.flux.transformer import FluxTransformer2DModel
from simpletuner_b200.shim import make_b200_family
from tests import flux_kontext_oracle as KO
from tests.test_shim_cpu import RefFlux, _ref_flux

GOLDEN = Path(__file__).resolve().parent / "golden" / "flux_kontext_golden.pt"


def _golden():
    return torch.load(GOLDEN, weights_only=False)


def _cfg(**over):
    kw = dict(lora_rank=4, model_type="lora", lora_type="standard", model_flavour="kontext")
    kw.update(over)
    return default_config(**kw)


def _wrapper(**over):
    return Flux(_cfg(**over), transformer=FluxTransformer2DModel(num_layers=1, num_single_layers=1, num_attention_heads=2,
                                                                 joint_attention_dim=64, pooled_projection_dim=32),
                device=torch.device("cpu"))


# ---- pinned against the reference ------------------------------------------------------------------------------------
def test_host_ids_equal_the_reference_bit_for_bit():
    cases = _golden()["pack"]
    assert any(float(c["ids"].float().max()) > 256 for c in cases)
    for c in cases:
        ids = kontext_ids(c["sizes"])
        ref = c["ids"]
        assert ref.dtype == torch.bfloat16 and ref.shape == (c["B"], ids.shape[0], 3)
        for b in range(c["B"]):
            assert torch.equal(ids, ref[b].float()), c["sizes"]


def test_oracle_packing_and_ids_equal_the_reference_bit_for_bit():
    for c in _golden()["pack"]:
        packed, ids = KO.build_kontext_inputs(c["latents"])
        assert torch.equal(packed, c["packed"]) and torch.equal(ids, c["ids"]), c["sizes"]


def test_oracle_timesteps_and_tokenwise_conditioning_match_the_reference():
    g = _golden()
    e = g["extend"]
    assert torch.equal(KO.extend_conditioning_timesteps(e["t"], e["S_scene"], e["S_c"]), e["out"])
    assert torch.equal(e["out"], torch.tensor([[0.1, 0.1, 0.1, 0.0, 0.0], [0.9, 0.9, 0.9, 0.0, 0.0]]))
    tw = g["tokenwise"]
    from oracle import flux_oracle as O
    cfg = O.FluxConfig(num_layers=0, num_single_layers=0, num_attention_heads=1, attention_head_dim=g["D"],
                       pooled_projection_dim=g["pooled_dim"], guidance_embeds=True)
    temb = KO.tokenwise_temb(tw["P"], cfg, tw["t2"], tw["guidance"], tw["pooled"])
    assert float((temb - tw["temb"]).abs().max()) <= 1e-5
    # the denoiser's closed form of the text stream's temb: the mean of the two distinct rows weighted by token counts
    S = tw["t2"].shape[1]
    S_c = int((tw["t2"][0] == 0).sum())
    scene, cond = temb[:, 0], temb[:, -1]
    closed = (scene * (S - S_c) + cond * S_c) / S
    assert float((closed - tw["temb_txt"]).abs().max()) <= 1e-5


def test_oracle_adaln_pieces_match_the_reference():
    a = _golden()["ada"]
    z = KO.ada_zero(a["zero"]["W"], a["zero"]["b"], a["x"], a["emb"], 6)
    zs = KO.ada_zero(a["single"]["W"], a["single"]["b"], a["x"], a["emb"], 3)
    c = KO.ada_continuous(a["continuous"]["W"], a["continuous"]["b"], a["x"], a["emb"])
    for got, ref in ((z, a["zero"]["out"]), (zs, a["single"]["out"])):
        assert len(got) == len(ref)
        for u, v in zip(got, ref):
            assert float((u - v).abs().max()) <= 1e-5
    assert float((c - a["continuous"]["out"]).abs().max()) <= 1e-5


def test_tokenwise_oracle_with_uniform_timesteps_is_the_plain_oracle():
    from oracle import flux_oracle as O
    from tests import flux_parity as FP
    cfg = FP.small_config(layers=1, single=1, hd=64)
    P = O.init_flux_params(cfg)
    b = FP.make_batch(2, 8, 8, 16, cfg)
    x = O.pack_latents(b["latent_batch"].float(), 2, 16, 8, 8)
    t = torch.tensor([0.3, 0.8])
    args = (b["prompt_embeds"].float(), b["add_text_embeds"].float())
    tok = KO.kontext_forward(P, cfg, x, *args, t[:, None].expand(-1, 16), O.prepare_latent_image_ids(8, 8),
                             torch.zeros(16, 3), torch.ones(2))
    plain = O.flux_forward(P, cfg, x, *args, t, O.prepare_latent_image_ids(8, 8), torch.zeros(16, 3), torch.ones(2))
    assert float((tok - plain).abs().max()) <= 1e-5


# ---- load-time rules and shim routing --------------------------------------------------------------------------------
@pytest.mark.parametrize("over", [dict(), dict(loss_type="huber", huber_schedule="constant"),
                                  dict(loss_type="smooth_l1", huber_schedule="constant")])
def test_kontext_configs_that_run(over):
    Flux.validate_config(_cfg(**over))


@pytest.mark.parametrize("lt,sched", [("huber", "snr"), ("huber", "exponential"), ("smooth_l1", "snr")])
def test_kontext_with_a_timestep_dependent_huber_schedule_raises(lt, sched):
    with pytest.raises(NotImplementedError, match="Kontext"):
        Flux.validate_config(_cfg(loss_type=lt, huber_schedule=sched))
    Flux.validate_config(_cfg(loss_type=lt, huber_schedule=sched, model_flavour=None))     # the plain step runs it


def test_shim_installs_the_h100_path_for_a_kontext_run():
    cls = make_b200_family(RefFlux, "flux")
    fam = cls(_cfg(), "cpu")
    fam.load_model()
    assert fam._b200 is not None and fam._b200_fallback_reason is None
    bad = cls(_cfg(loss_type="huber", huber_schedule="snr"), "cpu")
    bad.load_model()
    assert bad._b200 is None and "Kontext" in bad._b200_fallback_reason


# ---- batch conditions ------------------------------------------------------------------------------------------------
def _cond_batch(sizes, B=2):
    lat = [torch.randn(B, 16, h, w).bfloat16() for h, w in sizes]
    return {"latents": torch.zeros(B, 16, 16, 16), "conditioning_latents": list(lat)}, lat


@pytest.mark.parametrize("state", [{}, {"args": {}}, {"args": {"conditioning_multidataset_sampling": "random"}}])
def test_random_sampling_uses_the_first_conditioning_latent(state):
    w = _wrapper()
    batch, lat = _cond_batch([(8, 12), (16, 16)])
    conds, ids = w._kontext_conditions(batch, state)
    assert len(conds) == 1 and torch.equal(conds[0], lat[0])
    assert torch.equal(ids, kontext_ids([(8, 12)]))
    assert torch.equal(batch["conditioning_latents"], lat[0])      # the base class's list collapse


def test_combined_sampling_uses_every_conditioning_latent():
    w = _wrapper()
    batch, lat = _cond_batch([(8, 12), (16, 16), (6, 4)])
    batch["conditioning_type"] = "reference_strict"
    batch["conditioning_latents_type"] = ["reference_loose", "reference_strict", "reference_loose"]
    conds, ids = w._kontext_conditions(batch, {"args": {"conditioning_multidataset_sampling": "combined"}})
    assert [tuple(c.shape[2:]) for c in conds] == [(8, 12), (16, 16), (6, 4)]
    assert ids.shape == (4 * 6 + 8 * 8 + 3 * 2, 3) and torch.equal(ids, kontext_ids([(8, 12), (16, 16), (6, 4)]))
    # the base class then keeps the reference_strict element (common.py:4672-4683)
    assert torch.equal(batch["conditioning_latents"], lat[1])
    assert batch["conditioning_latents_type"] == "reference_strict"


def test_a_single_tensor_and_an_unbatched_latent_are_accepted():
    w = _wrapper()
    one = torch.randn(2, 16, 8, 8).bfloat16()
    conds, _ = w._kontext_conditions({"latents": torch.zeros(2, 16, 16, 16), "conditioning_latents": one}, {})
    assert len(conds) == 1 and torch.equal(conds[0], one)
    conds, _ = w._kontext_conditions({"latents": torch.zeros(1, 16, 16, 16), "conditioning_latents": one[0]}, {})
    assert conds[0].shape == (1, 16, 8, 8)
    with pytest.raises(ValueError, match="conditioning latents"):
        w._kontext_conditions({"latents": torch.zeros(3, 16, 16, 16), "conditioning_latents": one}, {})


def test_a_kontext_batch_without_conditioning_runs_the_plain_step():
    assert _wrapper()._kontext_conditions({"latents": torch.zeros(1, 16, 8, 8)}, {}) is None


# ---- model_predict's timesteps ---------------------------------------------------------------------------------------
class _Recorder(torch.nn.Module):
    def __init__(self, den):
        super().__init__()
        self.module = den
        self.kw = None

    def forward(self, **kw):
        self.kw = kw
        B, S = kw["hidden_states"].shape[:2]
        return (torch.zeros(B, S - kw.get("conditioning_tokens", 0), 64),)


def test_model_predict_leaves_the_reference_two_d_timesteps_in_the_batch():
    w = _wrapper()
    rec = _Recorder(w.model)
    w.model = rec
    B, Hh, Ww = 2, 4, 4                       # 4 scene tokens
    ids = kontext_ids([(2, 4)])               # 2 conditioning tokens
    pb = {"latents": torch.zeros(B, 16, Hh, Ww), "timesteps": torch.tensor([100.0, 900.0]),
          "encoder_hidden_states": torch.zeros(B, 3, 64), "added_cond_kwargs": {"text_embeds": torch.zeros(B, 32)},
          "_packed_noisy_latents": torch.zeros(B, 6, 64), "_kontext_ids": ids}
    out = w.model_predict(pb)
    assert torch.equal(pb["timesteps"], torch.tensor([[0.1, 0.1, 0.1, 0.1, 0.0, 0.0], [0.9, 0.9, 0.9, 0.9, 0.0, 0.0]]))
    assert rec.kw["conditioning_tokens"] == 2 and torch.equal(rec.kw["timestep"], torch.tensor([0.1, 0.9]))
    assert torch.equal(rec.kw["img_ids"][4:], ids) and rec.kw["img_ids"].shape == (6, 3)
    assert out["model_prediction"].shape == (B, 16, Hh, Ww)
    # a constant huber_c reads one value per sample from the 2-D timesteps
    w.config.loss_type, w.config.huber_schedule = "huber", "constant"
    kind, c = w._loss_kind(pb)
    assert kind == "huber" and c.shape == (B,)


# ---- guards ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["conditioning_latents", "conditioning_packed_latents", "conditioning_ids"])
def test_conditioning_inputs_outside_kontext_still_raise(key):
    w = _wrapper(model_flavour="dev")
    with pytest.raises(NotImplementedError, match="conditioning"):
        w.prepare_batch({"latent_batch": torch.zeros(1, 16, 4, 4), key: torch.zeros(1)}, {})


def test_prepacked_kontext_inputs_without_latents_raise():
    with pytest.raises(NotImplementedError, match="conditioning_latents"):
        _wrapper().prepare_batch({"latent_batch": torch.zeros(1, 16, 4, 4), "conditioning_packed_latents": torch.zeros(1)}, {})


def test_graphed_step_refuses_kontext_batches():
    from simpletuner_b200.training.step import GraphedTrainStep
    g = GraphedTrainStep.__new__(GraphedTrainStep)
    with pytest.raises(NotImplementedError, match="Kontext"):
        g({"conditioning_latents": torch.zeros(1)})


def test_masked_loss_still_raises_under_kontext():
    w = _wrapper()
    with pytest.raises(NotImplementedError, match="masked"):
        w.loss({"loss_mask_type": "mask"}, {"model_prediction": torch.zeros(1, 4, 64)}, apply_conditioning_mask=True)
