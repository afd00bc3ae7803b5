"""CPU: the Chroma host logic and oracle pieces against tests/golden/chroma_golden.pt (the reference's own functions), the
state-dict names, the LoRA target lists, the refusals, shim routing and the LoRA file round trip."""
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from simpletuner_b200.chroma.model import Chroma, default_config, lora_targets
from simpletuner_b200.chroma.transformer import (CHROMA_DEFAULT_LORA_TARGET, CHROMA_LORA_TARGETS, ChromaTransformer2DModel,
                                                 adjust_chroma_sigmas, chroma_input_vec, chroma_key_bias, chroma_mod_proj)
from tests import chroma_oracle as CO
from tests.shim_stub import StubFoundation

G = torch.load(Path(__file__).parent / "golden" / "chroma_golden.pt", weights_only=False)
TINY = dict(num_layers=1, num_single_layers=1, attention_head_dim=64, num_attention_heads=2, joint_attention_dim=32,
            approximator_hidden_dim=64, approximator_layers=1, axes_dims_rope=(8, 28, 28))


def test_mod_proj_and_approximator_input_equal_the_reference_bit_for_bit():
    iv = G["input_vec"]
    mp = chroma_mod_proj(iv["rows"], 16)
    assert torch.equal(mp, iv["mod_proj"])
    # the wrapper's chain: bf16 timesteps (adjusted sigma x 1000) / 1000 in bf16, then the forward's .to(bf16) * 1000
    assert torch.equal(iv["t"].to(torch.bfloat16) * 1000, iv["t_model"])
    vec = chroma_input_vec(iv["t_model"], mp)
    assert vec.dtype == iv["vec"].dtype and torch.equal(vec, iv["vec"])


def _approx_replay(p, x, cfg, dtype, eps):
    """The reference's bf16 approximator chain with torch ops: a bf16 rounding after every module, RMSNorm eps `eps`.
    torch's RMSNorm multiplies by its weight in fp32 and rounds once."""
    P = {k: v.to(dtype) for k, v in p.items()}
    lin = lambda t, n: F.linear(t, P[n + ".weight"], P[n + ".bias"])
    h = lin(x.to(dtype), "in_proj")
    for i in range(cfg["n_layers"]):
        hf = h.float()
        n = (hf * torch.rsqrt(hf.pow(2).mean(-1, keepdim=True) + eps) * P[f"norms.{i}.weight"].float()).to(dtype)
        h = h + lin(F.silu(lin(n, f"layers.{i}.linear_1")), f"layers.{i}.linear_2")
    return lin(h, "out_proj")


def test_approximator_matches_the_reference_and_pins_the_rmsnorm_epsilon():
    a = G["approximator"]
    assert a["rmsnorm_eps"] is None                      # nn.RMSNorm(hidden_dim): eps left to torch
    P = {"distilled_guidance_layer." + k: v for k, v in a["params"].items()}
    cfg = CO.ChromaConfig(approximator_hidden_dim=a["config"]["hidden_dim"], approximator_layers=a["config"]["n_layers"])
    assert torch.allclose(CO.approximator(P, cfg, a["x"]), a["out_fp32"], rtol=1e-5, atol=1e-5)
    # bf16: torch takes the fp32 epsilon (2^-23), not torch.finfo(bfloat16).eps (2^-7); row [1, 4] is small enough to tell
    got = _approx_replay(a["params"], a["x"], a["config"], torch.bfloat16, torch.finfo(torch.float32).eps)
    assert torch.equal(got, a["out_bf16"])
    wrong = _approx_replay(a["params"], a["x"], a["config"], torch.bfloat16, torch.finfo(torch.bfloat16).eps)
    assert not torch.equal(wrong[1, 4], a["out_bf16"][1, 4])


def test_pruned_norms_chunk_order():
    n = G["norms"]
    x = n["x"]
    ln = lambda t: F.layer_norm(t, (t.shape[-1],), eps=1e-6)
    e6 = n["zero"]["emb"]           # image / text rows of a double block: shift, scale, gate, shift, scale, gate
    out, g, sh_m, sc_m, g_m = n["zero"]["out"]
    assert torch.allclose(out, ln(x) * (1 + e6[:, 1, None]) + e6[:, 0, None], atol=1e-6)
    assert torch.equal(g, e6[:, 2]) and torch.equal(sh_m, e6[:, 3]) and torch.equal(sc_m, e6[:, 4]) and torch.equal(g_m, e6[:, 5])
    e3 = n["single"]["emb"]         # single block: shift, scale, gate
    out, g = n["single"]["out"]
    assert torch.allclose(out, ln(x) * (1 + e3[:, 1, None]) + e3[:, 0, None], atol=1e-6) and torch.equal(g, e3[:, 2])
    e2 = n["continuous"]["emb"]     # norm_out: shift, then scale (the reverse of Flux's AdaLayerNormContinuous)
    assert torch.allclose(n["continuous"]["out"], ln(x) * (1 + e2[:, 1, None]) + e2[:, 0, None], atol=1e-6)
    # the forward passes TailFn (scale | shift): the rows flipped
    mod = e2.flip(1).reshape(e2.shape[0], -1)
    D = x.shape[-1]
    assert torch.equal(mod[:, :D], e2[:, 1]) and torch.equal(mod[:, D:], e2[:, 0])


def test_adjust_sigmas_bit_for_bit():
    s = G["sigmas"]
    assert torch.equal(adjust_chroma_sigmas(s["sigmas"].to(torch.bfloat16)), s["bf16"])
    assert torch.equal(adjust_chroma_sigmas(s["sigmas"]), s["fp32"])


@pytest.mark.parametrize("case", ["b2_ragged_2d", "b1_3d"])
def test_model_predict_mask_extension_and_timesteps(case):
    c = G["predict"][case]
    mask = c["mask"].squeeze(1) if c["mask"].dim() == 3 else c["mask"]
    B, L = mask.shape
    S_img = c["attention_mask"].shape[1] - L
    joint = torch.cat([mask > 0, torch.ones(B, S_img, dtype=torch.bool)], 1)
    assert torch.equal(joint, c["attention_mask"])
    bias = chroma_key_bias(joint, B, L + S_img, torch.bfloat16)
    assert torch.equal(torch.isinf(bias), ~c["attention_mask"]) and bool((bias[c["attention_mask"]] == 0).all())
    # Chroma.model_predict's timestep chain
    t = c["timesteps"].to(torch.bfloat16) / 1000
    assert torch.equal(t, c["timestep"])
    from simpletuner_b200.flux.model import prepare_latent_image_ids
    assert torch.equal(prepare_latent_image_ids(4, 6), c["img_ids"].float())
    assert not c["txt_ids"].any()


def test_modulation_rows_are_the_rows_the_reference_forward_hands_each_block():
    """The golden ran the reference's own forward with an approximator whose row r holds r and recorded the rows every
    block and norm_out received; ChromaTransformer2DModel.modulations must hand out the same rows, as views."""
    ro = G["row_offsets"]
    m = ChromaTransformer2DModel(**dict(TINY, num_layers=ro["n_double"], num_single_layers=ro["n_single"]))
    rows, D = m.mod_rows, m.inner_dim
    assert rows == 3 * ro["n_single"] + 12 * ro["n_double"] + 2 and G["input_vec"]["rows"] == 344 == 3 * 38 + 12 * 19 + 2
    pooled = torch.arange(rows, dtype=torch.float32)[None, :, None].expand(2, rows, D).contiguous()
    double, single, tail = m.modulations(pooled)
    ids = lambda t, k: t.view(2, k, D)[0, :, 0].tolist()
    assert [(ids(a, 6), ids(b, 6)) for a, b in double] == [tuple(x) for x in ro["double"]]
    assert [ids(t, 3) for t in single] == ro["single"]
    assert ids(tail, 2) == ro["norm_out"][::-1]              # TailFn reads (scale | shift)
    assert all(t.stride(0) == rows * D for pair in double for t in pair + tuple(single))


def test_state_dict_names_of_a_reference_shaped_model():
    ps = G["param_shapes"]
    cfg = dict(ps["config"])
    m = ChromaTransformer2DModel(**cfg)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == ps["shapes"]
    oc = CO.ChromaConfig(num_layers=cfg["num_layers"], num_single_layers=cfg["num_single_layers"],
                         attention_head_dim=cfg["attention_head_dim"], num_attention_heads=cfg["num_attention_heads"],
                         joint_attention_dim=cfg["joint_attention_dim"], approximator_hidden_dim=cfg["approximator_hidden_dim"],
                         approximator_layers=cfg["approximator_layers"])
    assert CO.param_shapes(oc) == ps["shapes"]
    sd = {k: torch.randn(v) for k, v in ps["shapes"].items()}
    m.load_state_dict({k: v.bfloat16() for k, v in sd.items()}, strict=True)


def _linear_names(m):
    from simpletuner_b200.flux.transformer import Linear
    return [n for n, mod in m.named_modules() if isinstance(mod, Linear)]


def _peft_selection(names, targets):
    return sorted(n for n in names if any(n == t or n.endswith("." + t) for t in targets))


@pytest.mark.parametrize("target", [None] + sorted(CHROMA_LORA_TARGETS))
def test_every_target_list_adapts_what_peft_would(target):
    c = default_config(flux_lora_target=target, lora_rank=4)
    want = CHROMA_DEFAULT_LORA_TARGET if target is None else CHROMA_LORA_TARGETS[target]
    assert lora_targets(c) == want
    Chroma.validate_config(c)
    w = Chroma(c, transformer=ChromaTransformer2DModel(**TINY), device=torch.device("cpu"))
    n = w.add_lora_adapter()
    den = w._denoiser()
    assert sorted(den.lora_linears()) == _peft_selection(_linear_names(den), want) and n == len(den.lora_linears())
    assert not any(k.startswith(("distilled_guidance_layer", "context_embedder")) for k in den.lora_linears())


def test_target_lists_differ_from_flux_where_the_reference_does():
    from simpletuner_b200.flux.transformer import FLUX_LORA_TARGETS
    assert CHROMA_LORA_TARGETS["tiny"] != FLUX_LORA_TARGETS["tiny"]
    assert "tiny+embedder" not in FLUX_LORA_TARGETS
    m = ChromaTransformer2DModel(**TINY)
    names = _linear_names(m)
    # ai-toolkit's adaLN names match nothing on Chroma: the same Linears as all+ffs
    assert _peft_selection(names, CHROMA_LORA_TARGETS["ai-toolkit"]) == _peft_selection(names, CHROMA_LORA_TARGETS["all+ffs"])
    assert lora_targets(default_config(flux_lora_target="no-such-list")) == CHROMA_DEFAULT_LORA_TARGET


@pytest.mark.parametrize("over,what", [
    (dict(lora_type="lycoris"), "lora_type"), (dict(use_dora=True), "DoRA"), (dict(slider_lora_target=True), "slider"),
    (dict(model_type="full"), "model_type"), (dict(controlnet=True), "ControlNet"), (dict(tread_config={"a": 1}), "TREAD"),
    (dict(mixflow_enabled=True), "mixflow"), (dict(crepa_enabled=True), "crepa"), (dict(twinflow_enabled=True), "twinflow"),
    (dict(flowmap_enabled=True), "flowmap"), (dict(flow_cubic_schedule=True), "cubic"),
    (dict(musubi_blocks_to_swap=2), "musubi"), (dict(distillation_method="dmd"), "distillation"),
    (dict(model_flavour="kontext"), "model_flavour"), (dict(peft_lora_target_modules=["linear_1"]), "linear_1"),
    (dict(peft_lora_target_modules=["context_embedder"]), "context_embedder"),
])
def test_unsupported_options_are_refused_at_load(over, what):
    """What the shim refuses at load: validate_config, then the denoiser's rule for the resolved LoRA targets."""
    c = default_config(**over)
    with pytest.raises(NotImplementedError, match=what):
        Chroma.validate_config(c)
        ChromaTransformer2DModel(**TINY).lora_target_linears(Chroma.lora_targets(c))


def test_model_and_batch_refusals():
    for k in ("enable_time_sign_embed", "musubi_blocks_to_swap", "deltatime_type"):
        with pytest.raises(NotImplementedError):
            ChromaTransformer2DModel(**TINY, **{k: {"deltatime_type": "r"}.get(k, True)})
    m = ChromaTransformer2DModel(**TINY)
    hs = torch.zeros(1, 4, 64)
    for kw in (dict(timestep_sign=torch.ones(1)), dict(r_timestep=torch.ones(1)), dict(grounding_kwargs={}),
               dict(controlnet_block_samples=[hs]), dict(force_keep_mask=torch.ones(1, 4)), dict(skip_layers=[0]),
               dict(joint_attention_kwargs={"ip_adapter_image_embeds": 1})):
        with pytest.raises(NotImplementedError):
            m(hs, torch.zeros(1, 2, 32), torch.ones(1), **kw)
    with pytest.raises(NotImplementedError, match="token-wise"):
        m(hs, torch.zeros(1, 2, 32), torch.ones(1, 4))
    w = Chroma(default_config(), transformer=m, device=torch.device("cpu"))
    with pytest.raises(NotImplementedError):
        w.add_lycoris_adapter({})
    for k in ("conditioning_latents", "twinflow_time_sign", "crepa_self_flow_mask"):
        with pytest.raises(NotImplementedError, match=k):
            w.prepare_batch({"latent_batch": torch.zeros(1, 16, 4, 4), k: torch.ones(1)}, {})
    with pytest.raises(ValueError, match="No attention mask"):
        w.model_predict({"latents": torch.zeros(1, 16, 4, 4)})
    with pytest.raises(NotImplementedError, match="masked"):
        w.loss({"loss_mask_type": "mask"}, {})


def test_graphed_train_step_refuses_chroma_batches():
    from simpletuner_b200.training.step import GraphedTrainStep, TrainStep
    w = Chroma(default_config(), transformer=ChromaTransformer2DModel(**TINY), device=torch.device("cpu"))
    w.add_lora_adapter()
    g = GraphedTrainStep(TrainStep(w, torch.optim.AdamW(w._denoiser().trainable_parameters())))
    with pytest.raises(NotImplementedError, match="Chroma"):
        g({"latent_batch": torch.zeros(1, 16, 4, 4), "prompt_embeds": torch.zeros(1, 4, 32)})


def test_sigma_schedule_is_skipped_for_fast_beta_and_uniform_schedules():
    lat = torch.zeros(2, 16, 4, 4, dtype=torch.bfloat16)
    s = torch.tensor([0.3, 0.8])
    w = Chroma(default_config(), transformer=ChromaTransformer2DModel(**TINY), device=torch.device("cpu"))
    sig, ts = w._model_sigmas(s, s * 1000, lat)
    assert sig.dtype == torch.bfloat16 and torch.equal(sig, adjust_chroma_sigmas(s.bfloat16()))
    assert torch.equal(ts, sig * 1000.0)
    for k in ("flux_fast_schedule", "flow_use_beta_schedule", "flow_use_uniform_schedule"):
        w.config = default_config(**{k: True})
        sig, ts = w._model_sigmas(s, s * 1000, lat)
        assert torch.equal(sig, s) and torch.equal(ts, s * 1000)


def _ref_chroma():
    torch.manual_seed(0)
    m = ChromaTransformer2DModel(**TINY)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02)
    return m


class RefChroma(StubFoundation):
    MODEL_CLASS = staticmethod(_ref_chroma)
    LORA_TARGETS = CHROMA_DEFAULT_LORA_TARGET


def test_shim_routes_chroma_only_when_named_and_keeps_the_reference_on_refusal():
    from simpletuner_b200.shim import foundation as FD
    from simpletuner_b200.shim import make_b200_family
    assert "chroma" not in FD.FAMILIES and FD.family_spec("chroma").registry_key == "chroma"
    kw = dict(lora_rank=4, model_type="lora", lora_type="standard")
    fam = make_b200_family(RefChroma, "chroma")(default_config(**kw), "cpu")
    fam.load_model()
    assert isinstance(fam._b200, Chroma) and isinstance(fam.model, ChromaTransformer2DModel)
    assert all(torch.equal(fam.model.state_dict()[k], v) for k, v in _ref_chroma().state_dict().items())
    fam.add_lora_adapter()
    assert len(fam.model.lora_linears()) == 4 + 3      # double block q, k, v, out; single block q, k, v
    fam = make_b200_family(RefChroma, "chroma")(default_config(use_dora=True, **kw), "cpu")
    fam.load_model()
    assert fam._b200 is None and "DoRA" in fam._b200_fallback_reason
    fam.prepare_batch({"x": 1}, {})
    assert fam.calls[-1] == "ref.prepare_batch"


def test_lora_io_round_trip(tmp_path):
    from simpletuner_b200.training import lora_io
    targets = CHROMA_LORA_TARGETS["all+ffs+embedder"]
    m = ChromaTransformer2DModel(**TINY)
    m.add_adapter(rank=4, target_modules=targets)
    with torch.no_grad():
        for p in m.trainable_parameters():
            p.normal_()
    state = lora_io.get_peft_model_state_dict(m)
    assert "single_transformer_blocks.0.proj_mlp.lora_A.weight" in state and "x_embedder.lora_B.weight" in state
    lora_io.save_lora_weights(str(tmp_path), transformer_lora_layers=state)
    from safetensors.torch import load_file
    raw = load_file(str(tmp_path / "pytorch_lora_weights.safetensors"))
    assert set(raw) == {"transformer." + k for k in state}
    m2 = ChromaTransformer2DModel(**TINY)
    m2.add_adapter(rank=4, target_modules=targets)
    lora_io.set_peft_model_state_dict(m2, lora_io.load_lora_weights(str(tmp_path)))
    assert all(torch.equal(a, b) for a, b in zip(m.trainable_parameters(), m2.trainable_parameters()))
