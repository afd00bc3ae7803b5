"""CPU: the Qwen-Image host logic and oracle pieces against tests/golden/qwen_image_golden.pt (the reference's own
functions), the config refusals, shim routing and the LoRA file round trip."""
from pathlib import Path

import pytest
import torch

from simpletuner_b200.qwen_image.model import QwenImage, default_config
from simpletuner_b200.qwen_image.transformer import (QwenImageTransformer2DModel, mask_hides_keys, qwen_key_bias,
                                                     qwen_rope_tables, qwen_timestep_proj)
from tests import qwen_image_oracle as QO
from tests.shim_stub import StubFoundation

G = torch.load(Path(__file__).parent / "golden" / "qwen_image_golden.pt", weights_only=False)
TINY = dict(num_layers=1, attention_head_dim=128, num_attention_heads=2, joint_attention_dim=64)


def test_rope_tables_equal_the_reference_bit_for_bit():
    for c in G["rope"]:
        cos, sin = qwen_rope_tables(c["h"], c["w"], c["S_txt"])
        L = c["S_txt"]
        assert torch.equal(cos[:L], c["txt_cos"]) and torch.equal(sin[:L], c["txt_sin"]), (c["h"], c["w"], L)
        assert torch.equal(cos[L:], c["img_cos"]) and torch.equal(sin[L:], c["img_sin"]), (c["h"], c["w"], L)
        ocos, osin = QO.rope(c["h"], c["w"], L)
        assert torch.equal(ocos, cos) and torch.equal(osin, sin)


def test_timestep_embedding_input_and_output_match_the_reference():
    te = G["temb"]
    proj = qwen_timestep_proj(te["t"])
    assert torch.equal(proj, te["proj"])
    assert torch.equal(QO.timestep_proj(te["t"]), te["proj"])
    p = {k: v.float() for k, v in te["params"].items()}
    x = proj.to(torch.bfloat16).float()
    ref = torch.nn.functional.linear(torch.nn.functional.silu(torch.nn.functional.linear(x, p["linear_1.weight"], p["linear_1.bias"])),
                                     p["linear_2.weight"], p["linear_2.bias"])
    assert torch.allclose(ref, te["temb"].float(), rtol=2e-2, atol=2e-2)


def test_modulate_matches_the_reference():
    m = G["modulate"]
    shift, scale, gate = m["mod"].chunk(3, dim=-1)
    assert torch.allclose(m["x"] * (1 + scale[:, None]) + shift[:, None], m["out"], atol=1e-6)
    assert torch.equal(gate[:, None], m["gate"])


def test_text_seq_len_rule_is_the_sum_rule_used_by_the_key_bias():
    for k, c in G["seq_len"].items():
        assert c["text_seq_len"] == c["mask"].shape[1]
        assert torch.equal(c["bool_mask"], c["mask"].bool())


@pytest.mark.parametrize("case", ["b1_full", "b1_padded", "b3_ragged", "b2_non_prefix", "b2_all_zero"])
def test_key_bias_reproduces_the_reference_processor(case):
    a, c = G["attn"], G["attn"]["cases"][case]
    H, hd = a["H"], a["hd"]
    P = {"p.attn." + k: v.float() for k, v in a["params"].items()}
    cfg = QO.QwenConfig(num_layers=0, attention_head_dim=hd, num_attention_heads=H)
    B, L = c["mask"].shape
    S_img = c["img"].shape[1]
    icos, isin, tcos, tsin = c["rope"]
    cosin = (torch.cat([tcos, icos]), torch.cat([tsin, isin]))
    bias = QO.key_bias(c["mask"], B, L, S_img)
    io, to = QO.attention(P, cfg, "p.attn.", c["img"], c["txt"], cosin, bias, None, 1.0)
    assert torch.allclose(io, c["img_out"], atol=2e-5, rtol=1e-4)
    # text query rows: the kept ones agree; padded ones differ on purpose (B > 1: the reference zeroes them)
    kept = ~torch.isinf(bias[:, :L]) if B > 1 else torch.ones(B, L, dtype=torch.bool)
    assert torch.allclose(to[kept], c["txt_out"][kept], atol=2e-5, rtol=1e-4)
    # the product's bias equals the oracle's, and the host decision agrees with it
    pb = qwen_key_bias(c["mask"], S_img, torch.float32)
    assert torch.equal(pb, bias)
    assert mask_hides_keys(c["mask"]) == bool(torch.isinf(bias).any())


def test_parameter_names_and_shapes_match_the_reference():
    ps = G["param_shapes"]
    m = QwenImageTransformer2DModel(**ps["config"])
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == ps["shapes"]
    assert QO.param_shapes(QO.QwenConfig(**{k: v for k, v in ps["config"].items()})) == ps["shapes"]


def test_qkv_parameters_share_one_fused_tensor():
    m = QwenImageTransformer2DModel(**TINY)
    D = m.inner_dim
    sd = {k: torch.randn(v.shape).bfloat16() for k, v in m.state_dict().items()}
    for phase in ("init", "load", "to"):
        if phase == "load":
            m.load_state_dict(sd, strict=True)
        if phase == "to":
            m.to(torch.bfloat16)
        a = m.transformer_blocks[0].attn
        for name, (q, k, v) in a.streams().items():
            w, b = a.fused[name]
            es = w.element_size()
            assert q.weight.data_ptr() == w.data_ptr()
            assert k.weight.data_ptr() - q.weight.data_ptr() == D * D * es
            assert v.weight.data_ptr() - k.weight.data_ptr() == D * D * es
            assert v.bias.data_ptr() - q.bias.data_ptr() == 2 * D * b.element_size()
    assert torch.equal(m.transformer_blocks[0].attn.to_k.weight, sd["transformer_blocks.0.attn.to_k.weight"])


@pytest.mark.parametrize("over,needle", [
    (dict(model_flavour="edit-v1"), "model_flavour"),
    (dict(model_flavour="edit-v2+"), "model_flavour"),
    (dict(model_type="full"), "model_type"),
    (dict(lora_type="lycoris"), "lora_type"),
    (dict(use_dora=True), "DoRA"),
    (dict(peft_lora_target_modules=["to_q", "img_mod.1"]), "img_mod.1"),
    (dict(peft_lora_target_modules=["proj_out"]), "proj_out"),
    (dict(peft_lora_target_modules=["norm_out.linear"]), "norm_out"),
    (dict(peft_lora_target_modules=["img_in"]), "img_in"),
    (dict(peft_lora_target_modules=["txt_in"]), "txt_in"),
    (dict(peft_lora_target_modules=["to_k", "txt_mod.1"]), "txt_mod.1"),
    (dict(tread_config={"routes": []}), "TREAD"),
    (dict(twinflow_enabled=True), "twinflow"),
    (dict(crepa_enabled=True), "crepa"),
    (dict(musubi_blocks_to_swap=10), "musubi"),
    (dict(controlnet=True), "controlnet"),
])
def test_unsupported_options_are_refused_at_load(over, needle):
    """What the shim refuses at load: validate_config, then the denoiser's rule for the resolved LoRA targets."""
    c = default_config(**over)
    with pytest.raises(NotImplementedError, match=needle):
        QwenImage.validate_config(c)
        QwenImageTransformer2DModel(**TINY).lora_target_linears(QwenImage.lora_targets(c))


def test_supported_flavours_validate():
    for fl in ("v1.0", "v2.0", None):
        QwenImage.validate_config(default_config(model_flavour=fl, peft_lora_target_modules=QO.ATTN + QO.MLP))


def test_per_batch_refusals():
    w = QwenImage(default_config(), transformer=QwenImageTransformer2DModel(**TINY), device=torch.device("cpu"))
    with pytest.raises(NotImplementedError, match="control_latent_list"):
        w.prepare_batch({"latent_batch": torch.zeros(1, 16, 4, 4), "prompt_embeds": torch.zeros(1, 4, 64),
                         "control_latent_list": [torch.zeros(1)]}, {})
    with pytest.raises(NotImplementedError, match="masked"):
        w.loss({"loss_mask_type": "mask"}, {})
    m = w._denoiser()
    for kw in ({"timestep_sign": torch.ones(1)}, {"modulate_index": torch.zeros(1)}):
        with pytest.raises(NotImplementedError):
            m(torch.zeros(1, 4, 64), torch.zeros(1, 4, 64), None, torch.zeros(1), [(1, 2, 2)], **kw)
    with pytest.raises(NotImplementedError, match="token-wise"):
        m(torch.zeros(1, 4, 64), torch.zeros(1, 4, 64), None, torch.zeros(1, 4), [(1, 2, 2)])
    for t in ("img_mod.1", "txt_mod.1", "img_in", "txt_in", "proj_out", "norm_out.linear"):
        with pytest.raises(NotImplementedError, match="not supported"):
            m.add_adapter(rank=4, target_modules=[t])
    with pytest.raises(NotImplementedError, match="scale|attention_kwargs"):
        m(torch.zeros(1, 4, 64), torch.zeros(1, 4, 64), None, torch.zeros(1), [(1, 2, 2)], attention_kwargs={"x": 1})


def test_load_state_dict_assign_and_replaced_parameters_are_refused():
    m = QwenImageTransformer2DModel(**TINY)
    D = m.inner_dim
    sd = {k: torch.randn(v.shape).bfloat16() for k, v in m.state_dict().items()}
    m.load_state_dict(sd, strict=True, assign=True)
    a = m.transformer_blocks[0].attn
    w, b = a.fused["img"]
    assert a.to_k.weight.data_ptr() - w.data_ptr() == D * D * 2 and torch.equal(w[D:2 * D], sd["transformer_blocks.0.attn.to_k.weight"])
    # a parameter replaced behind the module's back (as accelerate's set_module_tensor_to_device does) is re-fused by the
    # next plan build, so the projection reads the new weights
    new = torch.randn(D, D).bfloat16()
    a.add_v_proj.weight = torch.nn.Parameter(new, requires_grad=False)
    pl = m.transformer_blocks[0].plans()
    assert torch.equal(pl["txt_attn"].w_qkv[2 * D:], new)
    assert a.add_v_proj.weight.data_ptr() == pl["txt_attn"].w_qkv.data_ptr() + 2 * D * D * 2


def test_graphed_train_step_refuses_qwen_batches():
    from simpletuner_b200.training.step import GraphedTrainStep, TrainStep
    w = QwenImage(default_config(), transformer=QwenImageTransformer2DModel(**TINY), device=torch.device("cpu"))
    w.add_lora_adapter()
    g = GraphedTrainStep(TrainStep(w, torch.optim.AdamW(w._denoiser().trainable_parameters())))
    with pytest.raises(NotImplementedError, match="Qwen-Image"):
        g({"latent_batch": torch.zeros(1, 16, 4, 4), "prompt_embeds": torch.zeros(1, 4, 64)})


@pytest.mark.parametrize("schedule", ["constant", "exponential", "snr"])
def test_scheduled_huber_c_reads_the_unscaled_timesteps(schedule):
    """The reference's Qwen model_predict divides a copy of `timesteps` by 1000 (qwen_image/model.py:1281, :1177), so the
    loss's scheduled huber_c sees the raw [0, 1000] values (Flux overwrites them with t / 1000 first)."""
    from oracle import flux_oracle as O
    c = default_config(loss_type="huber", huber_c=0.1, huber_schedule=schedule)
    w = QwenImage(c, transformer=QwenImageTransformer2DModel(**TINY), device=torch.device("cpu"))
    t = torch.tensor([937.5, 120.0, 500.0])
    kind, hc = w._loss_kind({"timesteps": t.clone()})
    assert kind == "huber"
    assert torch.allclose(hc.float().reshape(-1).cpu(), O.scheduled_huber_c(t, 0.1, schedule, "flow_matching").reshape(-1))


def _ref_qwen():
    torch.manual_seed(0)
    m = QwenImageTransformer2DModel(**TINY)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02)
    return m


class RefQwen(StubFoundation):
    MODEL_CLASS = staticmethod(_ref_qwen)
    LORA_TARGETS = ["to_k", "to_q", "to_v", "to_out.0"]


def test_shim_swaps_in_the_qwen_path_and_keeps_the_reference_on_refusal():
    from simpletuner_b200.shim import make_b200_family
    kw = dict(lora_rank=4, model_type="lora", lora_type="standard")
    fam = make_b200_family(RefQwen, "qwen_image")(default_config(**kw), "cpu")
    fam.load_model()
    assert fam._b200 is not None and isinstance(fam._b200, QwenImage) and isinstance(fam.model, QwenImageTransformer2DModel)
    assert all(torch.equal(fam.model.state_dict()[k], v) for k, v in _ref_qwen().state_dict().items())
    fam.add_lora_adapter()
    assert len(fam.model.lora_linears()) == 4
    fam = make_b200_family(RefQwen, "qwen_image")(default_config(model_flavour="edit-v3", **kw), "cpu")
    fam.load_model()
    assert fam._b200 is None and "model_flavour" in fam._b200_fallback_reason
    fam.prepare_batch({"x": 1}, {})
    assert fam.calls[-1] == "ref.prepare_batch"


def test_lora_io_round_trip(tmp_path):
    from simpletuner_b200.training import lora_io
    m = QwenImageTransformer2DModel(**TINY)
    m.add_adapter(rank=4, target_modules=QO.ATTN + QO.MLP)
    with torch.no_grad():
        for p in m.trainable_parameters():
            p.normal_()
    state = lora_io.get_peft_model_state_dict(m)
    assert "transformer_blocks.0.img_mlp.net.0.proj.lora_A.weight" in state and len(state) == 2 * 12
    lora_io.save_lora_weights(str(tmp_path), transformer_lora_layers=state)
    from safetensors.torch import load_file
    raw = load_file(str(tmp_path / "pytorch_lora_weights.safetensors"))
    assert set(raw) == {"transformer." + k for k in state}
    loaded = lora_io.load_lora_weights(str(tmp_path))
    m2 = QwenImageTransformer2DModel(**TINY)
    m2.add_adapter(rank=4, target_modules=QO.ATTN + QO.MLP)
    lora_io.set_peft_model_state_dict(m2, loaded)
    assert all(torch.equal(a, b) for a, b in zip(m.trainable_parameters(), m2.trainable_parameters()))
