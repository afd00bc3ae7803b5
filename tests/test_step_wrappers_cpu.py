"""CPU: the step-wrapper surface the families share (simpletuner_b200/family.py) on tiny models — the options each family
refuses at load, the LoRA-target rule, LoRA attach, the shim's load-time target check, the packed layouts and the
constructors the benchmark uses.  Plumbing only: no kernel runs."""
import pytest
import torch

from simpletuner_b200.chroma import model as chroma_model
from simpletuner_b200.chroma.transformer import CHROMA_DEFAULT_LORA_TARGET, CHROMA_LORA_TARGETS, ChromaTransformer2DModel
from simpletuner_b200.flux import model as flux_model
from simpletuner_b200.flux.transformer import FLUX_LORA_TARGETS, FluxTransformer2DModel, Linear
from simpletuner_b200.pixart import model as pixart_model
from simpletuner_b200.pixart.transformer import PIXART_LORA_TARGETS, PixArtTransformer2DModel
from simpletuner_b200.qwen_image import model as qwen_model
from simpletuner_b200.qwen_image.transformer import QWEN_DEFAULT_LORA_TARGETS, QwenImageTransformer2DModel
from simpletuner_b200.sd3.model import SD3
from simpletuner_b200.sd3.transformer import SD3_LORA_TARGETS, SD3Transformer2DModel
from simpletuner_b200.sdxl import model as sdxl_model
from tests.shim_stub import StubFoundation
from tests.test_denoiser_surface_cpu import FLUX_TINY, PIXART_TINY, QWEN_TINY, SD3_TINY

CHROMA_TINY = dict(num_layers=1, num_single_layers=1, attention_head_dim=64, num_attention_heads=2, joint_attention_dim=32,
                   approximator_hidden_dim=64, approximator_layers=1, axes_dims_rope=(8, 28, 28))
CPU = torch.device("cpu")

# family -> (shim family key, step class, default_config, tiny denoiser)
FAMILIES = {
    "flux": ("flux", flux_model.Flux, flux_model.default_config, lambda: FluxTransformer2DModel(**FLUX_TINY)),
    "sd3": ("sd3", SD3, flux_model.default_config, lambda: SD3Transformer2DModel(**SD3_TINY)),
    "pixart": ("pixart_sigma", pixart_model.PixartSigma, pixart_model.default_config,
               lambda: PixArtTransformer2DModel(**PIXART_TINY)),
    "qwen": ("qwen_image", qwen_model.QwenImage, qwen_model.default_config, lambda: QwenImageTransformer2DModel(**QWEN_TINY)),
    "chroma": ("chroma", chroma_model.Chroma, chroma_model.default_config, lambda: ChromaTransformer2DModel(**CHROMA_TINY)),
}
ALL = set(FAMILIES)

# option -> the families whose validate_config refuses it
MATRIX = [
    *[(dict(**{k: v}), ALL) for k, v in (
        ("controlnet", True), ("model_type", "full"), ("lora_type", "loha"), ("use_dora", True), ("tread_config", {"a": 1}),
        ("flow_cubic_schedule", True), ("twinflow_enabled", True), ("crepa_enabled", True), ("layersync_enabled", True),
        ("diff2flow_enabled", True), ("scheduled_sampling_max_step_offset", 4), ("distillation_method", "dmd"),
        ("slider_lora_target", True))],
    (dict(control=True), {"chroma"}),
    (dict(lora_type="lycoris"), {"sd3", "pixart", "qwen", "chroma"}),
    *[(dict(**{k: v}), {"qwen", "chroma"}) for k, v in (
        ("musubi_blocks_to_swap", 2), ("flowmap_enabled", True), ("flow_map_enabled", True), ("mixflow_enabled", True))],
    (dict(enable_time_sign_embed=True), {"chroma"}),
    (dict(flux_attention_masked_training=True), {"flux"}),
    (dict(flux_lora_target="ai-toolkit"), {"flux"}),
    (dict(model_flavour="kontext"), {"qwen", "chroma"}),
    (dict(prediction_type="sample"), {"pixart"}),
]


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_validate_config_matrix(family):
    _, cls, cfg, _ = FAMILIES[family]
    cls.validate_config(cfg())
    for over, refused_by in MATRIX:
        if family in refused_by:
            with pytest.raises(NotImplementedError):
                cls.validate_config(cfg(**over))
        else:
            cls.validate_config(cfg(**over))


@pytest.mark.parametrize("mod,build", [
    (pixart_model, lambda c: pixart_model.PixartSigma(c, transformer=PixArtTransformer2DModel(**PIXART_TINY), device=CPU)),
    (sdxl_model, lambda c: sdxl_model.SDXL(c, device=CPU)),
], ids=["pixart", "sdxl"])
def test_prediction_type_rule_is_shared_by_pixart_and_sdxl(mod, build):
    bad = mod.default_config(prediction_type="sample")
    for refuse in (lambda: type(build(mod.default_config())).validate_config(bad), lambda: build(bad)):
        with pytest.raises(NotImplementedError, match="prediction_type"):
            refuse()
    w = build(mod.default_config(prediction_type="v_prediction"))
    assert w.PREDICTION_TYPE == "v_prediction" == w.noise_schedule.config.prediction_type
    assert type(w).PREDICTION_TYPE == "epsilon"


DEFAULTS = {"flux": FLUX_LORA_TARGETS["all"], "sd3": SD3_LORA_TARGETS, "pixart": PIXART_LORA_TARGETS,
            "qwen": QWEN_DEFAULT_LORA_TARGETS, "chroma": CHROMA_DEFAULT_LORA_TARGET}


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_lora_targets(family):
    _, cls, cfg, _ = FAMILIES[family]
    default = DEFAULTS[family]
    assert cls.lora_targets(cfg()) == default
    for raw in (None, "", "None", [], [None, "", "None", "  "]):
        assert cls.lora_targets(cfg(peft_lora_target_modules=raw)) == default
    assert cls.lora_targets(cfg(peft_lora_target_modules=[" to_q ", None, "", "None", "to_k"])) == ["to_q", "to_k"]
    assert cls.lora_targets(cfg(peft_lora_target_modules=("to_v",))) == ["to_v"]
    # manual targets are read for a standard LoRA only
    assert cls.lora_targets(cfg(peft_lora_target_modules=["to_q"], lora_type="lycoris")) == default
    for bad in ("to_q", ["to_q", 3]):
        with pytest.raises(ValueError, match="peft_lora_target_modules"):
            cls.lora_targets(cfg(peft_lora_target_modules=bad))
    with pytest.raises(NotImplementedError, match="slider"):
        cls.lora_targets(cfg(slider_lora_target=True))
    assert cls.lora_targets(cfg(slider_lora_target=True, peft_lora_target_modules=["to_q"])) == ["to_q"]


def test_flux_and_chroma_defaults_follow_flux_lora_target():
    for name, targets in FLUX_LORA_TARGETS.items():
        assert flux_model.Flux.lora_targets(flux_model.default_config(flux_lora_target=name)) == targets
    for name, targets in CHROMA_LORA_TARGETS.items():
        assert chroma_model.Chroma.lora_targets(chroma_model.default_config(flux_lora_target=name)) == targets
    # the other families do not read flux_lora_target
    assert SD3.lora_targets(flux_model.default_config(flux_lora_target="context")) == SD3_LORA_TARGETS


def _peft_selection(model, targets):
    return sorted(n for n, m in model.named_modules()
                  if isinstance(m, Linear) and any(n == t or n.endswith("." + t) for t in targets))


@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("manual", [None, ["to_q", "to_out.0"], [" to_k", "to_v"]])
def test_add_lora_adapter_adapts_the_peft_selection_of_the_resolved_targets(family, manual):
    _, cls, cfg, build = FAMILIES[family]
    c = cfg(lora_rank=4, peft_lora_target_modules=manual)
    w = cls(c, transformer=build(), device=CPU)
    den = w._denoiser()
    want = _peft_selection(den, cls.lora_targets(c))
    assert w.add_lora_adapter() == len(want)
    assert sorted(den.lora_linears()) == want


def _ref_family(family, targets):
    key, cls, cfg, build = FAMILIES[family]

    def make():
        torch.manual_seed(0)
        m = build()
        with torch.no_grad():
            for p in m.parameters():
                p.normal_(0, 0.02)
        return m

    ref = type("Ref", (StubFoundation,), {"MODEL_CLASS": staticmethod(make), "LORA_TARGETS": targets})
    from simpletuner_b200.shim import make_b200_family
    fam = make_b200_family(ref, key)(cfg(lora_rank=4, model_type="lora", lora_type="standard",
                                         peft_lora_target_modules=targets), "cpu")
    fam.load_model()
    return fam


@pytest.mark.parametrize("family,target,linear", [
    ("flux", "norm1.linear", "transformer_blocks.0.norm1.linear"),
    ("sd3", "ff.net.2", "transformer_blocks.0.ff.net.2"),
    ("pixart", "ff.net.2", "transformer_blocks.0.ff.net.2"),
    ("qwen", "img_mod.1", "transformer_blocks.0.img_mod.1"),
    ("chroma", "context_embedder", "context_embedder"),
])
def test_shim_falls_back_at_load_for_an_unadaptable_manual_target(family, target, linear):
    fam = _ref_family(family, ["to_q", target])
    assert fam._b200 is None and f"LoRA target {linear} " in fam._b200_fallback_reason
    fam.prepare_batch({"x": 1}, {})
    assert fam.calls[-1] == "ref.prepare_batch"


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_shim_installs_for_a_supported_manual_target(family):
    _, cls, _, _ = FAMILIES[family]
    fam = _ref_family(family, ["to_q"])
    assert isinstance(fam._b200, cls) and fam._b200_fallback_reason is None
    fam.add_lora_adapter()
    assert sorted(fam.model.lora_linears()) == _peft_selection(fam.model, ["to_q"])


@pytest.mark.parametrize("cls,order", [(flux_model.Flux, "cdydx"), (SD3, "dydxc"), (pixart_model.PixartSigma, "dydxc")])
def test_packed_layouts(cls, order):
    from simpletuner_b200.flux.functional import pack_latents, unpack_latents
    x = torch.randn(2, 16, 6, 8)
    packed = cls._pack(x)
    if order == "cdydx":
        assert torch.equal(packed, pack_latents(x, 2, 16, 6, 8))
        assert torch.equal(cls._unpack(packed, x.shape), unpack_latents(packed, 6 * 8, 8 * 8, 16))
    else:
        want = x.reshape(2, 16, 3, 2, 4, 2).permute(0, 2, 4, 3, 5, 1).reshape(2, 12, 64)
        assert torch.equal(packed, want)
    assert torch.equal(cls._unpack(packed, x.shape), x)


def test_bench_constructors_build():
    fx = flux_model.Flux(flux_model.default_config(lora_rank=4), transformer=FluxTransformer2DModel(**FLUX_TINY), device=CPU)
    assert fx.add_lora_adapter() == len(_peft_selection(fx.model, FLUX_LORA_TARGETS["all"]))
    lokr = flux_model.Flux(flux_model.default_config(lora_type="lycoris"), transformer=FluxTransformer2DModel(**FLUX_TINY),
                           device=CPU)
    assert len(lokr.add_lycoris_adapter({"algo": "lokr", "linear_dim": 10000, "factor": 4}).loras) > 0
    m = SD3Transformer2DModel(**SD3_TINY)
    m.enable_full_finetune()
    sd3 = SD3(flux_model.default_config(model_type="full"), transformer=m, device=CPU)
    assert sd3.model is m and sd3.PACKED_LAYOUT == "packed_dydxc"
    px = pixart_model.PixartSigma(pixart_model.default_config(lora_rank=4), transformer=PixArtTransformer2DModel(**PIXART_TINY),
                                  device=CPU)
    assert px.add_lora_adapter() == len(_peft_selection(px.model, PIXART_LORA_TARGETS))
    assert px.PREDICTION_TYPE == "epsilon" and px.noise_schedule.config.num_train_timesteps == 1000
