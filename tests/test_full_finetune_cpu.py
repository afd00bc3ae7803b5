"""CPU: the trainer-facing surface of full fine-tuning (model_type=full) for SD3 and PixArt — which families admit it at
load, the shim turning it on with one process-wide optimizer post-hook, and the diffusers checkpoint layout of
`save_pretrained` / `from_config` / `register_to_config`.  Plumbing only: no kernel runs."""
import json
from dataclasses import replace

import pytest
import torch
from safetensors.torch import load_file

from oracle import pixart_oracle as PO
from oracle import sd3_oracle as SO
from simpletuner_b200.pixart.transformer import PixArtTransformer2DModel
from simpletuner_b200.pretrained import CONFIG_NAME, WEIGHTS_NAME
from simpletuner_b200.sd3.transformer import SD3Transformer2DModel
from simpletuner_b200.shim import foundation
from tests.shim_stub import StubFoundation
from tests.test_denoiser_surface_cpu import PIXART_TINY, SD3_TINY
from tests.test_step_wrappers_cpu import FAMILIES, MATRIX

FULL_FT = {"sd3", "pixart"}


@pytest.mark.parametrize("family", sorted(FULL_FT))
def test_full_finetune_validation_matrix(family):
    """`validate_full_finetune` admits model_type=full where the family can fine-tune every weight, with the shared refusal
    matrix on top; `validate_config` stays the LoRA run's check and refuses it."""
    _, cls, cfg, _ = FAMILIES[family]
    assert cls.FULL_FINETUNE
    with pytest.raises(NotImplementedError, match="only LoRA training"):
        cls.validate_config(cfg(model_type="full"))
    cls.validate_full_finetune(cfg(model_type="full"))
    for over, refused_by in MATRIX:
        cfg_over = cfg(**{"model_type": "full", **over})
        if over.get("model_type") == "full" or family not in refused_by:
            cls.validate_full_finetune(cfg_over)
        else:
            with pytest.raises(NotImplementedError):
                cls.validate_full_finetune(cfg_over)


@pytest.mark.parametrize("family", sorted(set(FAMILIES) - FULL_FT))
def test_full_finetune_stays_refused_elsewhere(family):
    _, cls, cfg, _ = FAMILIES[family]
    assert not cls.FULL_FINETUNE
    for check in (cls.validate_config, cls.validate_full_finetune):
        with pytest.raises(NotImplementedError, match="only LoRA training"):
            check(cfg(model_type="full"))


@pytest.mark.parametrize("family", sorted(FULL_FT))
@pytest.mark.parametrize("over", [dict(lora_type="lycoris"), dict(use_dora=True), dict(controlnet=True)],
                         ids=["lycoris", "dora", "controlnet"])
def test_full_finetune_with_an_adapter_option_is_refused(family, over):
    _, cls, cfg, _ = FAMILIES[family]
    with pytest.raises(NotImplementedError):
        cls.validate_full_finetune(cfg(model_type="full", **over))


def _random(m):
    torch.manual_seed(0)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02)
    return m


def _full_family(family):
    key, cls, cfg, build = FAMILIES[family]
    ref = type("Ref", (StubFoundation,), {"MODEL_CLASS": staticmethod(lambda: _random(build())), "LORA_TARGETS": None})
    fam = foundation.make_b200_family(ref, key)(cfg(model_type="full", peft_lora_target_modules=["ff.net.2"]), "cpu")
    fam.load_model()
    return fam


def test_shim_enables_full_finetune_and_registers_one_optimizer_hook(monkeypatch):
    monkeypatch.setattr(foundation, "_STEP_HOOK", None)
    monkeypatch.setattr(foundation, "_FULL_FT_MODELS", foundation.weakref.WeakSet())
    from torch.optim import optimizer
    registered = []
    real = optimizer.register_optimizer_step_post_hook

    def register(hook):
        registered.append(hook)
        return real(hook)

    monkeypatch.setattr(optimizer, "register_optimizer_step_post_hook", register)
    fams = [_full_family(f) for f in sorted(FULL_FT)]
    try:
        assert len(registered) == 1
        for fam in fams:
            den = fam.model
            # a LoRA target left in the config does not matter for a full fine-tune
            assert fam._b200 is not None and fam._b200_fallback_reason is None, fam._b200_fallback_reason
            assert den._full_ft and all(p.requires_grad for p in den.parameters())
            assert den in foundation._FULL_FT_MODELS
            for blk in den.transformer_blocks:
                blk._plans = {"stale": True}
        # any optimizer step of the process drops the derived layouts of every tracked model
        p = torch.nn.Parameter(torch.ones(3))
        p.grad = torch.ones(3)
        torch.optim.SGD([p], lr=0.1).step()
        assert all(blk._plans is None for fam in fams for blk in fam.model.transformer_blocks)
        # weakly referenced: a dropped model leaves the set
        n = len(foundation._FULL_FT_MODELS)
        del fams[0].model, fams[0]._b200, fams[0]
        import gc
        gc.collect()
        assert len(foundation._FULL_FT_MODELS) == n - 1
    finally:
        foundation._STEP_HOOK.remove()


def test_lora_run_does_not_enable_full_finetune():
    key, cls, cfg, build = FAMILIES["pixart"]
    ref = type("Ref", (StubFoundation,), {"MODEL_CLASS": staticmethod(lambda: _random(build())), "LORA_TARGETS": None})
    fam = foundation.make_b200_family(ref, key)(cfg(lora_rank=4), "cpu")
    fam.load_model()
    assert not getattr(fam.model, "_full_ft", False) and fam.model not in foundation._FULL_FT_MODELS


def _reference_names(kind):
    if kind == "sd3":
        c = SD3_TINY
        cfg = SO.SD3Config(sample_size=c["sample_size"], num_layers=c["num_layers"], attention_head_dim=c["attention_head_dim"],
                           num_attention_heads=c["num_attention_heads"], joint_attention_dim=c["joint_attention_dim"],
                           caption_projection_dim=c["caption_projection_dim"], pooled_projection_dim=c["pooled_projection_dim"],
                           out_channels=c["out_channels"], pos_embed_max_size=c["pos_embed_max_size"],
                           dual_attention_layers=c["dual_attention_layers"], qk_norm=c["qk_norm"])
        return set(SO.sd3_param_shapes(cfg)) | {"pos_embed.pos_embed"}     # the persistent sincos buffer
    c = PIXART_TINY
    cfg = replace(PO.PixArtConfig(), num_attention_heads=c["num_attention_heads"], attention_head_dim=c["attention_head_dim"],
                  num_layers=c["num_layers"], cross_attention_dim=c["cross_attention_dim"], sample_size=c["sample_size"],
                  caption_channels=c["caption_channels"])
    return set(PO.pixart_param_shapes(cfg))


@pytest.mark.parametrize("kind,cls,tiny", [("sd3", SD3Transformer2DModel, SD3_TINY), ("pixart", PixArtTransformer2DModel, PIXART_TINY)])
@pytest.mark.parametrize("shard", [None, 20_000])
def test_save_pretrained_round_trip(tmp_path, kind, cls, tiny, shard):
    m = _random(cls(**tiny)).enable_full_finetune()
    for blk in m.transformer_blocks:                # derived layouts exist: none of them may be written
        blk.plans()
    kw = {} if shard is None else {"max_shard_size": shard}
    m.save_pretrained(str(tmp_path), **kw)
    cfg = json.loads((tmp_path / CONFIG_NAME).read_text())
    assert cfg["_class_name"] == cls.__name__
    if shard is None:
        sd = load_file(str(tmp_path / WEIGHTS_NAME))
    else:
        index = json.loads((tmp_path / (WEIGHTS_NAME + ".index.json")).read_text())
        files = sorted(set(index["weight_map"].values()))
        assert len(files) > 1 and all((tmp_path / f).exists() for f in files)
        sd = {}
        for f in files:
            sd.update(load_file(str(tmp_path / f)))
        assert index["metadata"]["total_size"] == sum(v.numel() * v.element_size() for v in sd.values())
    assert set(sd) == _reference_names(kind)
    fresh = cls.from_config(cfg)
    fresh.load_state_dict(sd)
    want = m.state_dict()
    assert set(fresh.state_dict()) == set(want)
    for k, v in fresh.state_dict().items():
        assert v.dtype == want[k].dtype and torch.equal(v, want[k]), k


@pytest.mark.parametrize("cls,tiny", [(SD3Transformer2DModel, SD3_TINY), (PixArtTransformer2DModel, PIXART_TINY)])
def test_config_surface_for_resume_and_ema(tmp_path, cls, tiny):
    m = cls(**tiny)
    # resume (save_hooks.py:1258-1264): model.register_to_config(**load_model.config)
    other = cls(**tiny)
    m.register_to_config(**other.config, _diffusers_version="0.36.0")
    assert m.config._diffusers_version == "0.36.0" and dict(m.config)["num_layers"] == tiny["num_layers"]
    # EMAModel.save_pretrained: from_config(model.config), register_to_config(**ema_state), save_pretrained
    ema = cls.from_config(m.config)
    assert type(ema) is cls and dict(ema.config) == {k: v for k, v in dict(m.config).items() if not k.startswith("_")}
    ema.register_to_config(decay=0.999, optimization_step=7)
    _random(ema).save_pretrained(str(tmp_path))
    cfg = json.loads((tmp_path / CONFIG_NAME).read_text())
    assert cfg["decay"] == 0.999 and cfg["optimization_step"] == 7
    rebuilt = cls.from_config(cfg)               # the EMA entries are not constructor arguments
    assert {k: v.shape for k, v in rebuilt.state_dict().items()} == {k: v.shape for k, v in ema.state_dict().items()}


def test_load_state_dict_drops_the_full_finetune_layouts():
    m = _random(PixArtTransformer2DModel(**PIXART_TINY)).enable_full_finetune()
    for blk in m.transformer_blocks:
        blk.plans()
    m.load_state_dict({k: v.clone() for k, v in m.state_dict().items()})
    assert all(blk._plans is None for blk in m.transformer_blocks)
    m.after_optimizer_step()
    m.after_optimizer_step()       # a second drop in the same step is a no-op
    assert all(blk._plans is None for blk in m.transformer_blocks)


SLOT_CASES = [(SD3Transformer2DModel, SD3_TINY, ("norm1.", "norm1_context.")),
              (SD3Transformer2DModel, dict(SD3_TINY, dual_attention_layers=(), qk_norm=None), ("norm1.", "norm1_context.")),
              (PixArtTransformer2DModel, PIXART_TINY, ("scale_shift_table",))]
SLOT_IDS = ["sd3_dual_qknorm_pre_only", "sd3_no_qknorm", "pixart"]


def _attn_linears(blk):
    """The adapted Linears in the order of the LoRA slot list: attn to_q, to_k, to_v, to_out.0, then SD3's add_q / add_k /
    add_v / to_add_out and attn2's projections, or PixArt's attn2 projections."""
    if hasattr(blk, "attn1"):
        return [lin for a in (blk.attn1, blk.attn2) for lin in (a.to_q, a.to_k, a.to_v, a.to_out[0])]
    a, b = blk.attn, getattr(blk, "attn2", None)
    lins = [a.to_q, a.to_k, a.to_v, a.to_out[0], a.add_q_proj, a.add_k_proj, a.add_v_proj, getattr(a, "to_add_out", None)]
    return lins + ([b.to_q, b.to_k, b.to_v, b.to_out[0]] if b is not None else [None] * 4)


@pytest.mark.parametrize("cls,tiny,autograd", SLOT_CASES, ids=SLOT_IDS)
def test_full_finetune_slots_name_every_block_parameter_once(cls, tiny, autograd):
    """The full fine-tune slot list of each block holds every block parameter exactly once, outside the modulation path
    that torch autograd differentiates: a parameter left out would silently get no gradient."""
    m = cls(**tiny).enable_full_finetune()
    for blk in m.transformer_blocks:
        slots = [t for t in blk.block_slots() if t is not None]
        names = {id(p): n for n, p in blk.named_parameters()}
        assert len({id(t) for t in slots}) == len(slots), "a parameter sits in two slots"
        assert all(id(t) in names for t in slots)
        assert sorted(names[id(t)] for t in slots) == sorted(n for n in names.values() if not n.startswith(autograd))


@pytest.mark.parametrize("cls,tiny,autograd", SLOT_CASES, ids=SLOT_IDS)
def test_lora_slots_and_the_full_finetune_slots_that_replace_them(cls, tiny, autograd):
    """LoRA slots: the (A, B) of the attention projections in schedule order.  Full fine-tune puts each Linear's (weight,
    bias) in that Linear's LoRA slots."""
    m = cls(**tiny)
    for blk in m.transformer_blocks:
        for lin in _attn_linears(blk):
            if lin is not None:
                lin.add_lora(4, 4.0)
    for blk in m.transformer_blocks:
        lins = _attn_linears(blk)
        lora = blk.block_slots()
        assert len(lora) == 2 * len(lins) and all(x is y for x, y in zip(lora, [t for lin in lins for t in (
            lin.lora_tensors() if lin is not None else (None, None))]))
        blk._full_ft = True
        full = blk.block_slots()
        for k, lin in enumerate(lins):
            w, b = (lin.weight, lin.bias) if lin is not None else (None, None)
            assert full[2 * k] is w and full[2 * k + 1] is b, k
