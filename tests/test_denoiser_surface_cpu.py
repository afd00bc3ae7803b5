"""CPU: the adapter, gradient-checkpointing and plan-lifecycle surface the denoisers share (AdapterModelAPI), on tiny SD3
and PixArt models (SD3 with an SD3.5 second attention in block 0 and the `context_pre_only` last block), plus the
derived weight layouts of the SD3 block plans.  Plumbing only: no kernel runs."""
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from simpletuner_b200 import ops
from simpletuner_b200.flux.transformer import FluxTransformer2DModel, Linear
from simpletuner_b200.pixart.transformer import PixArtTransformer2DModel
from simpletuner_b200.qwen_image.transformer import QwenImageTransformer2DModel
from simpletuner_b200.sd3.transformer import SD3Transformer2DModel
from tests.shim_stub import StubFoundation

ROOT = Path(__file__).resolve().parents[1]

SD3_TINY = dict(sample_size=8, num_layers=2, attention_head_dim=64, num_attention_heads=1, joint_attention_dim=32,
                caption_projection_dim=64, pooled_projection_dim=32, out_channels=16, pos_embed_max_size=8,
                dual_attention_layers=(0,), qk_norm="rms_norm")
PIXART_TINY = dict(num_attention_heads=2, attention_head_dim=40, in_channels=4, out_channels=8, num_layers=2,
                   cross_attention_dim=80, sample_size=8, caption_channels=32)
FLUX_TINY = dict(in_channels=64, num_layers=1, num_single_layers=1, attention_head_dim=64, num_attention_heads=1,
                 joint_attention_dim=32, pooled_projection_dim=32, axes_dims_rope=(8, 28, 28))
QWEN_TINY = dict(num_layers=1, attention_head_dim=64, num_attention_heads=1, joint_attention_dim=32)


def _sd3(**over):
    return SD3Transformer2DModel(**{**SD3_TINY, **over})


def _pixart():
    return PixArtTransformer2DModel(**PIXART_TINY)


def _blocks(prefix, n, names):
    return {f"transformer_blocks.{i}.{prefix}{t}" for i in n for t in names}


_QKVO = ("to_q", "to_k", "to_v", "to_out.0")
# the Linears each model adapts for its default targets and for each single attention target; recorded from the
# per-model add_adapter implementations these models had before they shared AdapterModelAPI
SD3_SELECTED = {
    None: _blocks("attn.", (0, 1), _QKVO) | _blocks("attn2.", (0,), _QKVO),
    **{t: _blocks("attn.", (0, 1), (t,)) | _blocks("attn2.", (0,), (t,)) for t in _QKVO},
    **{t: _blocks("attn.", (0, 1), (t,)) for t in ("add_q_proj", "add_k_proj", "add_v_proj")},
    "to_add_out": {"transformer_blocks.0.attn.to_add_out"},           # block 1 is context_pre_only
}
PIXART_SELECTED = {
    None: _blocks("attn1.", (0, 1), _QKVO) | _blocks("attn2.", (0, 1), _QKVO),
    **{t: _blocks("attn1.", (0, 1), (t,)) | _blocks("attn2.", (0, 1), (t,)) for t in _QKVO},
    **{t: None for t in ("add_q_proj", "add_k_proj", "add_v_proj", "to_add_out")},   # no such Linear: ValueError
}


@pytest.mark.parametrize("build,selected", [(_sd3, SD3_SELECTED), (_pixart, PIXART_SELECTED)], ids=["sd3", "pixart"])
def test_adapted_linears_per_target(build, selected):
    for target, expected in selected.items():
        m = build()
        targets = None if target is None else [target]
        if expected is None:
            with pytest.raises(ValueError, match="no module matched"):
                m.add_adapter(rank=4, target_modules=targets)
            assert not m.lora_linears()
            continue
        assert m.add_adapter(rank=4, target_modules=targets) == len(expected), target
        assert set(m.lora_linears()) == expected, target


@pytest.mark.parametrize("build,default", [(_sd3, ["to_k", "to_q", "to_v", "to_out.0"]),
                                           (_pixart, ["to_k", "to_q", "to_v", "to_out.0"])], ids=["sd3", "pixart"])
def test_peft_config_scaling_and_argument_errors(build, default):
    m = build()
    cfg = SimpleNamespace(r=4, lora_alpha=8, target_modules=None, lora_dropout=0.1)
    m.add_adapter(cfg)
    pc = m.peft_config["default"]
    assert (pc.r, pc.lora_alpha, pc.target_modules, pc.lora_dropout) == (4, 8.0, default, 0.1)
    assert m._lora_scaling == 2.0 and m._lora_dropout_p == 0.1
    assert all(lin.scaling["default"] == 2.0 and lin.lora_A["default"].weight.shape == (4, lin.in_features)
               for lin in m.lora_linears().values())
    names = [n for n, p in m.named_parameters() if p.requires_grad]
    assert names and all(".lora_A.default." in n or ".lora_B.default." in n for n in names)
    assert len(m.trainable_parameters()) == len(names)
    m.disable_lora()
    assert not any(lin.lora_enabled for lin in m.lora_linears().values())
    m.enable_lora()
    assert all(lin.lora_enabled for lin in m.lora_linears().values())
    for kw, exc in ((dict(rank=4, lora_dropout=1.0), ValueError), (dict(rank=4, lora_dropout=-0.1), ValueError),
                    (dict(rank=0), NotImplementedError), (dict(rank=129), NotImplementedError),
                    (dict(rank=None), ValueError)):
        fresh = build()
        with pytest.raises(exc):
            fresh.add_adapter(**kw)
        assert not fresh.lora_linears(), kw


@pytest.mark.parametrize("build,targets", [(_sd3, ["to_q", "ff.net.2"]), (_pixart, ["ff.net.2"]),
                                           (_pixart, ["to_q", "adaln_single.linear"])], ids=["sd3", "pixart", "pixart-adaln"])
def test_unadaptable_target_raises_before_anything_is_attached(build, targets):
    m = build()
    with pytest.raises(NotImplementedError, match="not supported by the fused path"):
        m.add_adapter(rank=4, target_modules=targets)
    assert not m.lora_linears()
    assert not any(isinstance(mod, Linear) and mod.lora_A is not None for mod in m.modules())
    assert "default" not in m.peft_config


def test_sd3_qualified_target_follows_the_peft_suffix_rule():
    m = _sd3()
    assert m.add_adapter(rank=4, target_modules=["attn.to_q"]) == 2
    assert set(m.lora_linears()) == {"transformer_blocks.0.attn.to_q", "transformer_blocks.1.attn.to_q"}
    m = _sd3()
    m.add_adapter(rank=4, target_modules=["transformer_blocks.0.attn2.to_out.0"])
    assert set(m.lora_linears()) == {"transformer_blocks.0.attn2.to_out.0"}


@pytest.mark.parametrize("build", [_sd3, _pixart, lambda: FluxTransformer2DModel(**FLUX_TINY)], ids=["sd3", "pixart", "flux"])
@pytest.mark.parametrize("interval,expected", [(None, [0, 1, 2, 3, 4]), (2, [0, 2, 4]), (3, [0, 3])])
def test_run_block_checkpoints_every_interval_th_block(monkeypatch, build, interval, expected):
    import torch.utils.checkpoint as tuc
    calls = []

    def fake_checkpoint(fn, *args, use_reentrant):
        calls.append(args[0])
        assert use_reentrant is False
        return fn(*args)

    monkeypatch.setattr(tuc, "checkpoint", fake_checkpoint)
    m = build()
    block = lambda i: i + 10
    assert [m._run_block(i, block, i) for i in range(5)] == [10, 11, 12, 13, 14]      # off by default
    m.enable_gradient_checkpointing()
    if interval is not None:
        m.set_gradient_checkpointing_interval(interval)
    assert [m._run_block(i, block, i) for i in range(5)] == [10, 11, 12, 13, 14]
    assert calls == expected
    with torch.no_grad():
        m._run_block(0, block, 0)
    m.disable_gradient_checkpointing()
    m._run_block(0, block, 0)
    assert calls == expected


def _random(m):
    """Stands in for a loaded checkpoint (the constructors leave the weights uninitialised)."""
    torch.manual_seed(0)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02)
    return m


def _ref_sd3():
    return _random(_sd3())


def _ref_pixart():
    return _random(_pixart())


class RefSD3(StubFoundation):
    MODEL_CLASS = staticmethod(_ref_sd3)
    LORA_TARGETS = ["to_k", "to_q", "to_v", "to_out.0"]


class RefPixArt(StubFoundation):
    MODEL_CLASS = staticmethod(_ref_pixart)
    LORA_TARGETS = ["to_k", "to_q", "to_v", "to_out.0"]


@pytest.mark.parametrize("family", ["sd3", "pixart_sigma"])
def test_shim_carries_the_checkpointing_interval_over(family):
    from simpletuner_b200.shim import make_b200_family
    if family == "sd3":
        from simpletuner_b200.flux.model import default_config
        ref, den_cls = RefSD3, SD3Transformer2DModel
    else:
        from simpletuner_b200.pixart.model import default_config
        ref, den_cls = RefPixArt, PixArtTransformer2DModel
    cfg = default_config(lora_rank=4, model_type="lora", lora_type="standard", gradient_checkpointing=True,
                         gradient_checkpointing_interval=2)
    fam = make_b200_family(ref, family)(cfg, "cpu")
    fam.load_model()
    assert fam._b200_fallback_reason is None and fam._b200 is not None
    assert isinstance(fam.model, den_cls) and fam._b200.model is fam.model
    assert fam.model.gradient_checkpointing is True and fam.model.gradient_checkpointing_interval == 2
    fam.add_lora_adapter()
    assert set(fam.model.lora_linears()) == (SD3_SELECTED if family == "sd3" else PIXART_SELECTED)[None]


def _same_storage(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.untyped_storage().data_ptr() == b.untyped_storage().data_ptr()


@pytest.mark.parametrize("qk_norm", [None, "rms_norm"])
def test_sd3_plan_layouts(qk_norm):
    m = _random(_sd3(qk_norm=qk_norm))
    m.add_adapter(rank=4)
    blk = m.transformer_blocks[0]
    pl = blk.plans()
    assert set(pl) == {"img_attn", "txt_attn", "img_mlp", "txt_mlp", "img_attn2"}
    assert set(m.transformer_blocks[1].plans()) == {"img_attn", "txt_attn", "img_mlp"}     # context_pre_only
    a, ff = blk.attn, blk.ff
    w_qkv = torch.cat([a.to_q.weight, a.to_k.weight, a.to_v.weight], 0)
    p = pl["img_attn"]
    assert (p.norm_q is None) == (qk_norm is None) and (p.norm_k is None) == (qk_norm is None)
    assert torch.equal(p.w_qkv, w_qkv)
    # LoRA: the base weights are frozen, so each dgrad operand is a transposed copy
    for t, ref in ((p.w_qkv_t, w_qkv), (p.w_out_t, a.to_out[0].weight), (pl["img_mlp"].w1_t, ff.net[0].proj.weight),
                   (pl["img_mlp"].w2_t, ff.net[2].weight)):
        assert isinstance(t, torch.Tensor) and t.is_contiguous() and torch.equal(t, ref.t())
    assert m.transformer_blocks[1].plans()["txt_attn"].w_out is None
    # full fine-tune: the weights change every step, so each dgrad operand is a view of the forward weight
    m = _random(_sd3(qk_norm=qk_norm))
    m.enable_full_finetune()
    blk = m.transformer_blocks[0]
    pl = blk.plans()
    a, ff = blk.attn, blk.ff
    for name in ("img_attn", "txt_attn", "img_attn2"):
        p = pl[name]
        assert isinstance(p.w_qkv_t, ops.WT) and p.w_qkv_t.w is p.w_qkv
        assert isinstance(p.w_out_t, ops.WT)
    assert _same_storage(pl["img_attn"].w_out_t.w, a.to_out[0].weight)
    assert _same_storage(pl["txt_attn"].w_out_t.w, a.to_add_out.weight)
    assert _same_storage(pl["img_attn2"].w_out_t.w, blk.attn2.to_out[0].weight)
    for key, f in (("img_mlp", ff), ("txt_mlp", blk.ff_context)):
        mp = pl[key]
        assert isinstance(mp.w1_t, ops.WT) and isinstance(mp.w2_t, ops.WT)
        assert _same_storage(mp.w1_t.w, f.net[0].proj.weight) and _same_storage(mp.w2_t.w, f.net[2].weight)


def _fill_caches(m):
    blocks = list(m.transformer_blocks) + list(getattr(m, "single_transformer_blocks", []))
    for blk in blocks:
        if hasattr(blk, "_plans"):
            blk._plans = {"stale": True}
    if hasattr(m, "_tail_plan"):
        m._tail_plan = {"stale": True}
    for cache in ("_rope_cache", "_pos_cache"):
        if hasattr(m, cache):
            getattr(m, cache)["stale"] = True
    if hasattr(m, "_pad_index"):
        m._pad_index = torch.zeros(1)


def _assert_reset(m, kind):
    blocks = list(m.transformer_blocks) + list(getattr(m, "single_transformer_blocks", []))
    if kind == "qwen":
        assert m._rope_cache == {}
        assert all(blk.attn._is_fused() for blk in blocks)
        return
    assert all(blk._plans is None for blk in blocks)
    assert not m._tail_plan
    if kind == "flux":
        assert m._rope_cache == {}
    else:
        assert m._pos_cache == {}
    if kind == "pixart":
        assert m._pad_index is None


@pytest.mark.parametrize("kind,build", [("flux", lambda: FluxTransformer2DModel(**FLUX_TINY)), ("sd3", _sd3),
                                        ("pixart", _pixart), ("qwen", lambda: QwenImageTransformer2DModel(**QWEN_TINY))])
def test_to_and_load_state_dict_reset_every_cached_plan(kind, build):
    m = build()
    _fill_caches(m)
    m.to("cpu")
    _assert_reset(m, kind)
    _fill_caches(m)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    m.load_state_dict(sd)
    _assert_reset(m, kind)
    _fill_caches(m)
    m.load_state_dict(sd, assign=True)          # replaces the parameters (Qwen-Image re-fuses q|k|v)
    _assert_reset(m, kind)


def test_denoiser_code_reads_no_environment_switch():
    pkg = ROOT / "simpletuner_b200"
    paths = [pkg / "ops.py"] + [p for sub in ("flux", "sd3", "pixart", "qwen_image", "chroma") for p in (pkg / sub).glob("*.py")]
    for path in paths:
        assert "environ" not in path.read_text(), path
