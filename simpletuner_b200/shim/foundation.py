"""Seams B1 / B9 / B10: swap the denoiser after `ModelFoundation.load_model` and route the three step methods.

Reference call order this relies on (helpers/models/common.py:3543-3548): `load_model` builds `self.model` with
`MODEL_CLASS.from_pretrained`, moves it to the device, then calls `configure_chunked_feed_forward()`,
`apply_gradient_checkpointing_settings()`, `fuse_qkv_projections()` and finally `post_model_load_setup()` — the hook
used here.  `add_lora_adapter` (common.py:1049-1117) afterwards calls `self.model.add_adapter(self.lora_config)`, which the
B200 denoisers implement for a `peft.LoraConfig`-shaped object, so LoRA attach needs no override.  The trainer then calls
`self.model.prepare_batch(batch, state)` (trainer.py:6429), `self.model.model_predict(prepared_batch=...)`
(trainer.py:6085-6087) and `self.model.loss_with_logs(prepared_batch, model_output, apply_conditioning_mask=True)`
(trainer.py:6113-6117) on the FAMILY WRAPPER — the three methods routed below.

Unsupported configurations raise NotImplementedError inside the B200 classes; `post_model_load_setup` catches that,
records the reason in `self._b200_fallback_reason` and leaves the reference model in place (the family then behaves
exactly like the unmodified reference).
"""
from __future__ import annotations

import logging
import weakref
from dataclasses import dataclass
from typing import Any, Callable, Dict, Optional, Sequence, Tuple

logger = logging.getLogger("simpletuner_b200.shim")


@dataclass
class FamilySpec:
    registry_key: str                  # ModelRegistry key of the reference family (registry.py:73-77)
    reference_module: str              # module that defines the reference family class
    reference_class: str
    denoiser: Callable[[], type]       # lazy: B200 denoiser class
    step: Callable[[], type]           # lazy: B200 step wrapper class
    config_keys: Sequence[str]         # ctor arguments copied from the reference model's `.config`


def _flux():
    from ..flux.transformer import FluxTransformer2DModel
    return FluxTransformer2DModel


def _flux_step():
    from ..flux.model import Flux
    return Flux


def _sd3():
    from ..sd3.transformer import SD3Transformer2DModel
    return SD3Transformer2DModel


def _sd3_step():
    from ..sd3.model import SD3
    return SD3


def _pixart():
    from ..pixart.transformer import PixArtTransformer2DModel
    return PixArtTransformer2DModel


def _pixart_step():
    from ..pixart.model import PixartSigma
    return PixartSigma


def _qwen_image():
    from ..qwen_image.transformer import QwenImageTransformer2DModel
    return QwenImageTransformer2DModel


def _qwen_image_step():
    from ..qwen_image.model import QwenImage
    return QwenImage


def _chroma():
    from ..chroma.transformer import ChromaTransformer2DModel
    return ChromaTransformer2DModel


def _chroma_step():
    from ..chroma.model import Chroma
    return Chroma


FAMILIES: Dict[str, FamilySpec] = {
    # registry keys: flux/model.py:1504, sd3/model.py:900, pixart/model.py:858 ("pixart_sigma"), qwen_image/model.py:1874
    "flux": FamilySpec("flux", "simpletuner.helpers.models.flux.model", "Flux", _flux, _flux_step,
                       ("patch_size", "in_channels", "num_layers", "num_single_layers", "attention_head_dim",
                        "num_attention_heads", "joint_attention_dim", "pooled_projection_dim", "guidance_embeds",
                        "axes_dims_rope")),
    "sd3": FamilySpec("sd3", "simpletuner.helpers.models.sd3.model", "SD3", _sd3, _sd3_step,
                      ("sample_size", "patch_size", "in_channels", "num_layers", "attention_head_dim", "num_attention_heads",
                       "joint_attention_dim", "caption_projection_dim", "pooled_projection_dim", "out_channels",
                       "pos_embed_max_size", "dual_attention_layers", "qk_norm")),
    "pixart_sigma": FamilySpec("pixart_sigma", "simpletuner.helpers.models.pixart.model", "PixartSigma", _pixart, _pixart_step,
                               ("num_attention_heads", "attention_head_dim", "in_channels", "out_channels", "num_layers",
                                "cross_attention_dim", "sample_size", "patch_size", "caption_channels", "interpolation_scale",
                                "use_additional_conditions", "norm_eps")),
}
# Opt-in families: `install()` registers them only when named (`install(["qwen_image"])`, `install(["chroma"])`), so an
# existing setup that calls `install()` keeps exactly the families it had.  Registry key of Chroma: chroma/model.py:969.
OPT_IN_FAMILIES: Dict[str, FamilySpec] = {
    "qwen_image": FamilySpec("qwen_image", "simpletuner.helpers.models.qwen_image.model", "QwenImage", _qwen_image,
                             _qwen_image_step,
                             ("patch_size", "in_channels", "out_channels", "num_layers", "attention_head_dim",
                              "num_attention_heads", "joint_attention_dim", "guidance_embeds", "axes_dims_rope")),
    "chroma": FamilySpec("chroma", "simpletuner.helpers.models.chroma.model", "Chroma", _chroma, _chroma_step,
                         ("patch_size", "in_channels", "out_channels", "num_layers", "num_single_layers",
                          "attention_head_dim", "num_attention_heads", "joint_attention_dim", "axes_dims_rope",
                          "approximator_num_channels", "approximator_hidden_dim", "approximator_layers",
                          "enable_time_sign_embed", "musubi_blocks_to_swap", "deltatime_type")),
}


def family_spec(family: str) -> FamilySpec:
    spec = FAMILIES.get(family) or OPT_IN_FAMILIES.get(family)
    if spec is None:
        raise KeyError(f"unknown family {family!r}; known: {sorted(FAMILIES) + sorted(OPT_IN_FAMILIES)}")
    return spec


def _cfg_get(cfg: Any, key: str, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def _cfg_has(cfg: Any, key: str) -> bool:
    return (key in cfg) if isinstance(cfg, dict) else hasattr(cfg, key)


class B200FoundationMixin:
    """Put in FRONT of the reference family class: `class FluxB200(B200FoundationMixin, Flux)`."""

    B200_FAMILY: str = ""
    _b200 = None
    _b200_fallback_reason: Optional[str] = None

    # ---- B10: load-time hook -----------------------------------------------------------------------------------
    def post_model_load_setup(self):
        parent = getattr(super(), "post_model_load_setup", None)
        if callable(parent):
            parent()
        self._b200 = None
        self._b200_fallback_reason = None
        try:
            self._b200_install()
        except NotImplementedError as exc:   # unsupported option -> keep the reference module (SURVEY 8b "Errors")
            self._b200 = None
            self._b200_fallback_reason = str(exc)
            logger.warning("libstb200 path not used for %s: %s", self.B200_FAMILY, exc)

    def _b200_install(self):
        import torch

        from ..family import lora_type

        spec = family_spec(self.B200_FAMILY)
        ref = self.model
        if ref is None:
            raise NotImplementedError("no denoiser loaded")
        cfg = getattr(ref, "config", None)
        kwargs = {k: _cfg_get(cfg, k) for k in spec.config_keys if _cfg_has(cfg, k)}
        dtype = getattr(self.config, "weight_dtype", torch.bfloat16)
        if dtype != torch.bfloat16:
            raise NotImplementedError(f"libstb200 computes in bf16; weight_dtype={dtype}")
        step_cls = spec.step()
        full = str(getattr(self.config, "model_type", "lora")) == "full"
        # both raise NotImplementedError on unsupported options (full fine-tuning: outside SD3 / PixArt too)
        (step_cls.validate_full_finetune if full else step_cls.validate_config)(self.config)
        if lora_type(self.config) == "lycoris" and not _LYCORIS_ROUTED:
            # trainer.py:3391 calls the third-party `lycoris.create_lycoris` on the trained component; that wrapper only knows
            # torch.nn modules.  Only with `install_lycoris()` (which routes B200 denoisers to simpletuner_b200.lycoris) may
            # the swap happen for a LyCORIS run (validate_config admits it only where the block schedules carry LoKr).
            raise NotImplementedError("LyCORIS run: call simpletuner_b200.shim.install_lycoris() first (Flux LoKr only)")
        den = spec.denoiser()(**kwargs)
        if not full:
            den.lora_target_linears(step_cls.lora_targets(self.config))  # a target the fused path cannot adapt raises here
        missing, unexpected = den.load_state_dict(ref.state_dict(), strict=False)
        missing = [k for k in missing if "lora_" not in k]
        unexpected = [k for k in unexpected if "lora_" not in k]
        if missing or unexpected:
            raise NotImplementedError(f"state-dict mismatch (missing {missing[:3]}, unexpected {unexpected[:3]})")
        if full:
            den.enable_full_finetune()
            track_full_finetune(den)
        den.to(self.accelerator.device)
        # apply_gradient_checkpointing_settings() ran BEFORE this hook on the reference module (common.py:3545): carry over
        if getattr(ref, "gradient_checkpointing", False):
            den.enable_gradient_checkpointing()
        interval = getattr(ref, "gradient_checkpointing_interval", None) or getattr(self.config, "gradient_checkpointing_interval", None)
        if interval:
            den.set_gradient_checkpointing_interval(int(interval))
        step = step_cls(self.config, transformer=den, device=self.accelerator.device)
        sched = getattr(self, "noise_schedule", None)
        if sched is not None and hasattr(sched, "config") and hasattr(step, "adopt_noise_schedule"):
            step.adopt_noise_schedule(sched)
        self.model = den
        self._b200 = step

    def _b200_step(self):
        """The B200 step bound to whatever `self.model` currently is (accelerator.prepare may have wrapped it in DDP)."""
        step = self._b200
        if step is not None:
            step.model = self.model
        return step

    # ---- B9: step-level methods the trainer calls ----------------------------------------------------------------
    def prepare_batch(self, batch, state):
        step = self._b200_step()
        if step is None:
            return super().prepare_batch(batch, state)
        return step.prepare_batch(batch, state)

    def model_predict(self, prepared_batch, **kwargs):
        step = self._b200_step()
        if step is None:
            return super().model_predict(prepared_batch, **kwargs)
        if kwargs.get("custom_timesteps") is not None:
            raise NotImplementedError("custom_timesteps is not supported by the libstb200 step")
        return step.model_predict(prepared_batch)

    def loss(self, prepared_batch, model_output, apply_conditioning_mask: bool = True):
        step = self._b200_step()
        if step is None:
            return super().loss(prepared_batch, model_output, apply_conditioning_mask=apply_conditioning_mask)
        return step.loss(prepared_batch, model_output, apply_conditioning_mask=apply_conditioning_mask)

    def loss_with_logs(self, prepared_batch, model_output, apply_conditioning_mask: bool = True):
        step = self._b200_step()
        if step is None:
            return super().loss_with_logs(prepared_batch, model_output, apply_conditioning_mask=apply_conditioning_mask)
        return step.loss_with_logs(prepared_batch, model_output, apply_conditioning_mask=apply_conditioning_mask)


# Full fine-tune denoisers whose derived weight layouts must follow every optimizer step.  The reference trainer steps its
# optimizer itself (trainer.py:7239), so one process-wide optimizer post-hook calls `after_optimizer_step()` on each; the
# parameters' version counters cannot stand in for it, because the fused AdamW kernels write through `data_ptr`.
_FULL_FT_MODELS: "weakref.WeakSet" = weakref.WeakSet()
_STEP_HOOK = None


def _after_optimizer_step(optimizer, args, kwargs):
    for den in list(_FULL_FT_MODELS):
        den.after_optimizer_step()


def track_full_finetune(den) -> None:
    """Rebuild `den`'s derived layouts after every optimizer step of this process (weakly referenced: a freed model is
    dropped).  TrainStep's own `after_optimizer_step()` call comes on top; the second drop of the layouts is a no-op."""
    global _STEP_HOOK
    from torch.optim import optimizer

    _FULL_FT_MODELS.add(den)
    if _STEP_HOOK is None:
        _STEP_HOOK = optimizer.register_optimizer_step_post_hook(_after_optimizer_step)


def make_b200_family(reference_cls: type, family: str) -> type:
    """`class <Ref>B200(B200FoundationMixin, reference_cls)` with B200_FAMILY set."""
    family_spec(family)
    return type(reference_cls.__name__ + "B200", (B200FoundationMixin, reference_cls), {"B200_FAMILY": family})


_LYCORIS_ROUTED = False


def install_lycoris(lycoris_module=None):
    """Route `lycoris.create_lycoris` / `LycorisNetwork.apply_preset` (trainer.py:202, 3391-3497) to simpletuner_b200.lycoris
    when the trained component is a libstb200 denoiser; every other module still reaches the third-party implementation.
    `lycoris_module`: the imported `lycoris` package (default: import it)."""
    global _LYCORIS_ROUTED
    from .. import lycoris as b200_lycoris

    if lycoris_module is None:
        import importlib
        lycoris_module = importlib.import_module("lycoris")
    orig_create = lycoris_module.create_lycoris
    orig_net = lycoris_module.LycorisNetwork
    orig_preset = orig_net.apply_preset

    def create_lycoris(module, *a, **k):
        if type(module).__module__.startswith("simpletuner_b200."):
            return b200_lycoris.create_lycoris(module, *a, **k)
        return orig_create(module, *a, **k)

    def apply_preset(preset):
        b200_lycoris.LycorisNetwork.apply_preset(preset)      # both sides see the preset; the one that builds the network uses it
        return orig_preset(preset)

    lycoris_module.create_lycoris = create_lycoris
    orig_net.apply_preset = staticmethod(apply_preset)
    _LYCORIS_ROUTED = True
    return create_lycoris


def install(families: Optional[Sequence[str]] = None) -> Dict[str, type]:
    """Register the B200 subclasses under the reference's own family keys (`ModelRegistry.register`, registry.py:73-77).
    Imports the reference — call it from the reference process (e.g. at the top of simpletuner/train.py)."""
    import importlib

    registry = importlib.import_module("simpletuner.helpers.models.registry").ModelRegistry
    out = {}
    for fam in (families or list(FAMILIES)):
        spec = family_spec(fam)
        ref_cls = getattr(importlib.import_module(spec.reference_module), spec.reference_class)
        cls = make_b200_family(ref_cls, fam)
        registry.register(spec.registry_key, cls)
        out[fam] = cls
    return out
