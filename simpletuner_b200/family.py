"""The step-wrapper surface every model family shares: the methods the reference Trainer and the shim call on a family
object (SURVEY.md §8b seam B9) — `prepare_batch`, `model_predict`, `loss` / `loss_with_logs`, `add_lora_adapter` and the
load-time `validate_config`.

A family sets class attributes and writes only the steps that are its own:

  * `NAME`, `PREDICTION_TYPE`, `GRAPH_REPLAY`, `DENOISER` (built from `**transformer_kwargs` when no denoiser is passed),
    `DEFAULT_CONFIG` and the `_noise_schedule()` hook;
  * `PACKED_LAYOUT`, the feature order of a packed token, which picks `_pack` / `_unpack`, `model_prediction_layout` and the
    loss kernel's layout;
  * `FLAVOURS`, `LORA_TYPES`, `REFUSED_OPTIONS` and `REFUSED_BATCH_KEYS`: what `validate_config` and `_check_supported`
    refuse, so that the shim keeps the reference class for it (INTEGRATION.md §2);
  * `PREDICTION_TYPES`: the `prediction_type` values a DDPM family's loss implements;
  * `FULL_FINETUNE`: whether `model_type="full"` runs on this path (the denoiser has `enable_full_finetune()`); such a run
    is checked by `validate_full_finetune`.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Dict, Optional, Sequence

import torch

from . import ops
from .flux.blocks import FlowLossFn
from .training.noise import sample_noise
from .training.schedule import FlowSigmaSampler

# packed [B, (H/2)(W/2), 4C] tokens as a permutation of [B, C, H/2, 2, W/2, 2]: "packed" orders a token's features
# (c, dy, dx) like Flux's pack_latents, "packed_dydxc" orders them (dy, dx, c) like the SD3 / PixArt patchify
_PACK_ORDER = {"packed": (0, 2, 4, 1, 3, 5), "packed_dydxc": (0, 2, 4, 3, 5, 1)}
LOSS_LAYOUT = {"packed": 0, "packed_dydxc": 1}          # the loss kernels' `layout` argument for each packed layout
# options of the reference that no family runs on this path
_REFUSED_FLAGS = ("twinflow_enabled", "crepa_enabled", "layersync_enabled", "scheduled_sampling_max_step_offset",
                  "diff2flow_enabled")
CONDITIONING_INPUTS = ("conditioning_packed_latents", "conditioning_ids", "conditioning_latents")


def lora_type(c) -> str:
    return str(getattr(c, "lora_type", "standard") or "standard").lower()


class StepWrapper:
    """Drop-in for the step methods of a reference `ImageModelFoundation` family.  `self.model` is the denoiser (optionally
    DDP-wrapped), `self.accelerator.device` the rank's CUDA device."""

    NAME = ""
    PREDICTION_TYPE = "flow_matching"
    GRAPH_REPLAY = True
    DENOISER: Optional[type] = None
    DEFAULT_CONFIG = None
    PACKED_LAYOUT = "packed"
    FLAVOURS: Sequence[str] = ()            # model_flavour values this path runs; empty: any
    LORA_TYPES: Sequence[str] = ("standard",)
    REFUSED_OPTIONS: Sequence[str] = ()     # the family's refusals on top of _REFUSED_FLAGS
    REFUSED_BATCH_KEYS: Sequence[str] = ()
    PREDICTION_TYPES: Sequence[str] = ()
    FULL_FINETUNE = False

    def __init__(self, config: Optional[SimpleNamespace] = None, transformer=None, device: Optional[torch.device] = None,
                 **transformer_kwargs):
        self.config = config or self.DEFAULT_CONFIG()
        dev = device or torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        self.accelerator = SimpleNamespace(device=dev)
        self.noise_schedule = self._noise_schedule()
        if transformer is None and self.DENOISER is not None:
            transformer = self.DENOISER(**transformer_kwargs)
        self.model = transformer
        pt = getattr(self.config, "prediction_type", None) if self.PREDICTION_TYPES else None
        if pt is not None:
            self._check_prediction_type(pt)
            self.PREDICTION_TYPE = pt
            self.noise_schedule.config.prediction_type = pt

    def _noise_schedule(self):
        """The flow-matching scheduler config of Flux, SD3 and Chroma (replaced by `adopt_noise_schedule` under the shim)."""
        return SimpleNamespace(config=SimpleNamespace(num_train_timesteps=1000, patch_size=2, base_image_seq_len=256,
                                                      max_image_seq_len=4096, base_shift=0.5, max_shift=1.15))

    @classmethod
    def _check_prediction_type(cls, pt) -> None:
        if pt is not None and pt not in cls.PREDICTION_TYPES:       # pixart/model.py:698-700
            raise NotImplementedError(f"prediction_type {pt} is not implemented for the libstb200 {cls.NAME} step")

    # ------------------------------------------------------------------------------------------
    def get_trained_component(self):
        return self.model

    def _denoiser(self):
        m = self.model
        return m.module if hasattr(m, "module") else m

    def adopt_noise_schedule(self, sched) -> None:
        """Use the reference family's scheduler object (its `.config` feeds the flow shift / timestep count)."""
        self.noise_schedule = sched

    @classmethod
    def lora_targets(cls, c) -> list:
        """get_lora_target_layers (common.py:952-1007): for a standard LoRA the `peft_lora_target_modules` entries with None,
        "" and "None" dropped and whitespace stripped, when any remain; else the family default.  The reference's slider
        lists are its own, so `slider_lora_target` raises NotImplementedError."""
        if lora_type(c) == "standard":
            raw = getattr(c, "peft_lora_target_modules", None)
            if raw not in (None, "", "None"):
                if not isinstance(raw, (list, tuple)):
                    raise ValueError(f"peft_lora_target_modules must be a list of module name strings. Received {type(raw)}.")
                manual = []
                for t in raw:
                    if t in (None, "", "None"):
                        continue
                    if not isinstance(t, str):
                        raise ValueError(f"peft_lora_target_modules entries must be strings. Received {type(t)}.")
                    if t.strip():
                        manual.append(t.strip())
                if manual:
                    return manual
            if getattr(c, "slider_lora_target", False):
                raise NotImplementedError(f"slider LoRA targets are not supported by the libstb200 {cls.NAME} path")
        return cls._default_lora_targets(c)

    @classmethod
    def _default_lora_targets(cls, c) -> list:
        return list(getattr(cls.DENOISER, "_DEFAULT_LORA_TARGETS", ()))

    def add_lora_adapter(self):
        """common.py:1049-1117: a PEFT LoRA on the Linears `lora_targets` names."""
        c = self.config
        return self._denoiser().add_adapter(rank=c.lora_rank, lora_alpha=c.lora_alpha, target_modules=self.lora_targets(c),
                                            lora_dropout=getattr(c, "lora_dropout", 0.0))

    def add_lycoris_adapter(self, lycoris_config):
        raise NotImplementedError(f"LyCORIS adapters on {self.NAME} are not supported by the libstb200 path")

    # ------------------------------------------------------------------------------------------
    @classmethod
    def validate_config(cls, c) -> None:
        """Load-time counterpart of the per-batch guards for a LoRA run: options of the reference this path does not
        implement raise NotImplementedError so that the shim (shim/foundation.py) keeps the reference module for such a run.
        Whether the resolved LoRA targets can be adapted is the denoiser's rule (`lora_target_linears`), which the shim
        applies.  A `model_type="full"` run is checked by `validate_full_finetune` instead."""
        cls._validate(c, full=False)

    @classmethod
    def validate_full_finetune(cls, c) -> None:
        """The load-time check of a `model_type="full"` run: admitted where the family sets `FULL_FINETUNE`, with the same
        refusals as a LoRA run (so LyCORIS, DoRA and controlnet still keep the reference module)."""
        cls._validate(c, full=True)

    @classmethod
    def _validate(cls, c, full: bool) -> None:
        g = lambda k, d=None: getattr(c, k, d)
        fl = g("model_flavour", None)
        if cls.FLAVOURS and fl and fl not in cls.FLAVOURS:
            raise NotImplementedError(f"{cls.NAME} model_flavour={fl!r} is not supported by the libstb200 path "
                                      f"(supported: {cls.FLAVOURS})")
        if g("controlnet", False):
            raise NotImplementedError("ControlNet (controlnet) training is not supported by the libstb200 path")
        model_type = str(g("model_type", "lora"))
        if model_type != "lora" and not (full and model_type == "full" and cls.FULL_FINETUNE):
            raise NotImplementedError(f"model_type={g('model_type')!r}: only LoRA training runs on the libstb200 path")
        if lora_type(c) not in cls.LORA_TYPES:
            raise NotImplementedError(f"lora_type={g('lora_type')!r} on {cls.NAME} is not supported by the libstb200 path")
        if g("use_dora", False):
            raise NotImplementedError("DoRA is not supported by the libstb200 path")
        cls.lora_targets(c)
        if g("tread_config", None):
            raise NotImplementedError("TREAD routing is not supported by the libstb200 path")
        if g("flow_cubic_schedule", None) or g("flow_cubic_schedule_weights", None):
            raise NotImplementedError("the cubic-spline flow schedule is not part of the libstb200 step")
        for flag in _REFUSED_FLAGS + tuple(cls.REFUSED_OPTIONS):
            if g(flag, None):
                raise NotImplementedError(f"{flag} is not supported by the libstb200 path")
        if g("distillation_method", None) not in (None, "", "None"):
            raise NotImplementedError("distillation is not supported by the libstb200 path")
        if cls.PREDICTION_TYPES:
            cls._check_prediction_type(g("prediction_type", None))

    def _check_supported(self, batch: Dict[str, Any]) -> None:
        """Batch inputs of the reference wrapper this path does not implement must RAISE, never be ignored, so that a shim
        can route such a config to the reference class (INTEGRATION.md 2)."""
        for k in self.REFUSED_BATCH_KEYS:
            if batch.get(k) is not None:
                raise NotImplementedError(f"{self.NAME} batch input `{k}` is not supported by the libstb200 path")

    def _check_loss_supported(self, prepared_batch: Dict[str, Any], apply_conditioning_mask: bool) -> None:
        """common.py:6400-6424: with `apply_conditioning_mask` the reference multiplies the loss by the conditioning mask
        when the dataset's `conditioning_type` is 'mask' or 'segmentation'.  Not implemented here -> raise."""
        if not apply_conditioning_mask:
            return
        lm = prepared_batch.get("loss_mask_type") or prepared_batch.get("conditioning_type")   # legacy fallback, :6403-6408
        if lm in ("mask", "segmentation"):
            raise NotImplementedError("masked / segmentation-weighted loss is not supported by the libstb200 loss kernels")

    # ---- flow matching: common.py:5862-6041 -----------------------------------------------------------------------
    def prepare_batch(self, batch: Dict[str, Any], state: Dict[str, Any]) -> Dict[str, Any]:
        """Batch dict keys are the collate contract of the reference (training/collate.py:1316-1349): `latent_batch`,
        `prompt_embeds`, `add_text_embeds`; this adds `latents`, `noise`, `input_noise`, `sigmas`, `timesteps`,
        `noisy_latents`, `encoder_hidden_states` and `added_cond_kwargs`."""
        if not batch:
            return batch
        c = self.config
        self._check_supported(batch)
        kw = {"device": self.accelerator.device, "dtype": c.weight_dtype}
        if batch.get("prompt_embeds") is not None:
            batch["encoder_hidden_states"] = batch["prompt_embeds"].to(**kw, non_blocking=True)
        pooled = batch.get("add_text_embeds")
        batch["added_cond_kwargs"] = {}
        if pooled is not None:
            batch["added_cond_kwargs"]["text_embeds"] = pooled.to(**kw, non_blocking=True)
        latents = batch.get("latent_batch")
        if not hasattr(latents, "to"):
            raise ValueError("Received invalid value for latents.")
        batch["latents"] = latents.to(**kw, non_blocking=True).contiguous()
        mask = batch.get("encoder_attention_mask")
        if mask is not None and hasattr(mask, "to"):   # common.py:5911-5913
            batch["encoder_attention_mask"] = mask.to(**kw, non_blocking=True)
        interp = self._flow_draw(batch, state, batch["latents"])
        return self._prep_pack(batch, state, interp)

    def _flow_draw(self, batch: Dict[str, Any], state: Dict[str, Any], latents: torch.Tensor) -> torch.Tensor:
        """The flow-matching draws with the reference's generators and order (common.py:5938, 5068, 4962-4991): the noise
        (`randn_like(latents)`), the sigmas, then MixFlow's `rand_like`, so a seeded run samples the same values.  Stores
        `noise`, `input_noise`, `timesteps` and `sigmas` ([B,1,1,1] after expand_sigmas); returns the sigmas the noisy
        latents interpolate with."""
        c = self.config
        noise, input_noise = sample_noise(c, latents, state, flow_matching=True)
        batch["noise"] = noise
        batch["input_noise"] = input_noise.to(latents.dtype).contiguous()
        if getattr(self, "_sigma_sampler", None) is None:   # keeps the round-robin cursor of custom timestep lists
            self._sigma_sampler = FlowSigmaSampler(c, self.noise_schedule, self.accelerator.device)
        sigmas, timesteps = self._model_sigmas(*self._sigma_sampler.sample(latents.shape[0], noise, state), latents)
        batch["timesteps"] = timesteps
        batch["sigmas"] = sigmas.view(-1, 1, 1, 1)  # expand_sigmas, common.py:6825-6828
        # MixFlow (common.py:4962-4991): the model sees `sigmas`, the interpolation uses the slowed-down
        # sigma + U * gamma * (1 - sigma)
        if getattr(c, "mixflow_enabled", False) is not True:
            return sigmas
        gamma = float(getattr(c, "mixflow_gamma", 0.8))
        if not 0.0 <= gamma <= 1.0:
            raise ValueError("mixflow_gamma must be between 0.0 and 1.0.")
        slow = torch.rand_like(sigmas) if gamma > 0.0 else torch.zeros_like(sigmas)
        interp = sigmas if gamma == 0.0 else sigmas + slow * gamma * (1.0 - sigmas)
        batch["mixflow_slowdown_factors"] = slow
        batch["mixflow_interpolation_sigmas"] = interp
        return interp

    def _model_sigmas(self, sigmas: torch.Tensor, timesteps: torch.Tensor, latents: torch.Tensor):
        """(sigmas, timesteps) the step trains at, from the sampler's draw: the drawn values (Chroma remaps them)."""
        return sigmas, timesteps

    def _prep_pack(self, batch: Dict[str, Any], state: Dict[str, Any], interp: torch.Tensor) -> Dict[str, Any]:
        # fused: noisy = (1 - s) x + s eps  AND  2x2 patchify  (common.py:4975-4992, flux/__init__.py:25-30)
        noisy, packed = ops.flow_prep_pack(batch["latents"], batch["input_noise"], interp.float().contiguous(),
                                           want_unpacked=True)
        batch["noisy_latents"] = noisy
        batch["_packed_noisy_latents"] = packed
        return batch

    def _batch_timesteps(self, t: torch.Tensor, B: int) -> torch.Tensor:
        """`t` as [B]: a scalar or one-element timestep is broadcast; token-wise timesteps are not implemented."""
        if t.ndim == 0 or (t.ndim == 1 and t.shape[0] == 1):
            return t.reshape(1).expand(B)
        if t.ndim != 1:
            raise NotImplementedError(f"token-wise timesteps are not supported by the libstb200 {self.NAME} path")
        if t.shape[0] != B:
            raise ValueError(f"{self.NAME} expected 1 timestep or {B} per-batch timesteps, got {tuple(t.shape)}.")
        return t

    # ---- DDPM (PixArt, SDXL): DDPMScheduler.add_noise coefficients --------------------------------------------------
    def _ddpm_coefs(self, timesteps: torch.Tensor, dev):
        cache = self.__dict__.setdefault("_sched_dev", {})
        tab = cache.get(dev)
        if tab is None:
            ac = self.noise_schedule.alphas_cumprod.to(dev)
            tab = (ac ** 0.5, (1 - ac) ** 0.5)   # DDPMScheduler.add_noise: fp32 tables, gathered per sample
            cache[dev] = tab
        t = timesteps.to(dev)
        return tab[0][t].contiguous(), tab[1][t].contiguous()

    # ---- the packed prediction -----------------------------------------------------------------------------------
    def _prediction_dict(self, out_packed: torch.Tensor, latent_shape) -> Dict[str, Any]:
        """The reference's dict (flux/model.py:855-864): `model_prediction` is the un-packed [B, C, H, W] tensor (seam B9).
        The packed token layout the loss kernel consumes rides along under the private key `_packed_prediction`; `loss()`
        uses it while the caller has not replaced `model_prediction`."""
        unpacked = self._unpack(out_packed, latent_shape)
        return {"model_prediction": unpacked, "_packed_prediction": out_packed, "_unpacked_ref": unpacked,
                "model_prediction_layout": self.PACKED_LAYOUT, "latent_shape": tuple(latent_shape),
                "crepa_hidden_states": None, "hidden_states_buffer": None}

    @classmethod
    def _pack(cls, pred: torch.Tensor) -> torch.Tensor:
        B, C, H, W = pred.shape
        x = pred.reshape(B, C, H // 2, 2, W // 2, 2).permute(_PACK_ORDER[cls.PACKED_LAYOUT])
        return x.reshape(B, (H // 2) * (W // 2), 4 * C)

    @classmethod
    def _unpack(cls, out_packed: torch.Tensor, latent_shape) -> torch.Tensor:
        B, C, H, W = latent_shape
        order = _PACK_ORDER[cls.PACKED_LAYOUT]
        dims = (B, C, H // 2, 2, W // 2, 2)
        x = out_packed.reshape([dims[i] for i in order]).permute(sorted(range(6), key=order.__getitem__))
        return x.reshape(B, C, H, W)

    @staticmethod
    def unpacked_prediction(model_output: Dict[str, Any]) -> torch.Tensor:
        return model_output["model_prediction"]

    def _packed_for_loss(self, model_output: Dict[str, Any]) -> torch.Tensor:
        """The packed prediction the loss kernels read.  A caller that REPLACED `model_prediction` (e.g. the x-prediction
        fix-up of trainer.py:6099-6105) is honoured: the private packed tensor is only used while it still describes the
        same object; a bare `{"model_prediction": packed_tensor}` (3-D) is accepted as already packed."""
        pred = model_output["model_prediction"]
        packed = model_output.get("_packed_prediction")
        if packed is not None and model_output.get("_unpacked_ref") is pred:
            return packed
        if pred.dim() == 3:
            return pred
        return self._pack(pred).contiguous()

    # ------------------------------------------------------------------------------------------
    def loss(self, prepared_batch: Dict[str, Any], model_output: Dict[str, Any], apply_conditioning_mask: bool = True):
        """common.py:6217-6430, flow-matching branch: target = noise - latents (common.py:4610-4611), the loss in fp32,
        mean over (C,H,W) then over the batch."""
        self._check_loss_supported(prepared_batch, apply_conditioning_mask)
        return FlowLossFn.apply(self._packed_for_loss(model_output), prepared_batch["latents"], prepared_batch["noise"],
                                LOSS_LAYOUT[self.PACKED_LAYOUT], *self._loss_kind(prepared_batch))

    def _loss_kind(self, prepared_batch):
        """loss_type / per-sample huber_c (common.py:6230-6284).  For flow matching the reference ignores snr_gamma."""
        c = self.config
        lt = getattr(c, "loss_type", "l2")
        if lt == "l2":
            return "l2", None
        if lt not in ("huber", "smooth_l1"):
            raise NotImplementedError(f"Unsupported Loss Type {lt}")
        from .training.noise import compute_scheduled_huber_c
        # NB: Flux.model_predict has overwritten `timesteps` with t / 1000 (flux/model.py:739-745) before loss() runs; the
        # reference feeds those scaled values to compute_scheduled_huber_c as they are, and so does this mirror.
        t = prepared_batch["timesteps"]
        if t.dim() == 2:        # Kontext [B, S_scene + S_c]: validate_config allows only the constant c here
            t = t[:, 0]
        return lt, compute_scheduled_huber_c(c, self.noise_schedule, t.to(self.accelerator.device), self.PREDICTION_TYPE)

    def loss_with_logs(self, prepared_batch, model_output, apply_conditioning_mask: bool = True):
        return self.loss(prepared_batch, model_output, apply_conditioning_mask), None
