"""SDXL step wrapper on libstb200 — the step-level plumbing of reference simpletuner/helpers/models/sdxl/model.py
(class SDXL): `prepare_batch` (common.py:5862-6041, epsilon / v-prediction branch: offset noise, weighted / segmented
integer timesteps, fp32 `DDPMScheduler.add_noise`), `_model_predict_single` (sdxl/model.py:306-373: the UNet call with
`add_text_embeds` + `added_cond_kwargs = {text_embeds, time_ids}`), `loss` (common.py:6217-6430 with min-SNR weighting) and
the micro-conditioning helpers (`compute_time_ids`, `gather_conditional_sdxl_size_features`, collate.py:59-98, 501-523).

Scope (BASELINE configs[0] is the reference's CPU plumbing case): the conv / cross-attention UNet itself is NOT re-implemented
here — `self.model` is whatever `UNet2DConditionModel`-shaped callable the caller loads (the reference's diffusers module);
what runs on libstb200 is the step AROUND it: the fused noisy-latent kernel (`stb_ddpm_prep_pack`, bit-exact with the eager
fp32 add_noise chain) and the weighted loss kernel on the UNet's NCHW output (`stb_target_mse_loss`, layout 2) including its
gradient.  Everything the UNet consumes / produces keeps the reference's shapes, dtypes and dict keys.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Dict, Optional

import torch

from .. import ops
from ..family import CONDITIONING_INPUTS, StepWrapper
from ..pixart.model import _TargetLossFn, default_config as _eps_defaults
from ..training.noise import (gather_conditional_sdxl_size_features, make_ddpm_schedule, min_snr_loss_weights)
from ..training.schedule import generate_timestep_weights, segmented_timestep_selection


def default_config(**over) -> SimpleNamespace:
    cfg = vars(_eps_defaults())
    cfg.update(max_grad_norm=2.0, snr_gamma=None, prediction_type="epsilon")
    cfg.update(over)
    return SimpleNamespace(**cfg)


class SDXL(StepWrapper):
    NAME = "Stable Diffusion XL"
    PREDICTION_TYPE = "epsilon"
    PREDICTION_TYPES = ("epsilon", "v_prediction")
    DEFAULT_CONFIG = staticmethod(default_config)
    REFUSED_BATCH_KEYS = CONDITIONING_INPUTS

    def __init__(self, config: Optional[SimpleNamespace] = None, unet=None, device: Optional[torch.device] = None):
        super().__init__(config, transformer=unet, device=device)

    def _noise_schedule(self):
        # SDXL scheduler_config.json: DDPM, 1000 steps, scaled_linear betas 0.00085 .. 0.012, epsilon (v for some finetunes)
        return make_ddpm_schedule(1000, 0.00085, 0.012, "scaled_linear")

    def add_lora_adapter(self):
        raise NotImplementedError("SDXL LoRA attaches to the reference UNet (PEFT); the libstb200 step only wraps the UNet call")

    # ---- prepare_batch: the epsilon branch of common.py:5862-6041 without the 2x2 patchify ---------------------------
    def prepare_batch(self, batch: Dict[str, Any], state: Dict[str, Any]) -> Dict[str, Any]:
        if not batch:
            return batch
        self._check_supported(batch)
        c = self.config
        dev = self.accelerator.device
        kw = {"device": dev, "dtype": c.weight_dtype}
        if batch.get("prompt_embeds") is not None:
            batch["encoder_hidden_states"] = batch["prompt_embeds"].to(**kw, non_blocking=True)
        pooled = batch.get("add_text_embeds")
        batch["added_cond_kwargs"] = {}
        if pooled is not None:
            batch["add_text_embeds"] = pooled.to(**kw, non_blocking=True)
            batch["added_cond_kwargs"]["text_embeds"] = batch["add_text_embeds"]
        time_ids = batch.get("batch_time_ids")
        if time_ids is None and batch.get("examples") is not None:
            time_ids = gather_conditional_sdxl_size_features(batch["examples"], batch["latent_batch"], c.weight_dtype)
        if time_ids is not None:      # common.py:5903-5908: [B, 1, 6] -> [B, 6]
            batch["added_cond_kwargs"]["time_ids"] = time_ids.to(**kw).reshape(time_ids.shape[0], -1)
        latents = batch.get("latent_batch")
        if not hasattr(latents, "to"):
            raise ValueError("Received invalid value for latents.")
        batch["latents"] = latents.to(**kw, non_blocking=True).contiguous()
        from ..training.noise import sample_noise
        noise, input_noise = sample_noise(c, batch["latents"], state, flow_matching=False)
        bsz = batch["latents"].shape[0]
        batch["noise"] = noise.to(batch["latents"].dtype).contiguous()
        batch["input_noise"] = input_noise.to(batch["latents"].dtype).contiguous()
        n_t = self.noise_schedule.config.num_train_timesteps
        weights = generate_timestep_weights(c, n_t).to(dev)
        if bsz > 1 and not c.disable_segmented_timestep_sampling:
            batch["timesteps"] = segmented_timestep_selection(n_t, bsz, weights, c, use_refiner_range=False).to(dev)
        else:
            batch["timesteps"] = torch.multinomial(weights, bsz, replacement=True).long()
        ca, cb = self._ddpm_coefs(batch["timesteps"], dev)
        noisy, _ = ops.ddpm_prep_pack(batch["latents"], batch["input_noise"], ca, cb, want_unpacked=True, want_packed=False)
        batch["noisy_latents"] = noisy
        return batch

    # ---- sdxl/model.py:306-373 ---------------------------------------------------------------------------------------
    def model_predict(self, prepared_batch: Dict[str, Any]) -> Dict[str, Any]:
        pb = prepared_batch
        dev = self.accelerator.device
        if self.model is None:
            raise RuntimeError("SDXL step has no UNet: pass the reference's UNet2DConditionModel as `unet=`")
        model_pred = self.model(
            pb["noisy_latents"].to(device=dev, dtype=self.config.base_weight_dtype),
            pb["timesteps"],
            pb["encoder_hidden_states"].to(device=dev, dtype=self.config.base_weight_dtype),
            pb["add_text_embeds"].to(device=dev, dtype=self.config.weight_dtype),
            added_cond_kwargs=pb["added_cond_kwargs"],
            cross_attention_kwargs=None,
            return_dict=False,
        )[0]
        return {"model_prediction": model_pred, "hidden_states_buffer": None, "urepa_hidden_states": None}

    def _packed_for_loss(self, model_output: Dict[str, Any]) -> torch.Tensor:
        return model_output["model_prediction"].contiguous()

    def loss(self, prepared_batch, model_output, apply_conditioning_mask: bool = True):
        c = self.config
        self._check_loss_supported(prepared_batch, apply_conditioning_mask)
        lt, hc = self._loss_kind(prepared_batch)
        snr_w = float(c.snr_weight) if (lt == "l2" and not c.snr_gamma) else 1.0
        weights = None
        if c.snr_gamma:
            weights = min_snr_loss_weights(prepared_batch["timesteps"].to(self.accelerator.device), self.noise_schedule,
                                           c.snr_gamma, self.PREDICTION_TYPE).float()
        if self.PREDICTION_TYPE == "v_prediction":
            from ..training.noise import get_velocity
            target = get_velocity(self.noise_schedule, prepared_batch["latents"], prepared_batch["noise"],
                                  prepared_batch["timesteps"]).contiguous()
        else:
            target = prepared_batch["noise"]
        return _TargetLossFn.apply(self._packed_for_loss(model_output), target, weights, snr_w, lt, hc, 2)
