"""PixArt-Sigma training wrapper on libstb200 — mirror of the step-level API of reference
simpletuner/helpers/models/pixart/model.py (class PixartSigma, family key "pixart_sigma"):

  * `prepare_batch`   reference common.py:5862-6041, epsilon branch: `randn_like` noise, integer timesteps from
                      `generate_timestep_weights` + `segmented_timestep_selection` (bsz > 1) or one `multinomial`
                      (custom_schedule.py:18-106), `DDPMScheduler.add_noise` in fp32 then `.to(weight_dtype)` (:5998-6002)
  * `model_predict`   reference pixart/model.py:274-319: raw integer timesteps, `encoder_attention_mask`,
                      resolution / aspect-ratio conditioning from the LATENT shape (quirk Q4, :360-379), and only the
                      first half of the 8 output channels kept (`.chunk(2, dim=1)[0]`, :313)
  * `loss`            reference common.py:6376-6398, 6426-6429: fp32 MSE against the noise, optional min-SNR weights.

The DDPM scheduler is the diffusers `DDPMScheduler` the checkpoint's scheduler_config.json describes (PixArt-Sigma:
1000 steps, linear betas 1e-4..0.02, epsilon) — restated in training/noise.py.  add_noise + 2x2 patchify and the
weighted MSE (+ its gradient) are single libstb200 kernels; because the learned-sigma half of `proj_out` never reaches
the loss, the tail GEMM only computes the 16 kept features.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Dict

import torch

from .. import ops
from ..family import LOSS_LAYOUT, StepWrapper
from ..flux.model import default_config as _flux_defaults
from ..training.noise import make_ddpm_schedule, min_snr_loss_weights
from ..training.schedule import generate_timestep_weights, segmented_timestep_selection
from .transformer import PixArtTransformer2DModel


def default_config(**over) -> SimpleNamespace:
    cfg = vars(_flux_defaults())
    cfg.update(flow_matching=False, prediction_type="epsilon", snr_weight=1.0, offset_noise=False,
               timestep_bias_strategy="none", timestep_bias_portion=0.25, timestep_bias_multiplier=1.0,
               timestep_bias_begin=0, timestep_bias_end=1000, disable_segmented_timestep_sampling=False,
               refiner_training=False, refiner_training_invert_schedule=False, refiner_training_strength=0.2,
               max_grad_norm=0.01)  # pixart/model.py:688-696 forces max_grad_norm to 0.01
    cfg.update(over)
    return SimpleNamespace(**cfg)


class _TargetLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred_packed, target, weights, snr_weight, loss_type="l2", huber_c=None, layout=1):
        loss, dpred = ops.target_mse_loss(pred_packed.contiguous(), target, weights, want_grad=True, grad_scale=snr_weight,
                                          layout=layout, loss_type=loss_type, huber_c=huber_c)
        ctx.save_for_backward(dpred)
        return loss[0] * snr_weight if snr_weight != 1.0 else loss[0]

    @staticmethod
    def backward(ctx, g):
        (dpred,) = ctx.saved_tensors
        return (dpred.float() * g.float()).to(dpred.dtype), None, None, None, None, None, None   # fp32 scale, see FlowLossFn


class PixartSigma(StepWrapper):
    NAME = "PixArt Sigma"
    PREDICTION_TYPE = "epsilon"
    PREDICTION_TYPES = ("epsilon", "v_prediction")
    LATENT_CHANNEL_COUNT = 4
    DENOISER = PixArtTransformer2DModel
    DEFAULT_CONFIG = staticmethod(default_config)
    PACKED_LAYOUT = "packed_dydxc"
    FULL_FINETUNE = True

    def _noise_schedule(self):
        # PixArt-Sigma scheduler_config.json: DDPM, 1000 steps, linear betas 1e-4 .. 0.02, epsilon
        return make_ddpm_schedule(1000, 0.0001, 0.02, "linear")

    def prepare_batch(self, batch: Dict[str, Any], state: Dict[str, Any]) -> Dict[str, Any]:
        if not batch:
            return batch
        c = self.config
        dev = self.accelerator.device
        kw = {"device": dev, "dtype": c.weight_dtype}
        if batch.get("prompt_embeds") is not None:
            batch["encoder_hidden_states"] = batch["prompt_embeds"].to(**kw, non_blocking=True)
        batch["added_cond_kwargs"] = {}
        latents = batch.get("latent_batch")
        if not hasattr(latents, "to"):
            raise ValueError("Received invalid value for latents.")
        batch["latents"] = latents.to(**kw, non_blocking=True).contiguous()
        mask = batch.get("encoder_attention_mask")
        if mask is not None and hasattr(mask, "to"):
            batch["encoder_attention_mask"] = mask.to(**kw)
        from ..training.noise import sample_noise
        noise, input_noise = sample_noise(c, batch["latents"], state, flow_matching=False)   # common.py:5936-5967
        bsz = batch["latents"].shape[0]
        batch["noise"] = noise.to(batch["latents"].dtype).contiguous()
        batch["input_noise"] = input_noise.to(batch["latents"].dtype).contiguous()
        n_t = self.noise_schedule.config.num_train_timesteps
        weights = generate_timestep_weights(c, n_t).to(dev)              # common.py:5982-5984
        if bsz > 1 and not c.disable_segmented_timestep_sampling:
            batch["timesteps"] = segmented_timestep_selection(n_t, bsz, weights, c, use_refiner_range=False).to(dev)
        else:
            batch["timesteps"] = torch.multinomial(weights, bsz, replacement=True).long()
        ca, cb = self._ddpm_coefs(batch["timesteps"], dev)
        noisy, packed = ops.ddpm_prep_pack(batch["latents"], batch["input_noise"], ca, cb, want_unpacked=True, want_packed=True)
        batch["noisy_latents"] = noisy
        batch["_packed_noisy_latents"] = packed
        return batch

    def _build_added_cond_kwargs(self, prepared_batch: dict) -> dict:
        """pixart/model.py:360-379."""
        dev = self.accelerator.device
        nl = prepared_batch["noisy_latents"]
        B, height, width = nl.shape[0], nl.shape[-2], nl.shape[-1]
        resolution = prepared_batch.get("resolution")
        aspect_ratio = prepared_batch.get("aspect_ratio")
        # (the fall-back constants are cached per latent shape: building a device tensor from a Python list is a pageable
        # host-to-device copy, which must not happen inside a CUDA-graph capture of this call)
        cache = self.__dict__.setdefault("_cond_const_cache", {})
        if resolution is None:
            key = ("res", height, width, str(dev))
            if key not in cache:
                cache[key] = torch.tensor([[height, width]], device=dev)
            resolution = cache[key].expand(B, -1)
        else:
            resolution = resolution.to(device=dev, dtype=self.config.base_weight_dtype)
        if aspect_ratio is None:
            key = ("ar", height, width, str(dev))
            if key not in cache:
                cache[key] = torch.tensor([[float(height / width)]], device=dev)
            aspect_ratio = cache[key].expand(B, -1)
        else:
            aspect_ratio = aspect_ratio.to(device=dev, dtype=self.config.base_weight_dtype)
        return {"resolution": resolution, "aspect_ratio": aspect_ratio}

    def model_predict(self, prepared_batch: Dict[str, Any]) -> Dict[str, Any]:
        pb = prepared_batch
        B, Cc, Hh, Ww = pb["noisy_latents"].shape
        if Cc != self.LATENT_CHANNEL_COUNT:
            raise ValueError(f"{self.NAME} requires a latent size of {self.LATENT_CHANNEL_COUNT} channels. "
                             "Ensure you are using the correct VAE cache path.")
        timesteps = self._batch_timesteps(pb["timesteps"].to(self.accelerator.device), B)
        mask = pb.get("encoder_attention_mask")
        out = self.model(
            pb["noisy_latents"], encoder_hidden_states=pb["encoder_hidden_states"], timestep=timesteps,
            encoder_attention_mask=mask, added_cond_kwargs=self._build_added_cond_kwargs(pb), return_dict=False,
            _packed_latents=pb.get("_packed_noisy_latents"), _packed_output="eps_half",
        )[0]
        return self._prediction_dict(out, (B, Cc, Hh, Ww))

    def loss(self, prepared_batch, model_output, apply_conditioning_mask: bool = True):
        c = self.config
        self._check_loss_supported(prepared_batch, apply_conditioning_mask)
        lt, hc = self._loss_kind(prepared_batch)
        # common.py:6376-6398: `snr_weight` multiplies the plain-l2 branch only; huber / smooth_l1 and the min-SNR
        # branch do not apply it
        snr_w = float(c.snr_weight) if (lt == "l2" and not c.snr_gamma) else 1.0
        weights = None
        if c.snr_gamma:
            weights = min_snr_loss_weights(prepared_batch["timesteps"].to(self.accelerator.device), self.noise_schedule,
                                           c.snr_gamma, self.PREDICTION_TYPE).float()
        if self.PREDICTION_TYPE == "v_prediction":              # common.py:4648-4653 (DDPMScheduler.get_velocity, latent dtype)
            from ..training.noise import get_velocity
            target = get_velocity(self.noise_schedule, prepared_batch["latents"], prepared_batch["noise"],
                                  prepared_batch["timesteps"]).contiguous()
        else:
            target = prepared_batch["noise"]
        return _TargetLossFn.apply(self._packed_for_loss(model_output), target, weights, snr_w, lt, hc,
                                   LOSS_LAYOUT[self.PACKED_LAYOUT])
