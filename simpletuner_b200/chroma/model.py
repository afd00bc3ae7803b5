"""Chroma training wrapper on libstb200: the step methods of reference `Chroma` (chroma/model.py) for the base, HD and
flash flavours, LoRA only.

  * `prepare_batch`   common.py:5862-6041 (flow-matching branch, as for Flux), then `_apply_chroma_flow_schedule`
                      (chroma/model.py:326-355, 854-865): sigma -> sigma^2 below 0.5, else 1 - (1 - sigma)^2, in the latents'
                      dtype, before the noisy latents are formed; the timesteps are the adjusted sigma x 1000.  No guidance.
  * `model_predict`   chroma/model.py:605-716 (`_model_predict_single`): the prompt mask is required, extended with ones over
                      the image tokens, and becomes a -inf per-key logit bias in every attention.
  * `loss` / `loss_with_logs`  common.py:6217-6430, the Flux loss path.

The batch contract is the reference's: `latent_batch` [B, 16, h, w], `prompt_embeds` (T5, padded to the tokenizer length)
and `encoder_attention_mask` [B, S_txt] (or [B, 1, S_txt]).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Dict, Optional

import torch

from ..flux.model import Flux, default_config as flux_default_config, prepare_latent_image_ids
from .transformer import (CHROMA_DEFAULT_LORA_TARGET, CHROMA_LORA_TARGETS, ChromaTransformer2DModel, adjust_chroma_sigmas,
                          chroma_target_supported)

FLAVOURS = ("base", "hd", "flash")          # reference chroma/model.py:65-70


def default_config(**over) -> SimpleNamespace:
    cfg = dict(model_flavour="base", flux_lora_target=None, lora_type="standard")
    cfg.update(over)
    return flux_default_config(**cfg)


def lora_targets(c) -> list:
    """Chroma.get_lora_target_layers (chroma/model.py:472-592) for standard LoRA: `peft_lora_target_modules` when given,
    else the `flux_lora_target` list; unset or unknown names take DEFAULT_LORA_TARGET, as the reference does."""
    manual = getattr(c, "peft_lora_target_modules", None)
    if manual:
        return list(manual)
    t = getattr(c, "flux_lora_target", None)
    return list(CHROMA_LORA_TARGETS.get(t, CHROMA_DEFAULT_LORA_TARGET) if t is not None else CHROMA_DEFAULT_LORA_TARGET)


class Chroma(Flux):
    """Drop-in for the reference `Chroma(ImageModelFoundation)` step methods.  Shares Flux's noise / sigma sampling,
    packing, prediction dict and loss; the denoiser, the sigma remapping and the prompt mask are Chroma's."""

    NAME = "Chroma 1"
    GRAPH_REPLAY = False

    def __init__(self, config: Optional[SimpleNamespace] = None, transformer: Optional[ChromaTransformer2DModel] = None,
                 device: Optional[torch.device] = None, **transformer_kwargs):
        self.config = config or default_config()
        dev = device or torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        self.accelerator = SimpleNamespace(device=dev)
        self.noise_schedule = SimpleNamespace(config=SimpleNamespace(num_train_timesteps=1000, patch_size=2,
                                                                       base_image_seq_len=256, max_image_seq_len=4096,
                                                                       base_shift=0.5, max_shift=1.15))
        self.model = transformer if transformer is not None else ChromaTransformer2DModel(**transformer_kwargs)

    def add_lora_adapter(self):
        c = self.config
        alpha = c.lora_alpha if c.lora_alpha is not None else c.lora_rank
        return self._denoiser().add_adapter(rank=c.lora_rank, lora_alpha=alpha, target_modules=lora_targets(c),
                                            lora_dropout=getattr(c, "lora_dropout", 0.0))

    def add_lycoris_adapter(self, lycoris_config):
        raise NotImplementedError("LyCORIS adapters on Chroma are not supported by the libstb200 path")

    @classmethod
    def validate_config(cls, c) -> None:
        """Every option of the reference this path does not run raises NotImplementedError, so that the shim keeps the
        reference class for it."""
        g = lambda k, d=None: getattr(c, k, d)
        fl = g("model_flavour", None) or "base"
        if fl not in FLAVOURS:
            raise NotImplementedError(f"Chroma model_flavour={fl!r} is not supported by the libstb200 path "
                                      f"(supported: {FLAVOURS})")
        if g("controlnet", False) or g("control", False):
            raise NotImplementedError("Chroma ControlNet / control training is not supported by the libstb200 path")
        if str(g("model_type", "lora")) != "lora":
            raise NotImplementedError(f"model_type={g('model_type')!r}: only LoRA training runs on the libstb200 path")
        lt = str(g("lora_type", "standard") or "standard").lower()
        if lt != "standard":
            raise NotImplementedError(f"lora_type={g('lora_type')!r} on Chroma is not supported by the libstb200 path")
        if g("use_dora", False):
            raise NotImplementedError("DoRA is not supported by the libstb200 path")
        if g("slider_lora_target", False):
            raise NotImplementedError("slider LoRA targets are not supported by the libstb200 Chroma path")
        for t in lora_targets(c):
            if not chroma_target_supported(t):
                raise NotImplementedError(f"LoRA target {t!r} is not supported by the libstb200 Chroma path (approximator, "
                                          "context embedder and other linears stay on the reference module)")
        if g("tread_config", None):
            raise NotImplementedError("TREAD routing is not supported by the libstb200 path")
        if g("musubi_blocks_to_swap", 0):
            raise NotImplementedError("musubi block swap is not supported by the libstb200 path")
        if g("flow_cubic_schedule", None) or g("flow_cubic_schedule_weights", None):
            raise NotImplementedError("the cubic-spline flow schedule is not part of the libstb200 step")
        for flag in ("twinflow_enabled", "crepa_enabled", "layersync_enabled", "scheduled_sampling_max_step_offset",
                     "diff2flow_enabled", "flowmap_enabled", "flow_map_enabled", "mixflow_enabled", "enable_time_sign_embed"):
            if g(flag, None):
                raise NotImplementedError(f"{flag} is not supported by the libstb200 path")
        if g("distillation_method", None) not in (None, "", "None"):
            raise NotImplementedError("distillation is not supported by the libstb200 path")

    def _check_supported(self, batch: Dict[str, Any]) -> None:
        for k in ("conditioning_latents", "conditioning_packed_latents", "conditioning_ids", "twinflow_time_sign",
                  "crepa_self_flow_mask", "crepa_teacher_sigmas"):
            if batch.get(k) is not None:
                raise NotImplementedError(f"Chroma batch input `{k}` is not supported by the libstb200 path")

    def _model_sigmas(self, sigmas: torch.Tensor, timesteps: torch.Tensor, latents: torch.Tensor):
        """_apply_chroma_flow_schedule (chroma/model.py:326-345, 854-865): the sigmas remapped in the latents' dtype and
        timesteps = adjusted sigma x 1000, unless a fast, beta or uniform schedule is configured."""
        c = self.config
        if any(getattr(c, k, False) for k in ("flux_fast_schedule", "flow_use_beta_schedule", "flow_use_uniform_schedule")):
            return sigmas, timesteps
        adjusted = adjust_chroma_sigmas(sigmas.to(device=latents.device, dtype=latents.dtype))
        return adjusted, adjusted * 1000.0

    def model_predict(self, prepared_batch: Dict[str, Any]) -> Dict[str, Any]:
        """chroma/model.py:605-716.  `timesteps` is left as it is (the reference divides a copy by 1000)."""
        pb = prepared_batch
        lat = pb["latents"]
        B, Cc, Hh, Ww = lat.shape
        dev = self.accelerator.device
        mask = pb.get("encoder_attention_mask")
        if mask is None:
            raise ValueError("No attention mask was found for Chroma training. Regenerate your text embedding cache to "
                             "include masks.")
        if mask.dim() == 3 and mask.size(1) == 1:
            mask = mask.squeeze(1)
        packed = pb.get("_packed_noisy_latents")
        if packed is None:
            packed = self._pack(pb["noisy_latents"])
        S_img = packed.shape[1]
        # _prepare_model_predict_timesteps (:357-400): the model dtype, then / num_train_timesteps in that dtype
        t = pb["timesteps"].to(device=dev, dtype=self.config.base_weight_dtype)
        if t.ndim == 0 or (t.ndim == 1 and t.shape[0] == 1):
            t = t.reshape(1).expand(B)
        if t.ndim != 1:
            raise NotImplementedError("token-wise timesteps are not supported by the libstb200 Chroma path")
        t = t / self.noise_schedule.config.num_train_timesteps
        # :649-665: the text mask as bool, extended with ones over the image tokens
        mask = mask.to(device=dev)
        mask = mask if mask.dtype == torch.bool else mask > 0
        joint = torch.cat([mask, torch.ones((B, S_img), device=dev, dtype=torch.bool)], dim=1)
        enc = pb["encoder_hidden_states"]
        out = self.model(hidden_states=packed, encoder_hidden_states=enc, timestep=t,
                         img_ids=prepare_latent_image_ids(Hh, Ww), txt_ids=torch.zeros(enc.shape[1], 3),
                         attention_mask=joint, return_dict=False)[0]
        return self._prediction_dict(out, (B, Cc, Hh, Ww))
