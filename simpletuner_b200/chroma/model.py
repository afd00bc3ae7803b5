"""Chroma training wrapper on libstb200: the step methods of reference `Chroma` (chroma/model.py) for the base, HD and
flash flavours, LoRA only.

  * `prepare_batch`   common.py:5862-6041 (flow-matching branch, the shared StepWrapper draw), then `_apply_chroma_flow_schedule`
                      (chroma/model.py:326-355, 854-865): sigma -> sigma^2 below 0.5, else 1 - (1 - sigma)^2, in the latents'
                      dtype, before the noisy latents are formed; the timesteps are the adjusted sigma x 1000.  No guidance.
  * `model_predict`   chroma/model.py:605-716 (`_model_predict_single`): the prompt mask is required, extended with ones over
                      the image tokens, and becomes a -inf per-key logit bias in every attention.
  * `loss` / `loss_with_logs`  common.py:6217-6430, the shared flow-matching loss.

The batch contract is the reference's: `latent_batch` [B, 16, h, w], `prompt_embeds` (T5, padded to the tokenizer length)
and `encoder_attention_mask` [B, S_txt] (or [B, 1, S_txt]).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Dict

import torch

from ..family import StepWrapper
from ..flux.model import default_config as flux_default_config, prepare_latent_image_ids
from .transformer import CHROMA_DEFAULT_LORA_TARGET, CHROMA_LORA_TARGETS, ChromaTransformer2DModel, adjust_chroma_sigmas


def default_config(**over) -> SimpleNamespace:
    cfg = dict(model_flavour="base", flux_lora_target=None, lora_type="standard")
    cfg.update(over)
    return flux_default_config(**cfg)


class Chroma(StepWrapper):
    """Drop-in for the reference `Chroma(ImageModelFoundation)` step methods.  The flow-matching draw, packing, prediction
    dict and loss are the shared StepWrapper's; the denoiser, the sigma remapping and the prompt mask are Chroma's."""

    NAME = "Chroma 1"
    GRAPH_REPLAY = False
    DENOISER = ChromaTransformer2DModel
    DEFAULT_CONFIG = staticmethod(default_config)
    FLAVOURS = ("base", "hd", "flash")          # reference chroma/model.py:65-70
    # Chroma's own options (control, the time-sign embedding) and, as for Qwen-Image, block swap, flow-map and MixFlow
    REFUSED_OPTIONS = ("control", "enable_time_sign_embed", "musubi_blocks_to_swap", "flowmap_enabled", "flow_map_enabled",
                       "mixflow_enabled")
    REFUSED_BATCH_KEYS = ("conditioning_latents", "conditioning_packed_latents", "conditioning_ids", "twinflow_time_sign",
                          "crepa_self_flow_mask", "crepa_teacher_sigmas")

    @classmethod
    def _default_lora_targets(cls, c) -> list:
        """Chroma.get_lora_target_layers (chroma/model.py:472-592): the `flux_lora_target` list; unset or unknown names take
        DEFAULT_LORA_TARGET, as the reference does."""
        return list(CHROMA_LORA_TARGETS.get(getattr(c, "flux_lora_target", None), CHROMA_DEFAULT_LORA_TARGET))

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
        t = self._batch_timesteps(pb["timesteps"].to(device=dev, dtype=self.config.base_weight_dtype), B)
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


def lora_targets(c) -> list:
    """`Chroma.lora_targets` as a module function."""
    return Chroma.lora_targets(c)
