"""Qwen-Image training wrapper on libstb200: the step methods of reference `QwenImage` (qwen_image/model.py) for the
text-to-image flavours v1.0 (Qwen/Qwen-Image) and v2.0 (Qwen/Qwen-Image-2512), LoRA only.

  * `prepare_batch`   common.py:5862-6041 (flow-matching branch), the shared StepWrapper draw
  * `model_predict`   qwen_image/model.py:1227-1345 (`_model_predict_standard`)
  * `loss` / `loss_with_logs`  common.py:6217-6430

The batch contract is the reference's: `latent_batch` ([B, 16, h, w] or [B, 16, 1, h, w]), `prompt_embeds` (Qwen2.5-VL
hidden states zero-padded to the longest prompt) and `encoder_attention_mask` (0/1 [B, S_txt]).  Whether the mask hides any
key is decided on the host from the collated mask before it is uploaded, so a batch whose keys are all kept (a typical
B = 1 batch) runs the attention kernels without a bias.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Dict

import torch

from .. import ops
from ..family import LOSS_LAYOUT, StepWrapper
from ..flux.blocks import FlowLossFn
from .transformer import QwenImageTransformer2DModel, mask_hides_keys


def default_config(**over) -> SimpleNamespace:
    cfg = dict(
        weight_dtype=torch.bfloat16, base_weight_dtype=torch.bfloat16, model_flavour="v2.0",
        flow_matching=True, flow_schedule_shift=3.0, flow_schedule_auto_shift=False, flow_sigmoid_scale=1.0,
        flow_use_uniform_schedule=False, flow_use_beta_schedule=False,
        input_perturbation=0.0, offset_noise=False, loss_type="l2", huber_c=0.1, huber_schedule="constant", snr_gamma=None,
        lora_rank=16, lora_alpha=None, lora_dropout=0.0, peft_lora_target_modules=None,
    )
    cfg.update(over)
    return SimpleNamespace(**cfg)


class QwenImage(StepWrapper):
    """Drop-in for the reference `QwenImage(ImageModelFoundation)` step methods.  The flow-matching draw, prediction dict and
    loss plumbing are the shared StepWrapper's; the denoiser, the 5-D latents and the prompt mask are Qwen's."""

    NAME = "Qwen-Image"
    # prepare_batch decides on the host whether the prompt mask hides a key, and the two answers take different kernels:
    # a replayed graph would keep the first batch's choice
    GRAPH_REPLAY = False
    DENOISER = QwenImageTransformer2DModel
    DEFAULT_CONFIG = staticmethod(default_config)
    FLAVOURS = ("v1.0", "v2.0")        # reference qwen_image/model.py:82-89; the edit flavours stay on the reference class
    # block swap is not implemented here, and flow-map and MixFlow training are not checked against the reference's Qwen step
    REFUSED_OPTIONS = ("musubi_blocks_to_swap", "flowmap_enabled", "flow_map_enabled", "mixflow_enabled")
    REFUSED_BATCH_KEYS = ("conditioning_latents", "conditioning_packed_latents", "control_latent_list",
                          "conditioning_image_embeds")      # the edit flavours' inputs

    def _noise_schedule(self):
        # reference setup_training_noise_schedule (qwen_image/model.py:348-370)
        return SimpleNamespace(config=SimpleNamespace(num_train_timesteps=1000, base_image_seq_len=256, max_image_seq_len=8192,
                                                      base_shift=0.5, max_shift=0.9))

    def prepare_batch(self, batch: Dict[str, Any], state: Dict[str, Any]) -> Dict[str, Any]:
        if not batch:
            return batch
        c = self.config
        self._check_supported(batch)
        dev = self.accelerator.device
        kw = {"device": dev, "dtype": c.weight_dtype}
        batch["encoder_hidden_states"] = batch["prompt_embeds"].to(**kw, non_blocking=True)
        latents = batch.get("latent_batch")
        if not hasattr(latents, "to"):
            raise ValueError("Received invalid value for latents.")
        if latents.dim() == 5 and latents.shape[2] != 1:
            raise NotImplementedError(f"Qwen-Image latents with {latents.shape[2]} frames are not supported")
        if latents.dim() not in (4, 5):
            raise ValueError(f"Qwen-Image latents must be [B, C, h, w] or [B, C, 1, h, w], got {tuple(latents.shape)}")
        lat = latents.to(**kw, non_blocking=True).contiguous()
        lat4 = lat.squeeze(2) if lat.dim() == 5 else lat
        batch["latents"] = lat
        mask = batch.get("encoder_attention_mask")
        if mask is not None and hasattr(mask, "to"):      # common.py:5911-5913
            if mask.dim() == 3 and mask.size(1) == 1:
                mask = mask.squeeze(1)
            # host decision before the upload: a mask that hides no key needs no bias (no device sync either way)
            batch["_qwen_masked_keys"] = True if mask.is_cuda else mask_hides_keys(mask)
            batch["encoder_attention_mask"] = mask.to(**kw, non_blocking=True)
        sigmas = self._flow_draw(batch, state, lat4)
        noisy, packed = ops.flow_prep_pack(lat4, batch["input_noise"], sigmas.float().contiguous(), want_unpacked=True)
        batch["noise"] = batch["noise"].view(lat.shape)
        batch["input_noise"] = batch["input_noise"].view(lat.shape)
        batch["noisy_latents"] = noisy.view(lat.shape)
        batch["_packed_noisy_latents"] = packed
        return batch

    def model_predict(self, prepared_batch: Dict[str, Any]) -> Dict[str, Any]:
        """qwen_image/model.py:1227-1345.  `timesteps` is left as it is (the reference divides a copy by 1000), and the
        mask's per-sample lengths are not read back to the host (the reference's `txt_seq_lens` does not change the
        result: RoPE spans the padded text length)."""
        pb = prepared_batch
        lat = pb["latents"]
        lat4 = lat.squeeze(2) if lat.dim() == 5 else lat
        B, Cc, Hh, Ww = lat4.shape
        if Hh // 2 < 1 or Ww // 2 < 1:
            raise ValueError(f"Packed latent grid is degenerate. Latent tensor shape: {tuple(lat4.shape)}")
        dev = self.accelerator.device
        packed = pb.get("_packed_noisy_latents")
        if packed is None:
            packed = self._pack(pb["noisy_latents"])
        t = self._batch_timesteps(pb["timesteps"].to(device=dev, dtype=torch.float32), B)
        mask = pb.get("encoder_attention_mask")
        if mask is not None and not pb.get("_qwen_masked_keys", True):
            mask = None
        if mask is not None and mask.dim() == 3 and mask.size(1) == 1:
            mask = mask.squeeze(1)
        out = self.model(hidden_states=packed, encoder_hidden_states=pb["encoder_hidden_states"],
                         encoder_hidden_states_mask=mask, timestep=t / 1000.0,
                         img_shapes=[(1, Hh // 2, Ww // 2)] * B, return_dict=False)[0]
        res = self._prediction_dict(out, (B, Cc, Hh, Ww))
        if lat.dim() == 5:      # the prediction gets the target's frame axis back
            res["model_prediction"] = res["_unpacked_ref"] = res["model_prediction"].unsqueeze(2)
        return res

    @classmethod
    def _pack(cls, pred: torch.Tensor) -> torch.Tensor:
        return super()._pack(pred.squeeze(2) if pred.dim() == 5 else pred)

    def loss(self, prepared_batch: Dict[str, Any], model_output: Dict[str, Any], apply_conditioning_mask: bool = True):
        self._check_loss_supported(prepared_batch, apply_conditioning_mask)
        lat, noise = prepared_batch["latents"], prepared_batch["noise"]
        if lat.dim() == 5:
            lat, noise = lat.squeeze(2), noise.squeeze(2)
        return FlowLossFn.apply(self._packed_for_loss(model_output), lat, noise, LOSS_LAYOUT[self.PACKED_LAYOUT],
                                *self._loss_kind(prepared_batch))


def lora_targets(c) -> list:
    """`QwenImage.lora_targets` as a module function."""
    return QwenImage.lora_targets(c)
