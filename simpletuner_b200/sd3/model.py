"""SD3 training wrapper on libstb200 — mirror of the step-level API of reference
simpletuner/helpers/models/sd3/model.py (class SD3): `prepare_batch` (common.py:5862-6041, flow-matching
branch — the shared StepWrapper's), `model_predict` (`_model_predict_single`, sd3/model.py:540-569) and `loss`
(common.py:6217-6430, l2).  Differences from Flux that are reproduced here: latents go to the denoiser
un-packed [B,16,H,W]; timesteps are passed RAW (0..1000) after a cast to the bf16 weight dtype (quirk Q8);
no guidance input; pooled projections are 2048-wide; the prediction is un-patchified in (dy, dx, c) order.
"""
from __future__ import annotations

from typing import Any, Dict

from ..family import CONDITIONING_INPUTS, StepWrapper
from ..flux.model import default_config
from .transformer import SD3Transformer2DModel


class SD3(StepWrapper):
    NAME = "Stable Diffusion 3.x"
    DENOISER = SD3Transformer2DModel
    DEFAULT_CONFIG = staticmethod(default_config)
    PACKED_LAYOUT = "packed_dydxc"
    FULL_FINETUNE = True
    REFUSED_BATCH_KEYS = CONDITIONING_INPUTS

    def model_predict(self, prepared_batch: Dict[str, Any]) -> Dict[str, Any]:
        pb = prepared_batch
        B, Cc, Hh, Ww = pb["latents"].shape
        dev = self.accelerator.device
        # sd3/model.py:542 — raw timesteps in the weight dtype (bf16 rounds most of 0..1000; quirk Q8)
        timesteps = pb["timesteps"].to(device=dev, dtype=self.config.weight_dtype)
        out = self.model(
            hidden_states=pb["noisy_latents"], timestep=timesteps, encoder_hidden_states=pb["encoder_hidden_states"],
            pooled_projections=pb["added_cond_kwargs"]["text_embeds"], return_dict=False,
            _packed_latents=pb.get("_packed_noisy_latents"), _packed_output=True,
        )[0]
        return self._prediction_dict(out, (B, Cc, Hh, Ww))
