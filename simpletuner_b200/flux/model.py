"""Flux training wrapper on libstb200 — mirror of the step-level API the reference Trainer calls
(SURVEY.md §8b seam B9):

  * `prepare_batch(batch, state)`   reference helpers/models/common.py:5862-6041 (flow-matching branch)
  * `model_predict(prepared_batch)` reference helpers/models/flux/model.py:630-864 (`_model_predict_single`)
  * `loss(prepared_batch, model_output)` / `loss_with_logs(...)`  common.py:6217-6430, xm_mixin.py:476-485

The flow-matching batch draw, the packed prediction and the loss are the shared StepWrapper's (family.py); what is Flux's
own is the guidance input, Kontext, attention-masked training, LyCORIS LoKr and the `flux_lora_target` lists.  All tensor
arithmetic is libstb200 (flow_prep_pack / flow_mse_loss / the transformer); the patchify / unpatchify index math is folded
into those two kernels.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Dict, Optional

import torch

from .. import ops
from ..family import CONDITIONING_INPUTS, StepWrapper, lora_type
from .transformer import FLUX_LORA_TARGETS, FluxTransformer2DModel


def default_config(**over) -> SimpleNamespace:
    """Hot-path-relevant reference defaults (SURVEY.md §5 'Config / flags')."""
    cfg = dict(
        weight_dtype=torch.bfloat16, base_weight_dtype=torch.bfloat16,
        flow_matching=True, flow_schedule_shift=3.0, flow_schedule_auto_shift=False, flow_sigmoid_scale=1.0,
        flow_use_uniform_schedule=False, flow_use_beta_schedule=False, flux_fast_schedule=False,
        flux_guidance_mode="constant", flux_guidance_value=1.0, flux_guidance_min=0.0, flux_guidance_max=4.0,
        input_perturbation=0.0, offset_noise=False, loss_type="l2", huber_c=0.1, huber_schedule="constant", snr_gamma=None,
        lora_rank=16, lora_alpha=None, lora_dropout=0.0, flux_lora_target="all",
        flux_attention_masked_training=False,
    )
    cfg.update(over)
    return SimpleNamespace(**cfg)


class Flux(StepWrapper):
    """Drop-in for the reference `Flux(ImageModelFoundation)` step methods."""

    NAME = "Flux.1"
    DENOISER = FluxTransformer2DModel
    DEFAULT_CONFIG = staticmethod(default_config)
    LORA_TYPES = ("standard", "lycoris")        # LyCORIS: LoKr only (validate_config)
    REFUSED_BATCH_KEYS = CONDITIONING_INPUTS    # outside model_flavour='kontext'

    def __init__(self, config: Optional[SimpleNamespace] = None, transformer: Optional[FluxTransformer2DModel] = None,
                 device: Optional[torch.device] = None, **transformer_kwargs):
        super().__init__(config, transformer, device, **transformer_kwargs)
        # set_attn_processor refuses the flash processors (key-padding semantics) while the additive mask is in use
        self._denoiser().attention_masked_training = bool(getattr(self.config, "flux_attention_masked_training", False))

    @classmethod
    def _default_lora_targets(cls, c) -> list:
        """The `flux_lora_target` list (flux/model.py:1235-1383)."""
        return list(FLUX_LORA_TARGETS[getattr(c, "flux_lora_target", None) or "all"])

    def add_lycoris_adapter(self, lycoris_config):
        """trainer.py:3390-3505 (`lora_type = "lycoris"`): LycorisNetwork.apply_preset + create_lycoris + apply_to.  Takes the
        parsed `lycoris_config.json` (or its path); returns the network whose `.parameters()` the optimizer trains."""
        from .. import lycoris as LY
        if isinstance(lycoris_config, str):
            import json
            with open(lycoris_config, "r") as f:
                lycoris_config = json.load(f)
        cfg = dict(lycoris_config)
        multiplier = int(cfg.pop("multiplier", 1))
        linear_dim = int(cfg.pop("linear_dim", 4))
        linear_alpha = int(cfg.pop("linear_alpha", 1))
        preset = cfg.pop("apply_preset", None)
        if preset:
            LY.LycorisNetwork.apply_preset(preset)
        net = LY.create_lycoris(self._denoiser(), multiplier, linear_dim, linear_alpha, **cfg)
        net.apply_to()
        self.lycoris_wrapped_network = net
        return net

    # ------------------------------------------------------------------------------------------
    @classmethod
    def validate_config(cls, c) -> None:
        """StepWrapper.validate_config plus Flux's own options: the `flux_lora_target` list, the LyCORIS algorithm,
        attention-masked training and Kontext's loss."""
        g = lambda k, d=None: getattr(c, k, d)
        tgt = g("flux_lora_target", "all") or "all"
        if tgt not in FLUX_LORA_TARGETS:       # "ai-toolkit" (adaLN linears) / "controlnet" stay on the reference module
            raise NotImplementedError(f"flux_lora_target={tgt!r} is not supported by the libstb200 path "
                                      f"(supported: {sorted(FLUX_LORA_TARGETS)})")
        super().validate_config(c)
        if lora_type(c) == "lycoris":
            cfg = g("lycoris_config", None)
            if isinstance(cfg, str):
                import json
                with open(cfg, "r") as f:
                    cfg = json.load(f)
            if isinstance(cfg, dict):       # only LoKr (the reference's documented default) runs here
                from ..lycoris import validate_lycoris_config
                validate_lycoris_config(cfg)
        check_masked_training(c)
        if is_kontext(c):
            lt = str(g("loss_type", "l2"))
            if lt in ("huber", "smooth_l1") and g("huber_schedule", "constant") != "constant":
                # the reference feeds Kontext's 2-D timesteps [B, S_scene + S_c] to compute_scheduled_huber_c
                raise NotImplementedError(f"Kontext with loss_type={lt!r} and huber_schedule={g('huber_schedule')!r} is not "
                                          "supported by the libstb200 path (l2 or a constant huber_c run)")

    def _check_supported(self, batch: Dict[str, Any]) -> None:
        """Masked training outside `check_masked_training`'s rule or without the batch's `encoder_attention_mask`
        (flux/model.py:813-822), conditioning latents outside the Kontext flavour, and pre-packed Kontext inputs that
        `prepare_batch` did not build (flux/model.py:757-786) raise."""
        if check_masked_training(self.config) and batch.get("encoder_attention_mask") is None:
            raise NotImplementedError("flux_attention_masked_training: the batch has no encoder_attention_mask (the text-embed "
                                      "cache must carry attention_masks)")
        if not is_kontext(self.config):
            return super()._check_supported(batch)
        for k in ("conditioning_packed_latents", "conditioning_ids"):
            if batch.get(k) is not None:
                raise NotImplementedError(f"Kontext input `{k}` without `conditioning_latents`: the libstb200 Flux path "
                                          "packs the reference latents itself")

    def _prep_pack(self, batch: Dict[str, Any], state: Dict[str, Any], interp: torch.Tensor) -> Dict[str, Any]:
        cond = self._kontext_conditions(batch, state) if is_kontext(self.config) else None
        if cond is None:
            return super()._prep_pack(batch, state, interp)
        # Kontext: the x_embedder input [B, S_scene + S_c, 64] is filled in place, the noisy scene tokens first and then each
        # reference image's packed tokens (flux/model.py:767-779 concatenates them), with no cat / permute copies
        conds, ids = cond
        dev = self.accelerator.device
        bsz, C, Hh, Ww = batch["latents"].shape
        S_scene = (Hh // 2) * (Ww // 2)
        S_c = ids.shape[0]
        joint = torch.empty((bsz, S_scene + S_c, 4 * C), device=dev, dtype=torch.bfloat16)
        noisy, _ = ops.flow_prep_pack(batch["latents"], batch["input_noise"], interp.float().contiguous(), want_unpacked=True,
                                      out=joint[:, :S_scene])
        off = S_scene
        for lat in conds:
            n = (lat.shape[2] // 2) * (lat.shape[3] // 2)
            ops.flow_prep_pack(lat, None, None, out=joint[:, off:off + n])
            off += n
        batch["noisy_latents"] = noisy
        batch["_packed_noisy_latents"] = joint
        batch["_kontext_ids"] = ids
        batch["conditioning_packed_latents"] = joint[:, S_scene:]
        batch["conditioning_ids"] = ids.to(dev, torch.bfloat16)[None].expand(bsz, -1, -1)   # the reference's dtype
        return batch

    def _kontext_conditions(self, batch: Dict[str, Any], state: Dict[str, Any]):
        """Flux.prepare_batch_conditions (flux/model.py:522-555) then the base class's list collapse (common.py:4668-4683).
        Returns None (plain step) or (the conditioning latents on the device, bf16 contiguous [B, 16, h, w] each, in
        sequence order; their ids [S_c, 3] built on the host from the shapes)."""
        cond = batch.get("conditioning_latents")
        if cond is None:
            return None
        args = state.get("args", {}) if isinstance(state, dict) else {}
        mode = args.get("conditioning_multidataset_sampling", "random") if isinstance(args, dict) else \
            getattr(args, "conditioning_multidataset_sampling", "random")
        if mode == "random" and isinstance(cond, list) and len(cond) >= 1:
            cond = cond[0]
        conds = list(cond) if isinstance(cond, list) else [cond]
        B, C = batch["latents"].shape[:2]
        dev = self.accelerator.device
        out = []
        for lat in conds:
            if lat.dim() == 3 and lat.shape[0] == C:          # (C, H, W): one image without a batch dimension
                lat = lat.unsqueeze(0)
            if lat.dim() != 4 or lat.shape[1] != C or lat.shape[0] != B or lat.shape[2] % 2 or lat.shape[3] % 2:
                raise ValueError(f"conditioning latents must be [{B}, {C}, h, w] with even h, w; got {tuple(lat.shape)}")
            out.append(lat.to(device=dev, dtype=torch.bfloat16, non_blocking=True).contiguous())
        ids = kontext_ids([tuple(t.shape[2:]) for t in out])
        cl = batch.get("conditioning_latents")
        if isinstance(cl, list) and len(cl) > 0:              # common.py:4672-4683
            types = batch.get("conditioning_latents_type")
            sel = 0
            if batch.get("conditioning_type") == "reference_strict" and isinstance(types, list) and "reference_strict" in types:
                sel = types.index("reference_strict")
            batch["conditioning_latents"] = cl[sel]
            if isinstance(types, list) and sel < len(types):
                batch["conditioning_latents_type"] = types[sel]
        return out, ids

    # ------------------------------------------------------------------------------------------
    def _guidance(self, bsz: int, device) -> Optional[torch.Tensor]:
        if not self._denoiser().config.guidance_embeds:
            return None
        c = self.config
        # flux/model.py:682-706 (`_flux_guidance_scales`): "constant" or one python `random.uniform` draw per sample
        if c.flux_guidance_mode == "constant":
            return torch.full((bsz,), float(c.flux_guidance_value), device=device, dtype=torch.float32)
        if c.flux_guidance_mode == "random-range":
            import random
            scales = [random.uniform(c.flux_guidance_min, c.flux_guidance_max) for _ in range(bsz)]
            return torch.tensor(scales, device=device, dtype=torch.float32)
        raise ValueError(f"Unsupported Flux guidance mode: {c.flux_guidance_mode!r}.")

    def model_predict(self, prepared_batch: Dict[str, Any]) -> Dict[str, Any]:
        """flux/model.py:707-864."""
        pb = prepared_batch
        lat = pb["latents"]
        B, Cc, Hh, Ww = lat.shape
        dev = self.accelerator.device
        packed = pb.get("_packed_noisy_latents")
        if packed is None:
            packed = self._pack(pb["noisy_latents"])
        img_ids = prepare_latent_image_ids(Hh, Ww)
        txt_ids = torch.zeros(pb["encoder_hidden_states"].shape[1], 3)
        # side effect kept from the reference: timesteps are overwritten with t / 1000 (flux/model.py:739-745)
        t = pb["timesteps"] = pb["timesteps"].to(device=dev, dtype=torch.float32) / self.noise_schedule.config.num_train_timesteps
        cond_ids = pb.get("_kontext_ids")
        S_c = 0 if cond_ids is None else cond_ids.shape[0]
        if S_c:
            if t.dim() != 1:
                raise NotImplementedError("Kontext with token-wise timesteps is not supported by the libstb200 Flux path")
            # _extend_conditioning_timesteps (flux/model.py:602-618): later readers of the batch see [B, S_scene + S_c]
            pb["timesteps"] = torch.cat([t[:, None].expand(-1, img_ids.shape[0]),
                                         torch.zeros(B, S_c, device=dev, dtype=torch.float32)], dim=1)
            img_ids = torch.cat([img_ids, cond_ids], dim=0)
        attention_mask = None
        if getattr(self.config, "flux_attention_masked_training", False):   # flux/model.py:813-822
            attention_mask = pb.get("encoder_attention_mask")
            if attention_mask is None:
                raise ValueError("No attention mask was discovered when attempting validation - this means you need to "
                                 "recreate your text embed cache.")
            if attention_mask.dim() == 3 and attention_mask.size(1) == 1:
                attention_mask = attention_mask.squeeze(1)   # [B, 1, S] -> [B, S]
        out = self.model(
            hidden_states=packed, timestep=t, guidance=self._guidance(B, dev),
            pooled_projections=pb["added_cond_kwargs"]["text_embeds"], encoder_hidden_states=pb["encoder_hidden_states"],
            txt_ids=txt_ids, img_ids=img_ids, joint_attention_kwargs=None, return_dict=False, attention_mask=attention_mask,
            **({"conditioning_tokens": S_c} if S_c else {}),
        )[0]
        return self._prediction_dict(out, (B, Cc, Hh, Ww))


def is_kontext(c) -> bool:
    """model_flavour "kontext" (flux/model.py:94, black-forest-labs/flux.1-kontext-dev)."""
    return getattr(c, "model_flavour", None) == "kontext"


def kontext_ids(sizes) -> torch.Tensor:
    """Position ids [S_c, 3] of the Kontext conditioning tokens for latents of the (h, w) `sizes`, in sequence order:
    build_kontext_inputs (flux/__init__.py:64-172) on the host from shapes alone.  (1, y, x) over each (h/2, w/2) patch
    grid, offset by the ComfyUI scheme (x0 / y0: the next image goes right of or below what is placed, whichever keeps
    max(x, y) smaller), then rounded through bf16 as the reference's `.to(weight_dtype)` does (so positions above 256
    lose their low bits), returned as float32 like the reference's cat with the fp32 scene ids."""
    x0 = y0 = 0
    out = []
    for H, W in sizes:
        x = y = 0
        if H + y0 > W + x0:
            x = x0
        else:
            y = y0
        iy = torch.arange(H // 2) + y // 2
        ix = torch.arange(W // 2) + x // 2
        grid = torch.stack(torch.meshgrid(iy, ix, indexing="ij"), dim=-1).reshape(-1, 2)
        out.append(torch.cat([torch.ones_like(grid[:, :1]), grid], dim=1))
        x0 = max(x0, W + x)
        y0 = max(y0, H + y)
    return torch.cat(out, 0).to(torch.bfloat16).to(torch.float32)


def check_masked_training(c) -> bool:
    """True when `flux_attention_masked_training` is on and this path reproduces the reference's mask semantics; raises
    NotImplementedError when it is on and the semantics are another's or unknown.

    The reference's default processor (attention_mechanism "diffusers", un-fused QKV: FluxAttnProcessor2_0) passes the
    float mask `(mask > 0).to(dtype)` to SDPA, which ADDS it to the logits: kept text keys and every image key get +1,
    padded text keys +0, and nothing is masked out (flux/transformer.py:170-173, 200-207; SURVEY.md quirk Q2).  That is
    what runs here.  A flash mechanism with fused QKV uses FluxFusedFlashAttnProcessor3, a varlen path with real key
    padding (flux/model.py:369-380, flux/attention.py:207-210, 307-311); other mechanisms swap SDPA for other kernels."""
    g = lambda k, d=None: getattr(c, k, d)
    if not g("flux_attention_masked_training", False):
        return False
    mech = g("attention_mechanism", None)
    if mech is None:
        raise NotImplementedError("flux_attention_masked_training: the config names no attention_mechanism, so the mask "
                                  "semantics the reference would apply are unknown; use the reference module")
    if mech != "diffusers":
        raise NotImplementedError(f"flux_attention_masked_training with attention_mechanism={mech!r}: only 'diffusers' "
                                  "(the additive SDPA mask) runs on the libstb200 Flux path")
    if g("fuse_qkv_projections", False):
        raise NotImplementedError("flux_attention_masked_training with fuse_qkv_projections: the reference then masks "
                                  "through a fused processor; only the un-fused 'diffusers' processor runs here")
    return True


def prepare_latent_image_ids(height: int, width: int) -> torch.Tensor:
    """flux/__init__.py:47-61: ids[S_img, 3] = (0, row, col) over the (H/2, W/2) patch grid, float32."""
    ids = torch.zeros(height // 2, width // 2, 3)
    ids[..., 1] = ids[..., 1] + torch.arange(height // 2)[:, None]
    ids[..., 2] = ids[..., 2] + torch.arange(width // 2)[None, :]
    return ids.reshape(-1, 3).to(torch.float32)
