"""Seam B8: VAE latent encode.  `load_vae` ends with `self.post_vae_load_setup()` (common.py:2747-2757) and
`VAECache.encode_images` reaches the VAE through `encode_cache_batch -> encode_with_vae(vae, samples)`
(common.py:2766-2779), accepting an object with `.latent_dist.sample()` (caching/vae.py:1331-1343).  Qwen-Image's
AutoencoderKLQwenImage is encoded by vae.qwen_image.QwenImageVAE for single-frame, untiled batches."""
from __future__ import annotations

import logging

logger = logging.getLogger("simpletuner_b200.shim")

_CFG = ("in_channels", "latent_channels", "block_out_channels", "layers_per_block", "norm_num_groups", "use_quant_conv",
        "scaling_factor", "shift_factor", "mid_block_add_attention")


# AutoencoderKLQwenImage (Wan 2.1); the last three only to refuse Wan 2.2 style configs
_QWEN_CFG = ("base_dim", "z_dim", "dim_mult", "num_res_blocks", "attn_scales", "temperal_downsample", "dropout",
             "latents_mean", "latents_std", "is_residual", "patch_size", "in_channels")


def build_b200_vae(ref_vae, device):
    """B200 encoder half carrying the reference VAE's encoder / quant_conv weights: QwenImageVAE for a Wan 2.1 config
    (`z_dim` / `base_dim`), AutoencoderKL otherwise."""
    c = ref_vae.config
    get = (lambda k, d=None: c.get(k, d)) if isinstance(c, dict) else (lambda k, d=None: getattr(c, k, d))
    if get("z_dim") is not None or get("base_dim") is not None:
        from ..vae.qwen_image import QwenImageVAE

        vae = QwenImageVAE(**{k: get(k) for k in _QWEN_CFG if get(k) is not None})
    else:
        from ..vae.autoencoder import AutoencoderKL

        vae = AutoencoderKL(**{k: get(k) for k in _CFG if get(k, None) is not None or k == "shift_factor"})
    enc = {k: v for k, v in ref_vae.state_dict().items() if k.startswith(("encoder.", "quant_conv."))}
    vae.load_state_dict(enc, strict=True)
    return vae.to(device)


class B200VAEMixin:
    _b200_vae = None

    def post_vae_load_setup(self):
        parent = getattr(super(), "post_vae_load_setup", None)
        if callable(parent):
            parent()
        self._b200_vae = None
        try:
            self._b200_vae = build_b200_vae(self.vae, self.accelerator.device)
        except (NotImplementedError, RuntimeError, KeyError, TypeError) as exc:   # unsupported VAE flavour -> reference path
            logger.warning("libstb200 VAE encode not used: %s", exc)

    def encode_with_vae(self, vae, samples):
        if self._b200_vae is None or vae is not getattr(self, "vae", None) or not _b200_encodes(self._b200_vae, vae, samples):
            return super().encode_with_vae(vae, samples)
        return self._b200_vae.encode(samples)


def _b200_encodes(b200_vae, ref_vae, samples) -> bool:
    """The Qwen-Image encoder takes single-frame [B, 3, 1, H, W] batches with H and W multiples of its downsampling
    factor, from a VAE without tiling: video and tiled encoding (different numbers at the tile seams) stay with the
    reference VAE."""
    from ..vae.qwen_image import QwenImageVAE

    if not isinstance(b200_vae, QwenImageVAE):
        return True
    m = b200_vae.spatial_multiple
    return (samples.dim() == 5 and samples.shape[2] == 1 and not getattr(ref_vae, "use_tiling", False)
            and samples.shape[3] % m == 0 and samples.shape[4] % m == 0)
