"""Reference-side shims: the code a SimpleTuner maintainer drops in to run the hot path on libstb200, shipped as
importable modules (INTEGRATION.md describes each seam; SURVEY.md 8b numbers them):

  foundation.py         B1 / B9 / B10  family wrapper mixin + `install()` (ModelRegistry.register under the same key)
  vae.py                B8             `post_vae_load_setup` / `encode_with_vae` mixin
  attention_backend.py  B3 / B4        packed-attention backend module + SDPA-signature wrapper (autograd-capable)

Nothing here imports the reference at module import time: `install()` does, and the mixins are ordinary classes that are
combined with the reference family class (`make_b200_family(RefFlux, "flux")`), so the same code is testable against a
stub that reproduces `ModelFoundation.load_model`'s hook order (tests/test_shim_cpu.py, tests/test_shim_gpu.py).
"""
from .foundation import (B200FoundationMixin, FAMILIES, OPT_IN_FAMILIES, install, install_lycoris, make_b200_family,  # noqa: F401
                         track_full_finetune)
from .vae import B200VAEMixin  # noqa: F401
