"""Text-encoder embed path (SURVEY.md 8f rank 4): the two encoders the reference's Flux pipeline runs when prompt embeddings are
not pre-cached — `T5EncoderModel` (T5 v1.1 XXL) and `CLIPTextModel` (CLIP-L), transformers classes called at
simpletuner/helpers/models/flux/pipeline.py:1085 and :1127-1130 (driven by Flux._encode_prompts, flux/model.py:497-520, and the
text-embed cache, helpers/caching/text_embeds.py) — on the libstb200 kernels: wgmma GEMMs with fused epilogues (residual add,
tanh-GELU, gated multiply, quick-GELU), the wgmma attention forward with an additive bias tile (T5 relative-position bias /
CLIP causal mask), and the row-norm kernels.  Inference only (the reference never trains these in the Flux recipes covered here);
tokenisation (sentencepiece / BPE) stays the caller's.
"""
from .clip import CLIPTextModel  # noqa: F401
from .t5 import T5EncoderModel  # noqa: F401
from .embed import encode_token_ids  # noqa: F401
