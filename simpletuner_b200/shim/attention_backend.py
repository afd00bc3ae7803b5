"""Seams B3 / B4: use only the wgmma attention under the unmodified diffusers model.

B4 — packed backend module.  The reference loads a module by name and calls whichever of these it exports
(helpers/training/attention_backend.py:236-254, 405-411): `flash_attn_qkvpacked_func(qkv[B,S,3,H,D], dropout_p,
softmax_scale, causal)` -> `out[B,S,H,D]` (:479-486).  Register it with
`_PACKED_BACKEND_ALIASES["b200"] = ("module", "simpletuner_b200.shim.attention_backend")` (:340-368).
The var-len entry points (:489-554) are deliberately NOT exported: the caller then keeps bool key-padding masks on its own
padded path (:456-476) instead of this module silently mis-handling them.

B3 — SDPA override.  `install_sdpa_override()` monkey-patches `torch.nn.functional.scaled_dot_product_attention` the way
the reference's SageAttention wrapper does (:1520-1587): same wrapper signature (:1554-1574), the original kept at
`F.scaled_dot_product_attention_sdpa` (:1160-1163), any exception -> fall back to the original (:1564-1572);
`restore_sdpa()` undoes it (:1149-1157).
"""
from __future__ import annotations

import logging
from typing import Optional

import torch
import torch.nn.functional as F

from ..attention import attention_bshd, attention_qkvpacked

logger = logging.getLogger("simpletuner_b200.shim")


def flash_attn_qkvpacked_func(qkv, dropout_p: float = 0.0, softmax_scale: Optional[float] = None, causal: bool = False,
                              **unused):
    if dropout_p:
        raise NotImplementedError("libstb200 attention has no attention dropout")
    if causal:
        raise NotImplementedError("libstb200 attention is non-causal (diffusion transformers)")
    return attention_qkvpacked(qkv, softmax_scale)


def key_bias_from_mask(attn_mask: torch.Tensor, B: int, H: int, Sq: int, Sk: int, dtype: torch.dtype) -> torch.Tensor:
    """The [B or 1, Sk] per-key view of an SDPA float `attn_mask` that is constant over heads and queries, decided from
    its shape and strides alone (values are never read: no device sync).  FluxAttnProcessor2_0 passes such a mask,
    [B, 1, 1, S] in the activation dtype (reference flux/transformer.py:170-173).  Any other mask raises
    NotImplementedError, so the override falls back to torch."""
    if attn_mask.dtype != dtype:
        raise NotImplementedError(f"libstb200 SDPA: attn_mask must be a float mask in the query dtype {dtype}, "
                                  f"got {attn_mask.dtype}")
    if not 1 <= attn_mask.dim() <= 4:
        raise NotImplementedError(f"libstb200 SDPA: attn_mask must have 1 to 4 dimensions, got {attn_mask.dim()}")
    m = attn_mask
    while m.dim() < 4:
        m = m.unsqueeze(0)
    mb, mh, mq, mk = m.shape
    if mb not in (1, B) or mk != Sk or m.stride(3) != 1 or any(n != 1 and s != 0 for n, s in ((mh, m.stride(1)),
                                                                                             (mq, m.stride(2)))):
        raise NotImplementedError(f"libstb200 SDPA: only a per-key attn_mask [B or 1, 1, 1, Sk] (heads / queries of size 1 "
                                  f"or stride 0, contiguous keys) is supported, got {tuple(attn_mask.shape)} strides "
                                  f"{attn_mask.stride()} for B={B} H={H} Sq={Sq} Sk={Sk}")
    if mh not in (1, H) or mq not in (1, Sq):
        raise NotImplementedError(f"libstb200 SDPA: attn_mask {tuple(attn_mask.shape)} does not broadcast to "
                                  f"[{B}, {H}, {Sq}, {Sk}]")
    return m[:, 0, 0, :]


def b200_sdpa(query, key, value, attn_mask=None, dropout_p=0.0, is_causal=False, scale=None, enable_gqa=False):
    """`F.scaled_dot_product_attention` signature, layout [B, H, S, D] (what the diffusers processors pass).  A float
    `attn_mask` runs when it is per-key (key_bias_from_mask); any other mask raises."""
    if dropout_p or is_causal or enable_gqa:
        raise NotImplementedError("libstb200 SDPA: dropout / causal / GQA are not supported")
    if query.dim() != 4 or key.shape[1] != query.shape[1]:
        raise NotImplementedError("libstb200 SDPA expects [B, H, S, D] with equal head counts")
    key_bias = None
    if attn_mask is not None:
        B, H, Sq, _ = query.shape
        key_bias = key_bias_from_mask(attn_mask, B, H, Sq, key.shape[2], query.dtype)
    q, k, v = (t.transpose(1, 2) for t in (query, key, value))   # [B, S, H, D] views: the kernels take strides, no copies
    if q.stride(-1) != 1 or k.stride(-1) != 1 or v.stride(-1) != 1:
        raise NotImplementedError("libstb200 SDPA needs a contiguous head dimension")
    return attention_bshd(q, k, v, scale, key_bias=key_bias).transpose(1, 2)


def install_sdpa_override() -> None:
    if getattr(F, "scaled_dot_product_attention_sdpa", None) is None:
        F.scaled_dot_product_attention_sdpa = F.scaled_dot_product_attention
    original = F.scaled_dot_product_attention_sdpa

    def wrapper(query, key, value, attn_mask=None, dropout_p=0.0, is_causal=False, scale=None, enable_gqa=False):
        try:
            return b200_sdpa(query, key, value, attn_mask=attn_mask, dropout_p=dropout_p, is_causal=is_causal, scale=scale,
                             enable_gqa=enable_gqa)
        except Exception as exc:   # the reference's convention (:1564-1572): log and fall back to the stock kernel
            logger.debug("libstb200 SDPA fell back to torch: %s", exc)
            kw = {"attn_mask": attn_mask, "dropout_p": dropout_p, "is_causal": is_causal, "scale": scale}
            if enable_gqa:
                kw["enable_gqa"] = True
            return original(query, key, value, **kw)

    wrapper._b200 = True
    F.scaled_dot_product_attention = wrapper


def restore_sdpa() -> None:
    original = getattr(F, "scaled_dot_product_attention_sdpa", None)
    if original is not None:
        F.scaled_dot_product_attention = original
