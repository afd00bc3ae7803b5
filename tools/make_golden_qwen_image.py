"""Writes tests/golden/qwen_image_golden.pt: the reference's own Qwen-Image functions on small inputs.

Runs, lifted from a SimpleTuner checkout by oracle/ref_extract (qwen_image/transformer.py), with torch stand-ins for the
diffusers layers (Attention / RMSNorm / FeedForward / TimestepEmbedding / AdaLayerNormContinuous parameter holders,
`Timesteps(scale=1000)` as diffusers' get_timestep_embedding, and SDPA with a bool key mask for the attention dispatch):
  * `QwenEmbedRope.forward` + `precompute_real_rope_qwen` (:351-368, :531-644): square, non-square and odd patch grids,
    two text lengths each;
  * `compute_text_seq_len_from_mask` (:371-394);
  * `QwenTimestepProjEmbeddings.forward` (:460-528) with the model's bf16 rounding of t (:1295);
  * `QwenImageTransformerBlock._modulate` (:867-910);
  * `QwenDoubleStreamAttnProcessor2_0.__call__` (:662-821): B = 1 unpadded and padded, B = 3 ragged prefix masks, B = 2
    with a non-prefix mask, and B = 2 with one all-zero mask;
  * the parameter names and shapes of `QwenImageTransformer2DModel.__init__` (:1045-1114) at a small config.

    SIMPLETUNER_SRC=<SimpleTuner checkout> python tools/make_golden_qwen_image.py
"""
from __future__ import annotations

import functools
import math
import sys
import types
from pathlib import Path

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import ref_extract as R  # noqa: E402

OUT = ROOT / "tests" / "golden" / "qwen_image_golden.pt"
TR = "helpers/models/qwen_image/transformer.py"
ROPE_CASES = [(8, 8), (6, 10), (9, 7)]          # (h, w) patch grids
TXT_LENS = (5, 12)


class Timesteps(nn.Module):
    """diffusers Timesteps -> get_timestep_embedding(t, C, flip_sin_to_cos, downscale_freq_shift, scale)."""

    def __init__(self, num_channels, flip_sin_to_cos, downscale_freq_shift, scale=1):
        super().__init__()
        self.c, self.flip, self.shift, self.scale = num_channels, flip_sin_to_cos, downscale_freq_shift, scale

    def forward(self, t):
        half = self.c // 2
        exponent = -math.log(10000) * torch.arange(0, half, dtype=torch.float32, device=t.device)
        exponent = exponent / (half - self.shift)
        emb = t[:, None].float() * torch.exp(exponent)[None, :]
        emb = self.scale * emb
        emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
        if self.flip:
            emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
        return emb


class TimestepEmbedding(nn.Module):
    def __init__(self, in_channels, time_embed_dim):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)

    def forward(self, x):
        return self.linear_2(self.act(self.linear_1(x)))


class RMSNorm(nn.Module):
    def __init__(self, dim, eps=1e-6, elementwise_affine=True):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(dim))

    def forward(self, x):
        var = x.float().pow(2).mean(-1, keepdim=True)
        return (x * torch.rsqrt(var + self.eps)) * self.weight


class Attention(nn.Module):
    """diffusers Attention(added_kv_proj_dim=dim, context_pre_only=False, bias=True, qk_norm="rms_norm")."""

    def __init__(self, query_dim, cross_attention_dim=None, added_kv_proj_dim=None, dim_head=64, heads=8, out_dim=None,
                 context_pre_only=None, bias=False, processor=None, qk_norm=None, eps=1e-5):
        super().__init__()
        inner = dim_head * heads
        self.heads = heads
        self.to_q, self.to_k, self.to_v = (nn.Linear(query_dim, inner, bias=bias) for _ in range(3))
        self.norm_q, self.norm_k = RMSNorm(dim_head, eps), RMSNorm(dim_head, eps)
        self.add_k_proj, self.add_v_proj, self.add_q_proj = (nn.Linear(added_kv_proj_dim, inner, bias=True) for _ in range(3))
        self.norm_added_q, self.norm_added_k = RMSNorm(dim_head, eps), RMSNorm(dim_head, eps)
        self.to_out = nn.ModuleList([nn.Linear(inner, out_dim, bias=True), nn.Dropout(0.0)])
        self.to_add_out = nn.Linear(inner, out_dim, bias=True)


class FeedForward(nn.Module):
    class _Proj(nn.Module):
        def __init__(self, d, inner):
            super().__init__()
            self.proj = nn.Linear(d, inner)

    def __init__(self, dim, dim_out=None, activation_fn="geglu"):
        super().__init__()
        self.net = nn.ModuleList([self._Proj(dim, 4 * dim), nn.Dropout(0.0), nn.Linear(4 * dim, dim_out)])


class AdaLayerNormContinuous(nn.Module):
    def __init__(self, embedding_dim, conditioning_embedding_dim, elementwise_affine=True, eps=1e-5):
        super().__init__()
        self.silu = nn.SiLU()
        self.linear = nn.Linear(conditioning_embedding_dim, 2 * embedding_dim)


def sdpa_dispatch(query, key, value, attn_mask=None, dropout_p=0.0, is_causal=False, backend=None, tile_size=1024):
    """dispatch_attention_fn on [B, S, H, D] with a bool [B, S_k] key mask (True = attend)."""
    q, k, v = (t.transpose(1, 2) for t in (query, key, value))
    m = None if attn_mask is None else attn_mask[:, None, None, :].to(q.device)
    return F.scaled_dot_product_attention(q, k, v, attn_mask=m).transpose(1, 2)


def _lift_module(name, methods, ns):
    lifted = R.methods(TR, name, methods, extra_ns=ns)
    return type(name, (lifted, nn.Module), {})


def main():
    if not R.available():
        raise SystemExit("set SIMPLETUNER_SRC to a SimpleTuner checkout")
    g = torch.Generator().manual_seed(0)
    fns = R.functions(TR, ["precompute_real_rope_qwen", "compute_text_seq_len_from_mask", "apply_rotary_emb_qwen"])
    ns = {"nn": nn, "functools": functools, "np": None, "Timesteps": Timesteps, "TimestepEmbedding": TimestepEmbedding,
          "RMSNorm": RMSNorm, "Attention": Attention, "FeedForward": FeedForward,
          "AdaLayerNormContinuous": AdaLayerNormContinuous, "MutableModuleList": nn.ModuleList,
          "register_to_config": lambda f: f, "attention_with_oom_fallback": sdpa_dispatch,
          "publish_attention_max_logits": lambda *a, **k: None, **fns}
    out = {}
    # ---- RoPE
    Rope = R.methods(TR, "QwenEmbedRope", ["__init__", "rope_params", "forward", "_compute_video_freqs"], extra_ns=ns)
    rope = Rope(theta=10000, axes_dim=[16, 56, 56], scale_rope=True)
    out["rope"] = []
    for h, w in ROPE_CASES:
        for L in TXT_LENS:
            rope.rope_cache = {}
            (icos, isin), (tcos, tsin) = fns["precompute_real_rope_qwen"](rope.forward([(1, h, w)], L, device=torch.device("cpu")))
            out["rope"].append({"h": h, "w": w, "S_txt": L, "img_cos": icos.clone(), "img_sin": isin.clone(),
                                "txt_cos": tcos.clone(), "txt_sin": tsin.clone()})
    # ---- text length from the mask
    masks = {"prefix": torch.tensor([[1, 1, 1, 0, 0], [1, 1, 1, 1, 1], [1, 0, 0, 0, 0]]),
             "non_prefix": torch.tensor([[1, 0, 1, 1, 0], [0, 0, 0, 0, 0]])}
    out["seq_len"] = {}
    for k, m in masks.items():
        enc = torch.zeros(m.shape[0], m.shape[1], 4)
        L, per, nm = fns["compute_text_seq_len_from_mask"](enc, m)
        out["seq_len"][k] = {"mask": m, "text_seq_len": L, "per_sample_len": per.clone(), "bool_mask": nm.clone()}
    # ---- timestep embedding: the model rounds t to bf16 (:1295) before time_text_embed
    D = 32
    TE = _lift_module("QwenTimestepProjEmbeddings", ["__init__", "forward"], ns)
    te = TE(D).to(torch.bfloat16)
    with torch.no_grad():
        for p in te.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    t = torch.tensor([0.0, 0.0137, 0.5, 0.731, 0.99961, 1.0])
    hs = torch.zeros(1, 1, D, dtype=torch.bfloat16)
    with torch.no_grad():
        proj = te.time_proj(t.to(torch.bfloat16))
        temb = te(t.to(torch.bfloat16), hs)
    out["temb"] = {"t": t, "proj": proj.clone(), "temb": temb.clone(),
                   "params": {k: v.detach().clone() for k, v in te.timestep_embedder.state_dict().items()}}
    # ---- _modulate
    Block = R.methods(TR, "QwenImageTransformerBlock", ["_modulate"], extra_ns=ns)
    x = torch.randn(2, 5, D, generator=g)
    mp = torch.randn(2, 3 * D, generator=g)
    mx, gate = Block()._modulate(x, mp)
    out["modulate"] = {"x": x, "mod": mp, "out": mx.clone(), "gate": gate.clone()}
    # ---- attention processor with padded prompts
    H, hd, S_img = 2, 32, 6
    Dm = H * hd
    Proc = R.methods(TR, "QwenDoubleStreamAttnProcessor2_0", ["__call__"], extra_ns=ns)
    Proc._attention_backend = None
    attn = Attention(Dm, added_kv_proj_dim=Dm, dim_head=hd, heads=H, out_dim=Dm, bias=True, eps=1e-6)
    with torch.no_grad():
        for n, p in attn.named_parameters():
            p.copy_(1.0 + 0.05 * torch.randn(p.shape, generator=g) if "norm" in n else torch.randn(p.shape, generator=g) * Dm ** -0.5)
    cases = {
        "b1_full": torch.tensor([[1, 1, 1, 1, 1, 1, 1]]),
        "b1_padded": torch.tensor([[1, 1, 1, 1, 0, 0, 0]]),
        "b3_ragged": torch.tensor([[1, 1, 1, 1, 1, 1, 1], [1, 1, 1, 0, 0, 0, 0], [1, 1, 1, 1, 1, 0, 0]]),
        "b2_non_prefix": torch.tensor([[1, 0, 1, 1, 0, 1, 0], [1, 1, 1, 1, 1, 1, 0]]),
        "b2_all_zero": torch.tensor([[0, 0, 0, 0, 0, 0, 0], [1, 1, 1, 0, 0, 0, 0]]),
    }
    out["attn"] = {"params": {k: v.detach().clone() for k, v in attn.state_dict().items()}, "H": H, "hd": hd, "cases": {}}
    for name, m in cases.items():
        B, L = m.shape
        img = torch.randn(B, S_img, Dm, generator=g)
        txt = torch.randn(B, L, Dm, generator=g)
        rope.rope_cache = {}
        (icos, isin), (tcos, tsin) = fns["precompute_real_rope_qwen"](rope.forward([(1, 2, 3)], L, device=torch.device("cpu")))
        # the model passes the joint bool mask as attention_mask only for B == 1 (:1360-1366)
        joint = torch.cat([m.bool(), torch.ones(B, S_img, dtype=torch.bool)], 1) if B == 1 else None
        with torch.no_grad():
            io, to = Proc()(attn, img, txt, encoder_hidden_states_mask=m.bool(), attention_mask=joint,
                            image_rotary_emb=((icos[:, :hd], isin[:, :hd]), (tcos[:, :hd], tsin[:, :hd])))
        out["attn"]["cases"][name] = {"mask": m, "img": img, "txt": txt, "img_out": io.clone(), "txt_out": to.clone(),
                                      "rope": (icos[:, :hd].clone(), isin[:, :hd].clone(), tcos[:, :hd].clone(),
                                               tsin[:, :hd].clone())}
    # ---- parameter names / shapes at a small config
    ns["QwenTimestepProjEmbeddings"] = TE
    ns["QwenEmbedRope"] = lambda **k: None
    ns["QwenDoubleStreamAttnProcessor2_0"] = lambda: None
    ns["logger"] = None
    ns["QwenImageTransformerBlock"] = _lift_module("QwenImageTransformerBlock", ["__init__"], ns)
    ns["MusubiBlockSwapManager"] = types.SimpleNamespace(build=lambda **k: None)
    Model = _lift_module("QwenImageTransformer2DModel", ["__init__"], ns)
    model = Model(num_layers=2, attention_head_dim=64, num_attention_heads=2, joint_attention_dim=48)
    out["param_shapes"] = {"config": dict(num_layers=2, attention_head_dim=64, num_attention_heads=2, joint_attention_dim=48),
                           "shapes": {k: tuple(v.shape) for k, v in model.state_dict().items()}}
    OUT.parent.mkdir(parents=True, exist_ok=True)
    torch.save(out, OUT)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
