"""Writes tests/golden/flux_attn_mask_golden.pt: the reference's own masked Flux attention on small fp32 inputs.

Runs `expand_flux_attention_mask` and `FluxAttnProcessor2_0.__call__` (reference flux/transformer.py:116-242), lifted
from a SimpleTuner checkout by oracle/ref_extract, with RoPE and ragged per-sample text masks (one of them shorter than
the text sequence, so `expand_flux_attention_mask` pads it with ones): one joint (double-block) call and one
single-block call.  The processor is given its collaborators as stubs: `Attention` (a type annotation only),
`maybe_metal_flash_rope_attention` returning None (the non-Metal path) and a no-op `publish_attention_max_logits`.

    SIMPLETUNER_SRC=<SimpleTuner checkout> python tools/make_golden_flux_mask.py
"""
from __future__ import annotations

import sys
import types
from pathlib import Path

import torch
import torch.nn as nn

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import flux_oracle as O  # noqa: E402
from oracle import ref_extract as R  # noqa: E402

REL = "helpers/models/flux/transformer.py"
OUT = ROOT / "tests" / "golden" / "flux_attn_mask_golden.pt"
H, HD = 2, 32
D = H * HD
EPS = 1e-6


class _RMSNorm(nn.Module):
    """diffusers RMSNorm(head_dim, eps=1e-6) with a weight, fp32 (the processor only calls it)."""

    def __init__(self, w):
        super().__init__()
        self.weight = nn.Parameter(w)

    def forward(self, x):
        return O.rms_norm(x, self.weight, EPS)


def _linear(g, name, P):
    lin = nn.Linear(D, D)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(D, D, generator=g) * D ** -0.5)
        lin.bias.copy_(torch.randn(D, generator=g) * 0.1)
    P[name + ".weight"], P[name + ".bias"] = lin.weight.detach().clone(), lin.bias.detach().clone()
    return lin


def _norm(g, name, P):
    w = 1.0 + 0.1 * torch.randn(HD, generator=g)
    P[name + ".weight"] = w.clone()
    return _RMSNorm(w)


def _attn(g, joint: bool, P):
    a = types.SimpleNamespace(heads=H)
    for n in ("to_q", "to_k", "to_v"):
        setattr(a, n, _linear(g, n, P))
    a.norm_q, a.norm_k = _norm(g, "norm_q", P), _norm(g, "norm_k", P)
    if joint:
        for n in ("add_q_proj", "add_k_proj", "add_v_proj"):
            setattr(a, n, _linear(g, n, P))
        a.norm_added_q, a.norm_added_k = _norm(g, "norm_added_q", P), _norm(g, "norm_added_k", P)
        a.to_out = [_linear(g, "to_out.0", P), nn.Identity()]
        a.to_add_out = _linear(g, "to_add_out", P)
    else:
        a.norm_added_q = a.norm_added_k = None
    return a


def main():
    if not R.available():
        raise SystemExit("set SIMPLETUNER_SRC to a SimpleTuner checkout")
    fns = R.functions(REL, ["expand_flux_attention_mask", "_apply_rotary_emb_anyshape"])
    ns = {"Attention": object, "maybe_metal_flash_rope_attention": lambda *a, **k: None,
          "publish_attention_max_logits": lambda *a, **k: None, **fns}
    Proc = R.methods(REL, "FluxAttnProcessor2_0", ["__call__"], extra_ns=ns)
    g = torch.Generator().manual_seed(0)
    B, S_txt, S_img = 3, 12, 20
    # ragged masks: sample 0 keeps 5 of 12 text tokens, sample 1 all of them, sample 2 the first 9 but token 3.  The
    # single-block call gets the same masks cut to 9 tokens (shorter than S_txt: columns 9..11 stay 1 when expanded).
    mask = torch.zeros(B, S_txt)
    mask[0, :5] = 1
    mask[1, :] = 1
    mask[2, :9] = 1
    mask[2, 3] = 0
    mask_short = mask[:, :9].clone()
    ids = torch.cat([torch.zeros(S_txt, 3), O.prepare_latent_image_ids(8, 10)], 0)
    cos, sin = O.rope_tables(ids, (8, 12, 12))
    out = {"H": H, "HD": HD, "B": B, "S_txt": S_txt, "S_img": S_img, "cos": cos, "sin": sin, "cases": []}
    for joint, m in ((True, mask), (False, mask_short)):
        P = {}
        attn = _attn(g, joint, P)
        x = torch.randn(B, S_img if joint else S_txt + S_img, D, generator=g)
        enc = torch.randn(B, S_txt, D, generator=g) if joint else None
        joint_hidden = torch.cat([enc, x], 1) if joint else x
        full = fns["expand_flux_attention_mask"](joint_hidden, m)
        with torch.no_grad():
            res = Proc().__call__(attn, x, enc, attention_mask=full, image_rotary_emb=(cos, sin))
        case = {"joint": joint, "mask": m.clone(), "expanded": full.clone(), "P": P, "x": x, "enc": enc}
        if joint:
            case["out_img"], case["out_txt"] = res[0].clone(), res[1].clone()
        else:
            case["out"] = res.clone()
        out["cases"].append(case)
    OUT.parent.mkdir(parents=True, exist_ok=True)
    torch.save(out, OUT)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes, {len(out['cases'])} cases)")


if __name__ == "__main__":
    main()
