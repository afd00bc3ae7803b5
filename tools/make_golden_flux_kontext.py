"""Writes tests/golden/flux_kontext_golden.pt: the reference's own Flux Kontext input and conditioning functions on small
inputs.

Runs, lifted from a SimpleTuner checkout by oracle/ref_extract:
  * `build_kontext_inputs` (+ `pack_latents`, flux/__init__.py:25-30, 64-172) with 1, 2 and 3 conditioning images, square
    and non-square sizes, a reference size different from the edit, B = 2, and one layout whose positions pass 256 (its
    latents have one channel so that the fixture stays small; the ids only depend on the sizes);
  * `Flux._extend_conditioning_timesteps` (flux/model.py:602-618);
  * `_flux_tokenwise_conditioning` (flux/transformer.py:245-294) with the oracle's time_text_embed as the conditioning
    module;
  * `_flux_apply_ada_layer_norm_zero`, `_flux_apply_ada_layer_norm_zero_single` and
    `_flux_apply_ada_layer_norm_continuous` (flux/transformer.py:386-412) on 3-D embeddings, with torch stand-ins for the
    diffusers norms (`linear`, `silu`, a LayerNorm without affine, eps 1e-6).

    SIMPLETUNER_SRC=<SimpleTuner checkout> python tools/make_golden_flux_kontext.py
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

OUT = ROOT / "tests" / "golden" / "flux_kontext_golden.pt"
# (B, C, [(h, w) of each conditioning latent])
PACK_CASES = [
    (2, 16, [(16, 16)]),                          # same size as the 16 x 16 edit
    (2, 16, [(12, 20)]),                          # non-square, another size
    (2, 16, [(16, 16), (8, 12)]),
    (2, 16, [(10, 14), (16, 8), (6, 6)]),
    (1, 1, [(8, 520), (600, 8)]),                 # positions above 256 on both axes
]
D, POOLED = 32, 16


def _norm(n_chunks, g):
    m = types.SimpleNamespace(linear=nn.Linear(D, n_chunks * D), silu=nn.SiLU(),
                              norm=nn.LayerNorm(D, elementwise_affine=False, eps=1e-6))
    with torch.no_grad():
        m.linear.weight.copy_(torch.randn(n_chunks * D, D, generator=g) * D ** -0.5)
        m.linear.bias.copy_(torch.randn(n_chunks * D, generator=g) * 0.1)
    return m


def main():
    if not R.available():
        raise SystemExit("set SIMPLETUNER_SRC to a SimpleTuner checkout")
    init = R.functions("helpers/models/flux/__init__.py", ["pack_latents"])
    kb = R.functions("helpers/models/flux/__init__.py", ["build_kontext_inputs"], extra_ns=init)["build_kontext_inputs"]
    Flux = R.methods("helpers/models/flux/model.py", "Flux", ["_extend_conditioning_timesteps"])
    tr = R.functions("helpers/models/flux/transformer.py", [
        "_flux_tokenwise_conditioning", "_flux_apply_ada_layer_norm_zero", "_flux_apply_ada_layer_norm_zero_single",
        "_flux_apply_ada_layer_norm_continuous"])
    g = torch.Generator().manual_seed(0)
    out = {"pack": [], "D": D, "pooled_dim": POOLED}
    for B, C, sizes in PACK_CASES:
        lats = [torch.randn(B, C, h, w, generator=g).bfloat16() for h, w in sizes]
        packed, ids = kb(lats, dtype=torch.bfloat16, device=torch.device("cpu"), latent_channels=C)
        out["pack"].append({"B": B, "C": C, "sizes": sizes, "latents": lats, "packed": packed.clone(), "ids": ids.clone()})
    # timesteps: per-sample t / 1000 over the scene, 0 over the conditioning tokens
    t = torch.tensor([0.1, 0.9])
    ext = Flux()._extend_conditioning_timesteps(t, batch_size=2, scene_sequence_length=3, conditioning_sequence_length=2,
                                                device=torch.device("cpu"), dtype=torch.float32)
    out["extend"] = {"t": t, "S_scene": 3, "S_c": 2, "out": ext.clone()}
    # token-wise conditioning with the oracle's CombinedTimestepGuidanceTextProjEmbeddings as the module
    cfg = O.FluxConfig(num_layers=0, num_single_layers=0, num_attention_heads=1, attention_head_dim=D,
                       pooled_projection_dim=POOLED, guidance_embeds=True)
    P = {k: v for k, v in O.init_flux_params(cfg, seed=3).items() if k.startswith("time_text_embed.")}
    module = lambda ts, gd, pooled: O.time_text_embed(P, cfg, ts, gd, pooled)
    S_scene, S_c = 5, 3
    t2 = torch.cat([torch.tensor([[371.0], [912.5]]).expand(-1, S_scene), torch.zeros(2, S_c)], 1)
    guid = torch.tensor([1000.0, 3500.0])
    pooled = torch.randn(2, POOLED, generator=g)
    temb = tr["_flux_tokenwise_conditioning"](module, t2, pooled, guid)
    out["tokenwise"] = {"P": P, "t2": t2, "guidance": guid, "pooled": pooled, "temb": temb.clone(),
                        "temb_txt": temb.mean(dim=1).clone()}
    # the 3-D adaLN branches on a per-token embedding
    x = torch.randn(2, S_scene + S_c, D, generator=g)
    emb = torch.randn(2, S_scene + S_c, D, generator=g)
    n6, n3, n2 = _norm(6, g), _norm(3, g), _norm(2, g)
    with torch.no_grad():
        z = tr["_flux_apply_ada_layer_norm_zero"](n6, x, emb)
        zs = tr["_flux_apply_ada_layer_norm_zero_single"](n3, x, emb)
        c = tr["_flux_apply_ada_layer_norm_continuous"](n2, x, emb)
    out["ada"] = {"x": x, "emb": emb,
                  "zero": {"W": n6.linear.weight.detach().clone(), "b": n6.linear.bias.detach().clone(), "out": [u.clone() for u in z]},
                  "single": {"W": n3.linear.weight.detach().clone(), "b": n3.linear.bias.detach().clone(), "out": [u.clone() for u in zs]},
                  "continuous": {"W": n2.linear.weight.detach().clone(), "b": n2.linear.bias.detach().clone(), "out": c.clone()}}
    OUT.parent.mkdir(parents=True, exist_ok=True)
    torch.save(out, OUT)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes, {len(out['pack'])} packing cases)")


if __name__ == "__main__":
    main()
