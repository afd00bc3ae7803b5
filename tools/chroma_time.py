#!/usr/bin/env python
"""Chroma 1 LoRA step on the GPU: full size (19 + 38 blocks, D = 3072, approximator width 5120), random weights, LoRA r16
on the default targets (to_k, to_q, to_v, to_out.0), AdamW through the eager TrainStep, 1024^2 latents, gradient
checkpointing on every block, T5 prompts padded to 512 tokens.  Arms, alternated for `--rounds` rounds in one session:
  chroma_p100   batch 1, a 100-token prompt (412 padded keys, -inf in the per-key bias)
  chroma_p300   batch 1, a 300-token prompt
Each arm runs twice per round, with the attention kernels skipping the key tiles whose bias is -inf throughout and with
every tile processed (the live list withheld from the kernels, as before the skip existed), so the two alternate in one
session on one library.  Per arm: ms per step (CUDA events over `--steps` steps after `--warmup`) and peak allocated
memory; the approximator's time per forward (CUDA events around ChromaTransformer2DModel.pooled_temb); and attention
forward and backward alone at B 1, H 24, S 4608 (512 text + 4096 image keys) with each prompt's key bias, both ways.  Prints one JSON object with the card's name,
power limit and max SM clock read in the same run; `--out FILE` also writes it there.

    python tools/chroma_time.py --out result.json
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from simpletuner_b200 import ops  # noqa: E402
from tools.masked_attention_time import card, events  # noqa: E402

_LIVE = ops._key_live


def skipping(on: bool) -> None:
    """on: the kernels get each bias's live list; off: they process every key tile."""
    ops._key_live = _LIVE if on else (lambda bias: None)


def attention_ms(kept, dev, n=20):
    """Forward and backward of one joint attention at B 1, H 24, S 4608, HD 128 with the bias of a `kept`-token prompt."""
    g = torch.Generator(device=dev).manual_seed(0)
    q, k, v, d_o = (torch.randn(1, 4608, 24, 128, device=dev, generator=g).bfloat16() for _ in range(4))
    bias = torch.zeros(1, 4608, device=dev, dtype=torch.bfloat16)
    bias[0, kept:512] = float("-inf")
    o, lse = ops.attn_fwd(q, k, v, key_bias=bias)
    fwd = events(lambda i: ops.attn_fwd(q, k, v, key_bias=bias), n)
    bwd = events(lambda i: ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=bias), n)
    return round(fwd, 3), round(bwd, 3)


def build(dev):
    from simpletuner_b200.chroma.model import Chroma, default_config
    from simpletuner_b200.chroma.transformer import ChromaTransformer2DModel
    with torch.device(dev):
        m = ChromaTransformer2DModel()
    g = torch.Generator(device=dev).manual_seed(0)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "norm" in n:
                p.fill_(1.0)
            elif n.startswith("distilled_guidance_layer") and n.endswith("weight"):
                p.normal_(0, p.shape[1] ** -0.5, generator=g)
            else:
                p.normal_(0, 0.02 if n.endswith("weight") else 0.01, generator=g)
    w = Chroma(default_config(lora_rank=16), transformer=m, device=dev)
    w.add_lora_adapter()
    m.enable_gradient_checkpointing()
    return w


def batch(kept, dev, S_txt=512, seed=0):
    g = torch.Generator().manual_seed(seed)
    mask = (torch.arange(S_txt)[None] < kept).long()
    emb = torch.randn(1, S_txt, 4096, generator=g) * mask[:, :, None]
    return {"latent_batch": torch.randn(1, 16, 128, 128, generator=g).bfloat16(), "prompt_embeds": emb.bfloat16(),
            "encoder_attention_mask": mask}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("chroma_time.py measures on the GPU; no CUDA device is visible")
    from simpletuner_b200.training.step import TrainStep
    dev = torch.device("cuda")
    w = build(dev)
    den = w._denoiser()
    step = TrainStep(w, torch.optim.AdamW(den.trainable_parameters(), lr=1e-4))
    prompts = {"p100": 100, "p300": 300}
    arms = {f"chroma_{k}_{s}": (batch(n, dev), s == "skip") for k, n in prompts.items() for s in ("skip", "noskip")}
    res = {"card": card(), "ms_per_step": {k: [] for k in arms}, "approximator_ms": None, "peak_gib": {},
           "attention_fwd_bwd_ms": {f"{k}_{s}": [] for k in prompts for s in ("skip", "noskip")}}
    for name, (b, on) in arms.items():
        skipping(on)
        for _ in range(args.warmup):
            step({k: v.clone() for k, v in b.items()})
    for _ in range(args.rounds):
        for name, (b, on) in arms.items():
            skipping(on)
            torch.cuda.reset_peak_memory_stats()
            ms = events(lambda i: step({k: v.clone() for k, v in b.items()}), args.steps)
            res["ms_per_step"][name].append(round(ms, 1))
            res["peak_gib"][name] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)
        for k, n in prompts.items():
            for s in ("skip", "noskip"):
                skipping(s == "skip")
                res["attention_fwd_bwd_ms"][f"{k}_{s}"].append(attention_ms(n, dev))
    skipping(True)
    t = torch.full((1,), 500.0, device=dev, dtype=torch.bfloat16)
    res["approximator_ms"] = round(events(lambda i: den.pooled_temb(t), 20), 2)
    print(json.dumps(res))
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
