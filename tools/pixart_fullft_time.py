#!/usr/bin/env python
"""PixArt-Sigma full fine-tune step against the PixArt LoRA r32 step on the GPU, alternating in one session, three rounds.

PixArt-Sigma 600M geometry (28 blocks, D 1152, 16 x 72 heads, T5 captions of 4096 channels) with random weights, 1024^2
latents (4096 tokens), batch 4, 300-token prompts with a ragged keep-mask (300 / 220 / 140 / 60 tokens), AdamWBF16 through
the eager TrainStep.  Arms:
  full_gc_off / full_gc_on   model_type=full, gradient checkpointing off / on every block
  lora_gc_off / lora_gc_on   LoRA r32 on to_k, to_q, to_v, to_out.0 of both attentions (the control)
Per arm: ms per step (CUDA events over `--steps` steps; the minimum over the rounds), algorithmic TFLOP per step and TFLOP/s
(`tflop_per_sample`: full fine-tune counts forward + dgrad + wgrad of every linear, LoRA forward + dgrad of the frozen
linears; attention 4 S Sk D forward and 8 S Sk D backward; the real head width 72, not the padded 128; recompute not
counted), peak allocated memory.  Then one instrumented full fine-tune step (checkpointing off): the GPU time of the padded
q / k / v / out weight gradients (wgrad_full on the 128-wide head layout plus the gather of the real rows / columns) as a
share of that step, and one torch.profiler step of each full arm: CUDA time by kernel family.  Prints one JSON object
with the card's name and power limit read in the same run; `--out FILE` also writes it there.

    python tools/pixart_fullft_time.py --out result.json
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
from tools.masked_attention_time import ROUNDS, card, events  # noqa: E402
from tools.qwen_image_time import profile_step  # noqa: E402

B, S, ST, D, CAP, L = 4, 4096, 300, 1152, 4096, 28
HP = 16 * 128                      # the padded head layout the projections run on


def tflop_per_sample(full: bool) -> float:
    """Algorithmic TFLOP of one training sample (multiply-add = 2 flops)."""
    blk = S * 14 * D * D + ST * 2 * D * D          # img: qkv 3, out 1, cross q 1, cross out 1, FF 8 (D^2 MACs); kv on captions
    att = 4 * S * S * D + 4 * S * ST * D           # forward QK^T + PV, self and cross
    lin = 2 * L * blk + 2 * S * 16 * D + 2 * S * D * 16         # + PatchEmbed (16 features) + kept proj_out rows
    cap = 2 * ST * (CAP * D + D * D)                             # caption projection
    if full:
        return (3 * (lin + cap) + 3 * L * att) / 1e12            # forward + dgrad + wgrad; attention forward + 2x backward
    return (2 * lin + cap + 3 * L * att) / 1e12                  # frozen caption projection: forward only


def build(dev, full: bool):
    from simpletuner_b200.pixart.model import PixartSigma, default_config
    from simpletuner_b200.pixart.transformer import PixArtTransformer2DModel
    with torch.device(dev):
        m = PixArtTransformer2DModel(caption_channels=CAP)
    g = torch.Generator(device=dev).manual_seed(0)
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.normal_(0, 0.02 if n.endswith("weight") else 0.01, generator=g)
    w = PixartSigma(default_config(lora_rank=32, lora_alpha=32), transformer=m, device=dev)
    if full:
        m.enable_full_finetune()
    else:
        w.add_lora_adapter()
        with torch.no_grad():
            for lin in m.lora_linears().values():
                lin.lora_B["default"].weight.normal_(0, 0.02, generator=g)
    return w


def make_batch():
    g = torch.Generator().manual_seed(0)
    mask = torch.zeros(B, ST, dtype=torch.int64)
    for i, n in enumerate((300, 220, 140, 60)):
        mask[i, :n] = 1
    return {"latent_batch": torch.randn(B, 4, 128, 128, generator=g).bfloat16(),
            "prompt_embeds": torch.randn(B, ST, CAP, generator=g).bfloat16() * mask[:, :, None],
            "encoder_attention_mask": mask}


def padded_wgrad_share(step_fn):
    """One full fine-tune step with the padded-layout weight gradients bracketed by CUDA events: (their ms, step ms)."""
    spans = []
    real_wgrad, real_sel = ops.wgrad_full, torch.Tensor.index_select

    def wgrad(dy, x, *a, **k):
        padded = dy.shape[-1] in (HP, 2 * HP, 3 * HP) or x.shape[-1] == HP
        if not padded:
            return real_wgrad(dy, x, *a, **k)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = real_wgrad(dy, x, *a, **k)
        e1.record()
        spans.append((e0, e1))
        return out

    def sel(t, dim, index):          # the gather of the real rows / columns out of a padded-layout gradient
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = real_sel(t, dim, index)
        e1.record()
        spans.append((e0, e1))
        return out

    ops.wgrad_full = wgrad
    torch.Tensor.index_select = sel
    try:
        ms = events(step_fn, 1)
    finally:
        ops.wgrad_full = real_wgrad
        torch.Tensor.index_select = real_sel
    return sum(a.elapsed_time(b) for a, b in spans), ms, len(spans)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from simpletuner_b200.training.optim import AdamWBF16
    from simpletuner_b200.training.step import TrainStep

    dev = torch.device("cuda", torch.cuda.current_device())
    batch = make_batch()
    steps = {}
    for kind in ("full", "lora"):
        w = build(dev, kind == "full")
        params = [p for p in w._denoiser().parameters() if p.requires_grad]
        steps[kind] = (w, TrainStep(w, AdamWBF16(params, lr=1e-5, weight_decay=0.01), max_grad_norm=0.01))
    arms = [f"{k}_gc_{g}" for k in ("full", "lora") for g in ("off", "on")]
    res = {"card": card(), "setup": f"PixArt-Sigma 600M, 1024^2, batch {B}, {ST}-token ragged prompts, AdamWBF16, eager TrainStep",
           "tflop_per_sample": {"full": round(tflop_per_sample(True), 3), "lora": round(tflop_per_sample(False), 3)},
           "ms": {a: [] for a in arms}, "peak_gb": {}}

    def runner(arm):
        kind, gc = arm.split("_gc_")
        w, step = steps[kind]
        den = w._denoiser()
        den.enable_gradient_checkpointing() if gc == "on" else den.disable_gradient_checkpointing()
        return lambda i: step({k: v.clone() for k, v in batch.items()})

    for r in range(ROUNDS):
        for arm in arms:
            fn = runner(arm)
            events(fn, args.warmup)
            if r == 0:
                torch.cuda.reset_peak_memory_stats()
                events(fn, 1)
                res["peak_gb"][arm] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
            res["ms"][arm].append(round(events(fn, args.steps), 1))
    for _, step in steps.values():
        step.check_finite()
    res["tflops"] = {a: round(B * tflop_per_sample(a.startswith("full")) / (min(v) / 1e3), 1) for a, v in res["ms"].items()}
    res["full_over_lora_ms"] = {g: round(min(res["ms"][f"full_gc_{g}"]) / min(res["ms"][f"lora_gc_{g}"]), 3) for g in ("off", "on")}
    pad_ms, step_ms, n = padded_wgrad_share(runner("full_gc_off"))
    res["padded_wgrad"] = {"ms": round(pad_ms, 2), "step_ms": round(step_ms, 1), "share": round(pad_ms / step_ms, 4),
                           "launches": n}
    res["profile"] = {arm: profile_step(runner(arm))["by_family_ms"] for arm in ("full_gc_off", "full_gc_on")}
    text = json.dumps(res)
    print(text)
    if args.out:
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
