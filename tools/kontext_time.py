#!/usr/bin/env python
"""Flux Kontext step against the plain flux_lora step on the GPU, alternating, three rounds each.

Both steps run bench.py's Flux.1-dev LoRA model (random weights, rank 16, flux_lora_target "all", AdamW), batch 1, a
1024^2 edit, with gradient checkpointing on every block (the reference's default for Kontext; S = 8704 does not fit an
80 GB card without it).  The Kontext step adds one 1024^2 reference image: 512 text + 4096 scene + 4096 reference tokens.
Per step: ms (CUDA events over `--steps` steps), algorithmic TFLOP/s by bench.py's counting (linear 57 S 24 D^2, attention
57 4 S^2 D, LoRA step = forward + dgrad + 2x attention backward; with recompute the hardware does more than this), peak
memory and kernel launches.  `--profile` adds one torch.profiler step per arm: the CUDA time of the top kernels.
Prints one JSON object with the card name and power limit; `--out FILE` also writes it there.

    python tools/kontext_time.py --out result.json
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

D = 3072


def step_tflop(S: int) -> float:
    """bench.py's algorithmic FLOP of one LoRA training sample at joint length S (57 blocks of Flux.1-dev)."""
    lin = 57 * S * 24 * D * D
    att = 57 * 4 * S * S * D
    return (2 * lin + 3 * att) / 1e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import bench
    from simpletuner_b200.training.step import TrainStep

    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(42)
    w = bench.build_model(dev, rank=16, seed=0)
    w._denoiser().enable_gradient_checkpointing()
    params = [p for p in w._denoiser().parameters() if p.requires_grad]
    step = TrainStep(w, torch.optim.AdamW(params, lr=1e-4), max_grad_norm=1.0)
    batch = bench.synth_batch(1, dev)
    g = torch.Generator(device="cuda").manual_seed(3)
    ref = torch.randn(batch["latent_batch"].shape, device=dev, generator=g).bfloat16()
    S_txt = batch["prompt_embeds"].shape[1]
    S_scene = (batch["latent_batch"].shape[2] // 2) * (batch["latent_batch"].shape[3] // 2)
    arms = {"plain": (None, S_txt + S_scene), "kontext": ("kontext", S_txt + 2 * S_scene)}

    def run(name):
        w.config.model_flavour = arms[name][0]
        b = dict(batch)
        if name == "kontext":
            b["conditioning_latents"] = [ref]
        return lambda i: step(dict(b))

    res = {"card": card(), "step": "Flux.1-dev LoRA r16 'all', batch 1, 1024^2 edit, gradient checkpointing, AdamW",
           "tflop_per_sample": {n: round(step_tflop(S), 1) for n, (_, S) in arms.items()},
           "S": {n: S for n, (_, S) in arms.items()}, "ms": {n: [] for n in arms}}
    for name in arms:
        events(run(name), args.warmup)
    for name in arms:
        torch.cuda.reset_peak_memory_stats()
        ops.reset_launch_count()
        events(run(name), 1)
        res.setdefault("launches", {})[name] = ops.launch_count()
        res.setdefault("peak_gb", {})[name] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    for r in range(ROUNDS):
        for name in arms:
            res["ms"][name].append(round(events(run(name), args.steps), 2))
    step.check_finite()
    for name in arms:
        res.setdefault("tflops", {})[name] = round(res["tflop_per_sample"][name] / (min(res["ms"][name]) / 1e3), 1)
    res["kontext_tflops_over_plain"] = round(res["tflops"]["kontext"] / res["tflops"]["plain"], 4)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        res["top_kernels_ms"] = {}
        for name in arms:
            fn = run(name)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn(0)
                torch.cuda.synchronize()
            rows = sorted(((e.key, e.device_time_total / 1e3, e.count) for e in prof.key_averages()),
                          key=lambda x: -x[1])
            res["top_kernels_ms"][name] = [(k[:90], round(t, 2), c) for k, t, c in rows[:25]]
            mod = [r for r in rows if any(s in r[0] for s in ("ln_modulate", "gate_mul"))]
            res.setdefault("modulation_kernels_ms", {})[name] = round(sum(t for _, t, _ in mod), 2)
    text = json.dumps(res)
    print(text)
    if args.out:
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
