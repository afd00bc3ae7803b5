#!/usr/bin/env python
"""Qwen-Image LoRA step against the plain flux_lora step on the GPU, alternating in one session, three rounds.

Both steps train LoRA r16 on their default targets (Flux: bench.py's Flux.1-dev model, flux_lora_target "all"; Qwen-Image:
to_k, to_q, to_v, to_out.0) with random weights, AdamW through the eager TrainStep, 1024^2 latents and gradient
checkpointing on every block.  Qwen-Image (20.4 B parameters) and Flux.1-dev (11.9 B) do not both fit an 80 GB card with
their activations, so each round builds Flux, times it, frees it, then builds Qwen-Image and times it.  Arms:
  flux       batch 1, 512 text tokens (S = 4608)
  qwen_256   batch 1, a 256-token prompt (no padding: the unbiased attention kernels)
  qwen_512   batch 1, a 512-token prompt (S = 4608, the Flux arm's shape)
  qwen_b4    batch 4, prompts of 512 / 384 / 256 / 128 tokens zero-padded to 512 (the per-key bias kernels)
Per arm: ms per step (CUDA events over `--steps` steps), algorithmic TFLOP per sample and TFLOP/s counted as bench.py counts
(GEMM 2MNK over the blocks' projections, attention 4 S^2 D forward and 8 S^2 D backward, recompute not counted; padded
text tokens count, since the kernels run them), peak allocated memory and kernel launches of one step.  `--profile` adds
one torch.profiler step per arm: CUDA time by kernel family and the top kernels.  Prints one JSON object with the card's
name and power limit read in the same run; `--out FILE` also writes it there.

    python tools/qwen_image_time.py --profile --out result.json
"""
from __future__ import annotations

import argparse
import gc
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from simpletuner_b200 import ops  # noqa: E402
from tools.masked_attention_time import ROUNDS, card, events  # noqa: E402

D = 3072
IMG = 4096          # 1024^2: 128 x 128 latents, 2 x 2 patches


def qwen_tflop(S: int) -> float:
    """One Qwen-Image LoRA training sample at joint length S: 60 double blocks, 24 D^2 MACs per token in the projections
    (q, k, v, out: 4 D^2; MLP: 8 D^2; doubled for multiply-add), forward + dgrad; attention forward + 2x backward."""
    lin = 60 * S * 24 * D * D
    att = 60 * 4 * S * S * D
    return (2 * lin + 3 * att) / 1e12


def flux_tflop(S: int) -> float:
    lin = 57 * S * 24 * D * D
    att = 57 * 4 * S * S * D
    return (2 * lin + 3 * att) / 1e12


def build_qwen(dev):
    from simpletuner_b200.qwen_image.model import QwenImage, default_config
    from simpletuner_b200.qwen_image.transformer import QwenImageTransformer2DModel
    with torch.device(dev):
        m = QwenImageTransformer2DModel()
    g = torch.Generator(device=dev).manual_seed(0)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "norm" in n and p.dim() == 1:
                p.fill_(1.0)
            else:
                p.normal_(0, 0.02 if n.endswith("weight") else 0.01, generator=g)
    w = QwenImage(default_config(lora_rank=16), transformer=m, device=dev)
    w.add_lora_adapter()
    with torch.no_grad():
        for lin in m.lora_linears().values():
            lin.lora_B["default"].weight.normal_(0, 0.02, generator=g)
    m.enable_gradient_checkpointing()
    return w


def qwen_batch(B, lengths, S_txt, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    b = {"latent_batch": torch.randn(B, 16, 128, 128, generator=g).bfloat16(),
         "prompt_embeds": torch.randn(B, S_txt, 3584, generator=g).bfloat16()}
    if lengths is not None:
        mask = torch.zeros(B, S_txt, dtype=torch.int64)
        for i, n in enumerate(lengths):
            mask[i, :n] = 1
        b["prompt_embeds"] = b["prompt_embeds"] * mask[:, :, None]
        b["encoder_attention_mask"] = mask
    return b


def families(dev):
    import bench
    fb = bench.synth_batch(1, dev)
    return {
        "flux": (lambda: _flux(bench, dev), {"flux": (fb, 1, flux_tflop(fb["prompt_embeds"].shape[1] + IMG))}),
        "qwen": (lambda: build_qwen(dev), {
            "qwen_256": (qwen_batch(1, None, 256, dev), 1, qwen_tflop(256 + IMG)),
            "qwen_512": (qwen_batch(1, None, 512, dev), 1, qwen_tflop(512 + IMG)),
            "qwen_b4": (qwen_batch(4, [512, 384, 256, 128], 512, dev), 4, qwen_tflop(512 + IMG)),
        }),
    }


def _flux(bench, dev):
    torch.manual_seed(42)
    w = bench.build_model(dev, rank=16, seed=0)
    w._denoiser().enable_gradient_checkpointing()
    return w


def profile_step(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(0)
        torch.cuda.synchronize()
    rows = sorted(((e.key, e.device_time_total / 1e3, e.count) for e in prof.key_averages()), key=lambda x: -x[1])
    fam = {}
    for k, t, _ in rows:
        name = ("gemm" if "gemm" in k else "attn_bwd" if "attn_bwd" in k or "bwd_dq" in k or "bwd_dkdv" in k
                else "attn_fwd" if "attn_fwd" in k else "wgrad / skinny" if ("wgrad" in k or "skinny" in k) else "other")
        fam[name] = round(fam.get(name, 0.0) + t, 2)
    return {"by_family_ms": fam, "top": [(k[:90], round(t, 2), c) for k, t, c in rows[:15]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from simpletuner_b200.training.step import TrainStep

    dev = torch.device("cuda", torch.cuda.current_device())
    fams = families(dev)
    res = {"card": card(),
           "step": "LoRA r16 on each model's default targets, 1024^2, gradient checkpointing on every block, AdamW, eager TrainStep",
           "tflop_per_sample": {a: round(t, 1) for _, arms in fams.values() for a, (_, _, t) in arms.items()},
           "ms": {a: [] for _, arms in fams.values() for a in arms}, "launches": {}, "peak_gb": {}, "errors": {}}
    for r in range(ROUNDS):
        for fam, (build, arms) in fams.items():
            w = build()
            params = [p for p in w._denoiser().parameters() if p.requires_grad]
            step = TrainStep(w, torch.optim.AdamW(params, lr=1e-4), max_grad_norm=1.0)
            for arm, (batch, B, _) in arms.items():
                if arm in res["errors"]:
                    continue
                fn = lambda i, b=batch: step({k: v.clone() for k, v in b.items()})
                try:
                    events(fn, args.warmup)
                    if r == 0:
                        torch.cuda.reset_peak_memory_stats()
                        ops.reset_launch_count()
                        events(fn, 1)
                        res["launches"][arm] = ops.launch_count()
                        res["peak_gb"][arm] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
                    res["ms"][arm].append(round(events(fn, args.steps), 1))
                    if args.profile and r == ROUNDS - 1:
                        res.setdefault("profile", {})[arm] = profile_step(fn)
                except torch.cuda.OutOfMemoryError as exc:
                    res["errors"][arm] = f"out of memory: {str(exc)[:200]}"
                    for p in params:
                        p.grad = None
                    gc.collect()
                    torch.cuda.empty_cache()
            step.check_finite()
            del w, step, params
            gc.collect()
            torch.cuda.empty_cache()
    res["tflops"] = {}
    for _, arms in fams.values():
        for arm, (_, B, tf) in arms.items():
            if res["ms"][arm]:
                res["tflops"][arm] = round(B * tf / (min(res["ms"][arm]) / 1e3), 1)
    if "flux" in res["tflops"]:
        res["over_flux"] = {a: round(v / res["tflops"]["flux"], 4) for a, v in res["tflops"].items() if a != "flux"}
    text = json.dumps(res)
    print(text)
    if args.out:
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
