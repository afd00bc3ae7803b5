#!/usr/bin/env python
"""Cost of Flux masked training (the per-key logit bias) on the GPU, masked and unmasked runs alternating, three rounds:

  * attention forward and backward at B 1, H 24, S 4608 (512 text + 4096 image tokens), HD 128, with and without a key
    bias (CUDA events, 20 forward / 10 backward calls per run);
  * the device-resident flux_lora step (bench.py's Flux.1-dev LoRA rank 16 model and batch, 1024^2, batch 1) with
    `flux_attention_masked_training` on and off (CUDA events over 4 steps per run).

Prints one JSON object with the card name and power limit; `--out FILE` also writes it there.

    python tools/masked_attention_time.py --out result.json
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from simpletuner_b200 import ops  # noqa: E402

ROUNDS = 3


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else "unknown"


def events(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def text_mask(B, S_txt, kept):
    m = torch.zeros(B, S_txt)
    m[:, :kept] = 1
    return m


def time_attention(res):
    B, H, S, HD, S_txt = 1, 24, 4608, 128, 512
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v, d_o = (torch.randn(B, S, H, HD, device="cuda", generator=g).bfloat16() for _ in range(4))
    bias = torch.ones(B, S, device="cuda", dtype=torch.bfloat16)
    bias[:, 97:S_txt] = 0          # a 97-token prompt
    arms = {"unmasked": None, "masked": bias}
    bufs = {}
    for name, kb in arms.items():  # warm-up: module load, smem attributes
        o, lse = ops.attn_fwd(q, k, v, key_bias=kb)
        bufs[name] = (o, lse, *ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=kb))
    for r in range(ROUNDS):
        for name, kb in arms.items():
            o, lse, dq, dk, dv = bufs[name]
            fwd = events(lambda i: ops.attn_fwd(q, k, v, out=o, key_bias=kb), 20)
            bwd = events(lambda i: ops.attn_bwd(q, k, v, o, d_o, lse, dq=dq, dk=dk, dv=dv, key_bias=kb), 10)
            res["attention"][name].append({"fwd_ms": round(fwd, 4), "bwd_ms": round(bwd, 4)})


def time_step(res, steps=4, warmup=2):
    import bench
    from simpletuner_b200.training.step import TrainStep

    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(42)
    w = bench.build_model(dev, rank=16, seed=0)
    params = [p for p in w._denoiser().parameters() if p.requires_grad]
    step = TrainStep(w, torch.optim.AdamW(params, lr=1e-4), max_grad_norm=1.0)
    batch = bench.synth_batch(1, dev)
    S_txt = batch["prompt_embeds"].shape[1]
    masked_batch = {**batch, "encoder_attention_mask": text_mask(1, S_txt, 97).to(dev)}

    def arm(masked):
        w.config.flux_attention_masked_training = masked
        w.config.attention_mechanism = "diffusers"
        w._denoiser().attention_masked_training = masked
        b = masked_batch if masked else batch
        return lambda i: step({k: v for k, v in b.items()})

    for masked in (False, True):
        events(arm(masked), warmup)
    for r in range(ROUNDS):
        for name, masked in (("unmasked", False), ("masked", True)):
            res["flux_lora_step"][name].append(round(events(arm(masked), steps), 2))
    step.check_finite()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--skip-step", action="store_true", help="attention kernels only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res = {"card": card(), "attention_shape": "B1 H24 S4608 HD128, key bias = 97-token text mask",
           "step": "flux_lora Flux.1-dev LoRA r16, 1024^2, batch 1, device-resident, AdamW",
           "attention": {"unmasked": [], "masked": []}, "flux_lora_step": {"unmasked": [], "masked": []}}
    time_attention(res)
    if not args.skip_step:
        time_step(res)
    for key in ("fwd_ms", "bwd_ms"):
        u = min(x[key] for x in res["attention"]["unmasked"])
        m = min(x[key] for x in res["attention"]["masked"])
        res[f"attention_{key}_masked_over_unmasked"] = round(m / u, 4)
    if res["flux_lora_step"]["masked"]:
        res["step_masked_over_unmasked"] = round(min(res["flux_lora_step"]["masked"]) / min(res["flux_lora_step"]["unmasked"]), 4)
    text = json.dumps(res)
    print(text)
    if args.out:
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
