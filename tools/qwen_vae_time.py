"""Qwen-Image VAE encode throughput at 1024^2: QwenImageVAE (libstb200) against the oracle's 3-D causal form run eagerly
in bf16 on the same GPU (cuDNN conv3d, as diffusers runs it), alternating in one process, CUDA events, warm-up, three
rounds.  Prints the card name and power limit read in the same run, images/s, algorithmic TFLOP/s, and the level-0
(96-channel) 3x3 convs timed alone.

Algorithmic FLOPs (2 per multiply-add, from the shapes; `encoder_flops`): at 1024^2 about 2.8 TFLOP per image, 0.4 of
it the mid-block attention (S = 128^2 pixels, head dim 384: 2 x 2 S^2 C).

    python tools/qwen_vae_time.py [--size 1024] [--batches 1 4] [--out bench_out/qwen_vae_time.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from oracle import qwen_vae_oracle as O  # noqa: E402
from simpletuner_b200 import ops  # noqa: E402


def encoder_flops(cfg, H, W):
    """(total, attention, level-0 3x3 convs) algorithmic FLOPs of one image's encode."""
    blocks, dims = O._layout(cfg)
    h, w = H, W
    tot = 2 * 27 * dims[0] * h * w           # conv_in
    lvl0 = 0
    for b in blocks:
        if b[0] == "res":
            _, cin, cout = b
            f = 2 * 9 * (cin * cout + cout * cout) * h * w + (2 * cin * cout * h * w if cin != cout else 0)
            tot += f
            if h == H:
                lvl0 += 2 * 9 * (cin * cout + cout * cout) * h * w
        else:
            c = b[1]
            h, w = h // 2, w // 2
            tot += 2 * 9 * c * c * h * w
            if h == H // 2:
                lvl0 += 2 * 9 * c * c * h * w
    c, S = dims[-1], h * w
    tot += 2 * 2 * 9 * c * c * S * 2        # mid resnets
    attn = 2 * 2 * S * S * c + 2 * 4 * c * c * S
    tot += attn
    tot += 2 * 9 * c * 2 * cfg.z_dim * S + 2 * (2 * cfg.z_dim) ** 2 * S
    return tot, attn, lvl0


def _time(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "qwen_vae_time needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    from tests.qwen_vae_checks import build_vae
    cfg = O.QwenVaeConfig()
    P = O.init_params(cfg, 0)
    vae = build_vae(cfg, P)
    Pb = {k: v.bfloat16().cuda() for k, v in P.items()}
    H = W = args.size
    flops, attn, lvl0 = encoder_flops(cfg, H, W)
    res = {"gpu": smi[0] if smi else "unknown", "size": H, "tflop_per_image": flops / 1e12, "attention_tflop": attn / 1e12,
           "level0_conv_tflop": lvl0 / 1e12, "rows": []}
    torch.backends.cudnn.benchmark = True
    for B in args.batches:
        x = (torch.rand(B, 3, 1, H, W, device="cuda") * 2 - 1).bfloat16()
        b200 = lambda: vae.encode(x).latent_dist.parameters
        eager = lambda: O.encode3d(x, Pb, cfg)
        with torch.no_grad():
            for f in (b200, eager):
                f(); f()
            torch.cuda.synchronize()
            for r in range(args.rounds):
                for nm, f in (("b200", b200), ("eager_bf16", eager)):
                    t = _time(f, args.reps)
                    res["rows"].append({"impl": nm, "batch": B, "round": r, "s_per_batch": t, "images_per_s": B / t,
                                        "tflops": flops * B / t / 1e12})
                    print(json.dumps(res["rows"][-1]), flush=True)
    # the level-0 3x3 convs alone (96 -> 96 channels at full size, zero-padded to 128 per tap)
    xs = torch.randn(1, H, W, 96, device="cuda").bfloat16()
    w9 = ops.conv_w9(torch.randn(96, 96, 3, 3, device="cuda").bfloat16() * 0.03)
    bias = torch.zeros(96, device="cuda", dtype=torch.bfloat16)
    f0 = lambda: ops.conv3x3_nhwc(xs, w9, bias)
    f0(); torch.cuda.synchronize()
    t0 = _time(f0, 20)
    res["level0_conv_96to96"] = {"s": t0, "tflops_algorithmic": 2 * 9 * 96 * 96 * H * W / t0 / 1e12,
                                 "tflops_issued_with_padding": 2 * 9 * 128 * 96 * H * W / t0 / 1e12}
    print(json.dumps({k: v for k, v in res.items() if k != "rows"}), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
