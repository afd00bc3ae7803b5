#!/usr/bin/env python
"""libstb200 attention forward / backward next to torch's F.scaled_dot_product_attention (the kernel the reference's
default `attention_mechanism="diffusers"` path calls, reference flux/transformer.py:200-207) on the same box, same
shapes, CUDA events, SM clocks recorded.  Writes bench_out/attn_vs_sdpa.json.

  python tools/attn_vs_sdpa.py [tag]
"""
import json
import os
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from simpletuner_b200 import ops  # noqa: E402


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def clocks():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,power.draw", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=5).stdout.strip()
        return [float(x) for x in out.split(",")]
    except Exception:
        return None


def one(B, H, S, HD):
    q, k, v, do = (torch.randn(B, S, H, HD, device="cuda").bfloat16() for _ in range(4))
    o, lse = ops.attn_fwd(q, k, v)
    dq, dk, dv = ops.attn_bwd(q, k, v, o, do, lse)
    fl = 4.0 * B * H * S * S * HD
    r = {"B": B, "H": H, "S": S, "HD": HD}
    r["stb_fwd_ms"] = round(timeit(lambda: ops.attn_fwd(q, k, v, out=o)), 4)
    r["clocks_during_stb_fwd"] = clocks()
    r["stb_bwd_ms"] = round(timeit(lambda: ops.attn_bwd(q, k, v, o, do, lse, dq=dq, dk=dk, dv=dv), iters=5), 4)
    # torch SDPA: [B, H, S, HD] views of the same buffers (what the reference's processor passes after its transpose)
    qt, kt, vt = (t.permute(0, 2, 1, 3).detach().requires_grad_(True) for t in (q, k, v))
    dot = do.permute(0, 2, 1, 3)
    r["sdpa_fwd_ms"] = round(timeit(lambda: F.scaled_dot_product_attention(qt.detach(), kt.detach(), vt.detach())), 4)
    r["clocks_during_sdpa_fwd"] = clocks()
    ot = F.scaled_dot_product_attention(qt, kt, vt)

    def bwd():
        torch.autograd.grad(ot, (qt, kt, vt), dot, retain_graph=True)

    r["sdpa_bwd_ms"] = round(timeit(bwd, iters=5), 4)
    # agreement of the two implementations (bf16 outputs)
    r["fwd_max_abs_diff"] = float((ot.detach().permute(0, 2, 1, 3).float() - o.float()).abs().max())
    gq, gk, gv = torch.autograd.grad(ot, (qt, kt, vt), dot, retain_graph=True)
    cos = lambda a, b: float(F.cosine_similarity(a.flatten().float(), b.flatten().float(), dim=0))
    r["bwd_cos"] = [round(cos(gq.permute(0, 2, 1, 3), dq), 6), round(cos(gk.permute(0, 2, 1, 3), dk), 6), round(cos(gv.permute(0, 2, 1, 3), dv), 6)]
    r["stb_fwd_tflops"] = round(fl / r["stb_fwd_ms"] / 1e9, 1)
    r["sdpa_fwd_tflops"] = round(fl / r["sdpa_fwd_ms"] / 1e9, 1)
    r["stb_bwd_tflops_alg"] = round(2.0 * fl / r["stb_bwd_ms"] / 1e9, 1)   # SURVEY 8(d): 8 S^2 D
    r["sdpa_bwd_tflops_alg"] = round(2.0 * fl / r["sdpa_bwd_ms"] / 1e9, 1)
    return r


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "run"
    res = {"tag": tag, "lib": os.environ.get("STB200_LIB", "default"), "env": {k: v for k, v in os.environ.items() if k.startswith("STB_")},
           "torch": torch.__version__, "gpu": torch.cuda.get_device_name(0), "shapes": []}
    for shp in [(4, 24, 4608, 128), (8, 24, 1255, 64), (4, 16, 4096, 128)]:
        try:
            res["shapes"].append(one(*shp))
        except Exception as e:  # noqa
            res["shapes"].append({"shape": shp, "error": str(e)[:300]})
        print(json.dumps(res["shapes"][-1]), flush=True)
    out = ROOT / "bench_out"
    out.mkdir(exist_ok=True)
    (out / f"attn_vs_sdpa_{tag}.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
