#!/usr/bin/env python
"""Launch a handful of isolated hot kernels (for `ncu --set full -k regex:...`)."""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402

from simpletuner_b200 import ops  # noqa: E402

which = sys.argv[1] if len(sys.argv) > 1 else "gemm"
torch.manual_seed(0)
if which == "gemm":
    M, N, K = 16384, 3072, 3072
    a = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    for _ in range(4):
        ops.gemm([a], [w])
elif which == "attn":
    q, k, v, do = (torch.randn(1, 4608, 24, 128, device="cuda").bfloat16() for _ in range(4))
    for _ in range(3):
        o, lse = ops.attn_fwd(q, k, v)
        ops.attn_bwd(q, k, v, o, do, lse)
elif which == "wgrad_full":          # Flux feed-forward weight gradient (LoKr / full fine-tune): [12288, 3072] from 2 x 4608 tokens
    dy = torch.randn(2, 4608, 12288, device="cuda").bfloat16()
    x = torch.randn(2, 4608, 3072, device="cuda").bfloat16()
    for _ in range(3):
        ops.wgrad_full(dy, x)
elif which == "conv":                # VAE encoder level 0: 3x3, 128 -> 128 channels at 1024^2 (one image)
    x = torch.randn(1, 1024, 1024, 128, device="cuda").bfloat16()
    w9 = (torch.randn(128, 9 * 128, device="cuda") * 0.02).bfloat16()
    b = torch.zeros(128, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        ops.conv3x3_nhwc(x, w9, b)
elif which == "optim":               # one launch: value clip + AdamW-bf16 + EMA over 532 LoRA tensors (26.1 M parameters)
    from simpletuner_b200.training.ema import EMAModel
    from simpletuner_b200.training.optim import AdamWBF16
    ps = [torch.nn.Parameter(torch.randn(16, 3072, device="cuda").bfloat16()) for _ in range(266)] + \
         [torch.nn.Parameter(torch.randn(3072, 16, device="cuda").bfloat16()) for _ in range(266)]
    opt, ema = AdamWBF16(ps, lr=1e-4, seed=0), EMAModel(ps)
    for k in range(4):
        for p in ps:
            p.grad = torch.randn_like(p)
        opt.step(grad_clamp=2.0, ema=ema, ema_global_step=k + 1)
elif which == "optim_big":           # the same kernel on full-fine-tune sized tensors (2.4 G parameters is too much here: 0.6 G)
    from simpletuner_b200.training.optim import AdamWBF16
    ps = [torch.nn.Parameter(torch.randn(3072, 12288, device="cuda").bfloat16()) for _ in range(16)]
    opt = AdamWBF16(ps, lr=1e-4, seed=0)
    for k in range(3):
        for p in ps:
            p.grad = torch.randn_like(p)
        opt.step(grad_clamp=2.0)
elif which == "lokr":                # LoKr rebuild + factor gradients of one Flux feed-forward projection [12288, 3072], factor 4
    W = (torch.randn(12288, 3072, device="cuda") * 0.02).bfloat16()
    w1 = torch.randn(4, 4, device="cuda").bfloat16()
    w2 = (torch.randn(3072, 768, device="cuda") * 0.02).bfloat16()
    out, out_t = torch.empty_like(W), torch.empty(3072, 12288, device="cuda", dtype=torch.bfloat16)
    dW = torch.randn(12288, 3072, device="cuda").bfloat16()
    for _ in range(3):
        ops.lokr_rebuild(W, w1, w2, 1.0, out, out_t)
        ops.lokr_factor_grads(dW, w1, w2, 1.0)
elif which == "gelu":
    pre = torch.randn(4, 4608, 12288, device="cuda").bfloat16()
    for _ in range(3):
        ops.gelu_tanh(pre)
elif which == "time_tail":
    # CUDA-event timings (not under a profiler) of the HBM-bound kernels at Flux shapes: ms and algorithmic GB/s
    import json
    B, S, H, HD, D = 4, 4608, 24, 128, 3072

    def timeit(fn, n=20):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    res = {}
    qkv = torch.randn(B, S, 3 * D, device="cuda").bfloat16()
    wq, wk = torch.ones(HD, device="cuda").bfloat16(), torch.ones(HD, device="cuda").bfloat16()
    cos, sin = torch.rand(S, HD, device="cuda"), torch.rand(S, HD, device="cuda")
    dq, dk = torch.randn(B, S, H, HD, device="cuda").bfloat16(), torch.randn(B, S, H, HD, device="cuda").bfloat16()
    dqkv = torch.empty_like(qkv)
    t = timeit(lambda: ops.qk_rmsnorm_rope_fwd(qkv, D, H, HD, wq, wk, None, None, 0, cos, sin, 1e-6))
    res["qk_rmsnorm_rope_fwd"] = {"ms": t, "GBps": 4 * B * S * D * 2 / t / 1e6}
    t = timeit(lambda: ops.qk_rmsnorm_rope_bwd(dq, dk, qkv, D, H, HD, wq, wk, None, None, 0, cos, sin, 1e-6, dsrc=dqkv))
    res["qk_rmsnorm_rope_bwd"] = {"ms": t, "GBps": 6 * B * S * D * 2 / t / 1e6}
    h = torch.randn(B, S, D, device="cuda").bfloat16()
    sh, sc = torch.randn(B, D, device="cuda").bfloat16(), torch.randn(B, D, device="cuda").bfloat16()
    t = timeit(lambda: ops.ln_modulate_fwd(h, sh, sc, 1e-6))
    res["ln_modulate_fwd"] = {"ms": t, "GBps": 2 * B * S * D * 2 / t / 1e6}
    dn = torch.randn(B, S, D, device="cuda").bfloat16()
    out = torch.empty_like(h)
    t = timeit(lambda: ops.ln_modulate_bwd(dn, h, sc, add=h, eps=1e-6, out=out))
    res["ln_modulate_bwd"] = {"ms": t, "GBps": 4 * B * S * D * 2 / t / 1e6}
    t = timeit(lambda: ops.gate_mul(h, sc))
    res["gate_mul"] = {"ms": t, "GBps": 2 * B * S * D * 2 / t / 1e6}
    from simpletuner_b200.training.optim import AdamWBF16
    ps = [torch.nn.Parameter(torch.randn(3072, 12288, device="cuda").bfloat16()) for _ in range(16)]
    opt = AdamWBF16(ps, lr=1e-4, seed=0)
    for p in ps:
        p.grad = torch.randn_like(p)
    n_el = sum(p.numel() for p in ps)
    t = timeit(lambda: opt.step(grad_clamp=2.0), n=5)
    res["adamw_bf16_multi"] = {"ms": t, "GBps": n_el * 18 / t / 1e6}
    print(json.dumps(res))
elif which == "time_rope_bwd":
    import json
    B, S, H, HD, D = 4, 4608, 24, 128, 3072
    qkv = torch.randn(B, S, 3 * D, device="cuda").bfloat16()
    wq, wk = torch.ones(HD, device="cuda").bfloat16(), torch.ones(HD, device="cuda").bfloat16()
    cos, sin = torch.rand(S, HD, device="cuda"), torch.rand(S, HD, device="cuda")
    dq, dk = torch.randn(B, S, H, HD, device="cuda").bfloat16(), torch.randn(B, S, H, HD, device="cuda").bfloat16()
    dqkv = torch.empty_like(qkv)
    fn = lambda: ops.qk_rmsnorm_rope_bwd(dq, dk, qkv, D, H, HD, wq, wk, None, None, 0, cos, sin, 1e-6, dsrc=dqkv)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = e0.elapsed_time(e1) / 20
    print(json.dumps({"kernel": "qk_rmsnorm_rope_bwd", "ms": t, "GBps": 6 * B * S * D * 2 / t / 1e6, "checksum": float(dqkv[:, :, :2 * D].float().abs().mean())}))
    fq = lambda: ops.qk_rmsnorm_rope_fwd(qkv, D, H, HD, wq, wk, None, None, 0, cos, sin, 1e-6)
    for _ in range(3):
        q_, k_ = fq()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(20):
        fq()
    e1.record()
    torch.cuda.synchronize()
    t = e0.elapsed_time(e1) / 20
    print(json.dumps({"kernel": "qk_rmsnorm_rope_fwd", "ms": t, "GBps": 4 * B * S * D * 2 / t / 1e6, "checksum": float(q_.float().abs().mean() + k_.float().abs().mean())}))
torch.cuda.synchronize()
print("done", which)
