#!/usr/bin/env python
"""Kernel micro-benchmarks (CUDA events, rotating buffers larger than L2) -> bench_out/microbench.json."""
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402

from simpletuner_b200 import ops  # noqa: E402


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_gemm(M, N, K, tile, nbuf=3, epi=ops.EPI_STORE):
    As = [torch.randn(M, K, device="cuda").bfloat16() for _ in range(nbuf)]
    Ws = [(torch.randn(N, K, device="cuda") * 0.02).bfloat16() for _ in range(nbuf)]
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    i = [0]

    def fn():
        j = i[0] % nbuf
        i[0] += 1
        ops.gemm([As[j]], [Ws[j]], out=out, tile=tile, epi=epi)

    ms = timeit(fn)
    tf = 2.0 * M * N * K / ms / 1e9

    def ref():
        j = i[0] % nbuf
        i[0] += 1
        torch.matmul(As[j], Ws[j].t(), out=out)

    ms_ref = timeit(ref)
    return {"kind": "gemm", "M": M, "N": N, "K": K, "tile": tile, "ms": round(ms, 4), "tflops": round(tf, 1),
            "cublas_ms": round(ms_ref, 4), "cublas_tflops": round(2.0 * M * N * K / ms_ref / 1e9, 1)}


def bench_attn(B, H, S, HD=128, bwd=True):
    q = torch.randn(B, S, H, HD, device="cuda").bfloat16()
    k = torch.randn(B, S, H, HD, device="cuda").bfloat16()
    v = torch.randn(B, S, H, HD, device="cuda").bfloat16()
    do = torch.randn(B, S, H, HD, device="cuda").bfloat16()
    o, lse = ops.attn_fwd(q, k, v)
    ms_f = timeit(lambda: ops.attn_fwd(q, k, v, out=o))
    fl = 4.0 * B * H * S * S * HD
    r = {"kind": "attn", "B": B, "H": H, "S": S, "HD": HD, "fwd_ms": round(ms_f, 4), "fwd_tflops": round(fl / ms_f / 1e9, 1)}
    if bwd:
        dq, dk, dv = ops.attn_bwd(q, k, v, o, do, lse)
        ms_b = timeit(lambda: ops.attn_bwd(q, k, v, o, do, lse, dq=dq, dk=dk, dv=dv), iters=5)
        r.update({"bwd_ms": round(ms_b, 4), "bwd_tflops_5gemm": round(2.5 * fl / ms_b / 1e9, 1)})
    # torch SDPA (library) for context
    qt, kt, vt = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    try:
        ms_t = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qt, kt, vt))
        r["torch_sdpa_fwd_ms"] = round(ms_t, 4)
    except Exception as e:  # noqa
        r["torch_sdpa_err"] = str(e)[:100]
    return r


def main():
    res = []
    which = sys.argv[1:] or ["gemm", "attn"]
    if "gemm" in which:
        for (M, N, K) in [(16384, 3072, 3072), (16384, 12288, 3072), (16384, 3072, 12288), (2048, 3072, 3072), (16384, 9216, 3072)]:
            for tile in [(1, 256), (2, 256), (3, 256)]:
                try:
                    r = bench_gemm(M, N, K, tile)
                except Exception as e:  # noqa
                    r = {"kind": "gemm", "M": M, "N": N, "K": K, "tile": tile, "error": str(e)[:200]}
                print(json.dumps(r), flush=True)
                res.append(r)
    if "attn" in which:
        for (B, H, S, HD) in [(4, 24, 4608, 128), (1, 24, 4608, 128), (8, 24, 1280, 64)]:
            try:
                r = bench_attn(B, H, S, HD)
            except Exception as e:  # noqa
                r = {"kind": "attn", "B": B, "H": H, "S": S, "error": str(e)[:200]}
            print(json.dumps(r), flush=True)
            res.append(r)
    out = ROOT / "bench_out"
    out.mkdir(exist_ok=True)
    (out / f"microbench_{int(time.time())}.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
