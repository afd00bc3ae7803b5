#!/usr/bin/env python
"""Kernel micro-benchmarks (CUDA events, rotating buffers larger than L2) -> bench_out/microbench.json.

python tools/microbench.py [flux] [gemm] [attn] [--out DIR]; `flux` times the large GEMMs of the batch-1 flux_lora step."""
import hashlib
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


# The large GEMMs of one batch-1 flux_lora step (1024^2: 4096 image + 512 text tokens; single blocks run both as
# 4608 rows).  K segments: a trailing 16 is the rank-16 LoRA k-block; w_kn marks the dgrads, which read the forward
# weight as [K, N].  Columns: block, name, M, N, K segments, w_kn, epilogue, bias, nan_to_num.
E = ops
FLUX_GEMMS = [
    ("single", "qkv", 4608, 9216, [3072, 16], False, E.EPI_STORE, True, False),
    ("single", "fc1", 4608, 12288, [3072], False, E.EPI_GELU, True, False),
    ("single", "proj_out", 4608, 3072, [3072, 12288], False, E.EPI_GATE_RES, True, True),
    ("single", "d_o", 4608, 3072, [3072], True, E.EPI_STORE, False, False),
    ("single", "d_pre", 4608, 12288, [3072], True, E.EPI_MUL_DGELU, False, False),
    ("single", "d_nh", 4608, 3072, [12288, 9216, 16], True, E.EPI_STORE, False, False),
] + [
    (blk, name, M, N, segs, kn, epi, bias, False)
    for blk, M in (("double_img", 4096), ("double_txt", 512))
    for name, N, segs, kn, epi, bias in (
        ("qkv", 9216, [3072, 16], False, E.EPI_STORE, True),
        ("out", 3072, [3072, 16], False, E.EPI_GATE_RES, True),
        ("fc1", 12288, [3072], False, E.EPI_GELU, True),
        ("fc2", 3072, [12288], False, E.EPI_GATE_RES, True),
        ("d_pre", 12288, [3072], True, E.EPI_MUL_DGELU, False),
        ("d_nh2", 3072, [12288], True, E.EPI_STORE, False),
        ("d_o", 3072, [3072, 16], True, E.EPI_STORE, False),
        ("d_nh", 3072, [9216, 16], True, E.EPI_STORE, False),
    )
]


def _digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()[:16]


def _tile_suffix(tile):
    mt, bn = tile
    return ("" if bn == 0 else f"_bn{bn}") + ("_single" if mt == 1 else "_cluster" if mt == 2 else "")


def bench_flux_gemm(blk, name, M, N, segs, kn, epi, bias, nan, nbuf=3, tiles=((0, 0),), iters=20, rounds=2):
    """Our kernel with the step's epilogue, the same with a plain store (no bias), and torch.matmul at the same M, N and
    summed K; rotating operand sets.  tiles: (mt, bn) requests of ops.gemm, timed in turn for `rounds` rounds (best
    round kept), so that the paths compared share the machine's state.  `digest` fingerprints each output on seeded
    inputs, for old-vs-new and single-vs-cluster comparison."""
    g = torch.Generator(device="cuda").manual_seed(1234)
    rnd = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=g) * sc).bfloat16()  # noqa: E731
    sets = []
    for _ in range(nbuf):
        A = [rnd(M, k) for k in segs]
        W = [ops.WT(rnd(k, N, sc=0.02)) if kn else rnd(N, k, sc=0.02) for k in segs]
        sets.append((A, W))
    K = sum(segs)
    b = rnd(N) if bias else None
    gate = rnd(1, N) if epi == E.EPI_GATE_RES else None
    res = rnd(M, N) if epi == E.EPI_GATE_RES else None
    aux = rnd(M, N) if epi in (E.EPI_GELU, E.EPI_MUL_DGELU) else None
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    flop = 2.0 * M * N * K
    r = {"kind": "flux_gemm", "block": blk, "name": name, "M": M, "N": N, "K": segs, "w_kn": kn, "epi": epi}
    i = [0]

    def run(j, tile, e, with_bias):
        A, W = sets[j]
        ops.gemm(A, W, b if with_bias else None, out=out, epi=e, gate=gate if e == E.EPI_GATE_RES else None,
                 res=res if e == E.EPI_GATE_RES else None, aux=aux if e in (E.EPI_GELU, E.EPI_MUL_DGELU) else None,
                 nan_to_num=nan, tile=tile)

    def rot(tile, e, with_bias):
        def fn():
            i[0] += 1
            run(i[0] % nbuf, tile, e, with_bias)
        return fn

    best = {t: (float("inf"), float("inf")) for t in tiles}
    for _ in range(rounds):
        for tile in tiles:
            ms = timeit(rot(tile, epi, bias), iters=iters, warm=5)
            ms_store = timeit(rot(tile, E.EPI_STORE, False), iters=iters, warm=5)
            best[tile] = (min(best[tile][0], ms), min(best[tile][1], ms_store))
    for tile in tiles:
        sfx = _tile_suffix(tile)
        ms, ms_store = best[tile]
        run(0, tile, epi, bias)
        if aux is not None and epi == E.EPI_GELU:
            r["digest_aux" + sfx] = _digest(aux)
        r["digest" + sfx] = _digest(out)
        run(0, tile, E.EPI_STORE, False)
        r["digest_store" + sfx] = _digest(out)
        r.update({"ms" + sfx: round(ms, 4), "tflops" + sfx: round(flop / ms / 1e9, 1),
                  "store_ms" + sfx: round(ms_store, 4), "store_tflops" + sfx: round(flop / ms_store / 1e9, 1)})
    A2 = [torch.cat(A, 1) for A, _ in sets]
    W2 = [torch.cat([w.w.t() if kn else w for w in W], 1) for _, W in sets]

    def ref():
        i[0] += 1
        j = i[0] % nbuf
        torch.matmul(A2[j], W2[j].t(), out=out)

    ms_ref = timeit(ref, iters=iters, warm=5)
    r.update({"cublas_ms": round(ms_ref, 4), "cublas_tflops": round(flop / ms_ref / 1e9, 1)})
    del sets, A2, W2
    torch.cuda.empty_cache()
    return r


def flux_gemms():
    res = []
    pair = ((1, 128), (2, 128))   # 128 x 128 tiles on single CTAs and on 2-CTA clusters
    for row in FLUX_GEMMS:
        # every tile width at M = 512 (text stream), the two wide ones elsewhere: the tile choice in stb_gemm_bf16
        tiles = ((0, 0), (0, 64), *pair, (0, 256)) if row[2] == 512 else ((0, 0), *pair, (0, 256))
        res.append(bench_flux_gemm(*row, tiles=tiles))
    # per-k-block slope and per-tile intercept: plain store at three depths, both 128 x 128 paths
    for N in (3072, 12288):
        for K in (3072, 6144, 12288):
            res.append(bench_flux_gemm("ksweep", f"k{K}", 4608, N, [K], False, E.EPI_STORE, False, False, tiles=pair))
    # M = 1 modulation GEMM (6 x 3072 outputs) at every tile width
    res.append(bench_flux_gemm("mod", "mod", 1, 18432, [3072], False, E.EPI_STORE, True, False,
                               tiles=((0, 0), (0, 64), (0, 128), (0, 256)), iters=100))
    return res


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
    args = sys.argv[1:]
    out = ROOT / "bench_out"
    if "--out" in args:
        k = args.index("--out")
        out = Path(args[k + 1])
        del args[k:k + 2]
    which = args or ["gemm", "attn"]
    if "flux" in which:
        for r in flux_gemms():
            print(json.dumps(r), flush=True)
            res.append(r)
    if "gemm" in which:
        for (M, N, K) in [(16384, 3072, 3072), (16384, 12288, 3072), (16384, 3072, 12288), (2048, 3072, 3072), (16384, 9216, 3072)]:
            for tile in [(1, 256), (1, 128), (2, 128)]:
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
    out.mkdir(parents=True, exist_ok=True)
    (out / f"microbench_{int(time.time())}.json").write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
