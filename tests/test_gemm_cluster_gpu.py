"""GPU (-m gpu): the 2-CTA cluster GEMM (tile_mt = 2) against the single-CTA kernel (tile_mt = 1) at BN 128.

Each output tile is still computed by one warpgroup over the same k-blocks in the same order, so the two paths must
agree bit for bit: every epilogue (with its aux output), [N, K] and [K, N] weights, three segments (200 + 72 + 16 = 7
k-blocks, the ring out of step at every tile boundary), row tails, and odd m-tile counts, where the last pair's second
tile is a phantom past the end.  The tile-count cases restate those of test_gemm_pingpong_gpu.py for pairs and
clusters, taking SMs / 2 as the number of clusters (the device may hold a few fewer)."""
import re

import pytest
import torch

from simpletuner_b200 import ops as E
from tests.kernel_checks import _rand, check_gemm

pytestmark = pytest.mark.gpu

SEG7 = [72, 16]    # with K = 200: 4 + 2 + 1 k-blocks


def _run(M, N, K, B=1, segs=(), epi=E.EPI_STORE, bias=True, nan_to_num=False, w_kn=False, mt=1):
    """Seeded inputs -> (out, aux or None) of one ops.gemm at tile (mt, 128)."""
    Ks = [K, *segs]
    a = [_rand(B, M, k, seed=10 + i) for i, k in enumerate(Ks)]
    w = [_rand(k, N, scale=0.5, seed=20 + i) if w_kn else _rand(N, k, scale=0.5, seed=20 + i) for i, k in enumerate(Ks)]
    b = _rand(N, seed=30) if bias else None
    gate = _rand(B, N, seed=31) if epi == E.EPI_GATE_RES else None
    res = _rand(B, M, N, seed=32) if epi in (E.EPI_GATE_RES, E.EPI_ADD_RES) else None
    aux = None
    if epi in (E.EPI_GELU, E.EPI_GATE_RES):
        aux = torch.zeros(B, M, N, dtype=torch.bfloat16, device="cuda")
    elif epi in (E.EPI_MUL_DGELU, E.EPI_MUL):
        aux = _rand(B, M, N, seed=33)
    out = torch.zeros(B, M, N, dtype=torch.bfloat16, device="cuda")
    E.gemm(a, w, b, out=out, epi=epi, gate=gate, res=res, aux=aux, nan_to_num=nan_to_num, tile=(mt, 128),
           w_kn=[w_kn] * len(Ks))
    torch.cuda.synchronize()
    return out, aux


def _same(**kw):
    single = _run(mt=1, **kw)
    cluster = _run(mt=2, **kw)
    assert torch.equal(single[0].view(torch.int16), cluster[0].view(torch.int16)), "outputs differ"
    if single[1] is not None:
        assert torch.equal(single[1].view(torch.int16), cluster[1].view(torch.int16)), "aux differs"


EPIS = {
    "store_bias": dict(epi=E.EPI_STORE),
    "gelu_aux": dict(epi=E.EPI_GELU),
    "gate_res_nan_aux": dict(epi=E.EPI_GATE_RES, nan_to_num=True),
    "mul_dgelu": dict(epi=E.EPI_MUL_DGELU, bias=False),
    "add_res": dict(epi=E.EPI_ADD_RES),
    "mul": dict(epi=E.EPI_MUL),
    "quick_gelu": dict(epi=E.EPI_QUICK_GELU),
}


@pytest.mark.parametrize("epi", list(EPIS))
@pytest.mark.parametrize("wkn", (False, True))
def test_cluster_bit_identical_every_epilogue(epi, wkn):
    # 300 rows: three m-tiles (odd, with a row tail); N = 328: a partial last n-tile whose second W half is out of range
    _same(M=300, N=328, K=200, segs=SEG7, w_kn=wkn, **EPIS[epi])


@pytest.mark.parametrize("M,B", [(128, 1), (300, 1), (300, 3), (100, 5), (200, 3), (4608, 1)])
@pytest.mark.parametrize("wkn", (False, True))
def test_cluster_bit_identical_pairs_and_batches(M, B, wkn):
    # (128, 1): one m-tile, a phantom partner only; (300, 3) and (100, 5): odd tiles_m with pairs across batches
    _same(M=M, N=384, K=200, B=B, segs=SEG7, w_kn=wkn, epi=E.EPI_GATE_RES, nan_to_num=True)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


CASES = {
    # (rows, N) as functions of the number of clusters: pairs of 128-row tiles at BN 128
    "one_pair_per_cluster": lambda cl: (256, 128 * cl),
    "fewer_pairs_than_clusters": lambda cl: (256 * 3, 128 * 7),
    "three_pairs_per_cluster": lambda cl: (256 * 3, 128 * cl),
    "one_extra_pair": lambda cl: (256, 128 * (cl + 1)),
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("wkn", (False, True))
def test_cluster_tile_counts(case, wkn):
    M, N = CASES[case](_sms() // 2)
    _same(M=M, N=N, K=200, segs=SEG7, w_kn=wkn, epi=E.EPI_GATE_RES, nan_to_num=True)
    r = check_gemm(M, N, 200, segs=SEG7, bias=True, epi=E.EPI_GATE_RES, nan_to_num=True, tile=(2, 128),
                   w_kn=[True] * 3 if wkn else None)
    assert r["ok"], r


@pytest.mark.parametrize("args", [
    dict(M=300, N=328, K=200, B=3, segs=SEG7, bias=True, epi=E.EPI_GELU),
    dict(M=4608, N=3072, K=3072, bias=True, epi=E.EPI_STORE),
    dict(M=700, N=384, K=456, B=2, w_kn=[True]),
    dict(M=128, N=256, K=128, bias=True),
], ids=["gelu_b3_tails", "flux_qkv", "wkn_b2", "phantom_only"])
def test_cluster_against_fp32(args):
    r = check_gemm(tile=(2, 128), **args)
    assert r["ok"], r


def _gemm_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "gemm_bf16_tn_kernel" in e.name]


def test_tile_mt_selects_the_kernel():
    a = _rand(4608, 3072, seed=1)
    w = _rand(3072, 3072, scale=0.02, seed=2)
    E.gemm([a], [w], tile=(2, 128))     # warm-up: module load and the cluster-count query
    names = _gemm_kernels(lambda: E.gemm([a], [w], tile=(2, 128)))
    assert names and all(re.search(r"gemm_bf16_tn_kernel<128, 0, false, 2>", n) for n in names), names
    # automatic: single CTAs for a plain store, clusters for the GELU epilogue at a Flux shape
    names = _gemm_kernels(lambda: E.gemm([a], [w]))
    assert names and all(re.search(r"gemm_bf16_tn_kernel<128, 0, false, 1>", n) for n in names), names
    aux = torch.empty(4608, 3072, dtype=torch.bfloat16, device="cuda")
    names = _gemm_kernels(lambda: E.gemm([a], [w], epi=E.EPI_GELU, aux=aux))
    assert names and all(re.search(r"gemm_bf16_tn_kernel<128, 1, false, 2>", n) for n in names), names
