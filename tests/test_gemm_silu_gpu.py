"""GPU (-m gpu): the SiLU GEMM epilogue (ops.EPI_SILU, D = y sigmoid(y) with y = bf16(acc + bias)) of the Chroma
approximator, against an fp64 reference element by element, and bit for bit between the shared-memory epilogue of the
128 x 128 tiles and the register epilogue of the other widths (tests/test_gemm_epilogue_tma_gpu.py's harness)."""
import pytest
import torch

from simpletuner_b200 import ops as E
from tests.kernel_checks import GEMM_C, _U, _acc_unit, _gen, _neighbour, _rand, _report, _slope, exact_bound_ok
from tests.test_gemm_epilogue_tma_gpu import _same

pytestmark = pytest.mark.gpu
TILES = [(0, 0), (1, 64), (1, 128), (2, 128), (1, 256)]


def silu64(y):
    return y * torch.sigmoid(y)


def dsilu64(y):
    s = torch.sigmoid(y)
    return s + y * s * (1.0 - s)


@pytest.mark.parametrize("tile", TILES)
def test_silu_epilogue_exact_inputs_is_a_bf16_neighbour_of_fp64(tile):
    # exact inputs: the fp32 accumulator equals the fp64 sum, so y = bf16(acc + bias) is known exactly and the output must
    # be one of the two bf16 neighbours of fp64 silu(y) (__expf and the division stay within that)
    B, M, N, K = 2, 300, 328, 200
    a, w, bias = _gen(B, M, K, seed=10, exact="int"), _gen(N, K, seed=20, exact="frac"), _rand(N, seed=30, scale=4.0)
    got = E.gemm([a], [w], bias, epi=E.EPI_SILU, tile=tile)
    torch.cuda.synchronize()
    acc = a.double() @ w.double().t()
    assert exact_bound_ok([a], [w], a.double().abs() @ w.double().abs().t())
    y = (acc.float() + bias.float()).to(torch.bfloat16).double()
    assert bool((y < -8).any() and (y > 8).any())              # both tails of the sigmoid are exercised
    r = _neighbour("out", got, silu64(y))
    assert r["ok"], r


@pytest.mark.parametrize("tile", TILES)
def test_silu_epilogue_realistic_inputs_against_fp64(tile):
    B, M, N, K = 1, 688, 640, 640          # 2 x 344 approximator rows at a small width
    a, w, bias = _gen(B, M, K, seed=11), _gen(N, K, seed=21, scale=K ** -0.5), _rand(N, seed=31)
    got = E.gemm([a], [w], bias, epi=E.EPI_SILU, tile=tile)
    torch.cuda.synchronize()
    f64 = a.double() @ w.double().t() + bias.double()
    atol = GEMM_C * _acc_unit(a.double().abs() @ w.double().abs().t(), K)
    r = _report("out", got, silu64(f64), atol=_slope(dsilu64, f64) * (atol + _U * f64.abs()), rtol=_U)
    assert r["ok"], r


def test_silu_smem_epilogue_matches_registers_across_batches():
    _same(300, 328, 200, B=3, epi=E.EPI_SILU)


def test_silu_smem_epilogue_cluster_phantom_tile():
    _same(384, 384, 200, paths=("smem_cluster",), epi=E.EPI_SILU)
