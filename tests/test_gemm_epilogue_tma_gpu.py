"""GPU (-m gpu): the 128 x 128 GEMM's shared-memory epilogue (TMA load of res / aux, TMA stores of D and aux) against the
register epilogue of the 128 x 64 tiles, which reads and stores global memory from the accumulator layout.

A is drawn from small integers and W from multiples of 2^-4, so every partial sum of the dot products is exact and both
tile widths hold the same fp32 accumulators; the epilogue arithmetic is shared, so every output must agree bit for bit.
D, res and aux are column windows of wider buffers, one row in from each batch slab's edges, with a sentinel halo:
rows_per_batch is not a multiple of 128 and B = 3, so a tile that read or wrote across a batch boundary or past the
window would show in the halo or in the outputs."""
import pytest
import torch

from simpletuner_b200 import ops as E
from tests.kernel_checks import _gen, _rand

pytestmark = pytest.mark.gpu

SENTINEL = 3.0
PATHS = {"smem": (1, 128), "smem_cluster": (2, 128), "regs": (0, 64)}


def _window(B, M, N, seed=None):
    """([B, M + 2, N + 24] buffer full of SENTINEL, its [B, M, N] window at rows 1.., columns 8..); seed: random window"""
    full = torch.full((B, M + 2, N + 24), SENTINEL, dtype=torch.bfloat16, device="cuda")
    if seed is not None:
        full[:, 1:M + 1, 8:8 + N] = _rand(B, M, N, seed=seed)
    return full, full[:, 1:M + 1, 8:8 + N]


def _run(tile, M, N, K, B=1, epi=E.EPI_STORE, aux_out=False, nan_to_num=False, special=False):
    """The full buffers of out and aux (None without one) after one ops.gemm at `tile`, on seeded exact inputs."""
    a = _gen(B, M, K, seed=10, exact="int")
    w = _gen(N, K, seed=20, exact="frac")
    bias = _rand(N, seed=30)
    gate = _rand(B, N, seed=31) if epi == E.EPI_GATE_RES else None
    res_full, res = _window(B, M, N, seed=32) if epi in (E.EPI_GATE_RES, E.EPI_ADD_RES) else (None, None)
    aux_full, aux = None, None
    if epi in (E.EPI_MUL_DGELU, E.EPI_MUL):
        aux_full, aux = _window(B, M, N, seed=33)
    elif aux_out:
        aux_full, aux = _window(B, M, N)
    if special:   # +-inf and NaN residuals, and +-bf16 max pushed past the range by a 2^120 gate
        big = torch.finfo(torch.bfloat16).max
        res[..., 0::8] = float("inf")
        res[..., 1::8] = float("-inf")
        res[..., 2::8] = float("nan")
        res[:, 0::2, 3::8] = big
        res[:, 1::2, 3::8] = -big
        gate[:, 3::8] = 2.0 ** 120
    out_full, out = _window(B, M, N)
    E.gemm([a], [w], bias, out=out, epi=epi, gate=gate, res=res, aux=aux, nan_to_num=nan_to_num, tile=tile)
    torch.cuda.synchronize()
    if res_full is not None:
        assert _halo_clean(res_full, M, N), "res was written"
    return out_full, (aux_full if aux_out else None)


def _halo_clean(full, M, N):
    halo = torch.ones_like(full, dtype=torch.bool)
    halo[:, 1:M + 1, 8:8 + N] = False
    return bool((full[halo] == SENTINEL).all())


def _same(M, N, K, B=1, paths=("smem", "smem_cluster"), **kw):
    ref = _run(PATHS["regs"], M, N, K, B, **kw)
    for name in paths:
        got = _run(PATHS[name], M, N, K, B, **kw)
        for what, g, r in (("out", got[0], ref[0]), ("aux", got[1], ref[1])):
            if r is None:
                continue
            assert _halo_clean(g, M, N), f"{name}: {what} halo written"
            assert torch.equal(g.view(torch.int16), r.view(torch.int16)), f"{name}: {what} differs from the register epilogue"


EPIS = {
    "store": dict(epi=E.EPI_STORE),
    "gelu": dict(epi=E.EPI_GELU),
    "gelu_aux": dict(epi=E.EPI_GELU, aux_out=True),
    "gate_res": dict(epi=E.EPI_GATE_RES),
    "gate_res_aux": dict(epi=E.EPI_GATE_RES, aux_out=True),
    "gate_res_nan": dict(epi=E.EPI_GATE_RES, nan_to_num=True, special=True),
    "gate_res_aux_nan": dict(epi=E.EPI_GATE_RES, aux_out=True, nan_to_num=True, special=True),
    "mul_dgelu": dict(epi=E.EPI_MUL_DGELU),
    "add_res": dict(epi=E.EPI_ADD_RES),
    "mul": dict(epi=E.EPI_MUL),
    "quick_gelu": dict(epi=E.EPI_QUICK_GELU),
}


@pytest.mark.parametrize("epi", list(EPIS))
def test_smem_epilogue_matches_registers_across_batches(epi):
    # 300 rows per batch (a 44-row tail tile in each of 3 batches); N = 328: the last n-tile's second half is 8 wide
    _same(300, 328, 200, B=3, **EPIS[epi])


@pytest.mark.parametrize("epi", ["gelu_aux", "gate_res_aux_nan", "mul_dgelu", "add_res"])
def test_smem_epilogue_one_kblock(epi):
    # K = 64: the operand load is issued after the tile's only k-block
    _same(200, 256, 64, B=2, **EPIS[epi])


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("per_cta", (1, 2, 3))
def test_smem_epilogue_tiles_per_cta(per_cta):
    # single CTAs: every CTA takes per_cta tiles, so both warpgroups' buffers run, once or twice each
    _same(128 * per_cta, 128 * _sms(), 64, paths=("smem",), epi=E.EPI_GATE_RES, nan_to_num=True, special=True)


@pytest.mark.parametrize("epi", ["gelu_aux", "gate_res", "mul_dgelu"])
def test_smem_epilogue_cluster_phantom_tile(epi):
    # three m-tiles: the last pair's second tile is past the end, its loads zero-filled and its stores skipped
    _same(384, 384, 200, paths=("smem_cluster",), **EPIS[epi])
