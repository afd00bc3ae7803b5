"""GPU (-m gpu): tile counts that the ping-pong GEMM schedules in special ways.

The two consumer warpgroups of a CTA take its persistent tiles in turn (tile 0, 2, 4, ... and 1, 3, 5, ...) and each
passes over the other's stages of the shared ring.  These shapes give every CTA at most one tile (the second
warpgroup never runs a mainloop), leave SMs without a tile, give every CTA three tiles (the two warpgroups end on
different laps of the ring), and give one CTA a second tile while every other CTA has one.  Segments of
200 + 72 + 16 = 7 k-blocks keep the ring phase out of step at every tile boundary."""
import pytest
import torch

from tests.kernel_checks import check_gemm
from simpletuner_b200 import ops as E

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _bm(bn):
    return 64 if bn == 256 else 128


CASES = {
    # (rows, N) as functions of the SM count and the tile width
    "one_tile_per_cta": lambda sms, bn: (_bm(bn) * 4, bn * (sms // 4)),
    "fewer_tiles_than_sms": lambda sms, bn: (_bm(bn) * 3, bn * 7),
    "three_tiles_per_cta": lambda sms, bn: (_bm(bn) * 3, bn * sms),
    "one_extra_tile": lambda sms, bn: (_bm(bn), bn * (sms + 1)),
}


@pytest.mark.parametrize("bn", (64, 128, 256))
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("wkn", (False, True))
def test_pingpong_tile_counts(case, bn, wkn):
    M, N = CASES[case](_sms(), bn)
    r = check_gemm(M, N, 200, segs=[72, 16], bias=True, epi=E.EPI_GATE_RES, nan_to_num=True, tile=(0, bn),
                   w_kn=[True, True, True] if wkn else None)
    assert r["ok"], r
