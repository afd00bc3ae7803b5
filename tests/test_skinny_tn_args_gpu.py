"""GPU (-m gpu): the LoRA weight gradient (stb_skinny_tn) refuses what its tensor-core kernel cannot take (STB_ERR_ARG),
before any launch: R not a multiple of 8 or above 128, N not a multiple of 8, operands that are not 16-byte aligned or
whose strides are not multiples of 8 elements, and a missing or short slab workspace.  `out` is left as it was."""
import pytest
import torch

from simpletuner_b200 import _lib, ops
from simpletuner_b200._lib import StbError

pytestmark = pytest.mark.gpu

B, S, R, N = 2, 100, 16, 256


def _bf(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).bfloat16().cuda()


def _flat_view(shape, offset, seed=0):
    """A contiguous view of `shape` that starts `offset` elements into a flat buffer."""
    n = 1
    for s in shape:
        n *= s
    return _bf(n + 8, seed=seed)[offset:offset + n].view(*shape)


def _out(r, n):
    return torch.randn(r, n, generator=torch.Generator().manual_seed(9)).cuda()


def _raw(L, Rm, out, ws, ws_elems):
    """stb_skinny_tn with a caller-chosen workspace (ops.skinny_tn always passes a large enough one)."""
    _lib.check(_lib.lib().stb_skinny_tn(L.data_ptr(), L.stride(0), L.stride(1), Rm.data_ptr(), Rm.stride(0), Rm.stride(1),
                                        out.data_ptr(), B, S, L.shape[2], Rm.shape[2], 1.0, ws, ws_elems,
                                        ops._stream()))


def test_skinny_tn_rejects_shapes_and_views_outside_the_tensor_core_domain():
    L, Rm = _bf(B, S, R, seed=1), _bf(B, S, N, seed=2)
    cases = {
        "R = 12": (_bf(B, S, 12, seed=3), Rm),
        "R = 136": (_bf(B, S, 136, seed=3), Rm),
        "N = 250": (L, _bf(B, S, 250, seed=4)),
        "L pointer + 4 elements": (_flat_view((B, S, R), 4, seed=5), Rm),
        "Rm pointer + 4 elements": (L, _flat_view((B, S, N), 4, seed=6)),
        "Rm row stride N + 4": (L, _bf(B, S, N + 4, seed=7)[..., :N]),
    }
    for what, (l, rm) in cases.items():
        out = _out(l.shape[2], rm.shape[2])
        before = out.clone()
        with pytest.raises(StbError):
            ops.skinny_tn(l, rm, out=out)
            pytest.fail(f"accepted: {what}")
        torch.cuda.synchronize()
        assert torch.equal(out, before), what


def test_skinny_tn_rejects_a_missing_or_short_workspace():
    L, Rm = _bf(B, S, R, seed=1), _bf(B, S, N, seed=2)
    need = int(_lib.lib().stb_skinny_tn_workspace(B, S, R, N))
    assert need >= R * N
    ws = torch.empty(need, device="cuda", dtype=torch.float32)
    out = _out(R, N)
    before = out.clone()
    for what, ptr, elems in (("one element short", ws.data_ptr(), need - 1), ("null", None, need)):
        with pytest.raises(StbError):
            _raw(L, Rm, out, ptr, elems)
            pytest.fail(f"accepted: {what} workspace")
        torch.cuda.synchronize()
        assert torch.equal(out, before), what
    _raw(L, Rm, out, ws.data_ptr(), need)   # the exact size passes
    torch.cuda.synchronize()
    assert not torch.equal(out, before)
