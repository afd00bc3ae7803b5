"""GPU (-m gpu): the row-wise entry points reject views their vector loads cannot take (STB_ERR_ARG), before any launch.

ln_modulate_bwd loads 16 bytes at row + c (pointers 16-byte aligned, strides multiples of 8 elements); the warp-per-token
q/k RMSNorm + RoPE kernels load HD / 32 consecutive elements per lane (8 bytes at HD 128, 4 at HD 64)."""
import pytest
import torch

from simpletuner_b200 import ops
from simpletuner_b200._lib import StbError

pytestmark = pytest.mark.gpu


def _bf(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).bfloat16().cuda()


def _flat_view(shape, offset):
    """A contiguous view of `shape` that starts `offset` elements into a flat buffer."""
    n = 1
    for s in shape:
        n *= s
    return _bf(n + 8)[offset:offset + n].view(*shape)


def test_ln_modulate_bwd_rejects_misaligned():
    B, S, D = 2, 8, 64
    x, dy = _bf(B, S, D, seed=1), _bf(B, S, D, seed=2)
    scale = _bf(B, 6 * D, seed=3)[:, D:2 * D]
    wide = _bf(B, S, D + 12, seed=4)
    cases = {
        "x row stride D + 12": dict(dy=dy, x=wide[..., :D]),
        "x pointer + 8 bytes": dict(dy=dy, x=wide[..., 4:4 + D]),
        "dy row stride D + 12": dict(dy=wide[..., :D], x=x),
        "add row stride D + 12": dict(dy=dy, x=x, add=wide[..., :D]),
        "out row stride D + 12": dict(dy=dy, x=x, out=torch.zeros_like(wide)[..., :D]),
        "scale batch stride 6 D + 4": dict(dy=dy, x=x, scale=_bf(B, 6 * D + 4, seed=5)[:, :D]),
    }
    for what, kw in cases.items():
        with pytest.raises(StbError):
            ops.ln_modulate_bwd(kw["dy"], kw["x"], kw.get("scale", scale), add=kw.get("add"), out=kw.get("out"))
            pytest.fail(f"accepted: {what}")
    ops.ln_modulate_bwd(dy, x, scale, add=_bf(B, S, D + 16, seed=6)[..., 8:8 + D])   # aligned windows pass
    torch.cuda.synchronize()


@pytest.mark.parametrize("HD", [64, 128])
def test_qk_rmsnorm_rope_fwd_rejects_misaligned(HD):
    B, S, H = 2, 16, 2
    D = H * HD
    shift = 1 if HD == 64 else 2                  # elements: 2 bytes at HD 64, 4 bytes at HD 128
    buf = _bf(B, S, 3 * D + 8, seed=1)
    with pytest.raises(StbError):
        ops.qk_rmsnorm_rope_fwd(buf[..., shift:shift + 3 * D], D, H, HD, None, None)
    with pytest.raises(StbError):
        ops.qk_rmsnorm_rope_fwd(buf, D + shift, H, HD, None, None)
    with pytest.raises(StbError):
        ops.qk_rmsnorm_rope_fwd(buf, D, H, HD, None, None, q_out=_flat_view((B, S, H, HD), shift))
    ops.qk_rmsnorm_rope_fwd(buf, D + 2 * shift, H, HD, None, None)   # the smallest legal k offset
    torch.cuda.synchronize()


@pytest.mark.parametrize("HD,dw", [(64, False), (64, True), (128, False), (128, True)])
def test_qk_rmsnorm_rope_bwd_rejects_misaligned(HD, dw):
    """Every path that runs the warp-per-token kernel: HD 64, and HD 128 with dw or a layout the flat kernel cannot read."""
    B, S, H = 2, 16, 2
    D = H * HD
    shift = 1 if HD == 64 else 2
    src = _bf(B, S, 3 * D + 8, seed=1)
    dq, dk = _bf(B, S, H, HD, seed=2), _bf(B, S, H, HD, seed=3)
    w = [_bf(HD, seed=4 + i) for i in range(4)] if dw else [None] * 4
    run = lambda **kw: ops.qk_rmsnorm_rope_bwd(kw.get("dq", dq), kw.get("dk", dk), kw.get("src", src), kw.get("k_off", D), H,
                                               HD, *w, 0, None, None, dsrc=kw.get("dsrc", torch.zeros_like(src)),
                                               dw=torch.zeros(4, HD, device="cuda") if dw else None)
    cases = {
        "src pointer": dict(src=src[..., shift:shift + 3 * D], dsrc=torch.zeros_like(src)[..., :3 * D]),
        "k offset": dict(k_off=D + shift),
        "dsrc pointer": dict(dsrc=torch.zeros_like(src)[..., shift:shift + 3 * D + 8 - shift]),
        "dq / dk pointers": dict(dq=_flat_view((B, S, H, HD), shift), dk=_flat_view((B, S, H, HD), shift)),
    }
    for what, kw in cases.items():
        with pytest.raises(StbError):
            run(**kw)
            pytest.fail(f"accepted: {what}")
    run(k_off=D + 2 * shift)
    torch.cuda.synchronize()
