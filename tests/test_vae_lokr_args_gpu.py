"""GPU (-m gpu): the VAE-encode, LoKr and LoRA-dropout entry points reject arguments their kernels cannot take, before
any launch.

stb_groupnorm_nhwc loads x, gamma and beta and stores out 16 bytes at a time; stb_softmax_rows takes the row max of the
unscaled logits, which is the max of the scaled ones only for scale > 0; the LoKr and dropout wrappers read their
operands as rows of unit inner stride, so a transposed view must be refused rather than read as if it were contiguous."""
import pytest
import torch

from simpletuner_b200 import _lib, ops
from simpletuner_b200._lib import StbError

pytestmark = pytest.mark.gpu


def _bf(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).bfloat16().cuda()


def _raw_groupnorm(x, gamma, beta, out, B, HW, C, G):
    stats = torch.empty(max(1, B) * G * 2, device="cuda", dtype=torch.float32)
    _lib.check(_lib.lib().stb_groupnorm_nhwc(x, gamma, beta, out, stats.data_ptr(), B, HW, C, G, 1e-6, 1,
                                             torch.cuda.current_stream().cuda_stream))


def test_groupnorm_rejects_misaligned_pointers_and_empty_shapes():
    B, HW, C, G = 2, 12, 64, 32
    x, out = _bf(B * HW * C + 8, seed=1), torch.zeros(B * HW * C + 8, device="cuda", dtype=torch.bfloat16)
    gm, bt = _bf(C + 8, seed=2), _bf(C + 8, seed=3)
    p = lambda t, off=0: t.data_ptr() + 2 * off
    cases = {
        "x + 2 bytes": (p(x, 1), p(gm), p(bt), p(out), B, HW),
        "out + 8 bytes": (p(x), p(gm), p(bt), p(out, 4), B, HW),
        "gamma + 2 bytes": (p(x), p(gm, 1), p(bt), p(out), B, HW),
        "beta + 4 bytes": (p(x), p(gm), p(bt, 2), p(out), B, HW),
        "B = 0": (p(x), p(gm), p(bt), p(out), 0, HW),
        "HW = 0": (p(x), p(gm), p(bt), p(out), B, 0),
        "null x": (None, p(gm), p(bt), p(out), B, HW),
    }
    for what, (xp, gp, bp, op, b, hw) in cases.items():
        with pytest.raises(StbError):
            _raw_groupnorm(xp, gp, bp, op, b, hw, C, G)
            pytest.fail(f"accepted: {what}")
    _raw_groupnorm(p(x, 8), p(gm, 8), p(bt), p(out, 8), B, HW, C, G)      # 16-byte offsets pass
    torch.cuda.synchronize()


def test_groupnorm_wrapper_checks_out():
    x = _bf(2, 4, 6, 64, seed=1)
    gm, bt = _bf(64, seed=2), _bf(64, seed=3)
    with pytest.raises(ValueError):
        ops.groupnorm_nhwc(x, gm, bt, 32, out=torch.empty(2, 4, 7, 64, device="cuda", dtype=torch.bfloat16)[:, :, :6])
    with pytest.raises(ValueError):
        ops.groupnorm_nhwc(x, gm, bt, 32, out=torch.empty(2, 24, 64, device="cuda", dtype=torch.bfloat16))
    with pytest.raises(TypeError):
        ops.groupnorm_nhwc(x, gm, bt, 32, out=torch.empty(2, 4, 6, 64, device="cuda", dtype=torch.float32))
    out = torch.empty_like(x)
    assert ops.groupnorm_nhwc(x, gm, bt, 32, out=out) is out
    torch.cuda.synchronize()


def test_softmax_rows_rejects_non_positive_scale_and_empty_rows():
    s = _bf(4, 64, seed=1)
    for scale in (0.0, -0.125, float("nan")):
        with pytest.raises(StbError):
            ops.softmax_rows_(s, scale)
    with pytest.raises(StbError):
        _lib.check(_lib.lib().stb_softmax_rows(s.data_ptr(), 64, 0, 64, 0.125, torch.cuda.current_stream().cuda_stream))
    before = s.clone()
    torch.cuda.synchronize()
    assert torch.equal(s, before)                                          # nothing was launched
    ops.softmax_rows_(s, 0.125)
    torch.cuda.synchronize()


def test_gaussian_sample_rejects_null_pointers_and_empty_sizes():
    m, eps = _bf(2, 3, 5, 8, seed=1), _bf(2, 4, 3, 5, seed=2)
    out = torch.empty(2, 4, 3, 5, device="cuda", dtype=torch.bfloat16)
    st = torch.cuda.current_stream().cuda_stream
    fn = _lib.lib().stb_gaussian_sample_scale
    for what, args in {"null moments": (None, eps.data_ptr(), out.data_ptr(), 2, 4, 15),
                       "null eps": (m.data_ptr(), None, out.data_ptr(), 2, 4, 15),
                       "null out": (m.data_ptr(), eps.data_ptr(), None, 2, 4, 15),
                       "B = 0": (m.data_ptr(), eps.data_ptr(), out.data_ptr(), 0, 4, 15),
                       "L = 0": (m.data_ptr(), eps.data_ptr(), out.data_ptr(), 2, 0, 15),
                       "hw = 0": (m.data_ptr(), eps.data_ptr(), out.data_ptr(), 2, 4, 0)}.items():
        with pytest.raises(StbError):
            _lib.check(fn(*args, 0.0, 1.0, 0, st))
            pytest.fail(f"accepted: {what}")
    with pytest.raises(TypeError):
        ops.gaussian_sample_scale(m.float(), eps, None, 1.0)
    ops.gaussian_sample_scale(m, eps, 0.1159, 0.3611)
    torch.cuda.synchronize()


def test_lokr_wrappers_reject_transposed_views():
    a, b, c, d = 4, 16, 2, 32
    W, w1, w2 = _bf(a * b, c * d, seed=1), _bf(a, c, seed=2), _bf(b, d, seed=3)
    Wt = _bf(c * d, a * b, seed=4).t()                    # [a b, c d] with unit row stride: a transposed view
    out = torch.empty(a * b, c * d, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.lokr_rebuild(Wt, w1, w2, 0.5, out)
    with pytest.raises(ValueError):
        ops.lokr_rebuild(W, w1, w2, 0.5, torch.empty(c * d, a * b, device="cuda", dtype=torch.bfloat16).t())
    with pytest.raises(ValueError):
        ops.lokr_rebuild(W, w1, w2, 0.5, out, torch.empty(a * b, c * d, device="cuda", dtype=torch.bfloat16).t())
    with pytest.raises(ValueError):
        ops.lokr_factor_grads(Wt, w1, w2, 0.5)
    ops.lokr_rebuild(W, w1, w2, 0.5, out)
    ops.lokr_factor_grads(W, w1, w2, 0.5)
    torch.cuda.synchronize()


def test_dropout_wrappers_reject_transposed_views():
    B, S, K = 2, 16, 64
    xt = _bf(B, K, S, seed=1).transpose(1, 2)             # [B, S, K] with a unit stride on S
    with pytest.raises(ValueError):
        ops.dropout_expand(xt, 2, 0.1, 1, 0)
    d = _bf(2, B, S, K, seed=2)
    with pytest.raises(ValueError):
        ops.dropout_accum_(torch.zeros(B, K, S, device="cuda", dtype=torch.bfloat16).transpose(1, 2), d, 0.1, 1, 0)
    ops.dropout_accum_(torch.zeros(B, S, K, device="cuda", dtype=torch.bfloat16), d, 0.1, 1, 0)
    torch.cuda.synchronize()
