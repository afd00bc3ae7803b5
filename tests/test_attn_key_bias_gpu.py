"""GPU: the per-key logit bias of the attention forward and backward (Flux masked training).  The numerical checks against
the fp64 reference are `attn_*_kb_*` in tests/kernel_checks.py; this file holds the invariants that hold bit for bit
between instantiations, the refused forms, and the entry points above the kernels."""
import math

import pytest
import torch
import torch.nn.functional as F

from simpletuner_b200 import ops
from tests.kernel_checks import _attn_ref, _key_bias, attn_compare

pytestmark = pytest.mark.gpu


def _rand(*shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g).bfloat16()


def _fwd_bwd(q, k, v, d_o, key_bias=None):
    o, lse = ops.attn_fwd(q, k, v, key_bias=key_bias)
    return (o, lse, *ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=key_bias))


def test_shared_row_matches_per_sample_rows_bit_for_bit():
    B, H, S, HD = 3, 2, 300, 128
    q, k, v, d_o = (_rand(B, S, H, HD, seed=i) for i in range(4))
    row = _key_bias("01", 1, S, seed=5)
    outs = [_fwd_bwd(q, k, v, d_o, bias) for bias in (row, row.expand(B, S), row.repeat(B, 1))]
    torch.cuda.synchronize()
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)


@pytest.mark.parametrize("HD", [64, 128])
@pytest.mark.parametrize("Sq,Sk", [(333, 333), (129, 191), (7, 65)])
def test_zero_key_bias_is_bit_identical_to_no_bias(HD, Sq, Sk):
    """The forward adds fmaf(0, 1 / scale, s) = s and the backward subtracts the LSE from a zero bias (0 - x = -x): every
    output of the key-bias instantiations equals the unbiased kernels' bit for bit, tail tiles included."""
    B, H = 2, 2
    q, k, v, d_o = _rand(B, Sq, H, HD, seed=1), _rand(B, Sk, H, HD, seed=2), _rand(B, Sk, H, HD, seed=3), _rand(B, Sq, H, HD, seed=4)
    zeros = torch.zeros(B, Sk, device="cuda", dtype=torch.bfloat16)
    plain, biased = _fwd_bwd(q, k, v, d_o), _fwd_bwd(q, k, v, d_o, zeros)
    torch.cuda.synchronize()
    for nm, a, b in zip(("o", "lse", "dq", "dk", "dv"), plain, biased):
        assert torch.equal(a, b), nm


@pytest.mark.parametrize("HD", [64, 128])
@pytest.mark.parametrize("B", [1, 3])
def test_key_row_is_bit_identical_to_the_materialized_general_bias(HD, B):
    """One key row shared by the batch and the same row written out as a contiguous [1, Sq, Sk] general bias give the same
    forward bits: both add fmaf(float(bf16), 1 / scale, s).  The general bias must be materialized: an expanded view has a
    zero query stride and is routed to the key-row kernel."""
    H, Sq, Sk = 2, 200, 333
    q, k, v = _rand(B, Sq, H, HD, seed=1), _rand(B, Sk, H, HD, seed=2), _rand(B, Sk, H, HD, seed=3)
    row = _key_bias("inf_straddle", 1, Sk, seed=4)
    general = row[:, None, :].expand(1, Sq, Sk).contiguous()
    o_key, lse_key = ops.attn_fwd(q, k, v, key_bias=row)
    o_gen, lse_gen = ops.attn_fwd(q, k, v, bias=general)
    torch.cuda.synchronize()
    assert torch.equal(o_key, o_gen) and torch.equal(lse_key, lse_gen)


def test_backward_is_deterministic():
    B, H, S, HD = 2, 4, 700, 128
    q, k, v, d_o = (_rand(B, S, H, HD, seed=i) for i in range(4))
    bias = _key_bias("01", B, S, seed=3)
    o, lse, dq, dk, dv = _fwd_bwd(q, k, v, d_o, bias)
    dq2, dk2, dv2 = ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=bias)
    torch.cuda.synchronize()
    assert torch.equal(dq, dq2) and torch.equal(dk, dk2) and torch.equal(dv, dv2)


def test_all_ones_bias_equals_no_bias_in_the_backward_exponent():
    """A constant bias shifts every logit of a row equally: the softmax and its gradients are those of no bias."""
    B, H, S, HD = 2, 2, 200, 64
    q, k, v, d_o = (_rand(B, S, H, HD, seed=10 + i) for i in range(4))
    ones = torch.ones(B, S, device="cuda", dtype=torch.bfloat16)
    o1, l1, *g1 = _fwd_bwd(q, k, v, d_o, ones)
    o0, l0, *g0 = _fwd_bwd(q, k, v, d_o)
    torch.cuda.synchronize()
    assert float((o1.float() - o0.float()).abs().max()) <= 1e-2 and torch.allclose(l1, l0 + 1.0, atol=1e-4)
    ref = _attn_ref(q, k, v, HD ** -0.5, d_o=d_o, o=o1)
    r = attn_compare("all_ones", dict(zip(("dq", "dk", "dv"), g1)), ref)
    assert r["ok"], r


def test_text_encoder_bias_still_works_with_the_batch_stride():
    """The [H, Sq, Sk] bias (T5 relative position bias / CLIP causal mask) shared by the batch: bias_b = 0."""
    B, H, S, HD = 2, 4, 77, 64
    q, k, v = (_rand(B, S, H, HD, seed=20 + i) for i in range(3))
    causal = torch.full((S, S), -math.inf, device="cuda").triu(1)
    bias = (_rand(H, S, S, seed=30).float() + causal).bfloat16()
    o, lse = ops.attn_fwd(q, k, v, bias=bias)
    torch.cuda.synchronize()
    r = attn_compare("text_encoder_bias", {"o": o, "lse": lse}, _attn_ref(q, k, v, HD ** -0.5, bias=bias))
    assert r["ok"], r


def test_unsupported_backward_bias_form_is_refused(monkeypatch):
    """The backward takes a per-key bias only: a batch stride between 0 and Sk is refused by the library."""
    from simpletuner_b200._lib import StbError
    B, H, S, HD = 2, 2, 64, 64
    q, k, v, d_o = (_rand(B, S, H, HD, seed=40 + i) for i in range(4))
    bias = torch.ones(B, S, device="cuda", dtype=torch.bfloat16)
    o, lse = ops.attn_fwd(q, k, v, key_bias=bias)
    monkeypatch.setattr(ops, "_key_bias_stride", lambda kb, B, Sk: 1)
    with pytest.raises(StbError, match="per-key"):
        ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=bias)


def test_sdpa_override_runs_per_key_masks():
    from simpletuner_b200.shim import attention_backend as AB

    stock = F.scaled_dot_product_attention
    try:
        AB.install_sdpa_override()
        B, H, S, HD = 2, 4, 300, 128
        q, k, v = (_rand(B, H, S, HD, seed=50 + i).requires_grad_(True) for i in range(3))
        mask = ((torch.arange(S, device="cuda")[None] < torch.tensor([[120], [250]], device="cuda"))
                | (torch.arange(S, device="cuda")[None] >= 200)).to(torch.bfloat16)[:, None, None, :]
        ops.reset_launch_count()
        out = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        assert ops.launch_count() >= 1
        g = _rand(B, H, S, HD, seed=60)
        out.backward(g)
        torch.cuda.synchronize()
        # the override takes [B, H, S, HD]; the reference works in [B, S, H, HD]
        t = lambda x: x.detach().transpose(1, 2)
        ref = _attn_ref(t(q), t(k), t(v), HD ** -0.5, key_bias=mask[:, 0, 0, :], d_o=t(g), o=t(out))
        r = attn_compare("sdpa_override", {"o": t(out), "dq": t(q.grad), "dk": t(k.grad), "dv": t(v.grad)}, ref)
        assert r["ok"], r
    finally:
        AB.restore_sdpa()
    assert F.scaled_dot_product_attention is stock
