"""GPU: the per-key logit bias of the attention forward and backward (Flux masked training) against fp32 torch."""
import math

import pytest
import torch
import torch.nn.functional as F

from simpletuner_b200 import ops

pytestmark = pytest.mark.gpu


def _rand(*shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g).bfloat16()


def _masks(B, Sk, kind, seed=0):
    """bf16 [B, Sk]: a different ragged mask per sample."""
    g = torch.Generator().manual_seed(seed)
    bias = torch.ones(B, Sk)
    for b in range(B):
        n = int(torch.randint(0, Sk, (1,), generator=g)) if Sk > 1 else 0
        if kind == "01":
            bias[b, n:min(Sk, n + 1 + Sk // (b + 2))] = 0.0
        elif kind == "neg":
            bias[b, n:min(Sk, n + 1 + Sk // (b + 2))] = -10000.0
        elif kind == "inf":
            # the whole first 128-key tile and whole 64-key blocks; at least one finite key remains per row
            bias[b, :min(128, Sk - 1)] = -math.inf
            for k0 in range(192, Sk - 64, 128 * (b + 1)):
                bias[b, k0:k0 + 64] = -math.inf
    return bias.to("cuda", torch.bfloat16)


def _ref(q, k, v, d_o, bias, scale):
    """fp32 torch on the bf16 inputs; [B, S, H, D] layout."""
    qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale
    if bias is not None:
        s = s + bias.float()[:, None, None, :]
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), vf)
    o.backward(d_o.float())
    return o.detach(), qf.grad, kf.grad, vf.grad


def _cos(a, b):
    return float(F.cosine_similarity(a.flatten().float(), b.flatten().float(), dim=0))


def _run(B, H, Sq, Sk, HD, kind, seed=0):
    q, k, v = _rand(B, Sq, H, HD, seed=seed), _rand(B, Sk, H, HD, seed=seed + 1), _rand(B, Sk, H, HD, seed=seed + 2)
    d_o = _rand(B, Sq, H, HD, seed=seed + 3)
    bias = _masks(B, Sk, kind, seed)
    o, lse = ops.attn_fwd(q, k, v, key_bias=bias)
    dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=bias)
    torch.cuda.synchronize()
    ro, rdq, rdk, rdv = _ref(q, k, v, d_o, bias, HD ** -0.5)
    assert torch.isfinite(o.float()).all() and torch.isfinite(lse).all()
    assert _cos(o, ro) >= 0.9999 and float((o.float() - ro).abs().max()) <= 2e-2
    for got, ref in ((dq, rdq), (dk, rdk), (dv, rdv)):
        assert torch.isfinite(got.float()).all()
        if float(ref.abs().max()) > 0:
            assert _cos(got, ref) >= 0.999
    if kind == "inf":
        dead = torch.isinf(bias.float())[:, :, None, None].expand_as(dk)
        assert bool((dk[dead] == 0).all()) and bool((dv[dead] == 0).all())
    return q, k, v, d_o, bias, o, lse, dq, dk, dv


@pytest.mark.parametrize("HD", [64, 128])
@pytest.mark.parametrize("S", [1, 17, 64, 77, 128, 129])
@pytest.mark.parametrize("kind", ["01", "neg"])
def test_key_bias_self_attention(HD, S, kind):
    _run(B=1 + S % 3, H=2, Sq=S, Sk=S, HD=HD, kind=kind, seed=S)


@pytest.mark.parametrize("HD", [64, 128])
@pytest.mark.parametrize("Sq,Sk,kind", [(100, 300, "01"), (300, 77, "01"), (129, 520, "01"),
                                        (100, 300, "inf"), (129, 520, "inf")])   # "inf" needs a key past the first tile
def test_key_bias_cross_lengths(HD, Sq, Sk, kind):
    _run(B=3, H=3, Sq=Sq, Sk=Sk, HD=HD, kind=kind, seed=Sq + Sk)


@pytest.mark.parametrize("kind", ["01", "inf"])
def test_key_bias_flux_shape(kind):
    """Flux.1: 24 heads of 128, 512 text + 4096 image tokens."""
    _run(B=1, H=24, Sq=4608, Sk=4608, HD=128, kind=kind, seed=7)


def test_shared_row_matches_per_sample_rows_bit_for_bit():
    B, H, S, HD = 3, 2, 300, 128
    q, k, v, d_o = (_rand(B, S, H, HD, seed=i) for i in range(4))
    row = _masks(1, S, "01", seed=5)
    outs = []
    for bias in (row, row.expand(B, S), row.repeat(B, 1)):
        o, lse = ops.attn_fwd(q, k, v, key_bias=bias)
        outs.append((o, lse, *ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=bias)))
    torch.cuda.synchronize()
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)


def test_backward_is_deterministic():
    q, k, v, d_o, bias, o, lse, dq, dk, dv = _run(B=2, H=4, Sq=700, Sk=700, HD=128, kind="01", seed=3)
    dq2, dk2, dv2 = ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=bias)
    torch.cuda.synchronize()
    assert torch.equal(dq, dq2) and torch.equal(dk, dk2) and torch.equal(dv, dv2)


def test_all_ones_bias_equals_no_bias_in_the_backward_exponent():
    """A constant bias shifts every logit of a row equally: the softmax and its gradients are those of no bias."""
    B, H, S, HD = 2, 2, 200, 64
    q, k, v, d_o = (_rand(B, S, H, HD, seed=10 + i) for i in range(4))
    ones = torch.ones(B, S, device="cuda", dtype=torch.bfloat16)
    o1, l1 = ops.attn_fwd(q, k, v, key_bias=ones)
    o0, l0 = ops.attn_fwd(q, k, v)
    g1 = ops.attn_bwd(q, k, v, o1, d_o, l1, key_bias=ones)
    g0 = ops.attn_bwd(q, k, v, o0, d_o, l0)
    torch.cuda.synchronize()
    assert float((o1.float() - o0.float()).abs().max()) <= 1e-2 and torch.allclose(l1, l0 + 1.0, atol=1e-4)
    for a, b in zip(g1, g0):
        assert _cos(a, b) >= 0.9999


def test_fused_qk_prep_with_key_bias_equals_the_separate_pass():
    B, S, H, HD, s_split = 2, 333, 3, 128, 77
    D = H * HD
    qkv = _rand(B, S, 3 * D, seed=1)
    d_o = _rand(B, S, H, HD, seed=2)
    w = [(1.0 + 0.1 * _rand(HD, seed=sd).float()).bfloat16() for sd in (3, 4, 5, 6)]
    pos = torch.arange(S, device="cuda", dtype=torch.float32)[:, None] * torch.linspace(0.01, 1.0, HD // 2, device="cuda")
    cos = pos.cos().repeat_interleave(2, 1).contiguous()
    sin = pos.sin().repeat_interleave(2, 1).contiguous()
    bias = _masks(B, S, "01", seed=9)
    q, k = ops.qk_rmsnorm_rope_fwd(qkv, D, H, HD, *w, s_split, cos, sin, 1e-6)
    v = qkv[:, :, 2 * D:].unflatten(-1, (H, HD))
    o, lse = ops.attn_fwd(q, k, v, key_bias=bias)
    dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=bias)
    ref = torch.zeros_like(qkv)
    ops.qk_rmsnorm_rope_bwd(dq, dk, qkv, D, H, HD, *w, s_split, cos, sin, 1e-6, dsrc=ref)
    ref[:, :, 2 * D:] = dv.reshape(B, S, D)
    got = torch.zeros_like(qkv)
    ops.attn_bwd(q, k, v, o, d_o, lse, dq=got[:, :, 0:D].unflatten(-1, (H, HD)), dk=got[:, :, D:2 * D].unflatten(-1, (H, HD)),
                 dv=got[:, :, 2 * D:].unflatten(-1, (H, HD)), key_bias=bias,
                 qk_prep=dict(src=qkv, k_off=D, wq=w[0], wk=w[1], wq_added=w[2], wk_added=w[3], s_split=s_split, cos=cos,
                              sin=sin, eps=1e-6))
    torch.cuda.synchronize()
    assert torch.equal(got[:, :, 2 * D:], ref[:, :, 2 * D:])
    # the separate pass rounds dq / dk to bf16 before the norm backward, the fused one does not
    err = (got.float() - ref.float()).abs()
    assert float(err.max()) <= 2e-2 * float(ref.float().abs().max()) + 1e-3 and _cos(got, ref) >= 0.9999


def test_text_encoder_bias_still_works_with_the_batch_stride():
    """The [H, Sq, Sk] bias (T5 relative position bias / CLIP causal mask) shared by the batch: bias_b = 0."""
    B, H, S, HD = 2, 4, 77, 64
    q, k, v = (_rand(B, S, H, HD, seed=20 + i) for i in range(3))
    causal = torch.full((S, S), -math.inf, device="cuda").triu(1)
    bias = (_rand(H, S, S, seed=30).float() + causal).bfloat16()
    o, _ = ops.attn_fwd(q, k, v, bias=bias)
    s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * HD ** -0.5 + bias.float()[None]
    ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v.float())
    torch.cuda.synchronize()
    assert _cos(o, ref) >= 0.9999 and float((o.float() - ref).abs().max()) <= 2e-2


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
        grads = [t.grad.clone() for t in (q, k, v)]
        qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
        ref = F.scaled_dot_product_attention_sdpa(qf, kf, vf, attn_mask=mask.float())
        ref.backward(g.float())
        assert _cos(out, ref) >= 0.9999 and float((out.float() - ref).abs().max()) <= 2e-2
        for a, b in zip(grads, (qf.grad, kf.grad, vf.grad)):
            assert _cos(a, b) >= 0.999
    finally:
        AB.restore_sdpa()
    assert F.scaled_dot_product_attention is stock
