"""GPU (-m gpu): the Chroma LoRA step (prepare_batch -> model_predict -> loss -> backward) against the fp32 oracle
(tests/chroma_oracle.py) with the tolerances of tests/flux_parity.py, the approximator against its fp32 restatement, and
bit-exact properties of the step."""
import pytest
import torch

from tests import chroma_oracle as CO
from tests import flux_parity as FP

pytestmark = pytest.mark.gpu
HD64 = CO.ChromaConfig(attention_head_dim=64, num_attention_heads=2, axes_dims_rope=(8, 28, 28))


def _ok(res):
    FP.record("chroma", res)
    assert res["loss_rel_err"] <= FP.LOSS_RTOL, res
    assert res["pred_cos"] >= FP.PRED_COS, res
    assert res["grad_cos_min"] >= FP.GRAD_COS, res


def _approx_replay(P, x, layers, eps, weight_first):
    """The approximator's bf16 chain in torch on the GPU: the library's RMSNorm order (round, then weight) or torch's
    (weight, then one rounding)."""
    a = "distilled_guidance_layer."
    W = {k[len(a):]: v.bfloat16().cuda() for k, v in P.items() if k.startswith(a)}
    lin = lambda t, n: torch.nn.functional.linear(t, W[n + ".weight"], W[n + ".bias"])
    h = lin(x, "in_proj")
    for i in range(layers):
        r = h.float() * torch.rsqrt(h.float().pow(2).mean(-1, keepdim=True) + eps)
        w = W[f"norms.{i}.weight"]
        n = (r * w.float()).bfloat16() if weight_first else r.bfloat16() * w
        h = h + lin(torch.nn.functional.silu(lin(n, f"layers.{i}.linear_1")), f"layers.{i}.linear_2")
    return lin(h, "out_proj").float()


def test_approximator_per_element():
    """Against a bf16 torch replay per element (the two differ only in GEMM summation order), and against fp32.  The
    in_proj bias is 0 and one row is scaled by 1e-3, so that its RMSNorm is decided by the epsilon: a wrong epsilon or
    a missing normalisation is far outside the bound."""
    from simpletuner_b200.chroma.transformer import ChromaTransformer2DModel, chroma_input_vec, chroma_mod_proj
    cfg = CO.ChromaConfig(approximator_hidden_dim=512, approximator_layers=5)
    P = {k: v.bfloat16().float() for k, v in CO.init_params(cfg, 3).items()}
    P["distilled_guidance_layer.in_proj.bias"].zero_()
    m = ChromaTransformer2DModel(**cfg.kwargs())
    m.load_state_dict({k: v.bfloat16() for k, v in P.items()})
    m.cuda()
    t = torch.tensor([0.0, 0.37, 0.999], dtype=torch.bfloat16) * 1000
    x = chroma_input_vec(t, chroma_mod_proj(cfg.mod_rows, 16)).clone()
    x[1, 7] *= 1e-3
    x = x.cuda()
    got = m.distilled_guidance_layer(x).float()
    eps = torch.finfo(torch.float32).eps
    ref = _approx_replay(P, x, cfg.approximator_layers, eps, weight_first=False)
    row_rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
    tol = 2 ** -6 * ref.abs() + 2 ** -8 * row_rms
    assert bool(((got - ref).abs() <= tol).all()), float(((got - ref).abs() / tol).max())
    # a 2^-7 epsilon is far outside the bound
    wrong = _approx_replay(P, x, cfg.approximator_layers, 2 ** -7, weight_first=False)
    assert not bool(((got - wrong).abs() <= tol).all())
    # torch's rounding order (the reference's: RMSNorm weight applied before its one rounding) moves the normalised
    # input of linear_1 by up to one bf16 step; after five residual layers that stays within 8x the bound above (6.0x
    # measured on an H100 80GB HBM3)
    ref_torch = _approx_replay(P, x, cfg.approximator_layers, eps, weight_first=True)
    ratio = float(((got - ref_torch).abs() / tol).max())
    print(f"approximator vs torch rounding order: max |diff| / tol = {ratio:.2f}")
    assert ratio <= 8.0
    ref32 = CO.approximator(P, cfg, x.float().cpu())
    assert float((got.cpu() - ref32).norm() / ref32.norm()) < 2e-2


@pytest.mark.parametrize("targets", sorted(CO.CHROMA_LORA_TARGETS))
def test_step_parity_every_target_list(targets):
    _ok(CO.run_parity(B=2, lens=(24, 9), targets=targets))


@pytest.mark.parametrize("B,lens", [(1, (13,)), (2, (32, 5))])
def test_step_parity_hd64_non_square(B, lens):
    _ok(CO.run_parity(HD64, B=B, Hh=18, Ww=12, lens=lens, targets="all+ffs"))


def test_step_parity_lora_dropout_checkpointing_huber():
    _ok(CO.run_parity(B=2, lens=(20, 7), targets="all+ffs+embedder", dropout=0.1))
    _ok(CO.run_parity(B=2, lens=(20, 7), targets="all", checkpoint=True))
    _ok(CO.run_parity(B=1, lens=(11,), targets="all", loss_type="huber"))


def test_checkpointing_and_padding_values_are_bit_identical():
    cfg = CO.ChromaConfig()
    P = {k: v.bfloat16().float() for k, v in CO.init_params(cfg, 0).items()}
    tl = CO.CHROMA_LORA_TARGETS["all+ffs"]
    L = {k: v.bfloat16().float() for k, v in CO.init_lora(cfg, 16, tl, 1).items()}
    w = CO.build_cuda(cfg, P, L, 16, "all+ffs")
    mask = CO.ragged_mask(2, 32, (32, 6))
    batch = CO.make_batch(2, 16, 16, mask, cfg)
    _, out0, l0, g0 = CO.run_step(w, batch)
    _, out1, l1, g1 = CO.run_step(w, batch, checkpoint=True)
    assert torch.equal(l0, l1) and all(torch.equal(g0[k], g1[k]) for k in g0)
    b2 = dict(batch)
    noise = torch.randn(batch["prompt_embeds"].shape, generator=torch.Generator().manual_seed(9)).bfloat16()
    b2["prompt_embeds"] = torch.where(mask[:, :, None] != 0, batch["prompt_embeds"], noise)
    _, out2, l2, g2 = CO.run_step(w, b2)
    assert torch.equal(l0, l2) and all(torch.equal(g0[k], g2[k]) for k in g0)
    assert torch.equal(out0["model_prediction"], out2["model_prediction"])
