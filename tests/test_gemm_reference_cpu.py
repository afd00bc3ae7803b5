"""CPU: the reference model of the GEMM-family checks in tests/kernel_checks.py.

The exact-input mode replays the GEMM epilogue with fp32 torch ops on an exact accumulator; here that replay is held bit
for bit against the eager bf16 module chains the kernel comments cite, and the input generator against its bound."""
import math

import pytest
import torch

import tests.kernel_checks as KC
from simpletuner_b200 import ops

F = torch.nn.functional


@pytest.fixture(autouse=True)
def _on_cpu(monkeypatch):
    monkeypatch.setattr(KC, "DEV", "cpu")


def _linear_inputs(B=2, S=48, K=200, N=72, seed=0):
    x = KC._gen(B, S, K, seed=seed, exact="int")
    w = KC._gen(N, K, seed=seed + 1, exact="frac")
    b = KC._rand(N, seed=seed + 2)
    acc = (x.double() @ w.double().t()).float()          # exact: the kernel's fp32 accumulator
    return x, w, b, acc


def _eq(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_store_is_the_bf16_linear():
    x, w, b, acc = _linear_inputs()
    out, pre = KC.replay_epilogue(ops.EPI_STORE, acc, b)
    assert _eq(out, F.linear(x, w, b)) and _eq(pre, out)


def test_gate_res_is_the_eager_chain():
    # flux/transformer.py: res + gate * linear(x), every step a bf16 tensor
    x, w, b, acc = _linear_inputs(seed=3)
    gate, res = KC._rand(2, 72, seed=4), KC._rand(2, 48, 72, seed=5)
    out, _ = KC.replay_epilogue(ops.EPI_GATE_RES, acc, b, gate=gate, res=res)
    assert _eq(out, res + gate[:, None, :] * F.linear(x, w, b))


def test_gate_res_nan_to_num_is_torch_nan_to_num():
    x, w, b, acc = _linear_inputs(seed=6)
    gate, res = KC._rand(2, 72, seed=7), KC._rand(2, 48, 72, seed=8)
    big = torch.finfo(torch.bfloat16).max
    res[..., 0::8], res[..., 1::8], res[..., 2::8] = float("inf"), float("-inf"), float("nan")
    res[:, 0::2, 3::8], res[:, 1::2, 3::8] = big, -big
    gate[:, 3::8] = 2.0 ** 120
    y = F.linear(x, w, b)
    chain = torch.nan_to_num(res + gate[:, None, :] * y, posinf=65504, neginf=-65504)
    out, _ = KC.replay_epilogue(ops.EPI_GATE_RES, acc, b, gate=gate, res=res, nan_to_num=True)
    assert _eq(out, chain)
    # the bf16 maximum is pushed past by gate * y in both directions, and 65504 is 65536 in bf16
    assert bool((out[..., 3::8] == 65536).any()) and bool((out[..., 3::8] == -65536).any())
    assert not bool(torch.isfinite(res + gate[:, None, :] * y)[..., 3::8].all())
    passed, _ = KC.replay_epilogue(ops.EPI_GATE_RES, acc, b, gate=gate, res=res, nan_to_num=False)
    assert bool(torch.isnan(passed[..., 2::8]).all()) and bool((passed[..., 0::8] == float("inf")).all())


def test_mul_is_the_t5_gated_product():
    # T5 gated feed-forward: gelu(x wi_0) * (x wi_1), the second factor a bf16 linear output
    x, w, b, acc = _linear_inputs(seed=9)
    g = KC._rand(2, 48, 72, seed=10)
    out, _ = KC.replay_epilogue(ops.EPI_MUL, acc, b, aux=g)
    assert _eq(out, F.linear(x, w, b) * g)


def test_add_res_rounds_once():
    # acc + bias + res in fp32 and one rounding (gradient accumulation); a bf16 `res + linear(x)` rounds twice and lands
    # on the other neighbour for some elements
    x, w, b, acc = _linear_inputs(seed=11)
    res = KC._rand(2, 48, 72, seed=12)
    out, _ = KC.replay_epilogue(ops.EPI_ADD_RES, acc, b, res=res)
    once = (acc.double() + b.double() + res.double()).float().bfloat16()
    assert float((out.float() - once.float()).abs().max()) <= float(once.float().abs().max()) * 2 ** -7
    chain = res + F.linear(x, w, b)
    assert KC._neighbour("add_res", out, acc.double() + b.double() + res.double())["ok"]
    assert not _eq(out, chain)


def test_gelu_module_is_a_neighbour_of_fp64():
    # nn.Linear -> nn.GELU(approximate="tanh"): the activation of a bf16 pre-activation lies next to the fp64 value (or,
    # far below zero, within the fp32 formula's cancellation error), so the criterion of the checks admits the module
    pre = KC._rand(4, 64, 256, seed=13) * 3
    act = torch.nn.GELU(approximate="tanh")(pre)
    x = pre.double()
    assert KC._neighbour("gelu", act, KC.gelu64(x), KC._gelu_atol(x)[0])["ok"]
    assert not KC._neighbour("gelu", act, KC.gelu64(x))["ok"]          # the cancellation is real
    unrounded = KC.gelu64(x + x.abs() * 2 ** -8)                          # GELU of a pre-activation off by half an ulp
    assert not KC._neighbour("gelu", act, unrounded, KC._gelu_atol(x)[0])["ok"]


def test_neighbour_criterion():
    one = torch.tensor([1.0], dtype=torch.bfloat16)
    dn, up = KC._bf16_steps(one)
    assert float(dn) == 1 - 2 ** -8 and float(up) == 1 + 2 ** -7
    dn, up = KC._bf16_steps(-one)
    assert float(dn) == -(1 + 2 ** -7) and float(up) == -(1 - 2 ** -8)
    dn, up = KC._bf16_steps(torch.zeros(1, dtype=torch.bfloat16))
    assert float(dn) < 0 < float(up)
    ref = torch.tensor([1.0 + 2 ** -9], dtype=torch.float64)
    assert KC._neighbour("n", one, ref)["ok"]
    assert KC._neighbour("n", torch.tensor([1.0 + 2 ** -7], dtype=torch.bfloat16), ref)["ok"]
    assert not KC._neighbour("n", torch.tensor([1.0 + 2 ** -6], dtype=torch.bfloat16), ref)["ok"]
    assert not KC._neighbour("n", torch.tensor([float("nan")], dtype=torch.bfloat16), ref)["ok"]


def test_bits_compares_nan_positions_not_payloads():
    a = torch.tensor([1.0, float("nan"), 2.0], dtype=torch.bfloat16)
    b = a.clone()
    b.view(torch.int16)[1] = 0x7FC1
    assert KC._bits("x", a, b)["ok"]
    b[2] = 2.015625
    assert not KC._bits("x", a, b)["ok"]


# The largest contraction each exact-mode family registers: gemm 12288 + 9216 + 48 (Flux dgrad), skinny_tn 4 x 4608
# tokens, wgrad_full 4608 tokens, conv 9 x 512 channels.
LARGEST_K = {"gemm": 12288 + 9216 + 48, "skinny": 4 * 4608, "wgrad": 4608, "conv": 9 * 512}


@pytest.mark.parametrize("family", list(LARGEST_K))
def test_exact_inputs_respect_the_bound(family):
    K = LARGEST_K[family]
    a = KC._gen(64, K, seed=1, exact="int")
    w = KC._gen(64, K, seed=2, exact="frac")
    mag = a.double().abs() @ w.double().abs().t()
    assert KC.exact_bound_ok([a], [w], mag)
    # every partial sum, in any order, is bounded by K max|a| max|w|, whichever rows are drawn
    assert K * float(a.abs().max()) * float(w.abs().max()) < KC.EXACT_BOUND
    assert float(a.abs().max()) == 2 and float(w.abs().max()) == 6 / 16


def test_exact_bound_rejects():
    a = torch.full((1, 8), 2.0, dtype=torch.bfloat16)
    assert not KC.exact_bound_ok([a * 0.5 + 0.25], [a], a.double() @ a.double().t())
    assert not KC.exact_bound_ok([a], [a / 64], a.double() @ a.double().t())
    big = torch.full((1, 8), 2.0 ** 19, dtype=torch.float64)
    assert not KC.exact_bound_ok([a], [a], big)


def test_exact_accumulator_is_order_free():
    # a multiple of 2^-4 below 2^19 is exact in fp32: any summation order gives the fp64 value
    x, w, _, acc = _linear_inputs(K=3072, seed=14)
    prods = (x.float()[0, :4, None, :] * w.float()[None, :8, :])
    fwd = prods.sum(-1)
    rev = torch.zeros_like(fwd)
    for k in reversed(range(prods.shape[-1])):
        rev = rev + prods[..., k]
    assert torch.equal(fwd, acc[0, :4, :8]) and torch.equal(rev, acc[0, :4, :8])
    assert math.isfinite(float(acc.abs().max()))
