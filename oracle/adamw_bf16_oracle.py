"""CPU oracle for the reference's default optimizer `adamw_bf16` — TEST INFRASTRUCTURE ONLY.

Restates reference simpletuner/helpers/training/optimizers/adamw_bfloat16/__init__.py:112-180 (`_make_step`) and
.../stochastic/__init__.py:48-121 (`copy_stochastic_`, `add_stochastic_`, `addcdiv_stochastic_`) with the random
16-bit integers of the four stochastic roundings passed in explicitly, so that results are reproducible bit for bit.
Pinned against the reference's own functions executed verbatim (oracle/make_golden_optim.py ->
tests/golden/adamw_bf16_golden.pt, tests/test_adamw_bf16.py).

Quirk kept on purpose (Q-opt): `add_stochastic_(exp_avg, grad, alpha=1 - beta1)` computes `grad + alpha * exp_avg`
(it adds alpha x INPUT to OTHER), so the first moment is `grad + (1 - beta1) * beta1 * exp_avg_old`, not Adam's EMA;
there is no first-moment bias correction either.  The optimizer state also carries `shift`, the running remainder of
the bf16 parameter (Kahan-style), and weight decay is applied to `shift` only when the accumulated decay passes 5e-3.
"""
from __future__ import annotations

from typing import Sequence

import torch

Tensor = torch.Tensor


def copy_stochastic(source_f32: Tensor, rnd_i32: Tensor) -> Tensor:
    """fp32 -> bf16 by adding a random 16-bit integer to the bit pattern and truncating (stochastic/__init__.py:48-72)."""
    r = rnd_i32.clone()
    r.add_(source_f32.view(dtype=torch.int32))
    r.bitwise_and_(-65536)
    return r.view(dtype=torch.float32).to(torch.bfloat16)


def adamw_bf16_step(p: Tensor, grad: Tensor, shift: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, *, beta1: float,
                    beta2: float, step: float, lr: float, eps: float, decay_this_iteration: float, rnd: Sequence[Tensor],
                    scalar_semantics: str = "cpu"):
    """One `_make_step` (in place on the bf16 tensors).  rnd: four int32 tensors in [0, 65536), in the order the reference
    draws them: exp_avg, shift (addcdiv), p, shift (truncation error).

    scalar_semantics: PyTorch itself evaluates three of these ops differently on CPU and CUDA —
      * bf16 `add_(scalar / alpha)`: the CPU kernels cast the Python scalar to bf16 first, the CUDA kernels keep it in fp32
        (`sqrt().add_(eps)`, `shift.add_(p, alpha=-decay)`);
      * `addcdiv_`: CPU computes `self + (value * t1) / t2`, CUDA `self + value * (t1 / t2)` (fused multiply-add);
      * `addcmul_`: CPU computes `self + (value * t1) * t2`, CUDA `self + value * (t1 * t2)`.
    "cpu" follows the former (bit-exact against the reference executed here, tests/golden/adamw_bf16_golden.pt),
    "cuda" the latter — what the reference does on a GPU and what `stb_adamw_bf16_multi` implements."""
    cuda = scalar_semantics == "cuda"
    exp_avg.mul_(beta1)
    res = grad.to(torch.float32)
    res.add_(exp_avg, alpha=1 - beta1)                       # other + alpha * input  (quirk Q-opt)
    exp_avg.copy_(copy_stochastic(res, rnd[0]))
    if cuda:   # CUDA addcmul is a + value * (b * c): g * g rounded alone, then one FMA (fp64 sum rounded to fp32)
        v1, gf = exp_avg_sq.mul_(beta2).double(), grad.float()
        value = float(torch.tensor(1 - beta2, dtype=torch.float32))
        exp_avg_sq.copy_((v1 + value * (gf * gf).double()).float().to(torch.bfloat16))
    else:
        exp_avg_sq.mul_(beta2).addcmul_(grad, grad.conj(), value=1 - beta2)
    denom_correction = (1 - beta2 ** step) ** 0.5
    res = shift.to(torch.float32)
    if cuda:
        denom = exp_avg_sq.sqrt().float().add_(eps).to(torch.bfloat16)
        res.add_(exp_avg.float() / denom.float(), alpha=-lr * denom_correction)
    else:
        res.addcdiv_(exp_avg, exp_avg_sq.sqrt().add_(eps, alpha=1), value=-lr * denom_correction)
    shift.copy_(copy_stochastic(res, rnd[1]))
    buffer = p.clone()
    res = shift.to(torch.float32)
    res.add_(p, alpha=1.0)
    p.copy_(copy_stochastic(res, rnd[2]))
    res = buffer.sub_(p).to(torch.float32)
    res.add_(shift, alpha=1.0)
    shift.copy_(copy_stochastic(res, rnd[3]))
    if decay_this_iteration > 0:
        if cuda:
            shift.copy_(shift.float().add_(p.float(), alpha=-decay_this_iteration).to(torch.bfloat16))
        else:
            shift.add_(p, alpha=-decay_this_iteration)
    return p, shift, exp_avg, exp_avg_sq


def decay_schedule(accumulated_decay: float, weight_decay: float, lr: float, threshold: float = 5e-3):
    """__init__.py:96-99: returns (decay_this_iteration, new accumulated_decay)."""
    accumulated_decay += weight_decay * lr
    decay_this_iteration = (accumulated_decay > threshold) * accumulated_decay
    return decay_this_iteration, accumulated_decay - decay_this_iteration
