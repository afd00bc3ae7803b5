"""TEST INFRASTRUCTURE ONLY — CPU restatement of the LyCORIS LoKr adapter the reference attaches with
`create_lycoris(component, multiplier, linear_dim, linear_alpha, **lycoris_config)` (simpletuner/helpers/training/trainer.py:
3390-3505; default config in documentation/LYCORIS.md: algo = "lokr", linear_dim = 10000, linear_alpha = 1, factor 10 / 4,
targets = modules of class `Attention` and `FeedForward`).

PARITY UNPINNED: the algorithm lives in the third-party package `lycoris-lora` (setup.py:319 pins `>=3.4.0`), which is not
vendored in the reference and not installed in this image, so it is restated here from its published definition
(lycoris/modules/lokr.py, lycoris/functional/general.py::factorization, lycoris/functional/lokr.py::make_kron) and anchored on
the reference's own use of the module's attributes (`lokr_w1`, `lokr_w2`, `org_weight`: helpers/training/peft_init.py:34-38):

    shape = ((a, b), (c, d)) with (a, b) = factorization(out_features, factor), (c, d) = factorization(in_features, factor)
    lokr_w1 [a, c] (kaiming_uniform(a = sqrt 5));  lokr_w2 [b, d] (zeros) when linear_dim >= max(b, d) / 2 ("full matrix"),
    else lokr_w2_a [b, linear_dim] (kaiming) @ lokr_w2_b [linear_dim, d] (zeros)
    scale = alpha / linear_dim, with alpha := linear_dim (scale = 1) when both factors are full matrices
    delta W = kron(w1, w2) * scale;  forward (bypass_mode off): y = linear(x, org_weight + delta W * multiplier, bias)

Only tests/ and bench.py's baseline legs may import this file.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def factorization(dimension: int, factor: int = -1) -> Tuple[int, int]:
    """lycoris.functional.general.factorization: (m, n), m <= n, m * n = dimension; `factor` divides -> (factor, dim / factor)
    (sorted), otherwise the divisor pair with the smallest sum whose smaller part does not exceed `factor` (-1: unbounded)."""
    if factor > 0 and dimension % factor == 0:
        m, n = factor, dimension // factor
        return (n, m) if m > n else (m, n)
    if factor < 0:
        factor = dimension
    m, n = 1, dimension
    length = m + n
    while m < n:
        new_m = m + 1
        while dimension % new_m != 0:
            new_m += 1
        new_n = dimension // new_m
        if new_m + new_n > length or new_m > factor:
            break
        m, n = new_m, new_n
    return (n, m) if m > n else (m, n)


def lokr_shapes(out_features: int, in_features: int, factor: int) -> Tuple[Tuple[int, int], Tuple[int, int]]:
    return factorization(out_features, factor), factorization(in_features, factor)


def init_lokr_params(shapes: Dict[str, Tuple[int, int]], linear_dim: int, factor_of, seed: int = 1, w2_std: float = 0.0,
                     dtype=torch.float32) -> Dict[str, Tensor]:
    """{name + ".lokr_w1" / ".lokr_w2" (or ".lokr_w2_a" / ".lokr_w2_b")}.  `factor_of(name)` -> factor.  w2_std > 0 replaces the
    zero init of w2 (w2_b) by N(0, w2_std) so that every gradient path is exercised."""
    g = torch.Generator().manual_seed(seed)
    out = {}

    def kaiming(shape):
        bound = 1.0 / math.sqrt(shape[1])
        return ((torch.rand(shape, generator=g) * 2 - 1) * bound).to(dtype)

    for name, (n_out, k_in) in shapes.items():
        (a, b), (c, d) = lokr_shapes(n_out, k_in, factor_of(name))
        out[name + ".lokr_w1"] = kaiming((a, c))
        if linear_dim >= max(b, d) / 2:
            out[name + ".lokr_w2"] = (w2_std * torch.randn((b, d), generator=g)).to(dtype)
        else:
            out[name + ".lokr_w2_a"] = kaiming((b, linear_dim))
            out[name + ".lokr_w2_b"] = (w2_std * torch.randn((linear_dim, d), generator=g)).to(dtype)
    return out


def lokr_scale(params: Dict[str, Tensor], name: str, linear_dim: int, linear_alpha: float) -> float:
    full = (name + ".lokr_w2") in params
    alpha = linear_dim if full else linear_alpha      # both factors full matrices: alpha is overridden, scale = 1
    return float(alpha) / float(linear_dim)


def lokr_delta(params: Dict[str, Tensor], name: str, linear_dim: int, linear_alpha: float) -> Optional[Tensor]:
    if (name + ".lokr_w1") not in params:
        return None
    w1 = params[name + ".lokr_w1"]
    w2 = params[name + ".lokr_w2"] if (name + ".lokr_w2") in params else params[name + ".lokr_w2_a"] @ params[name + ".lokr_w2_b"]
    return torch.kron(w1, w2) * lokr_scale(params, name, linear_dim, linear_alpha)


def lokr_linear(x: Tensor, weight: Tensor, bias: Optional[Tensor], params: Dict[str, Tensor], name: str, linear_dim: int,
                linear_alpha: float, multiplier: float = 1.0) -> Tensor:
    delta = lokr_delta(params, name, linear_dim, linear_alpha)
    w = weight if delta is None else weight + delta.to(weight.dtype) * multiplier
    return F.linear(x, w, bias)
