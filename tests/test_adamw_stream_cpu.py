"""CPU: statistics of the AdamW-bf16 stochastic-rounding integers, replayed in numpy by tests/kernel_checks.py
(`adamw_rnd_np`, which the adamw_* kernel checks hold to the kernel bit for bit): every 16-bit draw is uniform, the draws
of one element are independent of each other and of the same element in the next tensor, step, `only=` chunk and param
group, the rounding they drive is unbiased, and the counter's high 32 bits change the stream."""
import numpy as np
import pytest
import torch
from scipy import stats

from oracle import adamw_bf16_oracle as A
from tests.kernel_checks import adamw_rnd_np, adamw_seed

N = 1 << 22
P_CHI2 = 1e-6       # significance of each chi-square test
P_MATCH = 1e-9      # two-sided failure probability of each match count under independence
SEED = 1234


def _draws(seed64, t=0, n=N, first=0):
    return adamw_rnd_np(seed64, t, n, first)


def _matches_are_chance(a, b):
    """Equal 16-bit draws at the same index: Poisson(n / 65536) under independence, accepted at P_MATCH two-sided."""
    obs, lam = int((a == b).sum()), a.size / 65536.0
    lo, hi = stats.poisson.cdf(obs, lam), stats.poisson.sf(obs - 1, lam)
    return min(lo, hi) > P_MATCH / 2, (obs, lam)


@pytest.mark.parametrize("draw", range(4))
def test_every_draw_is_uniform_in_both_bytes(draw):
    r = _draws(adamw_seed(SEED, 1))[draw]
    assert r.min() >= 0 and r.max() <= 0xFFFF
    for name, byte in (("high", r >> 8), ("low", r & 0xFF)):
        counts = np.bincount(byte, minlength=256)
        stat = float(((counts - N / 256) ** 2).sum() / (N / 256))
        assert stats.chi2.sf(stat, 255) > P_CHI2, (draw, name, stat)


@pytest.mark.parametrize("a,b", [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)])
def test_draws_of_one_element_are_independent(a, b):
    r = _draws(adamw_seed(SEED, 1))
    ok, info = _matches_are_chance(r[a], r[b])
    assert ok, info


@pytest.mark.parametrize("kind", ["tensor", "step", "salt"])
def test_neighbouring_tensors_steps_and_chunks_draw_independent_streams(kind):
    base = _draws(adamw_seed(SEED, 7), t=3)
    other = {"tensor": lambda: _draws(adamw_seed(SEED, 7), t=4), "step": lambda: _draws(adamw_seed(SEED, 8), t=3),
             "salt": lambda: _draws(adamw_seed(SEED, 7, salt=1), t=3)}[kind]()
    for d in range(4):
        ok, info = _matches_are_chance(base[d], other[d])
        assert ok, (kind, d, info)


def test_param_groups_draw_independent_streams():
    """Tensor t of param group 0 and tensor t of group 1 are launched with the same index t; the group ordinal in the
    production launch seed must separate them, and group 0 must keep the single-group seed."""
    from simpletuner_b200.training.optim import launch_seed
    g0, g1 = _draws(launch_seed(SEED, 5, 0, 0), t=2), _draws(launch_seed(SEED, 5, 0, 1), t=2)
    for d in range(4):
        ok, info = _matches_are_chance(g0[d], g1[d])
        assert ok, (d, info)
    for seed, step, salt, group in ((SEED, 1, 0, 0), (0, 10 ** 6, 2, 1), (2 ** 31 - 2, 3, 1, 3), (7, 0, 0, 2)):
        assert launch_seed(seed, step, salt, group) == adamw_seed(seed, step, salt, group)
        if group == 0:
            assert launch_seed(seed, step, salt) == (seed * 0x9E3779B1 + step * 0x85EBCA77 + salt * 0xC2B2AE3D27D4EB4F) % 2 ** 64


@pytest.mark.parametrize("draw", range(4))
@pytest.mark.parametrize("frac", [1 / 8, 1 / 2, 7 / 8])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_stochastic_rounding_with_the_stream_is_unbiased(draw, frac, sign):
    """copy_stochastic of x = +-(1 + frac 2^-7), frac of a bf16 ulp above 1: the mean of the bf16 results is within
    6 sigma of x, sigma = 2^-7 sqrt(frac (1 - frac) / n)."""
    x = sign * (1.0 + frac * 2.0 ** -7)
    r = torch.from_numpy(_draws(adamw_seed(SEED, 2), t=1)[draw].copy())
    y = A.copy_stochastic(torch.full((N,), x), r).double()
    assert set(y.unique().tolist()) == {sign * 1.0, sign * (1.0 + 2.0 ** -7)}
    sigma = 2.0 ** -7 * (frac * (1 - frac) / N) ** 0.5
    assert abs(float(y.mean()) - x) <= 6 * sigma, (float(y.mean()) - x, sigma)


def test_counter_high_word_changes_the_stream():
    """Elements 2^32 + i and i of one tensor (a term of the counter only tensors of 2^32 elements or more reach)."""
    n = 1 << 20
    s = adamw_seed(SEED, 1)
    lo, hi, hi2 = _draws(s, n=n), _draws(s, n=n, first=1 << 32), _draws(s, n=n, first=1 << 33)
    for a, b in ((lo, hi), (hi, hi2), (lo, hi2)):
        for d in range(4):
            ok, info = _matches_are_chance(a[d], b[d])
            assert ok, (d, info)
    assert np.array_equal(_draws(s, n=16, first=(1 << 32) + 5), hi[:, 5:21])
