"""Generate tests/golden/adamw_bf16_golden.pt by running the reference's OWN `_make_step`
(helpers/training/optimizers/adamw_bfloat16/__init__.py:112-180) and stochastic helpers
(.../stochastic/__init__.py) verbatim, with `torch.randint_like` replaced by a recorded stream so that the same random
integers can be fed to the oracle / CUDA kernel.  TEST INFRASTRUCTURE ONLY.   python -m oracle.make_golden_optim
"""
from __future__ import annotations

from pathlib import Path

import torch

from . import ref_extract as rx

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "adamw_bf16_golden.pt"


class _TorchProxy:
    """`torch` for the lifted code: randint_like is recorded, everything else is the real module."""

    def __init__(self, gen):
        self._gen = gen
        self.draws = []

    def randint_like(self, source, dtype=None, low=0, high=None):
        r = torch.randint(low, high, source.shape, generator=self._gen, dtype=dtype)
        self.draws.append(r.clone())
        return r

    def __getattr__(self, name):
        return getattr(torch, name)


def main():
    assert rx.available(), "set SIMPLETUNER_SRC to a SimpleTuner checkout"
    gen = torch.Generator().manual_seed(2024)
    proxy = _TorchProxy(gen)
    st = rx.functions("helpers/training/optimizers/adamw_bfloat16/stochastic/__init__.py",
                      ["copy_stochastic_", "add_stochastic_", "addcdiv_stochastic_"],
                      extra_ns={"torch": proxy, "Tensor": torch.Tensor, "FloatTensor": torch.FloatTensor})
    mk = rx.functions("helpers/training/optimizers/adamw_bfloat16/__init__.py", ["_make_step"],
                      extra_ns={"torch": proxy, "add_stochastic_": st["add_stochastic_"],
                                "addcdiv_stochastic_": st["addcdiv_stochastic_"]})["_make_step"]
    shape = (257, 33)
    g = {"p0": (torch.randn(shape, generator=gen) * 0.05).bfloat16()}
    p = g["p0"].clone()
    shift, m, v = (torch.zeros_like(p) for _ in range(3))
    hp = dict(beta1=0.9, beta2=0.999, lr=1e-3, eps=1e-6)
    g["hp"] = hp
    decays = [0.0, 0.0, 7.5e-3, 0.0]          # a decay step in the middle (accumulated decay passed the 5e-3 threshold)
    g["decays"] = decays
    for k, dec in enumerate(decays):
        grad = (torch.randn(shape, generator=gen) * (0.02 if k != 1 else 3.0)).bfloat16()
        proxy.draws.clear()
        mk(grad, p, shift, m, v, beta1=hp["beta1"], beta2=hp["beta2"], step=float(k + 1), lr=hp["lr"], eps=hp["eps"],
           decay_this_iteration=dec, zero_grad=False)
        assert len(proxy.draws) == 4
        g[f"step{k}.grad"] = grad
        g[f"step{k}.rnd"] = torch.stack(proxy.draws).clone()
        g[f"step{k}.p"], g[f"step{k}.shift"], g[f"step{k}.exp_avg"], g[f"step{k}.exp_avg_sq"] = p.clone(), shift.clone(), m.clone(), v.clone()
    OUT.parent.mkdir(parents=True, exist_ok=True)
    torch.save(g, OUT)
    print(f"wrote {OUT}: {len(decays)} steps, p moved by {float((p.float() - g['p0'].float()).abs().max()):.4g} max")


if __name__ == "__main__":
    main()
