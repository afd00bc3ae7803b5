"""`adamw_bf16` — the reference's default optimizer — on libstb200 (SURVEY.md §8f rank 1).

Mirror of reference simpletuner/helpers/training/optimizers/adamw_bfloat16/__init__.py:21-110 (class AdamWBF16): same
constructor arguments, per-parameter state (`step`, `exp_avg`, `exp_avg_sq`, `shift`, `accumulated_decay`), delayed weight
decay (`decay_threshold = 5e-3`, random starting phase per tensor) and `step(zero_grad=False)` signature.  The reference
runs ~25 eager kernels per parameter tensor per step (13k launches for the 532 Flux LoRA matrices); here the whole step is
ONE `stb_adamw_bf16_multi` launch over a pointer table.  Arithmetic follows the reference's CUDA path rounding for
rounding (oracle/adamw_bf16_oracle.py, scalar_semantics="cuda"); the stochastic-rounding integers come from a
counter-based generator keyed by (seed, step, chunk salt, param group, tensor, element) instead of `torch.randint_like` per call, i.e. the same
distribution but not the same Philox stream.  bf16 CUDA parameters only; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Tuple

import torch
from torch.optim.optimizer import Optimizer

from .. import _lib
from ..ops import _stream, check


def launch_seed(seed: int, step: int, salt: int = 0, group: int = 0) -> int:
    """The 64-bit seed of one optimizer launch.  The kernel keys tensor t by its index within the launch, so every launch
    of one step (each `only=` chunk, each param group) needs its own seed: `salt` numbers the chunks and `group` is the
    param group's ordinal, whose term is zero for group 0 (a single-group run keeps its rounding stream)."""
    return (seed * 0x9E3779B1 + step * 0x85EBCA77 + salt * 0xC2B2AE3D27D4EB4F + group * 0xD6E8FEB86659FD93) & 0xFFFFFFFFFFFFFFFF


def build_block_map(sizes: List[int], chunk: int) -> Tuple[List[int], List[int]]:
    """block -> (tensor index, first element): every tensor is cut into `chunk`-element pieces."""
    blk_tensor, blk_off = [], []
    for t, n in enumerate(sizes):
        for off in range(0, n, chunk):
            blk_tensor.append(t)
            blk_off.append(off)
    return blk_tensor, blk_off


class AdamWBF16(Optimizer):
    decay_threshold = 5e-3
    _RING = 4   # pinned staging slots for the per-step pointer / decay tables

    def __init__(self, params, *, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, seed: Optional[int] = None):
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        super().__init__(params, dict(betas=betas, eps=eps, weight_decay=weight_decay, lr=lr))
        self._seed = int(seed) if seed is not None else int(torch.randint(0, 2 ** 31 - 1, (1,)).item())
        self._plans: Dict[Tuple[int, ...], dict] = {}

    # ------------------------------------------------------------------------------------------
    def _plan(self, ps: List[torch.Tensor]) -> dict:
        key = tuple(id(p) for p in ps)
        pl = self._plans.get(key)
        if pl is None:
            dev = ps[0].device
            sizes = [p.numel() for p in ps]
            chunk = int(_lib.lib().stb_adamw_bf16_chunk())
            bt, bo = build_block_map(sizes, chunk)
            T = len(ps)
            pl = {
                "T": T, "num_blocks": len(bt),
                "sizes": torch.tensor(sizes, dtype=torch.int64, device=dev),
                "blk_tensor": torch.tensor(bt, dtype=torch.int32, device=dev),
                "blk_off": torch.tensor(bo, dtype=torch.int64, device=dev),
                # pinned staging ring: the async H2D copy reads host memory when it EXECUTES, and the host thread may be
                # several steps ahead of the GPU; a slot is rewritten only after the copy that last used it has completed
                "ptrs_host": [torch.empty((5, T), dtype=torch.int64).pin_memory() for _ in range(self._RING)],
                "decay_host": [torch.empty((T,), dtype=torch.float32).pin_memory() for _ in range(self._RING)],
                "ema_host": [torch.empty((T,), dtype=torch.int64).pin_memory() for _ in range(self._RING)],
                "ema": torch.empty((T,), dtype=torch.int64, device=dev),
                "copied": [None] * self._RING, "slot": 0,
                "ptrs": torch.empty((5, T), dtype=torch.int64, device=dev),
                "decay": torch.empty((T,), dtype=torch.float32, device=dev),
                "rnd_off": torch.tensor([0] + list(torch.tensor(sizes).cumsum(0)[:-1].tolist()), dtype=torch.int64, device=dev),
                "total": int(sum(sizes)),
            }
            self._plans[key] = pl
        return pl

    @torch.no_grad()
    def step(self, zero_grad: bool = False, _rnd: Optional[torch.Tensor] = None, *, grad_clamp: Optional[float] = None,
             ema=None, ema_global_step: Optional[int] = None, only=None, salt: int = 0):
        """Performs a single optimization step.  `_rnd` (tests only): int32 [4, total] random 16-bit integers, tensors
        concatenated in parameter order, replacing the internal generator.
        grad_clamp: fuse `clip_grad_value_(params, grad_clamp)` (the trainer's default clip, trainer.py:7188-7195) into the
        gradient read.  ema (+ ema_global_step): a training.ema.EMAModel whose update (trainer.py:7352-7357) runs inside the
        same kernel when it tracks exactly this group's tensors; otherwise `ema.step` runs after the launch.
        only (+ salt): update just these parameters (a chunk of a pipelined gradient exchange, training/dist.py); `salt`
        de-correlates the rounding streams of different chunks."""
        only_ids = None if only is None else {id(p) for p in only}
        if grad_clamp is not None and not grad_clamp > 0:
            grad_clamp = None
        ema_decay = ema.begin_step(ema_global_step) if ema is not None else None
        ema_done = ema is None or ema_decay is None
        for gi, group in enumerate(self.param_groups):
            beta1, beta2 = group["betas"]
            ps = [p for p in group["params"] if p.grad is not None and (only_ids is None or id(p) in only_ids)]
            if not ps:
                continue
            lr = group["lr"]
            steps = set()
            decays = []
            for p in ps:
                if not p.is_cuda:
                    raise _lib.StbError("AdamWBF16 (libstb200) needs CUDA parameters; there is no CPU fallback")
                state = self.state[p]
                if len(state) == 0:
                    assert p.dtype == torch.bfloat16, "only bfloat 16 is supported."
                    state["step"] = 0.0
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    state["shift"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    # each weight has its own starting point to avoid simultaneous decays (__init__.py:78-82)
                    state["accumulated_decay"] = float(torch.rand([]) * self.decay_threshold)
                state["step"] += 1
                steps.add(state["step"])
                state["accumulated_decay"] += group["weight_decay"] * lr
                acc = state["accumulated_decay"]
                dec = (acc > self.decay_threshold) * acc
                state["accumulated_decay"] -= dec
                decays.append(float(dec))
                if not (p.is_contiguous() and p.grad.is_contiguous() and p.grad.dtype == torch.bfloat16):
                    raise ValueError("AdamWBF16 (libstb200): parameters and gradients must be contiguous bf16")
            if len(steps) != 1:
                raise NotImplementedError("parameters of one group with different step counts are not supported")
            pl = self._plan(ps)
            slot = pl["slot"]
            pl["slot"] = (slot + 1) % self._RING
            if pl["copied"][slot] is not None:
                pl["copied"][slot].synchronize()     # normally long done (RING steps ago)
            ph, dh = pl["ptrs_host"][slot], pl["decay_host"][slot]
            for t, p in enumerate(ps):
                st = self.state[p]
                ph[0, t], ph[1, t] = p.data_ptr(), p.grad.data_ptr()
                ph[2, t], ph[3, t], ph[4, t] = st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(), st["shift"].data_ptr()
                dh[t] = decays[t]
            shadows = ema.fused_plan(ps) if (not ema_done and len(self.param_groups) == 1) else None
            if shadows is not None:
                eh = pl["ema_host"][slot]
                for t, sh in enumerate(shadows):
                    eh[t] = sh.data_ptr()
                pl["ema"].copy_(eh, non_blocking=True)
                ema_done = True
            pl["ptrs"].copy_(ph, non_blocking=True)
            pl["decay"].copy_(dh, non_blocking=True)
            ev = pl["copied"][slot] or torch.cuda.Event()
            ev.record()
            pl["copied"][slot] = ev
            stepf = float(next(iter(steps)))
            rnd_ptr, rnd_plane = None, 0
            if _rnd is not None:
                assert _rnd.dtype == torch.int32 and _rnd.is_cuda and _rnd.is_contiguous() and _rnd.shape == (4, pl["total"])
                rnd_ptr, rnd_plane = _rnd.data_ptr(), pl["total"]
            seed = launch_seed(self._seed, int(stepf), int(salt), gi)
            check(_lib.lib().stb_adamw_bf16_multi(
                pl["ptrs"].data_ptr(), pl["sizes"].data_ptr(), pl["decay"].data_ptr(), pl["blk_tensor"].data_ptr(),
                pl["blk_off"].data_ptr(), pl["num_blocks"], pl["T"], float(beta1), float(beta2), stepf, float(lr),
                float(group["eps"]), rnd_ptr, pl["rnd_off"].data_ptr(), rnd_plane, C.c_ulonglong(seed),
                float(grad_clamp or 0.0), pl["ema"].data_ptr() if shadows is not None else None,
                float(1.0 - ema_decay) if shadows is not None else 0.0, _stream()))
            if zero_grad:
                for p in ps:
                    p.grad.zero_()
        if not ema_done:       # several groups / fp32 or frozen shadows: the two foreach kernels of EMAModel.step
            ema.apply(ema_decay)
