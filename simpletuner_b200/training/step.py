"""One optimizer step of the diffusion training loop — the body of the reference's
`Trainer.train()` `while True:` loop (helpers/training/trainer.py:6951-7567; SURVEY.md §3.2) reduced
to the hot path:

    prepare_batch (6964) -> model_predict (6051) -> loss_with_logs (6113) -> backward (7126)
      -> grad clip (7138-7217, default: element clamp at max_grad_norm=2.0) -> optimizer.step (7239)
      -> zero_grad (7253)

What is deliberately different from the reference loop (and stated with every benchmark number):
  * no device->host sync inside the step: the non-finite-loss check (`trainer.py:7103`) is folded
    into a device-side flag that the caller polls when it logs (`check_finite()`), and the
    sample-weighted loss all-gather + `.item()` per micro-step (`:7114-7115`) is deferred to logging;
  * the gradient exchange is exactly one per optimizer step: either `training.dist.FlatGradSync` (default of bench.py:
    one flat NCCL all-reduce after backward on the compute stream) or torch DDP's bucketed all-reduce overlapped with the
    block-by-block backward (`wrap_ddp`, the reference's mechanism).
"""
from __future__ import annotations

from typing import Any, Dict, Iterable, Optional

import torch


class TrainStep:
    def __init__(self, model, optimizer: torch.optim.Optimizer, *, max_grad_norm: float = 2.0,
                 grad_clip_method: str = "value", gradient_accumulation_steps: int = 1, grad_sync=None, ema=None):
        self.model = model            # simpletuner_b200.flux.model.Flux (or another family wrapper)
        self.optimizer = optimizer
        self.max_grad_norm = max_grad_norm
        self.grad_clip_method = grad_clip_method
        self.accum = gradient_accumulation_steps
        self.state = {"global_step": 0, "micro_step": 0}
        self._params = [p for g in optimizer.param_groups for p in g["params"]]
        self._nonfinite = None
        self.grad_sync = grad_sync    # e.g. training.dist.FlatGradSync: called once per optimizer step, before the clip
        self.track_grad_norm = False  # True: keep the reference's logged `grad_norm` (inf-norm unless norm-clipping) as a device scalar
        self.grad_norm = None
        self.ema = ema                # training.ema.EMAModel over the trainable tensors (trainer.py:7351-7357), or None
        from .optim import AdamWBF16
        self._fused_opt = isinstance(optimizer, AdamWBF16)   # clamp + EMA ride inside the one optimizer launch
        # optimizers whose step() takes `grad_clamp=`, `only=`, `salt=` can run chunk by chunk behind a pipelined exchange
        self._chunked_opt = self._fused_opt or bool(getattr(optimizer, "supports_chunked_step", False))

    def _clip(self):
        """Gradient clip (trainer.py:7138-7217).  Returns the clamp value when the element clamp is left to the optimizer
        kernel (AdamWBF16 + `grad_clip_method = "value"`), else None."""
        clipping = self.max_grad_norm is not None and self.max_grad_norm > 0
        if self.track_grad_norm and (self.grad_clip_method != "norm" or not clipping):
            from .noise import max_grad_value       # trainer.py:7144-7147: self.grad_norm = self._max_grad_value()
            self.grad_norm = max_grad_value(self._params)
        if not clipping:
            return None
        if self.grad_clip_method == "value" and self._fused_opt:
            return float(self.max_grad_norm)
        grads = [p.grad for p in self._params if p.grad is not None]
        if not grads:
            return None
        if self.grad_clip_method == "value":
            torch._foreach_clamp_min_(grads, -self.max_grad_norm)
            torch._foreach_clamp_max_(grads, self.max_grad_norm)
        elif self.grad_clip_method == "norm":
            gn = torch.nn.utils.clip_grad_norm_(self._params, self.max_grad_norm)
            if self.track_grad_norm:
                self.grad_norm = gn
        else:
            raise ValueError(f"unknown grad_clip_method {self.grad_clip_method}")
        return None

    def _pipelined_ok(self) -> bool:
        gs = self.grad_sync
        clipping = self.max_grad_norm is not None and self.max_grad_norm > 0
        return (gs is not None and getattr(gs, "pipeline_chunks", 0) > 0 and self._chunked_opt and not self.track_grad_norm
                and (not clipping or self.grad_clip_method == "value"))

    def _sync_and_step_pipelined(self):
        """Full fine-tune sized gradient sets: chunk i's optimizer launch (clip fused) overlaps chunk i + 1's all-reduce."""
        clamp = float(self.max_grad_norm) if (self.max_grad_norm is not None and self.max_grad_norm > 0) else None
        ema_decay = self.ema.begin_step(self.state["global_step"] + 1) if self.ema is not None else None
        for i, (work, chunk) in enumerate(self.grad_sync.start_chunks()):
            if work is not None:
                work.wait()          # stream-level wait: the compute stream waits for this chunk's collective only
            self.optimizer.step(grad_clamp=clamp, only=chunk, salt=i)
        if ema_decay is not None:
            self.ema.apply(ema_decay)

    def _optimizer_step(self):
        """clip -> optimizer.step -> EMA (trainer.py:7138-7239, 7351-7357); one launch for all three with AdamWBF16."""
        clamp = self._clip()
        gs = self.state["global_step"] + 1
        if self._fused_opt:
            self.optimizer.step(grad_clamp=clamp, ema=self.ema, ema_global_step=gs)
        else:
            self.optimizer.step()
            if self.ema is not None:
                self.ema.step(self._params, global_step=gs)

    def __call__(self, batch: Dict[str, Any]) -> torch.Tensor:
        """Runs one micro-step (and the optimizer step when the accumulation boundary is reached).
        Returns the detached fp32 loss tensor (on device; no sync)."""
        prepared = self.model.prepare_batch(batch, self.state)
        sync = (self.state["micro_step"] + 1) % self.accum == 0
        ddp = self.model.model if hasattr(self.model.model, "no_sync") else None
        ctx = ddp.no_sync() if (ddp is not None and not sync) else _null()
        with ctx:
            out = self.model_predict(prepared)
            loss, _ = self.model.loss_with_logs(prepared, out, apply_conditioning_mask=True)
            (loss / self.accum if self.accum > 1 else loss).backward()
        ld = loss.detach()
        bad = ~torch.isfinite(ld)
        self._nonfinite = bad if self._nonfinite is None else (self._nonfinite | bad)
        self.state["micro_step"] += 1
        if sync:
            if self._pipelined_ok():
                self._sync_and_step_pipelined()
            else:
                if self.grad_sync is not None:
                    self.grad_sync()
                self._optimizer_step()
            self.optimizer.zero_grad(set_to_none=True)
            den = getattr(self.model, "model", None)
            den = getattr(den, "module", den)
            hook = getattr(den, "after_optimizer_step", None)
            if callable(hook):          # full fine-tune: derived weight layouts must be rebuilt from the updated weights
                hook()
            self.state["global_step"] += 1
        return ld

    def model_predict(self, prepared_batch):
        """`Trainer.model_predict` (trainer.py:6051-6107) for the plain training path: family `model_predict`, then the
        x-prediction fix-up (:6099-6105) — a scheduler with `prediction_type == "sample"` gets `prediction - noise`.  The
        reference applies the subtraction to whatever `model_predict` returned; here it is applied to the
        `model_prediction` entry of the dict (a new tensor, so the family's `loss()` re-packs it instead of using its
        private packed copy)."""
        out = self.model.model_predict(prepared_batch)
        sched = getattr(self.model, "noise_schedule", None)
        if sched is not None and getattr(getattr(sched, "config", None), "prediction_type", None) == "sample":
            if isinstance(out, dict):
                out = dict(out)
                out["model_prediction"] = out["model_prediction"] - prepared_batch["noise"]
            else:
                out = out - prepared_batch["noise"]
        return out

    def check_finite(self):
        """Host sync: raise like trainer.py:7103-7111 if any step since the last check saw a non-finite loss."""
        bad = self._nonfinite is not None and bool(self._nonfinite.item())
        self._nonfinite = None
        if bad:
            raise RuntimeError("Non-finite loss encountered during training.")


class GraphedTrainStep:
    """TrainStep whose micro-step body (prepare_batch -> model_predict -> loss -> backward) is captured ONCE per batch shape
    into a CUDA graph and replayed; gradient exchange, clip and optimizer stay eager.

    Why: with short kernels (SD3.5-medium full fine-tune: ~3000 launches of 20-50 us per step) the step is bound by the
    Python / launch path, not by the GPU.  A replay issues the same kernels from one `cudaGraphLaunch`.  The reference has
    no equivalent (its loop is eager); numerics are unchanged — the graph contains exactly the eager launches, and torch's
    CUDA generator is capture-aware, so noise / sigmas still advance every replay.
    Constraints: no torch DDP wrapper (use `FlatGradSync`), one uniform shape per call (aspect buckets -> one graph per
    bucket shape), gradients stay allocated between steps (their addresses are baked into the graph), the model must not
    change structure after the first call.  gradient_accumulation_steps > 1: every bucket graph ACCUMULATES into one shared,
    persistent set of gradient buffers (autograd's in-place accumulate is part of the capture); the buffers are zeroed at the
    start of each accumulation window and the loss is scaled by 1 / accum inside the graph, as TrainStep does eagerly."""

    def __init__(self, step: "TrainStep", warmup: int = 2, capture_prepare: bool = True):
        self._shared_grads = step.accum > 1
        # capture_prepare = False: `prepare_batch` runs eagerly every call and only model_predict -> loss -> backward is
        # replayed.  Needed by the epsilon / v families, whose timestep draw is host-side in the reference (one CPU
        # `torch.multinomial(...).item()` per segment, helpers/training/custom_schedule.py:18-58) and must not be frozen into a graph.
        self.capture_prepare = bool(capture_prepare)
        if hasattr(step.model.model, "no_sync"):
            raise NotImplementedError("GraphedTrainStep: wrap with FlatGradSync instead of torch DDP")
        den = getattr(step.model, "model", None)
        if float(getattr(den, "_lora_dropout_p", 0.0) or 0.0) > 0.0:
            # the dropout seed is drawn on the host once per forward: a captured graph would replay ONE mask forever
            raise NotImplementedError("GraphedTrainStep: lora_dropout > 0 draws a per-step host seed; run the eager TrainStep")
        if getattr(den, "_lycoris_network", None) is not None:
            raise NotImplementedError("GraphedTrainStep: LoKr rebuilds the projection layouts between steps; run the eager TrainStep")
        self.step = step
        self.warmup = warmup
        self._graphs: Dict[Any, Any] = {}
        self._pool = None          # one memory pool shared by the per-bucket graphs (they never replay concurrently)

    @property
    def state(self):
        return self.step.state

    def check_finite(self):
        return self.step.check_finite()

    def _body(self, batch):
        st = self.step
        prepared = st.model.prepare_batch(batch, st.state) if self.capture_prepare else batch
        out = st.model_predict(prepared)
        loss, _ = st.model.loss_with_logs(prepared, out, apply_conditioning_mask=True)
        (loss / st.accum if st.accum > 1 else loss).backward()
        return loss.detach()

    def _finish(self, ld):
        st = self.step
        bad = ~torch.isfinite(ld)
        st._nonfinite = bad if st._nonfinite is None else (st._nonfinite | bad)
        st.state["micro_step"] += 1
        if st.state["micro_step"] % st.accum != 0:
            return ld                      # inside an accumulation window: no exchange, no optimizer
        if st._pipelined_ok():
            st._sync_and_step_pipelined()
        else:
            if st.grad_sync is not None:
                st.grad_sync()
            st._optimizer_step()
        # NO zero_grad(set_to_none): the captured backward writes the same .grad tensors again on the next replay
        st.state["global_step"] += 1
        return ld

    def __call__(self, batch: Dict[str, Any]) -> torch.Tensor:
        if any(batch.get(k) is not None for k in ("conditioning_latents", "conditioning_packed_latents")):
            raise NotImplementedError("GraphedTrainStep: Flux Kontext batches (conditioning latents) run on the eager TrainStep")
        if not getattr(self.step.model, "GRAPH_REPLAY", True):
            raise NotImplementedError(f"GraphedTrainStep: {self.step.model.NAME} batches run on the eager TrainStep")
        if not self.capture_prepare:          # eager prepare (host-side draws stay live); its output is the graph's input
            batch = self.step.model.prepare_batch(batch, self.step.state)
        key = tuple((k, tuple(v.shape), v.dtype) for k, v in sorted(batch.items()) if torch.is_tensor(v))
        entry = self._graphs.get(key)
        if entry is None:
            static = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in batch.items()}
            shared = self._shared_grads
            if shared and getattr(self, "_grad_bufs", None) is None:
                self._grad_bufs = [torch.zeros_like(p) for p in self.step._params]     # outside every graph pool: persistent
            keep = [g.clone() for g in self._grad_bufs] if shared else None            # a capture may land mid-window
            for i, p in enumerate(self.step._params):
                p.grad = self._grad_bufs[i] if shared else None
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(self.warmup):          # lazy initialisation (weight layouts, tensor maps, smem attributes)
                    self._body(dict(static))
                    if not shared:
                        for p in self.step._params:
                            p.grad = None
            torch.cuda.current_stream().wait_stream(side)
            den = getattr(self.step.model, "model", None)
            hook = getattr(den, "before_graph_capture", None)
            if callable(hook):      # full fine-tune: the rebuild of the derived weight layouts must be PART of the graph
                hook()
            from .. import ops
            n0 = ops.launch_count()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, pool=self._pool):
                loss = self._body(dict(static))
            if self._pool is None:
                self._pool = graph.pool()
            if shared:       # warm-up runs and the capture pass itself added into the shared buffers: restore the window's state
                torch._foreach_copy_(self._grad_bufs, keep)
            entry = (graph, static, loss, [p.grad for p in self.step._params], ops.launch_count() - n0)
            self._graphs[key] = entry
        graph, static, loss, grads, n_kernels = entry
        for k, v in batch.items():
            if torch.is_tensor(v):
                static[k].copy_(v, non_blocking=True)
        for p, g in zip(self.step._params, grads):       # several bucket graphs own different gradient buffers (accum == 1)
            p.grad = g
        if self._shared_grads and self.step.state["micro_step"] % self.step.accum == 0:
            torch._foreach_zero_(self._grad_bufs)        # start of an accumulation window
        graph.replay()
        from .. import ops
        ops.note_graph_replay(n_kernels)
        return self._finish(loss.clone())


class _null:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


def wrap_ddp(model_wrapper, device_ids=None, bucket_cap_mb: int = 25):
    """Wrap the denoiser in torch DDP (reference: accelerator.prepare -> DDP, trainer.py:4571, 1026-1041).
    Only the trainable (LoRA) parameters carry gradients, so the per-step all-reduce is ~52 MB for Flux r=16."""
    from torch.nn.parallel import DistributedDataParallel as DDP

    model_wrapper.model = DDP(model_wrapper.model, device_ids=device_ids, bucket_cap_mb=bucket_cap_mb,
                              gradient_as_bucket_view=True, broadcast_buffers=False)
    return model_wrapper
