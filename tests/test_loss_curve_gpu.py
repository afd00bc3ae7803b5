"""GPU (-m gpu): loss-curve equivalence (BASELINE north_star: "loss-curve-equivalent to the reference").

50 optimizer steps of the libstb200 Flux LoRA step (prepare_batch -> model_predict -> loss -> backward -> value clip ->
adamw_bf16) against the CPU oracle trained the same way: oracle/flux_oracle.py for the model (fp32 math on the current bf16
LoRA weights), the reference's default clip (`torch.clamp` at max_grad_norm = 2.0 on bf16 gradients, trainer.py:7138-7217)
and oracle/adamw_bf16_oracle.py (pinned bit-exactly to the reference's `_make_step`) for the update.  Everything random is
REPLAYED: each step's noise / sigmas are the ones the CUDA path drew, and both optimizers consume the same stochastic-
rounding integers.  Stated tolerance: per-step |loss_cuda - loss_oracle| <= 3e-3 * loss_oracle (the two trajectories do
not share bf16 rounding inside the backward, so their weights drift apart by bf16-noise-sized updates); the test also
requires that training actually moved the loss, otherwise agreement would be vacuous."""
import pytest
import torch

from oracle import adamw_bf16_oracle as A
from oracle import flux_oracle as O
from tests import flux_parity as FP

pytestmark = pytest.mark.gpu

STEPS = 50
LOSS_CURVE_RTOL = 3e-3
LR = 1e-3
CLIP = 2.0


def test_flux_lora_loss_curve_matches_oracle_training():
    from simpletuner_b200.training.optim import AdamWBF16
    from simpletuner_b200.training.step import TrainStep

    cfg = FP.small_config(layers=1, single=1)
    rank = 8
    P = {k: v.bfloat16().float() for k, v in O.init_flux_params(cfg, seed=0).items()}
    L0 = {k: v.bfloat16() for k, v in O.init_lora_params(cfg, rank, seed=1, b_std=0.02).items()}
    batch = FP.make_batch(2, 16, 16, 32, cfg, seed=2)
    w = FP.build_cuda_model(cfg, P, {k: v.float() for k, v in L0.items()}, rank)
    den = w._denoiser()
    named = []      # (oracle key, cuda parameter) in the optimizer's parameter order
    for name, lin in den.lora_linears().items():
        named.append((f"{name}.lora_A.weight", lin.lora_A["default"].weight))
        named.append((f"{name}.lora_B.weight", lin.lora_B["default"].weight))
    params = [p for _, p in named]
    opt = AdamWBF16(params, lr=LR, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, seed=5)
    for p in params:
        opt.state[p].update(step=0.0, exp_avg=torch.zeros_like(p), exp_avg_sq=torch.zeros_like(p), shift=torch.zeros_like(p),
                            accumulated_decay=0.0)
    step = TrainStep(w, opt, max_grad_norm=CLIP, grad_clip_method="value")
    # oracle training state (bf16 tensors on the CPU, exactly the optimizer's view)
    Lo = {k: v.clone() for k, v in L0.items()}
    st = {k: [torch.zeros_like(v) for _ in range(3)] for k, v in Lo.items()}     # shift, exp_avg, exp_avg_sq
    sizes = [p.numel() for p in params]
    total = sum(sizes)
    grng = torch.Generator().manual_seed(99)
    losses, losses_ref = [], []
    for k in range(STEPS):
        rnd = torch.randint(0, 1 << 16, (4, total), dtype=torch.int32, generator=grng)
        torch.manual_seed(1000 + k); torch.cuda.manual_seed(1000 + k)
        # --- CUDA step (the optimizer consumes the replayed integers)
        orig = opt.step
        opt.step = lambda zero_grad=False, _r=rnd.cuda().contiguous(), **kw: orig(zero_grad=zero_grad, _rnd=_r, **kw)
        captured = {}
        prep0 = w.prepare_batch

        def prep_and_capture(b, s):
            out = prep0(b, s)
            captured.update(noise=out["noise"].float().cpu(), sigmas=out["sigmas"].flatten().float().cpu(),
                            latents=out["latents"].float().cpu())
            return out

        w.prepare_batch = prep_and_capture
        loss = step({kk: v.clone() for kk, v in batch.items()})
        w.prepare_batch, opt.step = prep0, orig
        losses.append(float(loss))
        # --- oracle step on the replayed noise / sigmas
        Lg = {kk: v.float().requires_grad_(True) for kk, v in Lo.items()}
        noisy = O.flow_noisy_latents(captured["latents"].bfloat16(), captured["noise"].bfloat16(), captured["sigmas"]).float()
        pred = O.flux_model_predict(P, cfg, noisy, captured["sigmas"] * 1000.0, batch["prompt_embeds"].float(),
                                    batch["add_text_embeds"].float(), 1.0, Lg, 1.0)
        lref = O.flow_loss(pred, O.flow_target(captured["latents"].bfloat16(), captured["noise"].bfloat16()))
        lref.backward()
        losses_ref.append(float(lref))
        off = 0
        for (key, _), n in zip(named, sizes):
            g = Lg[key].grad.to(torch.bfloat16).clamp_(-CLIP, CLIP)
            r = [rnd[i, off:off + n].reshape(Lo[key].shape) for i in range(4)]
            A.adamw_bf16_step(Lo[key], g, st[key][0], st[key][1], st[key][2], beta1=0.9, beta2=0.999, step=float(k + 1), lr=LR,
                              eps=1e-8, decay_this_iteration=0.0, rnd=r, scalar_semantics="cuda")
            off += n
    rel = [abs(a - b) / abs(b) for a, b in zip(losses, losses_ref)]
    worst = max(rel)
    # training did something: the weights moved by many bf16 ulps and the loss of the LAST step differs from what the
    # step-0 weights give on that step's noise (checked through the oracle, fp32)
    moved = max(float((Lo[k].float() - L0[k].float()).abs().max()) for k in Lo)
    cos = min(float(torch.nn.functional.cosine_similarity(p.detach().float().cpu().flatten(), Lo[key].float().flatten(), dim=0))
              for key, p in named)
    report = {"steps": STEPS, "worst_rel": worst, "mean_rel": sum(rel) / len(rel), "first": (losses[0], losses_ref[0]),
              "last": (losses[-1], losses_ref[-1]), "max_weight_move": moved, "min_weight_cos": cos}
    print("[loss-curve]", report)
    import os
    if os.environ.get("STB_LOSS_CURVE_REPORT"):   # optional: the full curves as JSON at that path
        import json
        with open(os.environ["STB_LOSS_CURVE_REPORT"], "w") as f:
            json.dump({**report, "cuda": losses, "oracle": losses_ref}, f, indent=1)
    assert worst <= LOSS_CURVE_RTOL, report
    assert moved >= 0.02, report           # 50 steps x lr 1e-3 of a sign-like update
    assert cos >= 0.99, report
