"""fp32 oracle of Flux masked training (`--flux_attention_masked_training`, default processor; SURVEY.md quirk Q2) and
the GPU parity harness for it.

The reference turns the text mask into a float mask that SDPA ADDS to the logits: `expand_flux_attention_mask` writes
the [B, L] mask into ones over the joint [text | image] sequence, and FluxAttnProcessor2_0 passes `(mask > 0)` in the
activation dtype as `attn_mask` [B, 1, 1, S] (reference flux/transformer.py:170-173, 200-207, 227-242).  Kept text keys
and every image key get +1, padded text keys +0.  `masked(mask)` evaluates oracle/flux_oracle.py with that bias added to
every attention's logits (its `sdpa` is swapped for the duration); the oracle itself stays the un-masked reference that
smoke() and the benchmark compare against.  Pinned against the reference's own processor by
tests/golden/flux_attn_mask_golden.pt (tools/make_golden_flux_mask.py)."""
from __future__ import annotations

import contextlib
from typing import Optional, Sequence

import torch

from oracle import flux_oracle as O
from tests import flux_parity as FP


def key_bias(mask: torch.Tensor, S: int) -> torch.Tensor:
    """[B, S] fp32: expand_flux_attention_mask + (mask > 0)."""
    bias = torch.ones(mask.shape[0], S)
    bias[:, :mask.shape[1]] = (mask.float().cpu() > 0).float()
    return bias


def sdpa_bias(q, k, v, bias: torch.Tensor):
    """softmax(q k^T * scale + bias[:, None, None, :]) v in fp32 (q / k / v [B, H, S, D])."""
    s = (q.float() @ k.float().transpose(-1, -2)) * q.shape[-1] ** -0.5 + bias[:, None, None, :].to(q.device)
    return (torch.softmax(s, dim=-1) @ v.float()).to(q.dtype)


@contextlib.contextmanager
def masked(mask: Optional[torch.Tensor]):
    """Within the block, every flux_oracle attention adds the per-key bias of `mask` [B, L] (None: unchanged)."""
    if mask is None:
        yield
        return
    plain = O.sdpa
    O.sdpa = lambda q, k, v: sdpa_bias(q, k, v, key_bias(mask, k.shape[2]))
    try:
        yield
    finally:
        O.sdpa = plain


def length_mask(lengths: Sequence[int], S_txt: int) -> torch.Tensor:
    m = torch.zeros(len(lengths), S_txt)
    for i, n in enumerate(lengths):
        m[i, :n] = 1
    return m


def masked_config(wrapper):
    """Turn masked training on for a model built by tests/flux_parity.build_cuda_model."""
    wrapper.config.flux_attention_masked_training = True
    wrapper.config.attention_mechanism = "diffusers"
    wrapper._denoiser().attention_masked_training = True
    return wrapper


def run_masked_parity(mask: Optional[torch.Tensor], cfg=None, B=3, Hh=16, Ww=16, S_txt=77, rank=16, seed=0,
                      checkpoint=False, interval=None, target="all", device="cuda"):
    """tests/flux_parity.run_parity with masked training: the CUDA step (mask in the batch) against the masked fp32
    oracle.  mask None: masked training off.  Returns the deviations and the CUDA loss."""
    from simpletuner_b200.flux.transformer import FLUX_LORA_TARGETS
    cfg = cfg or FP.small_config()
    P = {k: v.bfloat16().float() for k, v in O.init_flux_params(cfg, seed=seed).items()}
    L = {k: v.bfloat16().float() for k, v in O.init_lora_params(cfg, rank, seed=seed + 1, b_std=0.02,
                                                                targets=tuple(FLUX_LORA_TARGETS[target])).items()}
    batch = FP.make_batch(B, Hh, Ww, S_txt, cfg, seed=seed + 2)
    w = FP.build_cuda_model(cfg, P, L, rank, device, target=target)
    if mask is not None:
        masked_config(w)
        batch["encoder_attention_mask"] = mask.clone()
    if checkpoint:
        w._denoiser().enable_gradient_checkpointing()
        if interval:
            w._denoiser().set_gradient_checkpointing_interval(interval)
    torch.manual_seed(1234)
    torch.cuda.manual_seed(1234)
    prepared = w.prepare_batch({k: v.clone() for k, v in batch.items()}, {"global_step": 0})
    out = w.model_predict(prepared)
    loss = w.loss(prepared, out)
    loss.backward()
    torch.cuda.synchronize()
    lat, noise = prepared["latents"].float().cpu(), prepared["noise"].float().cpu()
    sig = prepared["sigmas"].flatten().float().cpu()
    Lg = {k: v.clone().requires_grad_(True) for k, v in L.items()}
    noisy_ref = O.flow_noisy_latents(lat.bfloat16(), noise.bfloat16(), sig).float()
    with masked(mask):
        pred_ref = O.flux_model_predict(P, cfg, noisy_ref, sig * 1000.0, batch["prompt_embeds"].float(),
                                        batch["add_text_embeds"].float(), 1.0, Lg, 1.0)
    loss_ref = O.flow_loss(pred_ref, O.flow_target(lat.bfloat16(), noise.bfloat16()))
    loss_ref.backward()
    pred = w.unpacked_prediction(out).float().cpu()
    res = {"loss": float(loss.item()), "loss_ref": float(loss_ref.item()),
           "loss_rel_err": abs(float(loss.item()) - float(loss_ref.item())) / abs(float(loss_ref.item())),
           "pred_cos": float(torch.nn.functional.cosine_similarity(pred.flatten(), pred_ref.detach().flatten(), dim=0))}
    cos_min, worst, n_txt_grads = 1.0, None, 0
    for name, lin in w._denoiser().lora_linears().items():
        for which, p in (("lora_A", lin.lora_A["default"].weight), ("lora_B", lin.lora_B["default"].weight)):
            gref = Lg[f"{name}.{which}.weight"].grad
            c = float(torch.nn.functional.cosine_similarity(p.grad.float().cpu().flatten(), gref.flatten(), dim=0))
            if c < cos_min:
                cos_min, worst = c, f"{name}.{which}"
            if "add_" in name or "ff_context" in name:
                n_txt_grads += int(p.grad.abs().sum().item() > 0)
    res.update({"grad_cos_min": cos_min, "grad_worst": worst, "text_stream_grads_nonzero": n_txt_grads})
    return res


def within_tolerance(res) -> bool:
    return res["loss_rel_err"] <= FP.LOSS_RTOL and res["pred_cos"] >= FP.PRED_COS and res["grad_cos_min"] >= FP.GRAD_COS
