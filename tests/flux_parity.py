"""Model-level parity harness: simpletuner_b200 Flux (CUDA, bf16, libstb200) vs the fp32 CPU oracle.
Shared by tests/test_flux_parity_gpu.py, __graft_entry__.smoke() and bench.py's cpu_baseline leg."""
from __future__ import annotations

import torch

from oracle import flux_oracle as O

# Tolerances (stated, per BASELINE north_star "noise-prediction loss within a stated bf16 tolerance"; SURVEY.md 7):
#   compared against the fp32 oracle evaluated on the SAME bf16-rounded weights and inputs.  Measured on H100
#   (smoke()): toy width loss rel. err 6e-5 / pred cos 0.99999 / worst grad cos 0.9999; full width (D = 3072, S = 4608)
#   in tests/test_fullwidth_parity_gpu.py.  The bounds leave ~10x head-room over what was measured.
LOSS_RTOL = 2e-3      # |loss_cuda - loss_fp32| / loss_fp32
PRED_COS = 0.9995     # cosine(pred_cuda, pred_fp32) over all elements
GRAD_COS = 0.999      # cosine per LoRA gradient tensor (bf16 backward through ~10 GEMMs per block)


def record(tag: str, res: dict) -> dict:
    """Append the measured deviations to $STB_PARITY_REPORT (a .jsonl path) when that variable is set."""
    import os

    path = os.environ.get("STB_PARITY_REPORT")
    if path:
        import json

        with open(path, "a") as f:
            f.write(json.dumps({"case": tag, **{k: v for k, v in res.items() if isinstance(v, (int, float, str, bool))}}) + "\n")
    return res


def small_config(layers=2, single=2, heads=2, hd=128, joint=192, pooled=64):
    return O.FluxConfig(in_channels=64, num_layers=layers, num_single_layers=single, attention_head_dim=hd,
                        num_attention_heads=heads, joint_attention_dim=joint, pooled_projection_dim=pooled,
                        guidance_embeds=True, axes_dims_rope=(16, 56, 56) if hd == 128 else (8, 28, 28))


def make_batch(B, Hh, Ww, S_txt, cfg, seed=0, C=16):
    g = torch.Generator().manual_seed(seed)
    return {
        "latent_batch": torch.randn(B, C, Hh, Ww, generator=g).bfloat16(),
        "prompt_embeds": torch.randn(B, S_txt, cfg.joint_attention_dim, generator=g).bfloat16(),
        "add_text_embeds": torch.randn(B, cfg.pooled_projection_dim, generator=g).bfloat16(),
    }


def build_cuda_model(cfg, P, lora, rank, device="cuda", target="all"):
    from simpletuner_b200.flux.model import Flux, default_config
    from simpletuner_b200.flux.transformer import FluxTransformer2DModel

    m = FluxTransformer2DModel(in_channels=cfg.in_channels, num_layers=cfg.num_layers,
                               num_single_layers=cfg.num_single_layers, attention_head_dim=cfg.attention_head_dim,
                               num_attention_heads=cfg.num_attention_heads, joint_attention_dim=cfg.joint_attention_dim,
                               pooled_projection_dim=cfg.pooled_projection_dim, guidance_embeds=cfg.guidance_embeds,
                               axes_dims_rope=cfg.axes_dims_rope)
    sd = {k: v.bfloat16() for k, v in P.items()}
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert not missing, missing
    m.to(device)
    wrapper = Flux(default_config(lora_rank=rank, flux_lora_target=target), transformer=m, device=torch.device(device))
    if lora is not None:
        wrapper.add_lora_adapter()
        with torch.no_grad():
            for name, lin in m.lora_linears().items():
                lin.lora_A["default"].weight.copy_(lora[name + ".lora_A.weight"].bfloat16())
                lin.lora_B["default"].weight.copy_(lora[name + ".lora_B.weight"].bfloat16())
    return wrapper


def run_parity(cfg=None, B=2, Hh=16, Ww=16, S_txt=64, rank=16, seed=0, device="cuda", checkpoint=False, interval=None,
               target="all"):
    """Returns a dict of measured deviations (and asserts nothing).  `target` = the reference's flux_lora_target."""
    from simpletuner_b200.flux.transformer import FLUX_LORA_TARGETS
    cfg = cfg or small_config()
    P = {k: v.bfloat16().float() for k, v in O.init_flux_params(cfg, seed=seed).items()}
    L = {k: v.bfloat16().float() for k, v in O.init_lora_params(cfg, rank, seed=seed + 1, b_std=0.02,
                                                                targets=tuple(FLUX_LORA_TARGETS[target])).items()}
    batch = make_batch(B, Hh, Ww, S_txt, cfg, seed=seed + 2)
    w = build_cuda_model(cfg, P, L, rank, device, target=target)
    assert set(w._denoiser().lora_linears()) == set(O.lora_target_names(cfg, tuple(FLUX_LORA_TARGETS[target])))
    if checkpoint:   # reference --gradient_checkpointing (+ interval): selected blocks are re-run in backward
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
    # oracle on the SAME noise / sigmas (drawn by torch on the device, SURVEY.md §8d parity harness)
    ob = {"latents": prepared["latents"].float().cpu(), "noise": prepared["noise"].float().cpu(),
          "sigmas": prepared["sigmas"].flatten().float().cpu(), "prompt_embeds": batch["prompt_embeds"].float(),
          "pooled": batch["add_text_embeds"].float()}
    Lg = {k: v.clone().requires_grad_(True) for k, v in L.items()}
    # the reference builds noisy latents in bf16 (common.py:4953-4960); feed the oracle the same bf16 tensor
    noisy_ref = O.flow_noisy_latents(ob["latents"].bfloat16(), ob["noise"].bfloat16(), ob["sigmas"]).float()
    pred_ref = O.flux_model_predict(P, cfg, noisy_ref, ob["sigmas"] * 1000.0, ob["prompt_embeds"], ob["pooled"], 1.0, Lg, 1.0)
    loss_ref = O.flow_loss(pred_ref, O.flow_target(ob["latents"].bfloat16(), ob["noise"].bfloat16()))
    loss_ref.backward()
    pred = w.unpacked_prediction(out).float().cpu()
    res = {
        "noisy_bit_exact": bool(torch.equal(prepared["noisy_latents"].cpu(), noisy_ref.bfloat16())),
        "loss": float(loss.item()), "loss_ref": float(loss_ref.item()),
        "loss_rel_err": abs(float(loss.item()) - float(loss_ref.item())) / abs(float(loss_ref.item())),
        "pred_cos": float(torch.nn.functional.cosine_similarity(pred.flatten(), pred_ref.detach().flatten(), dim=0)),
        "pred_max_abs_err": float((pred - pred_ref.detach()).abs().max()),
    }
    cos_min, worst = 1.0, None
    rel_norm_max = 0.0
    for name, lin in w._denoiser().lora_linears().items():
        for which, p in (("lora_A", lin.lora_A["default"].weight), ("lora_B", lin.lora_B["default"].weight)):
            gref = Lg[f"{name}.{which}.weight"].grad
            g = p.grad.float().cpu()
            c = float(torch.nn.functional.cosine_similarity(g.flatten(), gref.flatten(), dim=0))
            rn = float((g - gref).norm() / (gref.norm() + 1e-12))
            rel_norm_max = max(rel_norm_max, rn)
            if c < cos_min:
                cos_min, worst = c, f"{name}.{which}"
    res.update({"grad_cos_min": cos_min, "grad_worst": worst, "grad_rel_l2_max": rel_norm_max,
                "n_lora_tensors": 2 * len(w._denoiser().lora_linears())})
    return res
