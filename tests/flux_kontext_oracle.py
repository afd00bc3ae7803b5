"""fp32 oracle of Flux Kontext training (model_flavour "kontext") and the GPU parity harness for it.

Kontext appends packed reference-image latents after the noisy scene tokens.  The reference conditions them at timestep 0
through 2-D timesteps and a per-token temb, then drops their outputs before the loss:
  * build_kontext_inputs                     flux/__init__.py:64-172      -> `build_kontext_inputs`
  * Flux._extend_conditioning_timesteps      flux/model.py:602-618        -> `extend_conditioning_timesteps`
  * _flux_tokenwise_conditioning             flux/transformer.py:245-294  -> `tokenwise_temb`
  * the 3-D adaLN branches                   flux/transformer.py:386-412  -> `ada_zero` / `ada_continuous`
  * temb_txt = temb.mean(1), temb_single     flux/transformer.py:1068-1085
  * model_predict (cat, scene slice)         flux/model.py:707-864        -> `kontext_model_predict`
The layers themselves are oracle/flux_oracle.py's, unchanged.  Pinned against the reference's own functions by
tests/golden/flux_kontext_golden.pt (tools/make_golden_flux_kontext.py)."""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn.functional as F

from oracle import flux_oracle as O
from tests import flux_mask_oracle as MO
from tests import flux_parity as FP


def build_kontext_inputs(conds: List[torch.Tensor], dtype=torch.bfloat16):
    """(packed [B, S_c, 4C], ids [B, S_c, 3] in `dtype`): each latent packed and placed by the ComfyUI offset scheme."""
    packed, ids = [], []
    x0 = y0 = 0
    for lat in conds:
        B, C, H, W = lat.shape
        packed.append(O.pack_latents(lat, B, C, H, W).to(dtype))
        x = y = 0
        if H + y0 > W + x0:
            x = x0
        else:
            y = y0
        iy, ix = torch.arange(H // 2) + y // 2, torch.arange(W // 2) + x // 2
        grid = torch.stack(torch.meshgrid(iy, ix, indexing="ij"), dim=-1)
        ids.append(torch.cat([torch.ones_like(grid[..., :1]), grid], -1).view(1, -1, 3).expand(B, -1, -1).to(dtype))
        x0, y0 = max(x0, W + x), max(y0, H + y)
    return torch.cat(packed, 1), torch.cat(ids, 1)


def extend_conditioning_timesteps(t: torch.Tensor, S_scene: int, S_c: int) -> torch.Tensor:
    return torch.cat([t[:, None].expand(-1, S_scene), torch.zeros(t.shape[0], S_c, dtype=t.dtype)], 1)


def tokenwise_temb(P, cfg, t2: torch.Tensor, guidance: Optional[torch.Tensor], pooled: torch.Tensor) -> torch.Tensor:
    """[B, S, D]: time_text_embed on every token's (timestep, guidance, pooled); t2 [B, S] and guidance [B] already x1000."""
    B, S = t2.shape
    g = None if guidance is None else guidance[:, None].expand(-1, S).reshape(-1)
    rep = pooled[:, None, :].expand(-1, S, -1).reshape(B * S, -1)
    return O.time_text_embed(P, cfg, t2.reshape(-1), g, rep).view(B, S, -1)


def ada_zero(W, b, x, emb, n):
    """AdaLayerNormZero(Single) with a per-token emb [B, S, D]: (LN(x) (1 + scale) + shift, the remaining chunks)."""
    mod = F.linear(F.silu(emb), W, b).chunk(n, dim=-1)
    return (O.layer_norm_noaffine(x) * (1 + mod[1]) + mod[0],) + mod[2:]


def ada_continuous(W, b, x, emb):
    """AdaLayerNormContinuous with a per-token emb: chunk order (scale, shift)."""
    scale, shift = torch.chunk(F.linear(F.silu(emb).to(x.dtype), W, b), 2, dim=-1)
    return O.layer_norm_noaffine(x) * (1 + scale) + shift


def _double(P, cfg, i, x, enc, temb_img, temb_txt, rope, lora, ls):
    p = f"transformer_blocks.{i}."
    nx, g_a, sh_m, sc_m, g_m = ada_zero(P[p + "norm1.linear.weight"], P[p + "norm1.linear.bias"], x, temb_img, 6)
    cmod = F.linear(F.silu(temb_txt), P[p + "norm1_context.linear.weight"], P[p + "norm1_context.linear.bias"])
    csh_a, csc_a, cg_a, csh_m, csc_m, cg_m = cmod.chunk(6, dim=1)
    nenc = O.layer_norm_noaffine(enc) * (1 + csc_a[:, None]) + csh_a[:, None]
    ao, eo = O.flux_attention(P, cfg, p + "attn.", nx, nenc, rope, lora, ls)
    x = x + g_a * ao
    enc = enc + cg_a.unsqueeze(1) * eo
    nx = O.layer_norm_noaffine(x) * (1 + sc_m) + sh_m
    ff = O.linear(F.gelu(O.linear(nx, P, p + "ff.net.0.proj", lora, ls), approximate="tanh"), P, p + "ff.net.2", lora, ls)
    x = x + g_m * ff
    nenc = O.layer_norm_noaffine(enc) * (1 + csc_m[:, None]) + csh_m[:, None]
    cff = O.linear(F.gelu(O.linear(nenc, P, p + "ff_context.net.0.proj", lora, ls), approximate="tanh"), P,
                   p + "ff_context.net.2", lora, ls)
    return O.nan_to_num_(enc + cg_m.unsqueeze(1) * cff), x


def _single(P, cfg, i, x, temb, rope, lora, ls):
    p = f"single_transformer_blocks.{i}."
    nx, gate = ada_zero(P[p + "norm.linear.weight"], P[p + "norm.linear.bias"], x, temb, 3)
    ao = O.flux_attention(P, cfg, p + "attn.", nx, None, rope, lora, ls)
    mlp = F.gelu(O.linear(nx, P, p + "proj_mlp", lora, ls), approximate="tanh")
    return O.nan_to_num_(x + gate * O.linear(torch.cat([ao, mlp], dim=2), P, p + "proj_out", lora, ls))


def kontext_forward(P, cfg, hidden, enc_hs, pooled, t2, img_ids, txt_ids, guidance=None, lora=None, ls=1.0):
    """FluxTransformer2DModel.forward with 2-D timesteps t2 [B, S_img] (in [0, 1]); returns every image row."""
    x = O.linear(hidden, P, "x_embedder", lora, ls)
    g = guidance.float() * 1000 if guidance is not None else None
    temb = tokenwise_temb(P, cfg, t2.float() * 1000, g, pooled)
    temb_txt = temb.mean(dim=1)
    enc = F.linear(enc_hs, P["context_embedder.weight"], P["context_embedder.bias"])
    S_txt = enc.shape[1]
    temb_single = torch.cat([temb_txt.unsqueeze(1).expand(-1, S_txt, -1), temb], dim=1)
    rope = O.rope_tables(torch.cat((txt_ids, img_ids), 0), cfg.axes_dims_rope)
    for i in range(cfg.num_layers):
        enc, x = _double(P, cfg, i, x, enc, temb, temb_txt, rope, lora, ls)
    h = torch.cat([enc, x], dim=1)
    for i in range(cfg.num_single_layers):
        h = _single(P, cfg, i, h, temb_single, rope, lora, ls)
    x = ada_continuous(P["norm_out.linear.weight"], P["norm_out.linear.bias"], h[:, S_txt:], temb)
    return O.linear(x, P, "proj_out", lora, ls)


def kontext_model_predict(P, cfg, noisy, timesteps, prompt_embeds, pooled, conds, guidance_value=1.0, lora=None, ls=1.0):
    """Flux._model_predict_single with conditioning latents: returns the unpacked scene prediction and the 2-D timesteps."""
    B, Cc, Hh, Ww = noisy.shape
    packed = O.pack_latents(noisy, B, Cc, Hh, Ww)
    cond_seq, cond_ids = build_kontext_inputs(conds)
    S_scene, S_c = packed.shape[1], cond_seq.shape[1]
    t2 = extend_conditioning_timesteps(timesteps.float() / 1000.0, S_scene, S_c)
    guidance = torch.full((B,), float(guidance_value)) if cfg.guidance_embeds else None
    img_ids = torch.cat([O.prepare_latent_image_ids(Hh, Ww), cond_ids[0].float()], 0)
    out = kontext_forward(P, cfg, torch.cat([packed, cond_seq.to(packed.dtype)], 1), prompt_embeds, pooled, t2, img_ids,
                          torch.zeros(prompt_embeds.shape[1], 3), guidance, lora, ls)
    return O.unpack_latents(out[:, :S_scene], Hh * 8, Ww * 8, 16), t2


def _cos(a: torch.Tensor, b: torch.Tensor) -> float:
    """Cosine in fp64 of two gradients.  F.cosine_similarity clamps |a| |b| at 1e-8, which scales down the cosine of small
    gradients (the text-stream projections of the last double block at HD 64 have norms near 1e-5)."""
    a, b = a.double().flatten(), b.double().flatten()
    return float(a @ b / (a.norm() * b.norm()).clamp_min(1e-300))


# ---- GPU parity harness ------------------------------------------------------------------------------------------------
def kontext_config(wrapper):
    wrapper.config.model_flavour = "kontext"
    return wrapper


def make_conds(B, sizes, seed, C=16):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, C, h, w, generator=g).bfloat16() for h, w in sizes]


def run_kontext_parity(sizes, cfg=None, B=2, Hh=16, Ww=16, S_txt=32, rank=16, seed=0, checkpoint=False, mask=None,
                       dropout=0.0, lokr=None, device="cuda"):
    """The Kontext CUDA step (prepare_batch -> model_predict -> loss -> backward, "combined" sampling over `sizes`) against
    the fp32 oracle, with the deviations tests/flux_parity.py reports.  lokr: a LyCORIS config (LoKr) instead of LoRA."""
    cfg = cfg or FP.small_config()
    P = {k: v.bfloat16().float() for k, v in O.init_flux_params(cfg, seed=seed).items()}
    batch = FP.make_batch(B, Hh, Ww, S_txt, cfg, seed=seed + 2)
    conds = make_conds(B, sizes, seed + 3)
    batch["conditioning_latents"] = [c.clone() for c in conds]
    if lokr is None:
        L = {k: v.bfloat16().float() for k, v in O.init_lora_params(cfg, rank, seed=seed + 1, b_std=0.02).items()}
        w = FP.build_cuda_model(cfg, P, None, rank, device)
        w.config.lora_dropout = dropout
        w.add_lora_adapter()
        with torch.no_grad():
            for name, lin in w._denoiser().lora_linears().items():
                lin.lora_A["default"].weight.copy_(L[name + ".lora_A.weight"].bfloat16())
                lin.lora_B["default"].weight.copy_(L[name + ".lora_B.weight"].bfloat16())
        params = {f"{n}.{which}.weight": getattr(lin, which)["default"].weight
                  for n, lin in w._denoiser().lora_linears().items() for which in ("lora_A", "lora_B")}
    else:       # as tests/test_flux_lokr_gpu.py sets LoKr up
        from oracle import lokr_oracle as LO
        shapes = O.flux_param_shapes(cfg)
        targets = [k[:-7] for k in shapes if k.endswith(".weight") and len(shapes[k]) == 2 and (".attn." in k or ".ff" in k)]
        factor = lambda n: 4 if (".ff." in n or ".ff_context." in n) else 10
        L = {k: v.bfloat16().float() for k, v in LO.init_lokr_params({n: shapes[n + ".weight"] for n in targets},
                                                                      lokr["linear_dim"], factor, seed=seed + 1,
                                                                      w2_std=0.02).items()}
        w = FP.build_cuda_model(cfg, P, None, rank, device)
        w.config.lora_type = "lycoris"
        net = w.add_lycoris_adapter(dict(lokr))
        net.to(device)
        params = {}
        with torch.no_grad():
            for mod in net.loras:
                oname = next(t for t in targets if "lycoris_" + t.replace(".", "_") == mod.lora_name)
                for pn, prm in mod.named_parameters():
                    prm.copy_(L[f"{oname}.{pn}"].bfloat16())
                    params[f"{oname}.{pn}"] = prm
        w._denoiser().invalidate_plans()
        O.LOKR = {"linear_dim": lokr["linear_dim"], "linear_alpha": lokr["linear_alpha"], "multiplier": 1.0}
    kontext_config(w)
    den = w._denoiser()
    if mask is not None:
        MO.masked_config(w)
        batch["encoder_attention_mask"] = mask.clone()
    if checkpoint:
        den.enable_gradient_checkpointing()
    den.train()
    torch.manual_seed(1234)
    torch.cuda.manual_seed(1234)
    prepared = w.prepare_batch({k: v for k, v in batch.items()}, {"global_step": 0,
                                                                  "args": {"conditioning_multidataset_sampling": "combined"}})
    out = w.model_predict(prepared)
    loss = w.loss(prepared, out)
    loss.backward()
    torch.cuda.synchronize()
    S_scene = (Hh // 2) * (Ww // 2)
    S_c = sum((h // 2) * (w_ // 2) for h, w_ in sizes)
    if dropout:
        from tests.test_lora_dropout_gpu import _masks_for_flux
        O.DROPOUT_MASKS = _masks_for_flux(den, cfg, B, S_scene + S_c, S_txt, dropout)
    lat, noise = prepared["latents"].float().cpu(), prepared["noise"].float().cpu()
    sig = prepared["sigmas"].flatten().float().cpu()
    Lg = {k: v.clone().requires_grad_(True) for k, v in L.items()}
    try:
        noisy = O.flow_noisy_latents(lat.bfloat16(), noise.bfloat16(), sig).float()
        with MO.masked(mask):
            pred_ref, t2 = kontext_model_predict(P, cfg, noisy, sig * 1000.0, batch["prompt_embeds"].float(),
                                                 batch["add_text_embeds"].float(), [c.float() for c in conds], 1.0, Lg, 1.0)
        loss_ref = O.flow_loss(pred_ref, O.flow_target(lat.bfloat16(), noise.bfloat16()))
        loss_ref.backward()
    finally:
        O.DROPOUT_MASKS = None
        O.LOKR = {"linear_dim": 10000, "linear_alpha": 1, "multiplier": 1.0}
    pred = w.unpacked_prediction(out).float().cpu()
    res = {"loss": float(loss.item()), "loss_ref": float(loss_ref.item()),
           "loss_rel_err": abs(float(loss.item()) - float(loss_ref.item())) / abs(float(loss_ref.item())),
           "pred_cos": float(F.cosine_similarity(pred.flatten(), pred_ref.detach().flatten(), dim=0)),
           # the reference form: t / 1000 over the scene tokens, exactly 0 over the conditioning tokens (the CUDA path divides
           # on the device, the oracle on the host: the scene values may differ in the last fp32 bit)
           "timesteps_match": bool(prepared["timesteps"].shape == t2.shape and not prepared["timesteps"][:, S_scene:].any()
                                   and torch.allclose(prepared["timesteps"].cpu(), t2, rtol=1e-6, atol=0)),
           "S_c": S_c}
    cos_min, worst, rel_max = 1.0, None, 0.0
    gmax = max(float(Lg[n].grad.norm()) for n in params)
    for name, p in params.items():
        gref = Lg[name].grad
        if lokr is not None and float(gref.norm()) < 1e-4 * gmax:
            continue        # below the bf16 noise floor of the backward pass (tests/test_flux_lokr_gpu.py)
        g = p.grad.float().cpu()
        c = _cos(g, gref)
        rel_max = max(rel_max, float((g - gref).norm() / (gref.norm() + 1e-12)))
        if c < cos_min:
            cos_min, worst = c, name
    res.update({"grad_cos_min": cos_min, "grad_worst": worst, "grad_rel_l2_max": rel_max, "n_tensors": len(params)})
    return res
