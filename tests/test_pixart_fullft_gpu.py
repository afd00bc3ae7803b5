"""GPU (-m gpu): PixArt-Sigma FULL fine-tune step (model_type=full) on libstb200 vs the fp32 CPU oracle with torch autograd:
prepare_batch -> model_predict -> loss -> backward with a gradient for EVERY parameter (attention and FeedForward weights and
biases in both attentions, the blocks' and the final scale_shift_table, PatchEmbed, caption projection, adaLN-single with
its size embedders, proj_out).  Then the trainer-facing surface: gradient checkpointing, gradient accumulation, the layout
rebuild after an optimizer step (TrainStep's own call, and the optimizer post-hook alone) and CUDA-graph replay.
Tolerances are the SD3 full fine-tune ones: loss / prediction as in tests/flux_parity.py; per-parameter gradient cosine
>= 0.995 for matrices, >= 0.99 for vectors."""
import pytest
import torch

from oracle import pixart_oracle as O
from tests import flux_parity as FP
from tests import pixart_parity as PP

pytestmark = pytest.mark.gpu

MAT_COS, VEC_COS = 0.995, 0.99


def _mask(B, S_txt, mode, g):
    if mode is None:
        return None
    mask = torch.ones(B, S_txt)
    if mode == "prefix":               # tokenizer padding on the right, a different length per sample
        for b in range(B):
            mask[b, max(1, S_txt // 3 + 7 * b):] = 0
        mask[B - 1] = 1
    else:                              # arbitrary keep-mask, including a fully masked leading tile
        mask = (torch.rand(B, S_txt, generator=g) > 0.4).float()
        mask[0, : S_txt // 2] = 0
        mask[:, -1] = 1
    return mask


def _setup(cfg, B=2, Hh=16, Ww=24, S_txt=40, seed=0, mask_mode="prefix"):
    P = {k: v.bfloat16().float() for k, v in O.init_pixart_params(cfg, seed=seed).items()}
    g = torch.Generator().manual_seed(seed + 2)
    batch = {"latent_batch": torch.randn(B, 4, Hh, Ww, generator=g).bfloat16(),
             "prompt_embeds": torch.randn(B, S_txt, cfg.caption_channels, generator=g).bfloat16()}
    mask = _mask(B, S_txt, mask_mode, g)
    if mask is not None:
        batch["encoder_attention_mask"] = mask
    return P, batch


def _full_model(cfg, P, checkpointing=False):
    w = PP.build_cuda_model(cfg, P, None)
    den = w._denoiser()
    den.enable_full_finetune()
    if checkpointing:
        den.enable_gradient_checkpointing()
    assert all(p.requires_grad for p in den.parameters())
    return w


def _prepare(w, batch, seed=1234):
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)
    return w.prepare_batch({k: v.clone() for k, v in batch.items()}, {"global_step": 0})


def _backward(w, prepared):
    out = w.model_predict(prepared)
    loss = w.loss(prepared, out)
    loss.backward()
    torch.cuda.synchronize()
    return loss, out


def _oracle(cfg, P, w, steps):
    """fp32 autograd over the summed loss of `steps` = [(prepared, batch)]; returns (grads by name, last pred, last loss)."""
    Pg = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    ac = w.noise_schedule.alphas_cumprod
    for prepared, batch in steps:
        lat, noise = prepared["latents"].float().cpu(), prepared["noise"].float().cpu()
        t = prepared["timesteps"].cpu().long()
        noisy = O.ddpm_add_noise(ac, lat, noise, t)
        pred = O.pixart_model_predict(Pg, cfg, noisy.bfloat16().float(), t, batch["prompt_embeds"].float(),
                                      batch.get("encoder_attention_mask"))
        loss = O.eps_loss(pred, noise)
        loss.backward()
    return {k: v.grad for k, v in Pg.items()}, pred.detach(), loss.detach()


def _sigma_rows(cfg):
    """proj_out rows of the learned-sigma half ((dy, dx, c) row order, c >= out_channels / 2)."""
    Co = cfg.out_channels
    return torch.tensor([r for r in range(4 * Co) if r % Co >= Co // 2])


def _compare(den, cfg, G, tag, res):
    cos = torch.nn.functional.cosine_similarity
    worst_m, worst_v, missing, n = (1.0, None), (1.0, None), [], 0
    gmax = max(float(v.norm()) for v in G.values() if v is not None)
    for name, p in den.named_parameters():
        if p.grad is None:
            missing.append(name)
            continue
        gref = G[name]
        if gref is None or float(gref.norm()) < 1e-7 * gmax:
            continue
        n += 1
        c = float(cos(p.grad.float().cpu().flatten(), gref.flatten(), dim=0))
        if p.dim() >= 2:
            if c < worst_m[0]:
                worst_m = (c, name)
        elif c < worst_v[0]:
            worst_v = (c, name)
    rows = _sigma_rows(cfg).to(den.proj_out.weight.device)
    sigma_zero = bool((den.proj_out.weight.grad[rows] == 0).all()) and bool((den.proj_out.bias.grad[rows] == 0).all())
    res.update({"n_param_grads": n, "n_params": len(list(den.parameters())), "grad_cos_min_matrix": worst_m[0],
                "worst_matrix": worst_m[1], "grad_cos_min_vector": worst_v[0], "worst_vector": worst_v[1],
                "learned_sigma_grad_zero": sigma_zero})
    FP.record(tag, res)
    print(f"[{tag}]", res)
    assert not missing, missing
    assert sigma_zero, res
    assert res["grad_cos_min_matrix"] >= MAT_COS and res["grad_cos_min_vector"] >= VEC_COS, res


@pytest.mark.parametrize("case", [
    dict(cfg=dict(), B=3, mask_mode="prefix", seed=0),                                  # hd 72 -> 128, size conditioning
    dict(cfg=dict(sample_size=64), B=1, Hh=24, Ww=16, S_txt=150, mask_mode="holes", seed=4),   # no size conditioning
    dict(cfg=dict(heads=6, hd=64), B=3, Hh=16, Ww=16, S_txt=77, mask_mode=None, seed=7),  # head width without padding
], ids=["hd72_prefix_b3", "hd72_holes_b1_no_size_cond", "hd64_unpadded_b3"])
def test_pixart_full_finetune_parity(case):
    cfg = PP.small_config(**case["cfg"])
    kw = {k: v for k, v in case.items() if k != "cfg"}
    P, batch = _setup(cfg, **kw)
    w = _full_model(cfg, P)
    prepared = _prepare(w, batch)
    loss, out = _backward(w, prepared)
    G, pred_ref, loss_ref = _oracle(cfg, P, w, [(prepared, batch)])
    pred = w.unpacked_prediction(out).detach().float().cpu()
    res = {"loss_rel_err": abs(float(loss) - float(loss_ref)) / abs(float(loss_ref)),
           "pred_cos": float(torch.nn.functional.cosine_similarity(pred.flatten(), pred_ref.flatten(), dim=0))}
    assert res["loss_rel_err"] <= FP.LOSS_RTOL and res["pred_cos"] >= FP.PRED_COS, res
    _compare(w._denoiser(), cfg, G, "pixart_fullft_" + "_".join(f"{k}{v}" for k, v in kw.items()), res)


def test_pixart_full_finetune_checkpointing_gives_the_same_bits():
    cfg = PP.small_config(layers=3)
    P, batch = _setup(cfg, B=2, seed=11)
    grads, outs = [], []
    for ckpt in (False, True):
        w = _full_model(cfg, P, checkpointing=ckpt)
        prepared = _prepare(w, batch)
        loss, out = _backward(w, prepared)
        outs.append((float(loss), out["model_prediction"].detach().clone()))
        grads.append({n: p.grad.clone() for n, p in w._denoiser().named_parameters()})
    assert outs[0][0] == outs[1][0] and torch.equal(outs[0][1], outs[1][1])
    assert grads[0].keys() == grads[1].keys()
    diff = [n for n in grads[0] if not torch.equal(grads[0][n], grads[1][n])]
    assert not diff, diff


def test_pixart_full_finetune_gradient_accumulation():
    """Two micro-steps accumulate into the live .grad tensors: the sum matches the oracle's summed gradient."""
    cfg = PP.small_config()
    P, batch = _setup(cfg, B=2, seed=3)
    w = _full_model(cfg, P)
    steps = []
    for seed in (21, 22):
        prepared = _prepare(w, batch, seed=seed)
        _backward(w, prepared)
        steps.append((prepared, batch))
    G, _, _ = _oracle(cfg, P, w, steps)
    _compare(w._denoiser(), cfg, G, "pixart_fullft_accum2", {})


def _fresh_forward(cfg, den, prepared):
    """The prediction of a newly built full fine-tune model loaded with `den`'s state dict."""
    from simpletuner_b200.pixart.model import PixartSigma, default_config
    from simpletuner_b200.pixart.transformer import PixArtTransformer2DModel
    m = PixArtTransformer2DModel.from_config(den.config)
    m.load_state_dict({k: v.clone() for k, v in den.state_dict().items()})
    m.to("cuda").enable_full_finetune()
    w = PixartSigma(default_config(), transformer=m, device=torch.device("cuda"))
    return w.model_predict(prepared)["model_prediction"].detach()


def test_pixart_full_finetune_layouts_follow_the_optimizer():
    from simpletuner_b200.shim import track_full_finetune
    from simpletuner_b200.training.optim import AdamWBF16
    from simpletuner_b200.training.step import TrainStep

    cfg = PP.small_config()
    P, batch = _setup(cfg, B=2, seed=5)
    probe = _prepare(_full_model(cfg, P), batch, seed=99)
    # TrainStep: its explicit after_optimizer_step() call
    w = _full_model(cfg, P)
    den = w._denoiser()
    step = TrainStep(w, AdamWBF16(list(den.parameters()), lr=1e-3, weight_decay=0.01, seed=3), max_grad_norm=2.0)
    w0 = den.transformer_blocks[0].attn1.to_q.weight.detach().clone()
    torch.manual_seed(5)
    torch.cuda.manual_seed(5)
    step({k: v.clone() for k, v in batch.items()})
    assert not torch.equal(w0, den.transformer_blocks[0].attn1.to_q.weight)
    assert torch.equal(w.model_predict(probe)["model_prediction"].detach(), _fresh_forward(cfg, den, probe))
    # a plain torch optimizer: only the process-wide post-hook rebuilds the layouts
    w = _full_model(cfg, P)
    den = w._denoiser()
    track_full_finetune(den)
    opt = torch.optim.AdamW(den.parameters(), lr=1e-3)
    _backward(w, _prepare(w, batch))
    assert den.transformer_blocks[0]._plans is not None
    opt.step()
    assert all(blk._plans is None for blk in den.transformer_blocks) and not den._tail_plan
    assert torch.equal(w.model_predict(probe)["model_prediction"].detach(), _fresh_forward(cfg, den, probe))


def test_pixart_full_finetune_graph_replay_matches_eager():
    """GraphedTrainStep replays the full fine-tune step (the layout rebuild is part of the captured graph): three steps
    give the same losses and parameters, bit for bit, as the eager TrainStep."""
    from simpletuner_b200.training.optim import AdamWBF16
    from simpletuner_b200.training.step import GraphedTrainStep, TrainStep

    cfg = PP.small_config()
    P, batch = _setup(cfg, B=2, seed=8)
    runs = []
    for graphed in (False, True):
        w = _full_model(cfg, P)
        den = w._denoiser()
        step = TrainStep(w, AdamWBF16(list(den.parameters()), lr=1e-3, weight_decay=0.01, seed=3), max_grad_norm=2.0)
        if graphed:
            step = GraphedTrainStep(step, capture_prepare=False)
        losses = []
        for i in range(3):
            torch.manual_seed(100 + i)
            torch.cuda.manual_seed(100 + i)
            losses.append(float(step({k: v.clone() for k, v in batch.items()})))
        torch.cuda.synchronize()
        runs.append((losses, {n: p.detach().clone() for n, p in den.named_parameters()}))
    assert runs[0][0] == runs[1][0], (runs[0][0], runs[1][0])
    diff = [n for n in runs[0][1] if not torch.equal(runs[0][1][n], runs[1][1][n])]
    assert not diff, diff
