"""fp32 CPU oracle of the Qwen-Image text-to-image training step and the GPU parity harness for it.

A restatement of reference qwen_image/transformer.py (QwenImageTransformer2DModel.forward :1208-1500, the block :912-997,
QwenDoubleStreamAttnProcessor2_0 :662-821) and qwen_image/model.py:1227-1345, on oracle/flux_oracle.py's `linear`,
`rms_norm`, `layer_norm_noaffine` and `apply_rope`.  The prompt mask is an additive per-key bias of 0 / -inf
(`key_bias`); the reference's B > 1 path instead slices each sample's first `sum(mask)` text tokens and zeroes the padded
text query rows before to_add_out.  The two agree on every image row and every kept text row; padded text query rows
differ and never reach the loss (masked keys carry P = 0, so their dK = dV = 0 and nothing reads their values).  Pinned
against the reference's own functions by tests/golden/qwen_image_golden.pt (tools/make_golden_qwen_image.py)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from oracle import flux_oracle as O


@dataclass
class QwenConfig:
    num_layers: int = 3
    attention_head_dim: int = 128
    num_attention_heads: int = 2
    joint_attention_dim: int = 192
    axes_dims_rope: Tuple[int, int, int] = (16, 56, 56)

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim


ATTN = ("to_q", "to_k", "to_v", "to_out.0", "add_q_proj", "add_k_proj", "add_v_proj", "to_add_out")
MLP = ("img_mlp.net.0.proj", "img_mlp.net.2", "txt_mlp.net.0.proj", "txt_mlp.net.2")
TARGETS = {"default": ("to_k", "to_q", "to_v", "to_out.0"), "attn": ATTN, "attn+mlp": ATTN + MLP}


def param_shapes(cfg: QwenConfig) -> Dict[str, Tuple[int, ...]]:
    D, hd = cfg.inner_dim, cfg.attention_head_dim
    s: Dict[str, Tuple[int, ...]] = {}

    def lin(n, o, i):
        s[n + ".weight"], s[n + ".bias"] = (o, i), (o,)

    lin("img_in", D, 64)
    s["txt_norm.weight"] = (cfg.joint_attention_dim,)
    lin("txt_in", D, cfg.joint_attention_dim)
    lin("time_text_embed.timestep_embedder.linear_1", D, 256)
    lin("time_text_embed.timestep_embedder.linear_2", D, D)
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}."
        lin(p + "img_mod.1", 6 * D, D)
        lin(p + "txt_mod.1", 6 * D, D)
        for n in ATTN:
            lin(p + "attn." + n, D, D)
        for n in ("norm_q", "norm_k", "norm_added_q", "norm_added_k"):
            s[p + f"attn.{n}.weight"] = (hd,)
        for st in ("img_mlp", "txt_mlp"):
            lin(p + st + ".net.0.proj", 4 * D, D)
            lin(p + st + ".net.2", D, 4 * D)
    lin("norm_out.linear", 2 * D, D)
    lin("proj_out", 64, D)
    return s


def init_params(cfg: QwenConfig, seed=0, std=0.02) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    out = {}
    for n, shp in param_shapes(cfg).items():
        if "norm" in n and n.endswith(".weight") and len(shp) == 1:
            t = 1.0 + 0.05 * torch.randn(shp, generator=g)
        elif n.endswith(".bias"):
            t = 0.5 * std * torch.randn(shp, generator=g)
        else:
            t = std * torch.randn(shp, generator=g)
        out[n] = t
    return out


def lora_names(cfg: QwenConfig, targets):
    return [k[:-7] for k, v in param_shapes(cfg).items() if k.endswith(".weight") and len(v) == 2
            and any(k[:-7] == t or k[:-7].endswith("." + t) for t in targets)]


def init_lora(cfg: QwenConfig, rank: int, targets, seed=1, b_std=0.02):
    g = torch.Generator().manual_seed(seed)
    shapes, out = param_shapes(cfg), {}
    for n in lora_names(cfg, targets):
        o, k = shapes[n + ".weight"]
        out[n + ".lora_A.weight"] = (torch.rand((rank, k), generator=g) * 2 - 1) / math.sqrt(k)
        out[n + ".lora_B.weight"] = b_std * torch.randn((o, rank), generator=g)
    return out


def timestep_proj(t: torch.Tensor) -> torch.Tensor:
    """t rounded to bf16 (reference :1295), then get_timestep_embedding(flip_sin_to_cos, shift 0, scale=1000)."""
    half = 128
    freqs = torch.exp(-math.log(10000) * torch.arange(0, half, dtype=torch.float32) / half)
    emb = 1000 * (t.to(torch.bfloat16).float()[:, None] * freqs[None, :])
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


def rope(h: int, w: int, S_txt: int, axes=(16, 56, 56), theta=10000):
    """(cos, sin) [S_txt + h w, sum(axes)]: text rows first at max(h//2, w//2) + i, then the centred image grid."""
    def freqs(idx, d):
        f = torch.outer(idx.float(), 1.0 / torch.pow(theta, torch.arange(0, d, 2).float().div(d)))
        return torch.polar(torch.ones_like(f), f)
    yy, xx = torch.meshgrid(torch.arange(h) - (h - h // 2), torch.arange(w) - (w - w // 2), indexing="ij")
    img = torch.cat([freqs(torch.zeros(h * w), axes[0]), freqs(yy.reshape(-1), axes[1]), freqs(xx.reshape(-1), axes[2])], 1)
    pos = torch.arange(S_txt) + max(h // 2, w // 2)
    txt = torch.cat([freqs(pos, d) for d in axes], 1)
    f = torch.cat([txt, img], 0)
    return f.real.repeat_interleave(2, -1), f.imag.repeat_interleave(2, -1)


def key_bias(mask: Optional[torch.Tensor], B: int, S_txt: int, S_img: int) -> Optional[torch.Tensor]:
    """[B, S_txt + S_img] fp32 0 / -inf: B == 1 keeps the set positions, B > 1 the first max(sum, 1) positions."""
    if mask is None:
        return None
    m = mask.reshape(B, S_txt).cpu() != 0
    if B > 1:
        n = m.sum(1, keepdim=True).clamp_min(1)
        m = torch.arange(S_txt)[None] < n
    bias = torch.zeros(B, S_txt + S_img)
    bias[:, :S_txt][~m] = float("-inf")
    return bias


def attention(P, cfg, p, x, enc, cosin, bias, lora, ls):
    """Joint [text | image] attention of one block (QwenDoubleStreamAttnProcessor2_0 with an additive key bias)."""
    H, hd = cfg.num_attention_heads, cfg.attention_head_dim
    B, S_txt = x.shape[0], enc.shape[1]

    def heads(t):
        return t.view(B, -1, H, hd).transpose(1, 2)
    q = O.rms_norm(heads(O.linear(x, P, p + "to_q", lora, ls)), P[p + "norm_q.weight"], 1e-6)
    k = O.rms_norm(heads(O.linear(x, P, p + "to_k", lora, ls)), P[p + "norm_k.weight"], 1e-6)
    v = heads(O.linear(x, P, p + "to_v", lora, ls))
    eq = O.rms_norm(heads(O.linear(enc, P, p + "add_q_proj", lora, ls)), P[p + "norm_added_q.weight"], 1e-6)
    ek = O.rms_norm(heads(O.linear(enc, P, p + "add_k_proj", lora, ls)), P[p + "norm_added_k.weight"], 1e-6)
    ev = heads(O.linear(enc, P, p + "add_v_proj", lora, ls))
    cos, sin = cosin
    q, k, v = (torch.cat([a, b], 2) for a, b in ((eq, q), (ek, k), (ev, v)))
    q, k = O.apply_rope(q, cos, sin), O.apply_rope(k, cos, sin)
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    if bias is not None:
        s = s + bias[:, None, None, :]
    o = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, -1, H * hd)
    return O.linear(o[:, S_txt:], P, p + "to_out.0", lora, ls), O.linear(o[:, :S_txt], P, p + "to_add_out", lora, ls)


def block(P, cfg, i, x, enc, temb, cosin, bias, lora, ls):
    p = f"transformer_blocks.{i}."
    im = F.linear(F.silu(temb), P[p + "img_mod.1.weight"], P[p + "img_mod.1.bias"]).chunk(6, 1)
    tm = F.linear(F.silu(temb), P[p + "txt_mod.1.weight"], P[p + "txt_mod.1.bias"]).chunk(6, 1)
    mod = lambda t, sh, sc: O.layer_norm_noaffine(t) * (1 + sc[:, None]) + sh[:, None]
    ao, eo = attention(P, cfg, p + "attn.", mod(x, im[0], im[1]), mod(enc, tm[0], tm[1]), cosin, bias, lora, ls)
    x = x + im[2][:, None] * ao
    enc = enc + tm[2][:, None] * eo
    ff = lambda t, s: O.linear(F.gelu(O.linear(t, P, p + s + ".net.0.proj", lora, ls), approximate="tanh"), P,
                               p + s + ".net.2", lora, ls)
    x = x + im[5][:, None] * ff(mod(x, im[3], im[4]), "img_mlp")
    enc = enc + tm[5][:, None] * ff(mod(enc, tm[3], tm[4]), "txt_mlp")
    return x, enc


def forward(P, cfg, hidden, enc_hs, mask, t, gh, gw, lora=None, ls=1.0):
    """QwenImageTransformer2DModel.forward on packed tokens [B, gh gw, 64]; t [B] in [0, 1]."""
    B, S_img, _ = hidden.shape
    x = O.linear(hidden, P, "img_in", lora, ls)
    tp = "time_text_embed.timestep_embedder."
    temb = F.linear(F.silu(F.linear(timestep_proj(t), P[tp + "linear_1.weight"], P[tp + "linear_1.bias"])),
                    P[tp + "linear_2.weight"], P[tp + "linear_2.bias"])
    enc = F.linear(O.rms_norm(enc_hs, P["txt_norm.weight"], 1e-6), P["txt_in.weight"], P["txt_in.bias"])
    cosin = rope(gh, gw, enc.shape[1], cfg.axes_dims_rope)
    bias = key_bias(mask, B, enc.shape[1], S_img)
    for i in range(cfg.num_layers):
        x, enc = block(P, cfg, i, x, enc, temb, cosin, bias, lora, ls)
    scale, shift = F.linear(F.silu(temb), P["norm_out.linear.weight"], P["norm_out.linear.bias"]).chunk(2, 1)
    x = O.layer_norm_noaffine(x) * (1 + scale[:, None]) + shift[:, None]
    return O.linear(x, P, "proj_out", lora, ls)


def model_predict(P, cfg, noisy, sigmas, prompt_embeds, mask, lora=None, ls=1.0):
    B, C, Hh, Ww = noisy.shape
    out = forward(P, cfg, O.pack_latents(noisy, B, C, Hh, Ww), prompt_embeds, mask, sigmas.float(), Hh // 2, Ww // 2, lora, ls)
    return O.unpack_latents(out, Hh * 8, Ww * 8, 16)


# ---- GPU parity harness ------------------------------------------------------------------------------------------------
def build_cuda(cfg, P, L, rank, targets, dropout=0.0, device="cuda", **config):
    from simpletuner_b200.qwen_image.model import QwenImage, default_config
    from simpletuner_b200.qwen_image.transformer import QwenImageTransformer2DModel
    m = QwenImageTransformer2DModel(num_layers=cfg.num_layers, attention_head_dim=cfg.attention_head_dim,
                                    num_attention_heads=cfg.num_attention_heads, joint_attention_dim=cfg.joint_attention_dim,
                                    axes_dims_rope=cfg.axes_dims_rope)
    m.load_state_dict({k: v.bfloat16() for k, v in P.items()}, strict=True)
    m.to(device)
    w = QwenImage(default_config(lora_rank=rank, lora_dropout=dropout, peft_lora_target_modules=list(targets), **config), transformer=m,
                  device=torch.device(device))
    w.add_lora_adapter()
    with torch.no_grad():
        for name, lin in m.lora_linears().items():
            lin.lora_A["default"].weight.copy_(L[name + ".lora_A.weight"].bfloat16())
            lin.lora_B["default"].weight.copy_(L[name + ".lora_B.weight"].bfloat16())
    return w


def make_batch(B, Hh, Ww, S_txt, cfg, mask=None, seed=2, five_d=False):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(B, 16, Hh, Ww, generator=g).bfloat16()
    b = {"latent_batch": lat.unsqueeze(2) if five_d else lat,
         "prompt_embeds": torch.randn(B, S_txt, cfg.joint_attention_dim, generator=g).bfloat16()}
    if mask is not None:
        b["prompt_embeds"] = b["prompt_embeds"] * (mask[:, :, None] != 0)      # collate zero-pads
        b["encoder_attention_mask"] = mask.clone()
    return b


def run_step(w, batch, checkpoint=False, seed=1234):
    den = w._denoiser()
    if checkpoint:
        den.enable_gradient_checkpointing()
    else:
        den.disable_gradient_checkpointing()
    den.train()
    for lin in den.lora_linears().values():
        lin.lora_A["default"].weight.grad = lin.lora_B["default"].weight.grad = None
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)
    prepared = w.prepare_batch({k: v.clone() for k, v in batch.items()}, {"global_step": 0})
    out = w.model_predict(prepared)
    loss = w.loss(prepared, out)
    loss.backward()
    torch.cuda.synchronize()
    grads = {f"{n}.{which}.weight": getattr(lin, which)["default"].weight.grad.clone()
             for n, lin in den.lora_linears().items() for which in ("lora_A", "lora_B")}
    return prepared, out, loss.detach(), grads


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float(a @ b / (a.norm() * b.norm()).clamp_min(1e-300))


def run_parity(cfg=None, B=2, Hh=16, Ww=16, S_txt=32, mask=None, targets="default", rank=16, dropout=0.0,
               checkpoint=False, seed=0, loss_type="l2"):
    cfg = cfg or QwenConfig()
    P = {k: v.bfloat16().float() for k, v in init_params(cfg, seed).items()}
    L = {k: v.bfloat16().float() for k, v in init_lora(cfg, rank, TARGETS[targets], seed + 1).items()}
    w = build_cuda(cfg, P, L, rank, TARGETS[targets], dropout, loss_type=loss_type)
    batch = make_batch(B, Hh, Ww, S_txt, cfg, mask, seed + 2)
    prepared, out, loss, grads = run_step(w, batch, checkpoint)
    if dropout:
        O.DROPOUT_MASKS = _qwen_dropout_masks(w._denoiser(), cfg, B, (Hh // 2) * (Ww // 2), S_txt, dropout)
    lat, noise = prepared["latents"].float().cpu(), prepared["noise"].float().cpu()
    sig = prepared["sigmas"].flatten().float().cpu()
    Lg = {k: v.clone().requires_grad_(True) for k, v in L.items()}
    try:
        noisy = O.flow_noisy_latents(lat.bfloat16(), noise.bfloat16(), sig).float()
        pred_ref = model_predict(P, cfg, noisy, sig, batch["prompt_embeds"].float(), mask, Lg, 1.0)
        loss_ref = O.model_loss(pred_ref, O.flow_target(lat.bfloat16(), noise.bfloat16()), loss_type, huber_c=0.1)
        loss_ref.backward()
    finally:
        O.DROPOUT_MASKS = None
    pred = w.unpacked_prediction(out).float().cpu()
    loss_ref = loss_ref.detach()
    res = {"loss": float(loss), "loss_ref": float(loss_ref),
           "loss_rel_err": abs(float(loss) - float(loss_ref)) / abs(float(loss_ref)),
           "pred_cos": float(F.cosine_similarity(pred.flatten(), pred_ref.detach().flatten(), dim=0))}
    cmin, worst, n_dead = 1.0, None, 0
    for n, gr in grads.items():
        if Lg[n].grad is None or not bool(Lg[n].grad.any()):
            # the last block's text rows feed nothing (no single blocks follow), so its text queries, to_add_out and text
            # MLP have no gradient: the CUDA gradient must be exactly 0 there
            n_dead += 1
            if bool(gr.any()):
                cmin, worst = -1.0, n
            continue
        c = _cos(gr.float().cpu(), Lg[n].grad)
        if c < cmin:
            cmin, worst = c, n
    res.update({"grad_cos_min": cmin, "grad_worst": worst, "n_tensors": len(grads), "n_zero_by_structure": n_dead})
    return res


def _qwen_dropout_masks(den, cfg, B, S_img, S_txt, p):
    """The CUDA path's PEFT dropout masks of the last forward, regenerated as tests/test_lora_dropout_gpu.py does for
    Flux: the block's mask streams are numbered as flux/blocks.DoubleBlockFn draws them (image q|k|v 0..2, fc1 3, fc2 4,
    out 6; text +8)."""
    from simpletuner_b200 import ops
    D = cfg.inner_dim

    def grab(S, drop, members, K=D):
        ones = torch.ones(B, S, K, device="cuda", dtype=torch.bfloat16)
        return ops.dropout_expand(ones, members, drop.p, drop.seed, drop.stream).float().cpu()

    masks = {}
    for i, blk in enumerate(den.transformer_blocks):
        drop = blk._lora_drop
        pre = f"transformer_blocks.{i}."
        for names, S, off in ((("to_q", "to_k", "to_v"), S_img, 0), (("add_q_proj", "add_k_proj", "add_v_proj"), S_txt, 8)):
            m = grab(S, drop.at(off), 3)
            for j, n in enumerate(names):
                masks[pre + "attn." + n] = m[j]
        masks[pre + "attn.to_out.0"] = grab(S_img, drop.at(6), 1)[0]
        masks[pre + "attn.to_add_out"] = grab(S_txt, drop.at(14), 1)[0]
        for nm, S, off, K in (("img_mlp.net.0.proj", S_img, 3, D), ("img_mlp.net.2", S_img, 4, 4 * D),
                              ("txt_mlp.net.0.proj", S_txt, 11, D), ("txt_mlp.net.2", S_txt, 12, 4 * D)):
            masks[pre + nm] = grab(S, drop.at(off), 1, K)[0]
    return masks
