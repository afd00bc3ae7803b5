"""fp32 CPU oracle of the Chroma training step and the GPU parity harness for it.

A restatement of reference chroma/transformer.py (ChromaTransformer2DModel.forward :821-1311, the blocks :316-616, the
approximator :297-313) and chroma/model.py:605-716, on oracle/flux_oracle.py's `linear`, `rms_norm`, `layer_norm_noaffine`,
`apply_rope` and `rope_tables`, with the modulations passed to every block explicitly as rows of the approximator output.
The prompt mask is an additive per-key bias of 0 / -inf; the reference's outer-product mask also blanks the padded text
query rows, which differ here and never reach the loss.  The approximator input is `chroma_input_vec`, pinned bit for bit
against the reference's own code by tests/golden/chroma_golden.pt (tools/make_golden_chroma.py)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from oracle import flux_oracle as O
from simpletuner_b200.chroma.transformer import CHROMA_LORA_TARGETS, chroma_input_vec, chroma_mod_proj


@dataclass
class ChromaConfig:
    num_layers: int = 2
    num_single_layers: int = 2
    attention_head_dim: int = 128
    num_attention_heads: int = 2
    joint_attention_dim: int = 64
    approximator_hidden_dim: int = 128
    approximator_layers: int = 2
    in_channels: int = 64
    axes_dims_rope: Tuple[int, int, int] = (16, 56, 56)

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim

    @property
    def mod_rows(self) -> int:
        return 3 * self.num_single_layers + 12 * self.num_layers + 2

    def kwargs(self):
        return dict(num_layers=self.num_layers, num_single_layers=self.num_single_layers,
                    attention_head_dim=self.attention_head_dim, num_attention_heads=self.num_attention_heads,
                    joint_attention_dim=self.joint_attention_dim, approximator_hidden_dim=self.approximator_hidden_dim,
                    approximator_layers=self.approximator_layers, axes_dims_rope=self.axes_dims_rope)


ATTN = ("to_q", "to_k", "to_v", "to_out.0", "add_q_proj", "add_k_proj", "add_v_proj", "to_add_out")


def param_shapes(cfg: ChromaConfig) -> Dict[str, Tuple[int, ...]]:
    D, hd, Hd = cfg.inner_dim, cfg.attention_head_dim, cfg.approximator_hidden_dim
    s: Dict[str, Tuple[int, ...]] = {}

    def lin(n, o, i):
        s[n + ".weight"], s[n + ".bias"] = (o, i), (o,)

    a = "distilled_guidance_layer."
    lin(a + "in_proj", Hd, 64)
    for i in range(cfg.approximator_layers):
        lin(a + f"layers.{i}.linear_1", Hd, Hd)
        lin(a + f"layers.{i}.linear_2", Hd, Hd)
        s[a + f"norms.{i}.weight"] = (Hd,)
    lin(a + "out_proj", D, Hd)
    lin("context_embedder", D, cfg.joint_attention_dim)
    lin("x_embedder", D, 64)
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}."
        for n in ("norm_q", "norm_k", "norm_added_q", "norm_added_k"):
            s[p + f"attn.{n}.weight"] = (hd,)
        for n in ATTN:
            lin(p + "attn." + n, D, D)
        for st in ("ff", "ff_context"):
            lin(p + st + ".net.0.proj", 4 * D, D)
            lin(p + st + ".net.2", D, 4 * D)
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}."
        lin(p + "proj_mlp", 4 * D, D)
        lin(p + "proj_out", D, 5 * D)
        s[p + "attn.norm_q.weight"], s[p + "attn.norm_k.weight"] = (hd,), (hd,)
        for n in ("to_q", "to_k", "to_v"):
            lin(p + "attn." + n, D, D)
    lin("proj_out", 64, D)
    return s


def init_params(cfg: ChromaConfig, seed=0, std=0.02) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    out = {}
    for n, shp in param_shapes(cfg).items():
        if "norm" in n and n.endswith(".weight") and len(shp) == 1:
            t = 1.0 + 0.05 * torch.randn(shp, generator=g)
        elif n.startswith("distilled_guidance_layer") and n.endswith(".weight"):
            t = torch.randn(shp, generator=g) * shp[1] ** -0.5       # modulations of order 1, as a trained approximator's
        elif n.endswith(".bias"):
            t = 0.5 * std * torch.randn(shp, generator=g)
        else:
            t = std * torch.randn(shp, generator=g)
        out[n] = t
    return out


def lora_names(cfg: ChromaConfig, targets):
    return [k[:-7] for k, v in param_shapes(cfg).items() if k.endswith(".weight") and len(v) == 2
            and any(k[:-7] == t or k[:-7].endswith("." + t) for t in targets)]


def init_lora(cfg: ChromaConfig, rank: int, targets, seed=1, b_std=0.02):
    g = torch.Generator().manual_seed(seed)
    shapes, out = param_shapes(cfg), {}
    for n in lora_names(cfg, targets):
        o, k = shapes[n + ".weight"]
        out[n + ".lora_A.weight"] = (torch.rand((rank, k), generator=g) * 2 - 1) / math.sqrt(k)
        out[n + ".lora_B.weight"] = b_std * torch.randn((o, rank), generator=g)
    return out


def approximator(P, cfg: ChromaConfig, x: torch.Tensor) -> torch.Tensor:
    """ChromaApproximator.forward in fp32 (nn.RMSNorm with eps=None: torch.finfo(float32).eps)."""
    a = "distilled_guidance_layer."
    lin = lambda t, n: F.linear(t, P[a + n + ".weight"], P[a + n + ".bias"])
    h = lin(x, "in_proj")
    for i in range(cfg.approximator_layers):
        n = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + torch.finfo(torch.float32).eps) * P[a + f"norms.{i}.weight"]
        h = h + lin(F.silu(lin(n, f"layers.{i}.linear_1")), f"layers.{i}.linear_2")
    return lin(h, "out_proj")


def _attention(P, cfg, p, x, enc, cosin, bias, lora, ls):
    H, hd = cfg.num_attention_heads, cfg.attention_head_dim
    B = x.shape[0]

    def heads(t):
        return t.view(B, -1, H, hd).transpose(1, 2)
    q = O.rms_norm(heads(O.linear(x, P, p + "to_q", lora, ls)), P[p + "norm_q.weight"], 1e-6)
    k = O.rms_norm(heads(O.linear(x, P, p + "to_k", lora, ls)), P[p + "norm_k.weight"], 1e-6)
    v = heads(O.linear(x, P, p + "to_v", lora, ls))
    if enc is not None:
        eq = O.rms_norm(heads(O.linear(enc, P, p + "add_q_proj", lora, ls)), P[p + "norm_added_q.weight"], 1e-6)
        ek = O.rms_norm(heads(O.linear(enc, P, p + "add_k_proj", lora, ls)), P[p + "norm_added_k.weight"], 1e-6)
        ev = heads(O.linear(enc, P, p + "add_v_proj", lora, ls))
        q, k, v = (torch.cat([a, b], 2) for a, b in ((eq, q), (ek, k), (ev, v)))
    cos, sin = cosin
    q, k = O.apply_rope(q, cos, sin), O.apply_rope(k, cos, sin)
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    if bias is not None:
        s = s + bias[:, None, None, :]
    o = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, -1, H * hd)
    if enc is None:
        return o
    S_txt = enc.shape[1]
    return O.linear(o[:, S_txt:], P, p + "to_out.0", lora, ls), O.linear(o[:, :S_txt], P, p + "to_add_out", lora, ls)


def _mod(t, sh, sc):
    return O.layer_norm_noaffine(t) * (1 + sc[:, None]) + sh[:, None]


def double_block(P, cfg, i, x, enc, im, tm, cosin, bias, lora, ls):
    """ChromaTransformerBlock.forward; im / tm: the six image / text modulation rows [B, 6, D]."""
    p = f"transformer_blocks.{i}."
    im, tm = im.unbind(1), tm.unbind(1)
    ao, eo = _attention(P, cfg, p + "attn.", _mod(x, im[0], im[1]), _mod(enc, tm[0], tm[1]), cosin, bias, lora, ls)
    x = x + im[2][:, None] * ao
    enc = enc + tm[2][:, None] * eo
    ff = lambda t, s: O.linear(F.gelu(O.linear(t, P, p + s + ".net.0.proj", lora, ls), approximate="tanh"), P,
                               p + s + ".net.2", lora, ls)
    x = x + im[5][:, None] * ff(_mod(x, im[3], im[4]), "ff")
    enc = enc + tm[5][:, None] * ff(_mod(enc, tm[3], tm[4]), "ff_context")
    return x, enc


def single_block(P, cfg, i, h, m, cosin, bias, lora, ls):
    p = f"single_transformer_blocks.{i}."
    sh, sc, gate = m.unbind(1)
    nx = _mod(h, sh, sc)
    ao = _attention(P, cfg, p + "attn.", nx, None, cosin, bias, lora, ls)
    mlp = F.gelu(O.linear(nx, P, p + "proj_mlp", lora, ls), approximate="tanh")
    return h + gate[:, None] * O.linear(torch.cat([ao, mlp], 2), P, p + "proj_out", lora, ls)


def forward(P, cfg, hidden, enc_hs, t, joint_mask, Hh, Ww, lora=None, ls=1.0):
    """ChromaTransformer2DModel.forward on packed tokens [B, S_img, 64]; t [B] as model_predict passes it (bf16 t / 1000)."""
    B, S_img, _ = hidden.shape
    x = O.linear(hidden, P, "x_embedder", lora, ls)
    vec = chroma_input_vec(t.to(torch.bfloat16) * 1000, chroma_mod_proj(cfg.mod_rows, 16))
    pooled = approximator(P, cfg, vec.float())
    enc = O.linear(enc_hs, P, "context_embedder")
    S_txt = enc.shape[1]
    ids = torch.cat([torch.zeros(S_txt, 3), O.prepare_latent_image_ids(Hh, Ww)], 0)
    cosin = O.rope_tables(ids, cfg.axes_dims_rope)
    bias = torch.zeros(B, S_txt + S_img).masked_fill(~joint_mask.cpu(), float("-inf"))
    i0, t0 = 3 * cfg.num_single_layers, 3 * cfg.num_single_layers + 6 * cfg.num_layers
    for i in range(cfg.num_layers):
        x, enc = double_block(P, cfg, i, x, enc, pooled[:, i0 + 6 * i:i0 + 6 * i + 6], pooled[:, t0 + 6 * i:t0 + 6 * i + 6],
                              cosin, bias, lora, ls)
    h = torch.cat([enc, x], 1)
    for i in range(cfg.num_single_layers):
        h = single_block(P, cfg, i, h, pooled[:, 3 * i:3 * i + 3], cosin, bias, lora, ls)
    shift, scale = pooled[:, -2], pooled[:, -1]
    return O.linear(_mod(h[:, S_txt:], shift, scale), P, "proj_out", lora, ls)


def model_predict(P, cfg, noisy, timesteps, prompt_embeds, mask, lora=None, ls=1.0):
    """_model_predict_single: timesteps are the batch's (adjusted sigma x 1000, bf16)."""
    B, C, Hh, Ww = noisy.shape
    packed = O.pack_latents(noisy, B, C, Hh, Ww)
    t = timesteps.to(torch.bfloat16) / 1000
    joint = torch.cat([mask.cpu() > 0, torch.ones(B, packed.shape[1], dtype=torch.bool)], 1)
    out = forward(P, cfg, packed, prompt_embeds, t, joint, Hh, Ww, lora, ls)
    return O.unpack_latents(out, Hh * 8, Ww * 8, 16)


# ---- GPU parity harness ------------------------------------------------------------------------------------------------
def build_cuda(cfg, P, L, rank, targets, dropout=0.0, device="cuda", **config):
    from simpletuner_b200.chroma.model import Chroma, default_config
    from simpletuner_b200.chroma.transformer import ChromaTransformer2DModel
    m = ChromaTransformer2DModel(**cfg.kwargs())
    m.load_state_dict({k: v.bfloat16() for k, v in P.items()}, strict=True)
    m.to(device)
    w = Chroma(default_config(lora_rank=rank, lora_dropout=dropout, flux_lora_target=targets, **config), transformer=m,
               device=torch.device(device))
    w.add_lora_adapter()
    with torch.no_grad():
        for name, lin in m.lora_linears().items():
            lin.lora_A["default"].weight.copy_(L[name + ".lora_A.weight"].bfloat16())
            lin.lora_B["default"].weight.copy_(L[name + ".lora_B.weight"].bfloat16())
    return w


def ragged_mask(B, S_txt, lens):
    return (torch.arange(S_txt)[None] < torch.tensor(lens)[:, None]).long()


def make_batch(B, Hh, Ww, mask, cfg, seed=2):
    g = torch.Generator().manual_seed(seed)
    S_txt = mask.shape[1]
    emb = torch.randn(B, S_txt, cfg.joint_attention_dim, generator=g) * (mask[:, :, None] != 0)     # T5 zero-pads
    return {"latent_batch": torch.randn(B, 16, Hh, Ww, generator=g).bfloat16(), "prompt_embeds": emb.bfloat16(),
            "encoder_attention_mask": mask.clone()}


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


def run_parity(cfg=None, B=2, Hh=16, Ww=16, lens=(24, 9), S_txt=32, targets="all", rank=16, dropout=0.0, checkpoint=False,
               seed=0, loss_type="l2"):
    cfg = cfg or ChromaConfig()
    tl = CHROMA_LORA_TARGETS[targets]
    P = {k: v.bfloat16().float() for k, v in init_params(cfg, seed).items()}
    L = {k: v.bfloat16().float() for k, v in init_lora(cfg, rank, tl, seed + 1).items()}
    w = build_cuda(cfg, P, L, rank, targets, dropout, loss_type=loss_type)
    mask = ragged_mask(B, S_txt, lens[:B])
    batch = make_batch(B, Hh, Ww, mask, cfg, seed + 2)
    prepared, out, loss, grads = run_step(w, batch, checkpoint)
    if dropout:
        from tests.test_lora_dropout_gpu import _masks_for_flux
        O.DROPOUT_MASKS = _masks_for_flux(w._denoiser(), cfg, B, (Hh // 2) * (Ww // 2), S_txt, dropout)
    lat, noise = prepared["latents"].float().cpu(), prepared["noise"].float().cpu()
    sig = prepared["sigmas"].flatten().float().cpu()
    Lg = {k: v.clone().requires_grad_(True) for k, v in L.items()}
    try:
        noisy = O.flow_noisy_latents(lat.bfloat16(), noise.bfloat16(), sig).float()
        pred_ref = model_predict(P, cfg, noisy, prepared["timesteps"].cpu(), batch["prompt_embeds"].float(), mask, Lg, 1.0)
        loss_ref = O.model_loss(pred_ref, O.flow_target(lat.bfloat16(), noise.bfloat16()), loss_type, huber_c=0.1)
        loss_ref.backward()
    finally:
        O.DROPOUT_MASKS = None
    pred = w.unpacked_prediction(out).float().cpu()
    res = {"loss": float(loss), "loss_ref": float(loss_ref.detach()),
           "loss_rel_err": abs(float(loss) - float(loss_ref)) / abs(float(loss_ref)),
           "pred_cos": float(F.cosine_similarity(pred.flatten(), pred_ref.detach().flatten(), dim=0))}
    cmin, worst = 1.0, None
    for n, gr in grads.items():
        ref = Lg[n].grad
        if ref is None or not bool(ref.any()):
            if bool(gr.any()):
                cmin, worst = -1.0, n
            continue
        c = _cos(gr.float().cpu(), ref)
        if c < cmin:
            cmin, worst = c, n
    res.update({"grad_cos_min": cmin, "grad_worst": worst, "n_tensors": len(grads)})
    return res
