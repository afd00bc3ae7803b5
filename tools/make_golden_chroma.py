"""Writes tests/golden/chroma_golden.pt: the reference's own Chroma functions on small inputs.

Runs, lifted from a SimpleTuner checkout by oracle/ref_extract (chroma/transformer.py, chroma/model.py,
flux/__init__.py), with torch stand-ins for the diffusers layers (`Timesteps` / `get_timestep_embedding`,
`PixArtAlphaTextProjection`, FluxAttention / FeedForward / FluxPosEmbed parameter holders):
  * `ChromaCombinedTimestepTextProjEmbeddings` (:263-294): the `mod_proj` buffer and the approximator input for bf16
    timesteps that went through the model's `timestep.to(dtype) * 1000` (:857);
  * `ChromaApproximator` (:297-313) at a small width, in fp32 and in bf16 (nn.RMSNorm with eps=None);
  * the three pruned norms (:133-260): which chunk of the modulation rows is shift, scale and gate;
  * `Chroma._adjust_chroma_sigmas` (model.py:309-314) in bf16 and fp32;
  * `Chroma._model_predict_single` (model.py:605-716) with the model replaced by a recorder: the extended attention mask
    and the timesteps the denoiser receives, for 2-D and 3-D masks;
  * the parameter names and shapes of `ChromaTransformer2DModel.__init__` (:650-762) at a small config.

    SIMPLETUNER_SRC=<SimpleTuner checkout> python tools/make_golden_chroma.py
"""
from __future__ import annotations

import math
import sys
import types
from pathlib import Path

import torch
import torch.nn as nn

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import ref_extract as R  # noqa: E402

OUT = ROOT / "tests" / "golden" / "chroma_golden.pt"
TR = "helpers/models/chroma/transformer.py"
MD = "helpers/models/chroma/model.py"


def get_timestep_embedding(timesteps, embedding_dim, flip_sin_to_cos=False, downscale_freq_shift=1, scale=1,
                           max_period=10000):
    half = embedding_dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32, device=timesteps.device)
    exponent = exponent / (half - downscale_freq_shift)
    emb = timesteps[:, None].float() * torch.exp(exponent)[None, :]
    emb = scale * emb
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
    return emb


class Timesteps(nn.Module):
    def __init__(self, num_channels, flip_sin_to_cos, downscale_freq_shift, scale=1):
        super().__init__()
        self.c, self.flip, self.shift, self.scale = num_channels, flip_sin_to_cos, downscale_freq_shift, scale

    def forward(self, t):
        return get_timestep_embedding(t, self.c, self.flip, self.shift, self.scale)


class PixArtAlphaTextProjection(nn.Module):
    def __init__(self, in_features, hidden_size, out_features=None, act_fn="gelu_tanh"):
        super().__init__()
        assert act_fn == "silu"
        self.linear_1 = nn.Linear(in_features, hidden_size, bias=True)
        self.act_1 = nn.SiLU()
        self.linear_2 = nn.Linear(hidden_size, out_features or hidden_size, bias=True)

    def forward(self, caption):
        return self.linear_2(self.act_1(self.linear_1(caption)))


class _RMS(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))


class FluxAttention(nn.Module):
    """diffusers FluxAttention parameter holder (bias=True, qk RMSNorm)."""

    def __init__(self, query_dim, heads=8, dim_head=64, dropout=0.0, bias=False, added_kv_proj_dim=None,
                 added_proj_bias=True, out_bias=True, eps=1e-5, out_dim=None, context_pre_only=None, pre_only=False,
                 processor=None):
        super().__init__()
        inner = dim_head * heads
        self.norm_q, self.norm_k = _RMS(dim_head), _RMS(dim_head)
        self.to_q, self.to_k, self.to_v = (nn.Linear(query_dim, inner, bias=bias) for _ in range(3))
        if not pre_only:
            self.to_out = nn.ModuleList([nn.Linear(inner, out_dim, bias=out_bias), nn.Dropout(dropout)])
        if added_kv_proj_dim is not None:
            self.norm_added_q, self.norm_added_k = _RMS(dim_head), _RMS(dim_head)
            self.add_q_proj, self.add_k_proj, self.add_v_proj = (nn.Linear(added_kv_proj_dim, inner, bias=added_proj_bias)
                                                                 for _ in range(3))
            self.to_add_out = nn.Linear(inner, query_dim, bias=out_bias)


class FeedForward(nn.Module):
    class _Proj(nn.Module):
        def __init__(self, d, inner):
            super().__init__()
            self.proj = nn.Linear(d, inner)

    def __init__(self, dim, dim_out=None, activation_fn="geglu"):
        super().__init__()
        self.net = nn.ModuleList([self._Proj(dim, 4 * dim), nn.Dropout(0.0), nn.Linear(4 * dim, dim_out)])


def _forward_row_offsets(ns, n_double=2, n_single=3):
    """The rows of `pooled_temb` each block and norm_out receive in the reference's own
    ChromaTransformer2DModel.forward (:821-1311): the approximator is replaced by one whose output row r holds the value r,
    and the blocks / norm_out record the rows they are given."""
    seen = {"double": [], "single": [], "norm_out": None}
    rows = 3 * n_single + 12 * n_double + 2

    class Double(nn.Module):
        def forward(self, hidden_states, encoder_hidden_states, image_temb, text_temb, **k):
            seen["double"].append((image_temb[0, :, 0].tolist(), text_temb[0, :, 0].tolist()))
            return encoder_hidden_states, hidden_states

    class Single(nn.Module):
        def forward(self, hidden_states, temb, **k):
            seen["single"].append(temb[0, :, 0].tolist())
            return hidden_states

    class NormOut(nn.Module):
        def forward(self, x, emb):
            seen["norm_out"] = emb[0, :, 0].tolist()
            return x

    fwd_ns = dict(ns, USE_PEFT_BACKEND=False, scale_lora_layers=None, unscale_lora_layers=None, np=None,
                  _store_hidden_state=lambda *a, **k: None, adjust_rotary_embedding_dim=lambda r, d: r,
                  activation_offload_context=None, should_checkpoint_block=lambda *a: False,
                  apply_grounding_fuser=None, Transformer2DModelOutput=None,
                  _chroma_tokenwise_time_conditioning=lambda m, t: m(t))
    Fwd = R.methods(TR, "ChromaTransformer2DModel", ["forward"], extra_ns=fwd_ns)
    self = types.SimpleNamespace(
        x_embedder=lambda x: x, context_embedder=lambda x: x, pos_embed=lambda ids: (ids, ids),
        time_text_embed=lambda t: torch.zeros(t.shape[0], rows, 4),
        distilled_guidance_layer=lambda v: torch.arange(rows, dtype=torch.float32)[None, :, None].expand(v.shape[0], -1, 1),
        delta_distilled_guidance_layer=None, time_sign_embed=None, config=types.SimpleNamespace(attention_head_dim=None),
        _tread_routes=None, _tread_router=None, training=False, _musubi_block_swap=None, gradient_checkpointing=False,
        gradient_checkpointing_offload_attention=False, transformer_blocks=[Double() for _ in range(n_double)],
        single_transformer_blocks=[Single() for _ in range(n_single)], norm_out=NormOut(), proj_out=lambda x: x)
    Fwd.forward(self, hidden_states=torch.zeros(1, 4, 1), encoder_hidden_states=torch.zeros(1, 2, 1),
                timestep=torch.zeros(1), img_ids=torch.zeros(4, 3), txt_ids=torch.zeros(2, 3), return_dict=False)
    return {"n_double": n_double, "n_single": n_single, **seen}


def main():
    if not R.available():
        raise SystemExit("set SIMPLETUNER_SRC to a SimpleTuner checkout")
    g = torch.Generator().manual_seed(0)
    ns = {"nn": nn, "Timesteps": Timesteps, "get_timestep_embedding": get_timestep_embedding,
          "PixArtAlphaTextProjection": PixArtAlphaTextProjection, "FluxAttention": FluxAttention,
          "FeedForward": FeedForward, "FluxAttnProcessor": lambda: None, "is_torch_npu_available": lambda: False,
          "FP32LayerNorm": None, "RMSNorm": None, "CombinedTimestepLabelEmbeddings": None}
    lift = lambda name, meths: type(name, (R.methods(TR, name, meths, extra_ns=ns), nn.Module), {})
    out = {}
    # ---- approximator input: mod_proj and the per-row [time | guidance | mod_proj] vector
    rows = 3 * 38 + 2 * 6 * 19 + 2
    TE = lift("ChromaCombinedTimestepTextProjEmbeddings", ["__init__", "forward"])
    te = TE(num_channels=64 // 4, out_dim=rows)
    t_in = torch.tensor([0.0, 0.0137, 0.25, 0.5, 0.731, 0.99961, 1.0])
    t_model = t_in.to(torch.bfloat16) * 1000                 # the forward's `timestep.to(hidden_states.dtype) * 1000`
    with torch.no_grad():
        vec = te(t_model)
    out["input_vec"] = {"rows": rows, "t": t_in, "t_model": t_model, "mod_proj": te.mod_proj.clone(), "vec": vec.clone()}
    # ---- approximator at a small width
    Approx = lift("ChromaApproximator", ["__init__", "forward"])
    ap = Approx(in_dim=64, out_dim=96, hidden_dim=128, n_layers=3)
    with torch.no_grad():
        for n, p in ap.named_parameters():
            p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g) if n.startswith("norms") else
                    torch.randn(p.shape, generator=g) * p.shape[-1] ** -0.5)
    x = torch.randn(2, 5, 64, generator=g)
    x[1, 4] *= 1e-3                                            # a row where the RMSNorm epsilon shows
    params = {k: v.detach().clone() for k, v in ap.state_dict().items()}
    with torch.no_grad():
        y32 = ap(x)
        ap16 = ap.to(torch.bfloat16)
        y16 = ap16(x.to(torch.bfloat16))
    out["approximator"] = {"config": dict(in_dim=64, out_dim=96, hidden_dim=128, n_layers=3), "x": x,
                           "params": params,
                           "out_fp32": y32.clone(), "out_bf16": y16.clone(), "rmsnorm_eps": ap16.norms[0].eps}
    # ---- pruned norms: chunk order of shift / scale / gate
    D = 8
    norms = {}
    Zero = lift("ChromaAdaLayerNormZeroPruned", ["__init__", "forward"])
    Single = lift("ChromaAdaLayerNormZeroSinglePruned", ["__init__", "forward"])
    Cont = lift("ChromaAdaLayerNormContinuousPruned", ["__init__", "forward"])
    xs = torch.randn(2, 3, D, generator=g)
    with torch.no_grad():
        e6, e3, e2 = (torch.randn(2, k, D, generator=g) for k in (6, 3, 2))
        norms["zero"] = {"emb": e6, "out": [t.clone() for t in Zero(D)(xs, emb=e6)]}
        norms["single"] = {"emb": e3, "out": [t.clone() for t in Single(D)(xs, emb=e3)]}
        norms["continuous"] = {"emb": e2, "out": Cont(D, D, elementwise_affine=False, eps=1e-6)(xs, e2).clone()}
    out["norms"] = {"x": xs, **norms}
    # ---- sigma adjustment
    Model = R.methods(MD, "Chroma", ["_adjust_chroma_sigmas", "_prepare_model_predict_timesteps", "_model_predict_single"],
                      extra_ns={**ns, **R.functions("helpers/models/flux/__init__.py",
                                                    ["pack_latents", "prepare_latent_image_ids", "unpack_latents"])})
    s = torch.cat([torch.linspace(0, 1, 257), torch.tensor([0.4999, 0.5, 0.5001, 1e-4, 0.9999])])
    out["sigmas"] = {"sigmas": s, "bf16": Model._adjust_chroma_sigmas(s.to(torch.bfloat16)).clone(),
                     "fp32": Model._adjust_chroma_sigmas(s).clone()}
    # ---- model_predict: the extended mask and the timesteps the denoiser receives
    seen = {}

    def model(**kw):
        seen.update(kw)
        return (torch.zeros_like(kw["hidden_states"]),)

    self = types.SimpleNamespace(
        _new_hidden_state_buffer=lambda: None, _build_grounding_position_net_kwargs=lambda b: None,
        _apply_flowmap_r_timestep_kwargs=lambda kw, b: None, _select_crepa_hidden_states=lambda b, h: None,
        config=types.SimpleNamespace(base_weight_dtype=torch.bfloat16, weight_dtype=torch.bfloat16, tread_config=None),
        accelerator=types.SimpleNamespace(device=torch.device("cpu")),
        noise_schedule=types.SimpleNamespace(config=types.SimpleNamespace(num_train_timesteps=1000)), model=model)
    self._prepare_model_predict_timesteps = types.MethodType(Model._prepare_model_predict_timesteps, self)
    out["predict"] = {}
    for name, mask in (("b2_ragged_2d", torch.tensor([[1, 1, 1, 0, 0, 0], [1, 1, 1, 1, 1, 0]])),
                       ("b1_3d", torch.tensor([[[1, 1, 0, 0, 0, 0]]]))):
        B = mask.shape[0]
        sig = Model._adjust_chroma_sigmas(torch.rand(B, generator=g).to(torch.bfloat16))
        batch = {"latents": torch.zeros(B, 16, 4, 6), "noisy_latents": torch.randn(B, 16, 4, 6, generator=g),
                 "timesteps": sig * 1000.0, "prompt_embeds": torch.zeros(B, mask.shape[-1], 8),
                 "encoder_attention_mask": mask}
        Model._model_predict_single(self, batch)
        out["predict"][name] = {"mask": mask, "timesteps": batch["timesteps"].clone(),
                                "attention_mask": seen["attention_mask"].clone(), "timestep": seen["timestep"].clone(),
                                "img_ids": seen["img_ids"].clone(), "txt_ids": seen["txt_ids"].clone()}
    # ---- parameter names / shapes at a small config
    ns["ChromaCombinedTimestepTextProjEmbeddings"] = TE
    ns["ChromaApproximator"] = Approx
    ns["FluxPosEmbed"] = lambda **k: nn.Identity()
    ns["ChromaAdaLayerNormZeroPruned"] = Zero
    ns["ChromaAdaLayerNormZeroSinglePruned"] = Single
    ns["ChromaAdaLayerNormContinuousPruned"] = Cont
    ns["ChromaTransformerBlock"] = lift("ChromaTransformerBlock", ["__init__"])
    ns["ChromaSingleTransformerBlock"] = lift("ChromaSingleTransformerBlock", ["__init__"])
    ns["MusubiBlockSwapManager"] = types.SimpleNamespace(build=lambda **k: None)
    Full = R.methods(TR, "ChromaTransformer2DModel", ["__init__"], extra_ns=ns)
    Full = type("ChromaTransformer2DModel", (Full, nn.Module), {"register_to_config": lambda self, **k: None})
    cfg = dict(num_layers=2, num_single_layers=3, attention_head_dim=64, num_attention_heads=2, joint_attention_dim=48,
               approximator_hidden_dim=96, approximator_layers=2)
    full = Full(**cfg)
    out["param_shapes"] = {"config": cfg, "shapes": {k: tuple(v.shape) for k, v in full.state_dict().items()}}
    out["row_offsets"] = _forward_row_offsets(ns)
    OUT.parent.mkdir(parents=True, exist_ok=True)
    torch.save(out, OUT)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
