"""Generate tests/golden/flux_step_golden.pt by running the reference's own functions
(via oracle/ref_extract.py, with $SIMPLETUNER_SRC naming a SimpleTuner checkout) on seeded inputs.  TEST INFRASTRUCTURE ONLY.

Run in the build container:   python -m oracle.make_golden
"""
from __future__ import annotations

from pathlib import Path
from types import SimpleNamespace

import torch

from . import ref_extract as rx

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "flux_step_golden.pt"


def main():
    assert rx.available(), "set SIMPLETUNER_SRC to a SimpleTuner checkout"
    g = {}
    gen = torch.Generator().manual_seed(1234)

    # ---- flux/__init__.py:25-61  pack / unpack / ids
    fx = rx.functions("helpers/models/flux/__init__.py", ["pack_latents", "unpack_latents", "prepare_latent_image_ids"])
    lat = torch.randn(2, 16, 8, 12, generator=gen)
    packed = fx["pack_latents"](lat, 2, 16, 8, 12)
    g["pack.in"] = lat
    g["pack.out"] = packed
    g["unpack.out"] = fx["unpack_latents"](packed, 8 * 8, 12 * 8, 16)
    g["ids.out_8x12"] = fx["prepare_latent_image_ids"](2, 8, 12, "cpu", torch.float32)

    # ---- custom_schedule.py: shift, timestep weights, segmented selection
    cs = rx.functions("helpers/training/custom_schedule.py",
                      ["apply_flow_schedule_shift", "generate_timestep_weights", "segmented_timestep_selection"],
                      extra_ns={"calculate_shift_flux": None})
    cfg = SimpleNamespace(flow_schedule_shift=3.0, flow_schedule_auto_shift=False)
    sig = torch.tensor([0.1, 0.5, 0.9, 0.0, 1.0, 0.3333])
    g["shift.in"] = sig
    g["shift.out_s3"] = cs["apply_flow_schedule_shift"](cfg, None, sig.clone(), None)
    cfg1 = SimpleNamespace(flow_schedule_shift=1.0, flow_schedule_auto_shift=False)
    g["shift.out_s1"] = cs["apply_flow_schedule_shift"](cfg1, None, sig.clone(), None)
    for strat, kw in (("none", {}), ("later", {}), ("earlier", {}), ("range", {"timestep_bias_begin": 200, "timestep_bias_end": 500})):
        a = SimpleNamespace(timestep_bias_strategy=strat, timestep_bias_portion=0.25, timestep_bias_multiplier=2.0,
                            timestep_bias_begin=kw.get("timestep_bias_begin", 0), timestep_bias_end=kw.get("timestep_bias_end", 1000))
        g[f"tsw.{strat}"] = cs["generate_timestep_weights"](a, 1000)
    scfg = SimpleNamespace(refiner_training=False, refiner_training_invert_schedule=False, refiner_training_strength=0.2)
    for bsz in (2, 4, 7):
        torch.manual_seed(42)
        w = torch.ones(1000)
        sel = cs["segmented_timestep_selection"](1000, bsz, w, scfg)
        g[f"segsel.bsz{bsz}"] = sel
        g[f"segsel.bsz{bsz}.weights_after"] = w  # quirk Q1: weights are normalised in place

    # ---- flux/transformer.py:73-106  RoPE application
    tr = rx.functions("helpers/models/flux/transformer.py", ["_apply_rotary_emb_anyshape"])
    x = torch.randn(2, 3, 10, 16, generator=gen)
    ang = torch.rand(10, 8, generator=gen) * 6.28
    cos = ang.cos().repeat_interleave(2, dim=-1)
    sin = ang.sin().repeat_interleave(2, dim=-1)
    g["rope.x"], g["rope.cos"], g["rope.sin"] = x, cos, sin
    g["rope.out"] = tr["_apply_rotary_emb_anyshape"](x, (cos, sin))
    g["rope.out_bf16"] = tr["_apply_rotary_emb_anyshape"](x.bfloat16(), (cos, sin))

    # ---- common.py: ModelFoundation methods lifted onto a dummy (as reference tests/test_mixflow.py does)
    M = rx.methods("helpers/models/common.py", "ModelFoundation",
                   ["_expand_sigma_values", "_prepare_flow_noisy_latents", "_mixflow_enabled",
                    "flow_matching_target", "noiseward_flow_to_prediction", "flow_matching_target_direction",
                    "sample_flow_sigmas", "_normalize_flow_custom_timesteps", "_flow_cubic_schedule_weights",
                    "_get_dataset_timestep_sampling_offset", "flow_matching_timesteps_from_sigmas"],
                   extra_ns={"apply_flow_schedule_shift": cs["apply_flow_schedule_shift"], "Beta": None,
                             "resolve_distributed_batch_layout": None,
                             # 1-line stand-in: no per-dataset timestep offset configured (config.get -> 0.0)
                             "StateTracker": SimpleNamespace(get_data_backend_config=lambda _id: {}),
                             **rx.functions("helpers/training/timestep_distribution.py", ["parse_cubic_spline_weights"])})
    I = rx.methods("helpers/models/common.py", "ImageModelFoundation", ["expand_sigmas"])
    M.expand_sigmas = I.expand_sigmas  # ImageModelFoundation.expand_sigmas (common.py:6825-6828)
    m = M.__new__(M)
    m.config = SimpleNamespace(mixflow_enabled=False, flow_schedule_shift=3.0, flow_schedule_auto_shift=False,
                               flow_custom_timesteps=None, flux_fast_schedule=False, flow_use_beta_schedule=False,
                               flow_use_uniform_schedule=False, flow_sigmoid_scale=1.0, flow_cubic_schedule=None,
                               flow_cubic_schedule_weights=None)
    m.accelerator = SimpleNamespace(device=torch.device("cpu"))
    m.noise_schedule = SimpleNamespace(config=SimpleNamespace(num_train_timesteps=1000))
    # known answer of reference tests/test_mixflow.py:76-87 (x=2, eps=6, sigma=.25 -> 3.0)
    b = {"latents": torch.tensor([[[[2.0]]]]), "input_noise": torch.tensor([[[[6.0]]]]),
         "sigmas": torch.tensor([0.25]), "timesteps": torch.tensor([250.0])}
    m._prepare_flow_noisy_latents(b)
    g["noisy.known_answer"] = b["noisy_latents"]
    for dt, tag in ((torch.float32, "f32"), (torch.bfloat16, "bf16")):
        lat4 = torch.randn(3, 16, 6, 10, generator=gen).to(dt)
        eps4 = torch.randn(3, 16, 6, 10, generator=gen).to(dt)
        sg = torch.tensor([0.123, 0.5, 0.987])
        b = {"latents": lat4, "input_noise": eps4, "sigmas": sg.clone(), "timesteps": sg * 1000}
        m._prepare_flow_noisy_latents(b)
        g[f"noisy.{tag}.latents"], g[f"noisy.{tag}.noise"], g[f"noisy.{tag}.sigmas"] = lat4, eps4, sg
        g[f"noisy.{tag}.out"] = b["noisy_latents"]
        g[f"target.{tag}.out"] = m.flow_matching_target(lat4, eps4)
    try:
        torch.manual_seed(42)
        sigmas, timesteps = m.sample_flow_sigmas({"latents": torch.zeros(4, 16, 8, 8), "noise": torch.zeros(4, 16, 8, 8)}, state={})
        g["sample_sigmas.seed42.sigmas"], g["sample_sigmas.seed42.timesteps"] = sigmas, timesteps
    except Exception as e:  # pragma: no cover - records why, the test then skips this vector
        g["sample_sigmas.error"] = repr(e)

    # ---- min_snr_gamma.py:4-43 compute_snr, collate.py:59-98 compute_time_ids
    snr = rx.functions("helpers/training/min_snr_gamma.py", ["compute_snr"])["compute_snr"]
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float32) ** 2
    sched = SimpleNamespace(alphas_cumprod=torch.cumprod(1.0 - betas, dim=0))
    ts = torch.tensor([0, 1, 250, 500, 731, 999])
    g["snr.timesteps"] = ts
    g["snr.out"] = snr(ts, sched)
    g["snr.out_softmin"] = snr(ts, sched, use_soft_min=True, sigma_data=0.5)
    cti = rx.functions("helpers/training/collate.py", ["compute_time_ids"],
                       extra_ns={"StateTracker": SimpleNamespace(is_sdxl_refiner=lambda: False)})["compute_time_ids"]
    g["time_ids.a"] = cti((1024, 768), (4, 96, 128), torch.float32, crop_coordinates=[0, 0])
    g["time_ids.b"] = cti((1536, 640), (4, 80, 192), torch.bfloat16, crop_coordinates=[12, 34])

    OUT.parent.mkdir(parents=True, exist_ok=True)
    torch.save(g, OUT)
    print(f"wrote {OUT} with {len(g)} entries")
    for k, v in g.items():
        print(" ", k, tuple(v.shape) if torch.is_tensor(v) else v)


if __name__ == "__main__":
    main()
