"""Generate tests/golden/loss_golden.pt by running the reference's OWN `ModelFoundation.loss`
(helpers/models/common.py:6217-6430, with `conditional_loss` :6132-6166, `compute_scheduled_huber_c` :6168-6215,
`get_prediction_target` :4635-4658, `compute_snr` min_snr_gamma.py:4-43) on seeded inputs, lifted verbatim with
oracle/ref_extract.py.  TEST INFRASTRUCTURE ONLY.    Run in the build container:  python -m oracle.make_golden_loss
"""
from __future__ import annotations

import enum
from pathlib import Path
from types import SimpleNamespace

import torch

from . import ref_extract as rx

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "loss_golden.pt"


class PredictionTypes(enum.Enum):   # same member values as reference common.py:368-373 (identity comparisons only)
    EPSILON = "epsilon"
    SAMPLE = "sample"
    V_PREDICTION = "v_prediction"
    FLOW_MATCHING = "flow_matching"


def lifted(prediction_type, alphas_cumprod=None, **cfg):
    snr = rx.functions("helpers/training/min_snr_gamma.py", ["compute_snr"])["compute_snr"]
    M = rx.methods("helpers/models/common.py", "ModelFoundation",
                   ["loss", "conditional_loss", "compute_scheduled_huber_c", "get_prediction_target",
                    "get_flow_matching_target", "flow_matching_target", "noiseward_flow_to_prediction",
                    "flow_matching_target_direction", "_mixflow_enabled"],
                   extra_ns={"PredictionTypes": PredictionTypes, "compute_snr": snr})
    m = M.__new__(M)
    m.PREDICTION_TYPE = prediction_type
    base = dict(loss_type="l2", huber_c=0.1, huber_schedule="constant", snr_gamma=None, snr_weight=1.0,
                diff2flow_loss=False, diff2flow_enabled=False, scheduled_sampling_reflexflow=False,
                masked_loss_probability=0.0, mixflow_enabled=False)
    base.update(cfg)
    m.config = SimpleNamespace(**base)
    m.diff2flow_bridge = None
    m.noise_schedule = SimpleNamespace(alphas_cumprod=alphas_cumprod,
                                       config=SimpleNamespace(num_train_timesteps=1000, prediction_type=prediction_type.value))
    return m


def main():
    assert rx.available(), "set SIMPLETUNER_SRC to a SimpleTuner checkout"
    gen = torch.Generator().manual_seed(4321)
    B, C, H, W = 3, 4, 8, 12
    g = {"pred": torch.randn(B, C, H, W, generator=gen).bfloat16(),
         "latents": torch.randn(B, C, H, W, generator=gen).bfloat16(),
         "noise": torch.randn(B, C, H, W, generator=gen).bfloat16(),
         "flow_timesteps": torch.tensor([35.0, 512.5, 940.0]),
         "eps_timesteps": torch.tensor([12, 480, 977]),
         "alphas_cumprod": torch.cumprod(1.0 - torch.linspace(0.0001, 0.02, 1000, dtype=torch.float32), dim=0)}
    cases = {}
    for lt in ("l2", "huber", "smooth_l1"):
        for sched in (("constant",) if lt == "l2" else ("constant", "exponential", "snr")):
            for c in ((0.1,) if lt == "l2" else (0.1, 0.02)):
                name = f"flow.{lt}.{sched}.c{c}"
                m = lifted(PredictionTypes.FLOW_MATCHING, loss_type=lt, huber_schedule=sched, huber_c=c)
                pb = {"latents": g["latents"], "noise": g["noise"], "timesteps": g["flow_timesteps"]}
                cases[name] = m.loss(pb, {"model_prediction": g["pred"]}).float()
                if lt != "l2":
                    g[name + ".huber_c"] = torch.stack([m.compute_scheduled_huber_c(g["flow_timesteps"][i:i + 1]).reshape(()).float()
                                                        for i in range(B)])
    for lt, sched, gamma in (("l2", "constant", None), ("l2", "constant", 5.0), ("huber", "constant", None),
                             ("huber", "snr", 5.0), ("smooth_l1", "exponential", None), ("smooth_l1", "snr", 1.0)):
        name = f"eps.{lt}.{sched}.g{gamma}"
        m = lifted(PredictionTypes.EPSILON, alphas_cumprod=g["alphas_cumprod"], loss_type=lt, huber_schedule=sched, snr_gamma=gamma)
        pb = {"latents": g["latents"], "noise": g["noise"], "timesteps": g["eps_timesteps"]}
        cases[name] = m.loss(pb, {"model_prediction": g["pred"]}).float()
        if lt != "l2":
            g[name + ".huber_c"] = torch.stack([m.compute_scheduled_huber_c(g["eps_timesteps"][i:i + 1]).reshape(()).float()
                                                for i in range(B)])
    for k, v in cases.items():
        g["loss." + k] = v
    OUT.parent.mkdir(parents=True, exist_ok=True)
    torch.save(g, OUT)
    print(f"wrote {OUT} with {len(g)} entries")
    for k, v in g.items():
        if k.startswith("loss.") or k.endswith(".huber_c"):
            print(" ", k, v.tolist() if v.numel() <= 4 else tuple(v.shape))


if __name__ == "__main__":
    main()
