"""Generate tests/golden/collate_golden.pt: the reference's own size-feature gathers (helpers/training/collate.py:59-98,
487-523) and `Trainer._max_grad_value` (helpers/training/trainer.py:6376-6398) executed verbatim on seeded inputs.
TEST INFRASTRUCTURE ONLY.   Run in the build container:   python -m oracle.make_golden_collate
"""
from __future__ import annotations

from pathlib import Path
from types import SimpleNamespace

import torch

from . import ref_extract as rx

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "collate_golden.pt"


def main():
    assert rx.available(), "set SIMPLETUNER_SRC to a SimpleTuner checkout"
    g = {}
    tracker = SimpleNamespace(is_sdxl_refiner=lambda: False, get_args=lambda: SimpleNamespace(data_aesthetic_score=7.0),
                              get_accelerator=lambda: SimpleNamespace(device="cpu"))
    fx = rx.functions("helpers/training/collate.py",
                      ["compute_time_ids", "gather_conditional_sdxl_size_features", "gather_conditional_pixart_size_features"],
                      extra_ns={"StateTracker": tracker})
    examples = [
        {"intermediary_size": (1024, 768), "crop_coordinates": [0, 0], "drop_conditioning": False},
        {"original_size": (1536, 640), "crop_coordinates": [12, 34], "drop_conditioning": False},
        {"intermediary_size": (800, 1200), "crop_coordinates": [5, 7], "drop_conditioning": True},
    ]
    latents = torch.zeros(3, 4, 96, 128)
    g["sdxl.examples"] = examples
    g["sdxl.latent_shape"] = tuple(latents.shape)
    g["sdxl.time_ids.bf16"] = fx["gather_conditional_sdxl_size_features"](examples, latents, torch.bfloat16)
    g["sdxl.time_ids.f32"] = fx["gather_conditional_sdxl_size_features"](examples, latents, torch.float32)
    px = fx["gather_conditional_pixart_size_features"](examples, torch.zeros(3, 4, 160, 96), torch.bfloat16)
    g["pixart.resolution"], g["pixart.aspect_ratio"] = px["resolution"], px["aspect_ratio"]
    # Trainer._max_grad_value: lifted method on a dummy with three "parameters"
    T = rx.methods("helpers/training/trainer.py", "Trainer", ["_max_grad_value"], extra_ns={"DTensor": type("DTensor", (), {}), "dist": None})
    gen = torch.Generator().manual_seed(3)
    grads = [torch.randn(5, 7, generator=gen).bfloat16(), torch.randn(11, generator=gen).bfloat16() * 3, None]
    params = [SimpleNamespace(grad=t) for t in grads]
    dummy = T()
    dummy._get_trainable_parameters = lambda: params
    g["maxgrad.grads"] = [t for t in grads if t is not None]
    g["maxgrad.out"] = dummy._max_grad_value()
    dummy._get_trainable_parameters = lambda: [SimpleNamespace(grad=None)]
    g["maxgrad.empty"] = dummy._max_grad_value()
    torch.save(g, OUT)
    print("wrote", OUT, sorted(g))


if __name__ == "__main__":
    main()
