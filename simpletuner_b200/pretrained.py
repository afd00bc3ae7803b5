"""The diffusers `ModelMixin` / `ConfigMixin` surface the reference's full-model checkpointing calls on a denoiser:

  * `save_pretrained(save_dir, max_shard_size=, state_dict=)`      save_hooks.py:1128 (full-model save) and the EMA save
  * `register_to_config(**cfg)` and `from_config(config)`          save_hooks.py:1258-1264 (resume) and EMAModel
                                                                   (helpers/training/ema.py:289-320)

Files are written in the diffusers layout: `config.json` (the class name and the constructor arguments) and
`diffusion_pytorch_model.safetensors`, or numbered shards with a `.safetensors.index.json` weight map when the tensors
exceed `max_shard_size`.  Only the module's state dict is written, under the reference's parameter names and dtypes;
the derived weight layouts the block schedules build are plain attributes, never part of it.
"""
from __future__ import annotations

import json
import os
import re
from types import SimpleNamespace
from typing import Any, Dict, Optional, Union

import torch

WEIGHTS_NAME = "diffusion_pytorch_model.safetensors"
CONFIG_NAME = "config.json"


class ModelConfig(SimpleNamespace):
    """A denoiser's `.config`: attribute access like before, and mapping access like diffusers' FrozenDict, so that
    `model.register_to_config(**other.config)` and `dict(model.config)` work."""

    def keys(self):
        return vars(self).keys()

    def __getitem__(self, key):
        return vars(self)[key]

    def __contains__(self, key):
        return key in vars(self)


def _shard_bytes(size: Union[int, str]) -> int:
    """`max_shard_size` as bytes: an int, or a string such as "10GB" / "500MB" / "2GiB" (diffusers' units)."""
    if isinstance(size, int):
        return size
    m = re.fullmatch(r"\s*(\d+(?:\.\d+)?)\s*([KMGT]?)(I?)B\s*", str(size).upper())
    if m is None:
        raise ValueError(f"max_shard_size must be an int or a size like '10GB', got {size!r}")
    base = 1024 if m.group(3) else 1000
    return int(float(m.group(1)) * base ** "_KMGT".index(m.group(2) or "_"))


class PretrainedIOAPI:
    """Mixed into a denoiser whose constructor takes its `.config` fields as keyword arguments."""

    def register_to_config(self, **kwargs):
        for k, v in kwargs.items():
            setattr(self.config, k, v)

    @classmethod
    def from_config(cls, config: Any, **kwargs):
        """A freshly initialised model of the configured architecture (weights are loaded afterwards)."""
        cfg = dict(vars(config) if isinstance(config, SimpleNamespace) else config)
        cfg.update(kwargs)
        return cls(**{k: v for k, v in cfg.items() if not k.startswith("_")})

    def save_pretrained(self, save_directory: str, max_shard_size: Union[int, str] = "10GB",
                        state_dict: Optional[Dict[str, torch.Tensor]] = None, **unused):
        from safetensors.torch import save_file

        os.makedirs(save_directory, exist_ok=True)
        sd = self.state_dict() if state_dict is None else state_dict
        tensors = {k: v.detach().to("cpu").contiguous() for k, v in sd.items()}
        cfg = {"_class_name": type(self).__name__, **{k: list(v) if isinstance(v, tuple) else v for k, v in vars(self.config).items()}}
        with open(os.path.join(save_directory, CONFIG_NAME), "w") as f:
            json.dump(cfg, f, indent=2, sort_keys=True)
        limit = _shard_bytes(max_shard_size)
        shards, cur, cur_bytes = [], {}, 0
        for k, v in tensors.items():
            n = v.numel() * v.element_size()
            if cur and cur_bytes + n > limit:
                shards.append(cur)
                cur, cur_bytes = {}, 0
            cur[k] = v
            cur_bytes += n
        shards.append(cur)
        if len(shards) == 1:
            save_file(shards[0], os.path.join(save_directory, WEIGHTS_NAME), metadata={"format": "pt"})
            return
        stem = WEIGHTS_NAME[: -len(".safetensors")]
        weight_map = {}
        for i, shard in enumerate(shards):
            name = f"{stem}-{i + 1:05d}-of-{len(shards):05d}.safetensors"
            save_file(shard, os.path.join(save_directory, name), metadata={"format": "pt"})
            weight_map.update({k: name for k in shard})
        index = {"metadata": {"total_size": sum(v.numel() * v.element_size() for v in tensors.values())}, "weight_map": weight_map}
        with open(os.path.join(save_directory, WEIGHTS_NAME + ".index.json"), "w") as f:
            json.dump(index, f, indent=2, sort_keys=True)
