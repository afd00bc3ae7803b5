"""LyCORIS LoKr on the libstb200 Flux path (BASELINE config 4: "Flux.1-dev LyCORIS LoKr").

Host mirror of the part of `lycoris-lora` (setup.py:319, >= 3.4.0; third-party, not vendored in the reference tree) that the
reference drives at simpletuner/helpers/training/trainer.py:3390-3505:

    LycorisNetwork.apply_preset(cfg["apply_preset"])
    net = create_lycoris(component, multiplier, linear_dim, linear_alpha, algo="lokr", factor=..., ...)
    net.apply_to(); net.to(device, dtype=weight_dtype); optimizer over net.parameters()
    net.set_multiplier(x)  (validation / prior-regularisation batches, trainer.py:6138-6143)
    net.save_weights(path, dtype, metadata)  (trainer.py:7733)
    for lora in net.loras: lora.lokr_w1, lora.lokr_w2, lora.org_weight  (helpers/training/peft_init.py:34-38)

Algorithm (restated in oracle/lokr_oracle.py): delta W = kron(lokr_w1 [a, c], lokr_w2 [b, d]) * scale, forward
y = linear(x, W + delta W * multiplier).  Kernel mapping: the adapted weight IS rebuilt — once per optimizer step, straight into
the fused / transposed projection layouts the block schedules read (flux/transformer.py `plans()`), so forward and dgrad are
the plain wgmma GEMMs of the un-adapted model with no adapter work at all.  Backward forms the full weight gradient with the
MN-major wgmma weight-gradient kernel (`stb_wgrad_full`, exactly what autograd computes through `torch.kron` in the
reference) and contracts it against the other Kronecker factor:
    d w1[i, k] = scale * sum_{j, l} dW[(i, j), (k, l)] w2[j, l];   d w2[j, l] = scale * sum_{i, k} dW[(i, j), (k, l)] w1[i, k].
Unsupported LyCORIS options raise NotImplementedError (other algos, dropout / rank_dropout / module_dropout, bypass_mode,
decompose_both, tucker, DoRA weight_decompose, conv layers).
"""
from __future__ import annotations

import math
from typing import Dict, Iterable, List, Optional, Tuple

import torch
import torch.nn as nn


def factorization(dimension: int, factor: int = -1) -> Tuple[int, int]:
    """lycoris.functional.general.factorization (see oracle/lokr_oracle.py for the restated definition)."""
    if factor > 0 and dimension % factor == 0:
        m, n = factor, dimension // factor
        return (n, m) if m > n else (m, n)
    if factor < 0:
        factor = dimension
    m, n = 1, dimension
    length = m + n
    while m < n:
        new_m = m + 1
        while dimension % new_m != 0:
            new_m += 1
        new_n = dimension // new_m
        if new_m + new_n > length or new_m > factor:
            break
        m, n = new_m, new_n
    return (n, m) if m > n else (m, n)


class LokrModule(nn.Module):
    """One adapted Linear: parameters `lokr_w1`, `lokr_w2` (or `lokr_w2_a`, `lokr_w2_b`), buffer `alpha` — LyCORIS names."""

    def __init__(self, lora_name: str, org_module, multiplier: float, lora_dim: int, alpha: float, factor: int):
        super().__init__()
        self.lora_name = lora_name
        self.multiplier = float(multiplier)
        self.lora_dim = int(lora_dim)
        n_out, k_in = org_module.out_features, org_module.in_features
        (a, b), (c, d) = factorization(n_out, factor), factorization(k_in, factor)
        self.shape = ((a, b), (c, d))
        dt, dev = org_module.weight.dtype, org_module.weight.device
        self.lokr_w1 = nn.Parameter(torch.empty((a, c), dtype=dt, device=dev))
        self.full_matrix = self.lora_dim >= max(b, d) / 2
        if self.full_matrix:
            self.lokr_w2 = nn.Parameter(torch.zeros((b, d), dtype=dt, device=dev))
            alpha = self.lora_dim                       # both factors are full matrices: scale = 1
        else:
            self.lokr_w2_a = nn.Parameter(torch.empty((b, self.lora_dim), dtype=dt, device=dev))
            self.lokr_w2_b = nn.Parameter(torch.zeros((self.lora_dim, d), dtype=dt, device=dev))
            nn.init.kaiming_uniform_(self.lokr_w2_a, a=math.sqrt(5))
        nn.init.kaiming_uniform_(self.lokr_w1, a=math.sqrt(5))
        self.register_buffer("alpha", torch.tensor(float(alpha)))
        self.scale = float(alpha) / float(self.lora_dim)
        self.__dict__["_org"] = org_module             # not a sub-module: the base Linear stays owned by the denoiser

    @property
    def org_weight(self) -> torch.Tensor:
        return self._org.weight

    def w2(self) -> torch.Tensor:
        return self.lokr_w2 if self.full_matrix else self.lokr_w2_a @ self.lokr_w2_b

    def factors(self):
        """(w1, w2) as the block schedules consume them (w2 = w2_a @ w2_b stays on torch autograd: a [b, r] x [r, d] product)."""
        return self.lokr_w1, self.w2()

    @torch.no_grad()
    def delta_weight(self) -> torch.Tensor:
        return torch.kron(self.lokr_w1.float(), self.w2().float()) * (self.scale * self.multiplier)

    @torch.no_grad()
    def effective_weight(self) -> torch.Tensor:
        """org_weight + kron(w1, w2) * scale * multiplier, rounded once to the weight dtype."""
        w = self._org.weight
        if w.is_cuda:
            return self.rebuild_into(torch.empty_like(w))
        return (w.float() + self.delta_weight()).to(w.dtype)

    @torch.no_grad()
    def rebuild_into(self, out: torch.Tensor, out_t: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One `stb_lokr_rebuild` pass: the adapted weight (and its transpose) written straight into (slices of) the fused
        projection / dgrad layouts."""
        from . import ops
        return ops.lokr_rebuild(self._org.weight.detach(), self.lokr_w1.detach().contiguous(), self.w2().detach().contiguous(),
                                self.scale * self.multiplier, out, out_t)


class LycorisNetwork(nn.Module):
    """`lycoris.wrapper.LycorisNetwork` surface used by the reference trainer."""

    _preset: Dict = {"target_module": ["Attention", "FeedForward"], "module_algo_map": {}}

    @classmethod
    def apply_preset(cls, preset: Dict) -> None:
        for k in preset:
            if k not in ("target_module", "module_algo_map", "enable_conv", "unet_target_module", "unet_target_name",
                         "target_name", "name_algo_map", "use_fnmatch"):
                raise NotImplementedError(f"LyCORIS preset key {k!r} is not supported by the libstb200 path")
        if preset.get("name_algo_map") or preset.get("target_name") or preset.get("unet_target_name"):
            raise NotImplementedError("LyCORIS name-based targets are not supported by the libstb200 path")
        cls._preset = {"target_module": list(preset.get("target_module", cls._preset["target_module"])),
                       "module_algo_map": dict(preset.get("module_algo_map", {}))}

    def __init__(self, model: nn.Module, multiplier: float = 1.0, lora_dim: int = 4, alpha: float = 1.0, factor: int = -1,
                 **unused):
        super().__init__()
        self.multiplier = float(multiplier)
        self.__dict__["_model"] = model
        preset = type(self)._preset
        loras: List[LokrModule] = []
        seen = set()
        for mod_name, mod in model.named_modules():
            cls_name = getattr(mod, "_lycoris_class_name", type(mod).__name__)
            if cls_name not in preset["target_module"]:
                continue
            over = preset["module_algo_map"].get(cls_name, {})
            if over.get("algo", "lokr") != "lokr":
                raise NotImplementedError("only algo='lokr' is supported by the libstb200 path")
            f = int(over.get("factor", factor))
            dim = int(over.get("linear_dim", over.get("dim", lora_dim)))
            al = float(over.get("linear_alpha", over.get("alpha", alpha)))
            for child_name, child in mod.named_modules():
                if not (hasattr(child, "in_features") and hasattr(child, "weight") and child.weight.ndim == 2) or id(child) in seen:
                    continue
                if not getattr(child, "_lokr_capable", False):
                    raise NotImplementedError(f"LyCORIS target {mod_name}.{child_name} is not adaptable on the libstb200 path")
                seen.add(id(child))
                full = f"{mod_name}.{child_name}" if child_name else mod_name
                loras.append(LokrModule("lycoris_" + full.replace(".", "_"), child, multiplier, dim, al, f))
        if not loras:
            raise ValueError(f"LyCORIS preset {preset['target_module']} matched no module")
        self.loras = nn.ModuleList(loras)

    def apply_to(self) -> None:
        for lora in self.loras:
            lora._org.lokr = lora
        inv = getattr(self._model, "invalidate_plans", None)
        if callable(inv):
            inv()
        setattr(self._model, "_lycoris_network", self)

    def restore(self) -> None:
        for lora in self.loras:
            lora._org.lokr = None
        inv = getattr(self._model, "invalidate_plans", None)
        if callable(inv):
            inv()

    def set_multiplier(self, multiplier: float) -> None:
        self.multiplier = float(multiplier)
        for lora in self.loras:
            lora.multiplier = float(multiplier)
        inv = getattr(self._model, "invalidate_plans", None)
        if callable(inv):           # the rebuilt weights embed the multiplier
            inv()

    def state_dict_lycoris(self, dtype=None) -> Dict[str, torch.Tensor]:
        out = {}
        for lora in self.loras:
            for k, v in lora.state_dict().items():
                v = v.detach().clone().to("cpu")
                out[f"{lora.lora_name}.{k}"] = v.to(dtype) if (dtype is not None and v.is_floating_point()) else v
        return out

    def save_weights(self, file: str, dtype=None, metadata: Optional[Dict[str, str]] = None) -> None:
        """`LycorisNetwork.save_weights(file, dtype, metadata)`: `<lora_name>.<param>` keys; safetensors or torch pickle."""
        sd = self.state_dict_lycoris(dtype)
        if str(file).endswith(".safetensors"):
            from safetensors.torch import save_file
            save_file({k: v.contiguous() for k, v in sd.items()}, file, metadata or None)
        else:
            torch.save(sd, file)

    def load_weights(self, file: str) -> None:
        if str(file).endswith(".safetensors"):
            from safetensors.torch import load_file
            sd = load_file(file)
        else:
            sd = torch.load(file, map_location="cpu")
        own = {f"{lora.lora_name}.{k}": v for lora in self.loras for k, v in lora.state_dict().items()}
        missing = [k for k in own if k not in sd]
        if missing:
            raise KeyError(f"LyCORIS weights miss {missing[:4]}")
        with torch.no_grad():
            for k, v in own.items():
                v.copy_(sd[k].to(device=v.device, dtype=v.dtype))
        inv = getattr(self._model, "invalidate_plans", None)
        if callable(inv):
            inv()


_UNSUPPORTED_TRUE = ("bypass_mode", "decompose_both", "use_tucker", "use_scalar", "weight_decompose", "dora_wd", "train_norm",
                     "rs_lora", "unbalanced_factorization", "wd_on_output")
_UNSUPPORTED_NONZERO = ("dropout", "rank_dropout", "module_dropout", "conv_dim")


def validate_lycoris_config(cfg: Dict) -> None:
    if str(cfg.get("algo", "lokr")).lower() != "lokr":
        raise NotImplementedError(f"LyCORIS algo={cfg.get('algo')!r}: only 'lokr' runs on the libstb200 path")
    for k in _UNSUPPORTED_TRUE:
        if cfg.get(k):
            raise NotImplementedError(f"LyCORIS option {k} is not supported by the libstb200 path")
    for k in _UNSUPPORTED_NONZERO:
        if cfg.get(k):
            raise NotImplementedError(f"LyCORIS option {k}={cfg[k]} is not supported by the libstb200 path")


def create_lycoris(module: nn.Module, multiplier: float = 1.0, linear_dim: int = 4, linear_alpha: float = 1.0, **kwargs
                   ) -> LycorisNetwork:
    """`lycoris.create_lycoris(module, multiplier, linear_dim, linear_alpha, **config)` for algo = "lokr"."""
    cfg = dict(kwargs)
    validate_lycoris_config(cfg)
    cfg.pop("algo", None)
    cfg.pop("full_matrix", None)      # LyCORIS: forces full matrices; with linear_dim >= dim / 2 they already are
    factor = int(cfg.pop("factor", -1))
    return LycorisNetwork(module, multiplier=multiplier, lora_dim=linear_dim, alpha=linear_alpha, factor=factor)


def lokr_factor_grads(dW: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor, scale: float):
    """(d w1, d w2) from the full weight gradient dW [a b, c d] (see the module docstring)."""
    (a, c), (b, d) = w1.shape, w2.shape
    if dW.is_cuda and d % 8 == 0 and dW.stride(0) % 8 == 0 and dW.stride(1) == 1 and a * c * 4 <= 48 * 1024:
        from . import ops
        dw1, dw2 = ops.lokr_factor_grads(dW, w1.detach().contiguous(), w2.detach().contiguous(), scale)
        return dw1.to(w1.dtype), dw2.to(w2.dtype)
    g = dW.reshape(a, b, c, d).float()
    dw1 = torch.einsum("ajcl,jl->ac", g, w2.float()) * scale
    dw2 = torch.einsum("ajcl,ac->jl", g, w1.float()) * scale
    return dw1.to(w1.dtype), dw2.to(w2.dtype)
