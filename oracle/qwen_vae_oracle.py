"""Restatement of the Qwen-Image VAE encoder (diffusers AutoencoderKLQwenImage, the Wan 2.1 causal 3-D VAE) in its
3-D causal form, for any float dtype and device, on seeded synthetic weights.

It runs real conv3d with the causal padding of QwenImageCausalConv3d (two zero frames in front, none behind), the
first-chunk cache rule of the chunked encode (no cache on chunk 0: `downsample3d` stores its input and skips time_conv),
the per-frame mid attention, then quant_conv, DiagonalGaussianDistribution.sample and Qwen-Image's
post_vae_encode_transform_sample ((z - latents_mean) * (1 / latents_std)).  `encode2d` is the direct 2-D restatement
with the last temporal tap of every conv; on one frame the two must agree bit for bit in fp64.

State-dict names and shapes (`key_shapes`) restate diffusers' module tree: encoder.conv_in, encoder.down_blocks.{i} as a
flat list of QwenImageResidualBlock (norm1.gamma, conv1, norm2.gamma, conv2, conv_shortcut) and QwenImageResample
(resample.1, and time_conv for downsample3d), encoder.mid_block.{resnets.0, attentions.0 (norm.gamma, to_qkv, proj),
resnets.1}, encoder.norm_out.gamma, encoder.conv_out, quant_conv.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

# diffusers AutoencoderKLQwenImage defaults (the Qwen-Image checkpoint's vae/config.json)
QWEN_LATENTS_MEAN = [-0.7571, -0.7089, -0.9113, 0.1075, -0.1745, 0.9653, -0.1517, 1.5508,
                     0.4134, -0.0715, 0.5517, -0.3632, -0.1922, -0.9497, 0.2503, -0.2921]
QWEN_LATENTS_STD = [2.8184, 1.4541, 2.3275, 2.6558, 1.2196, 1.7708, 2.6052, 2.0743,
                    3.2687, 2.1526, 2.8652, 1.5579, 1.6382, 1.1253, 2.8251, 1.9160]


@dataclass
class QwenVaeConfig:
    base_dim: int = 96
    z_dim: int = 16
    dim_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    attn_scales: Tuple[float, ...] = ()
    temperal_downsample: Tuple[bool, ...] = (False, True, True)
    latents_mean: List[float] = field(default_factory=lambda: list(QWEN_LATENTS_MEAN))
    latents_std: List[float] = field(default_factory=lambda: list(QWEN_LATENTS_STD))

    def as_dict(self):
        return dict(base_dim=self.base_dim, z_dim=self.z_dim, dim_mult=list(self.dim_mult), num_res_blocks=self.num_res_blocks,
                    attn_scales=list(self.attn_scales), temperal_downsample=list(self.temperal_downsample), dropout=0.0,
                    latents_mean=list(self.latents_mean), latents_std=list(self.latents_std))


def _layout(cfg: QwenVaeConfig):
    """The encoder's down_blocks as ("res", cin, cout) / ("down", c, temporal) entries, and the dims list."""
    dims = [cfg.base_dim * u for u in [1, *cfg.dim_mult]]
    blocks = []
    for i, (cin, cout) in enumerate(zip(dims[:-1], dims[1:])):
        for _ in range(cfg.num_res_blocks):
            blocks.append(("res", cin, cout))
            cin = cout
        if i != len(cfg.dim_mult) - 1:
            blocks.append(("down", cout, bool(cfg.temperal_downsample[i])))
    return blocks, dims


def _res_keys(out, pre, cin, cout):
    out[f"{pre}.norm1.gamma"] = (cin, 1, 1, 1)
    out[f"{pre}.conv1.weight"] = (cout, cin, 3, 3, 3)
    out[f"{pre}.conv1.bias"] = (cout,)
    out[f"{pre}.norm2.gamma"] = (cout, 1, 1, 1)
    out[f"{pre}.conv2.weight"] = (cout, cout, 3, 3, 3)
    out[f"{pre}.conv2.bias"] = (cout,)
    if cin != cout:
        out[f"{pre}.conv_shortcut.weight"] = (cout, cin, 1, 1, 1)
        out[f"{pre}.conv_shortcut.bias"] = (cout,)


def key_shapes(cfg: QwenVaeConfig) -> "OrderedDict[str, tuple]":
    """Every encoder / quant_conv state-dict key of AutoencoderKLQwenImage with its shape, in module order."""
    blocks, dims = _layout(cfg)
    out: "OrderedDict[str, tuple]" = OrderedDict()
    out["encoder.conv_in.weight"] = (dims[0], 3, 3, 3, 3)
    out["encoder.conv_in.bias"] = (dims[0],)
    for i, b in enumerate(blocks):
        pre = f"encoder.down_blocks.{i}"
        if b[0] == "res":
            _res_keys(out, pre, b[1], b[2])
        else:
            c = b[1]
            out[f"{pre}.resample.1.weight"] = (c, c, 3, 3)
            out[f"{pre}.resample.1.bias"] = (c,)
            if b[2]:
                out[f"{pre}.time_conv.weight"] = (c, c, 3, 1, 1)
                out[f"{pre}.time_conv.bias"] = (c,)
    c = dims[-1]
    _res_keys(out, "encoder.mid_block.resnets.0", c, c)
    out["encoder.mid_block.attentions.0.norm.gamma"] = (c, 1, 1)
    out["encoder.mid_block.attentions.0.to_qkv.weight"] = (3 * c, c, 1, 1)
    out["encoder.mid_block.attentions.0.to_qkv.bias"] = (3 * c,)
    out["encoder.mid_block.attentions.0.proj.weight"] = (c, c, 1, 1)
    out["encoder.mid_block.attentions.0.proj.bias"] = (c,)
    _res_keys(out, "encoder.mid_block.resnets.1", c, c)
    out["encoder.norm_out.gamma"] = (c, 1, 1, 1)
    out["encoder.conv_out.weight"] = (2 * cfg.z_dim, c, 3, 3, 3)
    out["encoder.conv_out.bias"] = (2 * cfg.z_dim,)
    out["quant_conv.weight"] = (2 * cfg.z_dim, 2 * cfg.z_dim, 1, 1, 1)
    out["quant_conv.bias"] = (2 * cfg.z_dim,)
    return out


def init_params(cfg: QwenVaeConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded synthetic fp32 weights, rounded to bf16 values: convs N(0, 1 / fan_in) (all temporal taps, so a wrong
    tap shows), biases N(0, 0.1^2), gammas 1 + N(0, 0.1^2)."""
    g = torch.Generator().manual_seed(seed)
    P = {}
    for k, shp in key_shapes(cfg).items():
        if k.endswith(".gamma"):
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith(".bias"):
            t = 0.1 * torch.randn(shp, generator=g)
        else:
            fan_in = shp[1] * (shp[-1] * shp[-2])
            t = torch.randn(shp, generator=g) * fan_in ** -0.5
        P[k] = t.bfloat16().float()
    return P


def rms_norm(x, gamma):
    """QwenImageRMS_norm (channel_first, no bias): F.normalize(x, dim=1) * sqrt(C) * gamma."""
    return F.normalize(x, dim=1) * x.shape[1] ** 0.5 * gamma


def _attend(x, P, pre):
    """QwenImageAttentionBlock on [N, C, h, w] frames: one head of width C."""
    n, c, h, w = x.shape
    t = rms_norm(x, P[f"{pre}.norm.gamma"].to(x))
    qkv = F.conv2d(t, P[f"{pre}.to_qkv.weight"].to(x), P[f"{pre}.to_qkv.bias"].to(x))
    qkv = qkv.reshape(n, 1, 3 * c, h * w).permute(0, 1, 3, 2)
    q, k, v = qkv.chunk(3, dim=-1)
    s = (q @ k.transpose(-1, -2)) * c ** -0.5
    o = s.softmax(-1) @ v
    o = o.squeeze(1).permute(0, 2, 1).reshape(n, c, h, w)
    return F.conv2d(o, P[f"{pre}.proj.weight"].to(x), P[f"{pre}.proj.bias"].to(x)) + x


# ---------------------------------------------------------------------------------------------- 3-D causal form
def _causal_conv3d(x, w, b, cache=None):
    """QwenImageCausalConv3d: pad (k_t - 1) frames in front (minus the cached frames prepended), none behind."""
    kt, kh = w.shape[2], w.shape[3]
    pt, ps = kt - 1, (kh - 1) // 2
    if cache is not None and pt > 0:
        x = torch.cat([cache, x], 2)
        pt -= cache.shape[2]
    return F.conv3d(F.pad(x, (ps, ps, ps, ps, pt, 0)), w, b)


def _res3d(x, P, pre, feat_cache):
    h = _causal_conv3d(x, P[f"{pre}.conv_shortcut.weight"].to(x), P[f"{pre}.conv_shortcut.bias"].to(x)) \
        if f"{pre}.conv_shortcut.weight" in P else x
    x = F.silu(rms_norm(x, P[f"{pre}.norm1.gamma"].to(x)))
    x = _causal_conv3d(x, P[f"{pre}.conv1.weight"].to(x), P[f"{pre}.conv1.bias"].to(x), feat_cache.pop(0))
    x = F.silu(rms_norm(x, P[f"{pre}.norm2.gamma"].to(x)))
    x = _causal_conv3d(x, P[f"{pre}.conv2.weight"].to(x), P[f"{pre}.conv2.bias"].to(x), feat_cache.pop(0))
    return x + h


def _per_frame(x, fn):
    b, c, t, h, w = x.shape
    y = fn(x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w))
    return y.view(b, t, *y.shape[1:]).permute(0, 2, 1, 3, 4)


def encode3d(pixels5: torch.Tensor, P: Dict[str, torch.Tensor], cfg: QwenVaeConfig) -> torch.Tensor:
    """moments [B, 2 z, 1, h, w] of the first chunk ([B, 3, 1, H, W] input) in the dtype and on the device of pixels5.
    Chunk 0 has no feature cache: every causal conv gets cache None, and downsample3d keeps its input for the next chunk
    instead of running time_conv."""
    assert pixels5.dim() == 5 and pixels5.shape[2] == 1, "the first chunk is one frame"
    blocks, dims = _layout(cfg)
    feat_cache: List[Optional[torch.Tensor]] = [None] * 64        # chunk 0: nothing cached yet
    x = _causal_conv3d(pixels5, P["encoder.conv_in.weight"].to(pixels5), P["encoder.conv_in.bias"].to(pixels5),
                       feat_cache.pop(0))
    for i, blk in enumerate(blocks):
        pre = f"encoder.down_blocks.{i}"
        if blk[0] == "res":
            x = _res3d(x, P, pre, feat_cache)
        else:
            w, b = P[f"{pre}.resample.1.weight"].to(x), P[f"{pre}.resample.1.bias"].to(x)
            x = _per_frame(x, lambda f: F.conv2d(F.pad(f, (0, 1, 0, 1)), w, b, stride=2))
            if blk[2] and feat_cache.pop(0) is not None:         # downsample3d: chunk 0 only caches x
                raise NotImplementedError("time_conv runs from the second chunk on")
    x = _res3d(x, P, "encoder.mid_block.resnets.0", feat_cache)
    x = _per_frame(x, lambda f: _attend(f, P, "encoder.mid_block.attentions.0"))
    x = _res3d(x, P, "encoder.mid_block.resnets.1", feat_cache)
    x = F.silu(rms_norm(x, P["encoder.norm_out.gamma"].to(x)))
    x = _causal_conv3d(x, P["encoder.conv_out.weight"].to(x), P["encoder.conv_out.bias"].to(x), feat_cache.pop(0))
    return _causal_conv3d(x, P["quant_conv.weight"].to(x), P["quant_conv.bias"].to(x))


# ---------------------------------------------------------------------------------------------- 2-D form
def _tap(w):
    """The temporal tap of a causal conv weight that meets the frame when two zero frames precede it: the last."""
    return w[:, :, -1]


def _res2d(x, P, pre):
    h = F.conv2d(x, _tap(P[f"{pre}.conv_shortcut.weight"]).to(x), P[f"{pre}.conv_shortcut.bias"].to(x)) \
        if f"{pre}.conv_shortcut.weight" in P else x
    x = F.silu(rms_norm(x, P[f"{pre}.norm1.gamma"].to(x)[..., 0]))
    x = F.conv2d(x, _tap(P[f"{pre}.conv1.weight"]).to(x), P[f"{pre}.conv1.bias"].to(x), padding=1)
    x = F.silu(rms_norm(x, P[f"{pre}.norm2.gamma"].to(x)[..., 0]))
    x = F.conv2d(x, _tap(P[f"{pre}.conv2.weight"]).to(x), P[f"{pre}.conv2.bias"].to(x), padding=1)
    return x + h


def encode2d(pixels: torch.Tensor, P: Dict[str, torch.Tensor], cfg: QwenVaeConfig) -> torch.Tensor:
    """moments [B, 2 z, h, w] of [B, 3, H, W] images by the 2-D network: tap-2 3x3 convs, ZeroPad2d + stride-2 convs."""
    blocks, _ = _layout(cfg)
    x = F.conv2d(pixels, _tap(P["encoder.conv_in.weight"]).to(pixels), P["encoder.conv_in.bias"].to(pixels), padding=1)
    for i, blk in enumerate(blocks):
        pre = f"encoder.down_blocks.{i}"
        if blk[0] == "res":
            x = _res2d(x, P, pre)
        else:
            x = F.conv2d(F.pad(x, (0, 1, 0, 1)), P[f"{pre}.resample.1.weight"].to(x), P[f"{pre}.resample.1.bias"].to(x), stride=2)
    x = _res2d(x, P, "encoder.mid_block.resnets.0")
    x = _attend(x, P, "encoder.mid_block.attentions.0")
    x = _res2d(x, P, "encoder.mid_block.resnets.1")
    x = F.silu(rms_norm(x, P["encoder.norm_out.gamma"].to(x)[..., 0]))
    x = F.conv2d(x, _tap(P["encoder.conv_out.weight"]).to(x), P["encoder.conv_out.bias"].to(x), padding=1)
    return F.conv2d(x, _tap(P["quant_conv.weight"]).to(x), P["quant_conv.bias"].to(x))


# ---------------------------------------------------------------------------------------------- sampling + normalisation
def sample_normalized(moments: torch.Tensor, eps: torch.Tensor, cfg: QwenVaeConfig) -> torch.Tensor:
    """DiagonalGaussianDistribution(moments).sample() with noise eps, then post_vae_encode_transform_sample's
    (z - latents_mean[c]) * (1 / latents_std[c]), in the dtype of moments ([B, 2z, ...] -> [B, z, ...])."""
    mean, logvar = moments.chunk(2, dim=1)
    z = mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * eps
    shape = (1, cfg.z_dim) + (1,) * (moments.dim() - 2)
    lm = torch.tensor(cfg.latents_mean, dtype=torch.float64).view(shape).to(moments)
    ls = torch.tensor(cfg.latents_std, dtype=torch.float64).view(shape).to(moments)
    return (z - lm) * (1.0 / ls)
