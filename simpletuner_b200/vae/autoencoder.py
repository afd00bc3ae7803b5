"""AutoencoderKL *encoder* on libstb200 — the B200-native drop-in for the VAE latent-encode path
(SURVEY.md §8b seam B8): reference `AUTOENCODER_CLASS` (flux/model.py:61, diffusers AutoencoderKL) as used by
`ModelFoundation.encode_with_vae` (common.py:2766-2772) from `VAECache.encode_images` (caching/vae.py:1238-1396).

`encode(samples[n,3,H,W])` returns an object with `.latent_dist.sample()` / `.latent_dist.parameters`, which is
what caching/vae.py:1331-1343 consumes; `encode_scaled(samples)` additionally fuses sampling with
`scale_vae_latents_for_cache` (foundation_mixins.py:68-81).  Parameter names follow the diffusers state_dict
(`encoder.down_blocks.0.resnets.0.conv1.weight`, `encoder.mid_block.attentions.0.to_q.weight`, `quant_conv.weight` …).

Layout: activations NHWC bf16.  Every 3x3 conv is the wgmma implicit-GEMM kernel (ops.conv3x3_nhwc; weights are
re-laid once to [C_out, (dy, dx, c_in)]); 1x1 shortcuts / attention projections are ops.gemm over pixels; the
mid-block single-head attention (head_dim 512) runs as score GEMM -> row softmax -> PV GEMM per image; GroupNorm+SiLU
is a two-kernel NHWC pass.  Inference only (the reference runs it under torch.no_grad).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from .. import ops


class _Conv(nn.Module):
    def __init__(self, cin, cout, k, dtype):
        super().__init__()
        self.weight = nn.Parameter(torch.empty((cout, cin, k, k), dtype=dtype), requires_grad=False)
        self.bias = nn.Parameter(torch.empty((cout,), dtype=dtype), requires_grad=False)
        self._w9 = None

    def w9(self):
        """[C_out, C_in, kh, kw] -> [C_out, (kh, kw, C_in)] contiguous (tap-major K for the implicit GEMM)."""
        if self._w9 is None or self._w9.device != self.weight.device:
            w = self.weight.detach()
            self._w9 = w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()
        return self._w9


class _Norm(nn.Module):
    def __init__(self, c, dtype):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c, dtype=dtype), requires_grad=False)
        self.bias = nn.Parameter(torch.zeros(c, dtype=dtype), requires_grad=False)


class _Lin(nn.Module):
    def __init__(self, cin, cout, dtype):
        super().__init__()
        self.weight = nn.Parameter(torch.empty((cout, cin), dtype=dtype), requires_grad=False)
        self.bias = nn.Parameter(torch.empty((cout,), dtype=dtype), requires_grad=False)


class _Resnet(nn.Module):
    """diffusers ResnetBlock2D(temb_channels=None, groups=32, eps=1e-6, silu, output_scale_factor=1)."""

    def __init__(self, cin, cout, groups, dtype):
        super().__init__()
        self.groups = groups
        self.norm1 = _Norm(cin, dtype)
        self.conv1 = _Conv(cin, cout, 3, dtype)
        self.norm2 = _Norm(cout, dtype)
        self.conv2 = _Conv(cout, cout, 3, dtype)
        if cin != cout:
            self.conv_shortcut = _Conv(cin, cout, 1, dtype)

    def forward(self, x):  # NHWC
        h = ops.groupnorm_nhwc(x, self.norm1.weight, self.norm1.bias, self.groups, 1e-6, True)
        h = ops.conv3x3_nhwc(h, self.conv1.w9(), self.conv1.bias)
        h = ops.groupnorm_nhwc(h, self.norm2.weight, self.norm2.bias, self.groups, 1e-6, True)
        if hasattr(self, "conv_shortcut"):
            B, H, W, C = x.shape
            sc = ops.gemm([x.view(B, H * W, C)], [self.conv_shortcut.w9()], self.conv_shortcut.bias).view(B, H, W, -1)
        else:
            sc = x
        return ops.conv3x3_nhwc(h, self.conv2.w9(), self.conv2.bias, res=sc)  # conv2 + bias + shortcut in the epilogue


class _Downsample(nn.Module):
    def __init__(self, c, dtype):
        super().__init__()
        self.conv = _Conv(c, c, 3, dtype)

    def forward(self, x):
        return ops.conv3x3_nhwc(x, self.conv.w9(), self.conv.bias, stride=2)  # F.pad(0,1,0,1) + stride 2


class _DownBlock(nn.Module):
    def __init__(self, cin, cout, layers, down, groups, dtype):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(cin if i == 0 else cout, cout, groups, dtype) for i in range(layers)])
        if down:
            self.downsamplers = nn.ModuleList([_Downsample(cout, dtype)])

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if hasattr(self, "downsamplers"):
            x = self.downsamplers[0](x)
        return x


class _MidAttention(nn.Module):
    """diffusers Attention(heads=1, dim_head=C, norm_num_groups=32, residual_connection=True) of UNetMidBlock2D."""

    def __init__(self, c, groups, dtype):
        super().__init__()
        self.c, self.groups = c, groups
        self.group_norm = _Norm(c, dtype)
        self.to_q = _Lin(c, c, dtype)
        self.to_k = _Lin(c, c, dtype)
        self.to_v = _Lin(c, c, dtype)
        self.to_out = nn.ModuleList([_Lin(c, c, dtype), nn.Identity()])
        self._qkv = None

    def forward(self, x):  # NHWC
        B, H, W, C = x.shape
        S = H * W
        if self._qkv is None or self._qkv[0].device != x.device:
            self._qkv = (torch.cat([self.to_q.weight, self.to_k.weight, self.to_v.weight], 0).detach().contiguous(),
                         torch.cat([self.to_q.bias, self.to_k.bias, self.to_v.bias], 0).detach().contiguous())
        t = ops.groupnorm_nhwc(x, self.group_norm.weight, self.group_norm.bias, self.groups, 1e-6, False).view(B, S, C)
        return single_head_attention(t, x, self._qkv[0], self._qkv[1], self.to_out[0].weight, self.to_out[0].bias)


def single_head_attention(t, x, w_qkv, b_qkv, w_out, b_out):
    """x + out_proj(softmax(q k^T / sqrt(C)) v) for one head of width C over each image's pixels: t [B, S, C] is the
    normalised input, x [B, H, W, C] the residual, w_qkv [3C, C] the q | k | v projection.  Returns [B, H, W, C]."""
    B, H, W, C = x.shape
    S = H * W
    qkv = ops.gemm([t], [w_qkv], b_qkv)                              # [B, S, 3C]
    out = torch.empty((B, S, C), device=x.device, dtype=torch.bfloat16)
    xr = x.view(B, S, C)
    for b in range(B):  # one image at a time: the score matrix is S x S (512 MB at 1024^2)
        q, k, v = qkv[b, :, 0:C], qkv[b, :, C:2 * C], qkv[b, :, 2 * C:]
        s = ops.gemm([q], [k])                                       # [S, S] = q k^T
        ops.softmax_rows_(s, C ** -0.5)
        vt = v.t().contiguous()                                      # [C, S]: K-major "weight" for P @ V
        o = ops.gemm([s], [vt])                                      # [S, C]
        ops.gemm([o], [w_out], b_out, out=out[b], epi=ops.EPI_ADD_RES, res=xr[b])
    return out.view(B, H, W, C)


class _MidBlock(nn.Module):
    def __init__(self, c, groups, attn, dtype):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(c, c, groups, dtype), _Resnet(c, c, groups, dtype)])
        self.attentions = nn.ModuleList([_MidAttention(c, groups, dtype)] if attn else [])

    def forward(self, x):
        x = self.resnets[0](x)
        if len(self.attentions):
            x = self.attentions[0](x)
        return self.resnets[1](x)


class _Encoder(nn.Module):
    def __init__(self, cfg, dtype):
        super().__init__()
        ch = cfg.block_out_channels
        G = cfg.norm_num_groups
        self.groups = G
        self.conv_in = _Conv(cfg.in_channels, ch[0], 3, dtype)
        blocks, prev = [], ch[0]
        for i, c in enumerate(ch):
            blocks.append(_DownBlock(prev, c, cfg.layers_per_block, i != len(ch) - 1, G, dtype))
            prev = c
        self.down_blocks = nn.ModuleList(blocks)
        self.mid_block = _MidBlock(ch[-1], G, cfg.mid_block_add_attention, dtype)
        self.conv_norm_out = _Norm(ch[-1], dtype)
        self.conv_out = _Conv(ch[-1], 2 * cfg.latent_channels, 3, dtype)

    def forward(self, pixels):  # NCHW in, NHWC moments out
        x = ops.conv_in_3ch(pixels.contiguous(), self.conv_in.weight.detach(), self.conv_in.bias.detach())
        for blk in self.down_blocks:
            x = blk(x)
        x = self.mid_block(x)
        x = ops.groupnorm_nhwc(x, self.conv_norm_out.weight, self.conv_norm_out.bias, self.groups, 1e-6, True)
        return ops.conv3x3_nhwc(x, self.conv_out.w9(), self.conv_out.bias)


class DiagonalGaussian:
    """What caching/vae.py:1331-1343 needs from `encode(...).latent_dist`: `.sample()` and `.parameters` (NCHW)."""

    def __init__(self, moments_nhwc: torch.Tensor):
        self._m = moments_nhwc

    @property
    def parameters(self) -> torch.Tensor:
        return self._m.permute(0, 3, 1, 2).contiguous()

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        B, h, w, L2 = self._m.shape
        eps = torch.randn((B, L2 // 2, h, w), device=self._m.device, dtype=self._m.dtype, generator=generator)
        return ops.gaussian_sample_scale(self._m, eps, None, 1.0)


class AutoencoderKL(nn.Module):
    def __init__(self, in_channels: int = 3, latent_channels: int = 16, block_out_channels: Tuple[int, ...] = (128, 256, 512, 512),
                 layers_per_block: int = 2, norm_num_groups: int = 32, use_quant_conv: bool = False,
                 scaling_factor: float = 0.3611, shift_factor: Optional[float] = 0.1159,
                 mid_block_add_attention: bool = True, dtype=torch.bfloat16, **unused):
        super().__init__()
        if in_channels != 3:
            raise NotImplementedError("libstb200 VAE encoder expects RGB input")
        self.config = SimpleNamespace(in_channels=in_channels, latent_channels=latent_channels,
                                      block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                      norm_num_groups=norm_num_groups, use_quant_conv=use_quant_conv,
                                      scaling_factor=scaling_factor, shift_factor=shift_factor,
                                      mid_block_add_attention=mid_block_add_attention)
        self.encoder = _Encoder(self.config, dtype)
        if use_quant_conv:
            self.quant_conv = _Conv(2 * latent_channels, 2 * latent_channels, 1, dtype)

    @property
    def dtype(self):
        return self.encoder.conv_in.weight.dtype

    @property
    def device(self):
        return self.encoder.conv_in.weight.device

    @torch.no_grad()
    def _moments(self, samples: torch.Tensor) -> torch.Tensor:
        if not samples.is_cuda:
            from .._lib import StbError
            raise StbError("AutoencoderKL (libstb200) needs CUDA tensors; there is no CPU fallback")
        m = self.encoder(samples.to(self.dtype))
        if self.config.use_quant_conv:
            B, h, w, C = m.shape
            m = ops.gemm([m.view(B, h * w, C)], [self.quant_conv.w9()], self.quant_conv.bias).view(B, h, w, C)
        return m

    @torch.no_grad()
    def encode(self, samples: torch.Tensor, return_dict: bool = True):
        return SimpleNamespace(latent_dist=DiagonalGaussian(self._moments(samples)))

    @torch.no_grad()
    def encode_scaled(self, samples: torch.Tensor, eps: Optional[torch.Tensor] = None) -> torch.Tensor:
        """encode -> latent_dist.sample() -> (z - shift) * scale in one pass (vae.py:1311, 1337, 1355)."""
        m = self._moments(samples)
        B, h, w, L2 = m.shape
        if eps is None:
            eps = torch.randn((B, L2 // 2, h, w), device=m.device, dtype=m.dtype)
        return ops.gaussian_sample_scale(m, eps.contiguous(), self.config.shift_factor, self.config.scaling_factor)
