"""Qwen-Image VAE *encoder* on libstb200: diffusers `AutoencoderKLQwenImage` (the Wan 2.1 causal 3-D VAE, reference
`AUTOENCODER_CLASS` at qwen_image/model.py:62) for single-frame images, as encoded by the latent cache
(`pre_vae_encode_transform_sample` unsqueezes [B, 3, H, W] to [B, 3, 1, H, W]; `post_vae_encode_transform_sample`
samples and normalises per channel, qwen_image/model.py:1744-1768).

For one frame the causal 3-D network is a 2-D one:
  * every QwenImageCausalConv3d with temporal kernel 3 pads two zero frames in front of the frame (the first chunk has
    no cache), so only its last temporal tap w[:, :, 2] meets data and the layer is a 3x3 conv;
  * `downsample3d` skips its `time_conv` on the first chunk (it only fills the cache), so it is `downsample2d`:
    ZeroPad2d(0, 1, 0, 1) and a stride-2 3x3 conv;
  * the mid-block attention runs per frame.
The parameters keep diffusers' names and 5-D shapes (`encoder.down_blocks.3.conv1.weight` [192, 96, 3, 3, 3],
`encoder.norm_out.gamma` [384, 1, 1, 1], `quant_conv.weight` …) so the reference state dict loads with strict=True;
the 2-D weights (the last temporal tap, NHWC tap-major) are derived once.

Layout: activations NHWC bf16.  RMS norm (+ SiLU): ops.rmsnorm_fwd(normalize=True); 3x3 convs: ops.conv3x3_nhwc (96-channel
inputs are zero-padded to 128 per tap); 1x1 shortcuts, q | k | v, proj and quant_conv: ops.gemm over pixels; the mid-block
attention (one head, head dim = C = 384): score GEMM -> row softmax -> PV GEMM per image.  Inference only.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional, Sequence

import torch
import torch.nn as nn

from .. import ops
from .autoencoder import DiagonalGaussian, single_head_attention


class _CausalConv(nn.Module):
    """QwenImageCausalConv3d parameters; w2d(): the [C_out, C_in, k, k] tap that sees the frame (the last one)."""

    def __init__(self, cin, cout, k, dtype, kt=None):
        super().__init__()
        kt = k if kt is None else kt
        self.weight = nn.Parameter(torch.empty((cout, cin, kt, k, k), dtype=dtype), requires_grad=False)
        self.bias = nn.Parameter(torch.empty((cout,), dtype=dtype), requires_grad=False)
        self._w = None

    def _derived(self):
        if self._w is None or self._w[0].device != self.weight.device:
            w = self.weight.detach()[:, :, -1].contiguous()
            k = w.shape[-1]
            self._w = (w, ops.conv_w9(w) if k == 3 else w.reshape(w.shape[0], -1).contiguous())
        return self._w

    def w2d(self):
        return self._derived()[0]

    def wk(self):
        """3x3: the conv3x3_nhwc weight (ops.conv_w9); 1x1: the [C_out, C_in] GEMM weight."""
        return self._derived()[1]


class _Conv2d(nn.Module):
    """nn.Conv2d parameters: a Resample's `resample.1` (3x3) or the attention's to_qkv / proj (1x1)."""

    def __init__(self, cin, cout, k, dtype):
        super().__init__()
        self.weight = nn.Parameter(torch.empty((cout, cin, k, k), dtype=dtype), requires_grad=False)
        self.bias = nn.Parameter(torch.empty((cout,), dtype=dtype), requires_grad=False)
        self._w9 = None

    def w9(self):
        if self._w9 is None or self._w9.device != self.weight.device:
            self._w9 = ops.conv_w9(self.weight)
        return self._w9

    def w(self):
        return self.weight.detach().view(self.weight.shape[0], -1)


class _RMSNorm(nn.Module):
    """QwenImageRMS_norm without bias: gamma [C, 1, 1, 1] (images=False) or [C, 1, 1] (images=True)."""

    def __init__(self, c, images, dtype):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones((c, 1, 1) if images else (c, 1, 1, 1), dtype=dtype), requires_grad=False)

    def forward(self, x, silu):
        C = x.shape[-1]
        return ops.rmsnorm_fwd(x.view(1, -1, C), self.gamma.detach().view(-1), 1e-12, normalize=True, silu=silu).view(x.shape)


def _gemm_1x1(x, conv, **kw):
    B, H, W, C = x.shape
    return ops.gemm([x.view(B, H * W, C)], [conv.wk()], conv.bias, **kw).view(B, H, W, -1)


class _Residual(nn.Module):
    """QwenImageResidualBlock: norm1 + SiLU -> conv1 -> norm2 + SiLU -> conv2, plus x or its 1x1 conv_shortcut."""

    def __init__(self, cin, cout, dtype):
        super().__init__()
        self.norm1 = _RMSNorm(cin, False, dtype)
        self.conv1 = _CausalConv(cin, cout, 3, dtype)
        self.norm2 = _RMSNorm(cout, False, dtype)
        self.conv2 = _CausalConv(cout, cout, 3, dtype)
        if cin != cout:
            self.conv_shortcut = _CausalConv(cin, cout, 1, dtype)

    def forward(self, x):  # NHWC
        sc = _gemm_1x1(x, self.conv_shortcut) if hasattr(self, "conv_shortcut") else x
        h = ops.conv3x3_nhwc(self.norm1(x, True), self.conv1.wk(), self.conv1.bias)
        return ops.conv3x3_nhwc(self.norm2(h, True), self.conv2.wk(), self.conv2.bias, res=sc)  # + shortcut in the epilogue


class _Resample(nn.Module):
    """QwenImageResample, downsample2d / downsample3d: ZeroPad2d(0, 1, 0, 1) + Conv2d(c, c, 3, stride 2).  The
    time_conv of downsample3d is held for the state dict; a single frame never reaches it."""

    def __init__(self, c, temporal, dtype):
        super().__init__()
        self.resample = nn.ModuleList([nn.ZeroPad2d((0, 1, 0, 1)), _Conv2d(c, c, 3, dtype)])
        if temporal:
            self.time_conv = _CausalConv(c, c, 1, dtype, kt=3)

    def forward(self, x):
        conv = self.resample[1]
        return ops.conv3x3_nhwc(x, conv.w9(), conv.bias, stride=2)


class _Attention(nn.Module):
    """QwenImageAttentionBlock: RMS norm, to_qkv (1x1), single-head attention with head dim C, proj (1x1), + x."""

    def __init__(self, c, dtype):
        super().__init__()
        self.norm = _RMSNorm(c, True, dtype)
        self.to_qkv = _Conv2d(c, 3 * c, 1, dtype)
        self.proj = _Conv2d(c, c, 1, dtype)

    def forward(self, x):
        B, H, W, C = x.shape
        t = self.norm(x, False).view(B, H * W, C)
        return single_head_attention(t, x, self.to_qkv.w(), self.to_qkv.bias, self.proj.w(), self.proj.bias)


class _MidBlock(nn.Module):
    def __init__(self, c, dtype):
        super().__init__()
        self.resnets = nn.ModuleList([_Residual(c, c, dtype), _Residual(c, c, dtype)])
        self.attentions = nn.ModuleList([_Attention(c, dtype)])

    def forward(self, x):
        return self.resnets[1](self.attentions[0](self.resnets[0](x)))


class _Encoder(nn.Module):
    """QwenImageEncoder3d: conv_in, a flat list of residual blocks and resamples, mid block, norm_out + SiLU, conv_out."""

    def __init__(self, cfg, dtype):
        super().__init__()
        dims = [cfg.base_dim * u for u in [1, *cfg.dim_mult]]
        self.conv_in = _CausalConv(3, dims[0], 3, dtype)
        blocks = []
        for i, (cin, cout) in enumerate(zip(dims[:-1], dims[1:])):
            for _ in range(cfg.num_res_blocks):
                blocks.append(_Residual(cin, cout, dtype))
                cin = cout
            if i != len(cfg.dim_mult) - 1:
                blocks.append(_Resample(cout, bool(cfg.temperal_downsample[i]), dtype))
        self.down_blocks = nn.ModuleList(blocks)
        self.mid_block = _MidBlock(dims[-1], dtype)
        self.norm_out = _RMSNorm(dims[-1], False, dtype)
        self.conv_out = _CausalConv(dims[-1], 2 * cfg.z_dim, 3, dtype)

    def forward(self, pixels):  # [B, 3, H, W] in, NHWC out
        x = ops.conv_in_3ch(pixels.contiguous(), self.conv_in.w2d(), self.conv_in.bias.detach())
        for blk in self.down_blocks:
            x = blk(x)
        x = self.mid_block(x)
        return ops.conv3x3_nhwc(self.norm_out(x, True), self.conv_out.wk(), self.conv_out.bias)


class QwenImageDiagonalGaussian(DiagonalGaussian):
    """`latent_dist` with the reference's 5-D shapes: parameters [B, 2z, 1, h, w], sample() [B, z, 1, h, w]."""

    @property
    def parameters(self) -> torch.Tensor:
        return super().parameters.unsqueeze(2)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        return super().sample(generator).unsqueeze(2)


class QwenImageVAE(nn.Module):
    """Encoder half of AutoencoderKLQwenImage for single-frame images (see the module docstring)."""

    def __init__(self, base_dim: int = 96, z_dim: int = 16, dim_mult: Sequence[int] = (1, 2, 4, 4), num_res_blocks: int = 2,
                 attn_scales: Sequence[float] = (), temperal_downsample: Sequence[bool] = (False, True, True),
                 dropout: float = 0.0, latents_mean: Optional[Sequence[float]] = None,
                 latents_std: Optional[Sequence[float]] = None, dtype=torch.bfloat16, **unused):
        super().__init__()
        if len(attn_scales):
            raise NotImplementedError("libstb200 Qwen-Image VAE encoder: attention in the down blocks (attn_scales) is not supported")
        if unused.get("is_residual") or unused.get("patch_size") or unused.get("in_channels", 3) != 3:
            raise NotImplementedError("libstb200 Qwen-Image VAE encoder: Wan 2.2 style configs are not supported")
        if len(temperal_downsample) != len(dim_mult) - 1:
            raise NotImplementedError("temperal_downsample needs one entry per downsampling level")
        latents_mean = [0.0] * z_dim if latents_mean is None else list(latents_mean)
        latents_std = [1.0] * z_dim if latents_std is None else list(latents_std)
        if len(latents_mean) != z_dim or len(latents_std) != z_dim:
            raise ValueError("latents_mean / latents_std need z_dim entries")
        self.config = SimpleNamespace(base_dim=base_dim, z_dim=z_dim, dim_mult=tuple(dim_mult), num_res_blocks=num_res_blocks,
                                      attn_scales=tuple(attn_scales), temperal_downsample=tuple(temperal_downsample),
                                      dropout=dropout, latents_mean=latents_mean, latents_std=latents_std)
        self.encoder = _Encoder(self.config, dtype)
        self.quant_conv = _CausalConv(2 * z_dim, 2 * z_dim, 1, dtype)
        self._norm = None

    @property
    def dtype(self):
        return self.encoder.conv_in.weight.dtype

    @property
    def device(self):
        return self.encoder.conv_in.weight.device

    @property
    def spatial_multiple(self) -> int:
        """H and W must be multiples of this (every stride-2 conv halves an even size)."""
        return 2 ** (len(self.config.dim_mult) - 1)

    def latent_norm(self):
        """(latents_mean, 1 / latents_std) as post_vae_encode_transform_sample forms them: the config lists become
        fp32 tensors, are cast to bf16, and the reciprocal is taken of the bf16 std (bf16 result)."""
        if self._norm is None or self._norm[0].device != self.device:
            mean = torch.tensor(self.config.latents_mean).to(self.device, torch.bfloat16)
            inv_std = 1.0 / torch.tensor(self.config.latents_std).to(self.device, torch.bfloat16)
            self._norm = (mean.contiguous(), inv_std.contiguous())
        return self._norm

    @torch.no_grad()
    def _moments(self, samples: torch.Tensor) -> torch.Tensor:
        if not samples.is_cuda:
            from .._lib import StbError
            raise StbError("QwenImageVAE (libstb200) needs CUDA tensors; there is no CPU fallback")
        if samples.dim() != 5 or samples.shape[1] != 3 or samples.shape[2] != 1:
            raise ValueError(f"QwenImageVAE encodes [B, 3, 1, H, W] (one frame), got {tuple(samples.shape)}")
        m = self.spatial_multiple
        if samples.shape[3] % m or samples.shape[4] % m:
            raise ValueError(f"QwenImageVAE needs H and W multiples of {m}, got {tuple(samples.shape[3:])}")
        x = self.encoder(samples[:, :, 0].to(self.dtype))
        return _gemm_1x1(x, self.quant_conv)

    @torch.no_grad()
    def encode(self, samples: torch.Tensor, return_dict: bool = True):
        return SimpleNamespace(latent_dist=QwenImageDiagonalGaussian(self._moments(samples)))

    @torch.no_grad()
    def encode_scaled(self, samples: torch.Tensor, eps: Optional[torch.Tensor] = None) -> torch.Tensor:
        """encode -> latent_dist.sample() -> (z - latents_mean) * (1 / latents_std) in one launch: [B, z, h, w], what
        post_vae_encode_transform_sample returns."""
        m = self._moments(samples)
        B, h, w, L2 = m.shape
        if eps is None:
            eps = torch.randn((B, L2 // 2, h, w), device=m.device, dtype=m.dtype)
        mean, inv_std = self.latent_norm()
        return ops.gaussian_sample_scale(m, eps.reshape(B, L2 // 2, h, w).contiguous(), mean, inv_std)
