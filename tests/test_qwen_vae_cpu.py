"""CPU: the Qwen-Image VAE oracle's 2-D reduction, the state-dict key list, the shim's routing, and the bf16 replays
of the RMS-norm chain and the per-channel latent normalisation against torch's eager chains."""
import logging
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from oracle import qwen_vae_oracle as O


def _pixels(B, H, W, dtype, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, 3, H, W, generator=g, dtype=torch.float64) * 2 - 1).to(dtype)


def test_causal_3d_encoder_on_one_frame_is_the_2d_tap2_network():
    """The whole encoder: the 3-D causal form and the 2-D form differ only in how conv3d and conv2d order their sums
    (fp64: 1e-12 relative to the largest moment)."""
    cfg = O.QwenVaeConfig(base_dim=16)
    P = {k: v.double() for k, v in O.init_params(cfg, 0).items()}
    x = _pixels(2, 32, 48, torch.float64)
    m3, m2 = O.encode3d(x.unsqueeze(2), P, cfg), O.encode2d(x, P, cfg)
    assert m3.shape == (2, 32, 1, 4, 6)
    assert (m3[:, :, 0] - m2).abs().max() <= 1e-12 * m2.abs().max()
    m3f = O.encode3d(x.float().unsqueeze(2), {k: v.float() for k, v in P.items()}, cfg)
    assert (m3f.double() - m3).abs().max() <= 1e-4 * m3.abs().max()


def test_causal_conv3d_first_chunk_is_the_last_tap_bit_for_bit():
    """Each causal conv alone, on exact inputs (integers, weights k / 16): every sum is exact, so the 3-D conv with
    its two zero frames in front equals conv2d with w[:, :, 2] bit for bit, and no other tap reaches the frame."""
    g = torch.Generator().manual_seed(3)
    x = torch.randint(-2, 3, (2, 24, 1, 9, 11), generator=g).double()
    w = torch.randint(-6, 7, (16, 24, 3, 3, 3), generator=g).double() / 16
    b = torch.randint(-6, 7, (16,), generator=g).double() / 16
    y3 = O._causal_conv3d(x, w, b)
    assert torch.equal(y3[:, :, 0], F.conv2d(x[:, :, 0], w[:, :, 2], b, padding=1))
    w2 = w.clone()
    w2[:, :, :2] = 1e6
    assert torch.equal(O._causal_conv3d(x, w2, b), y3)


def test_state_dict_keys_are_diffusers_names():
    from simpletuner_b200.vae.qwen_image import QwenImageVAE
    cfg = O.QwenVaeConfig()
    want = O.key_shapes(cfg)
    m = QwenImageVAE(**cfg.as_dict())
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == dict(want)
    assert len(want) == 86
    keys = list(want)
    assert keys[:4] == ["encoder.conv_in.weight", "encoder.conv_in.bias", "encoder.down_blocks.0.norm1.gamma",
                        "encoder.down_blocks.0.conv1.weight"]
    assert "encoder.down_blocks.2.resample.1.weight" in want and "encoder.down_blocks.2.time_conv.weight" not in want
    assert want["encoder.down_blocks.5.time_conv.weight"] == (192, 192, 3, 1, 1)
    assert want["encoder.down_blocks.3.conv_shortcut.weight"] == (192, 96, 1, 1, 1)
    assert want["encoder.mid_block.attentions.0.to_qkv.weight"] == (1152, 384, 1, 1)
    assert keys[-4:] == ["encoder.conv_out.weight", "encoder.conv_out.bias", "quant_conv.weight", "quant_conv.bias"]
    m.load_state_dict({k: torch.zeros(s) for k, s in want.items()}, strict=True)


class _RefVAE(torch.nn.Module):
    def __init__(self, config, sd, use_tiling=False):
        super().__init__()
        self.config, self._sd, self.use_tiling = config, sd, use_tiling

    def state_dict(self, *a, **k):
        return self._sd


class _Base:
    def post_vae_load_setup(self):
        pass

    def encode_with_vae(self, vae, samples):
        return "reference"


def _family(ref_vae):
    from simpletuner_b200.shim.vae import B200VAEMixin

    class Fam(B200VAEMixin, _Base):
        pass

    f = Fam()
    f.vae = ref_vae
    f.accelerator = SimpleNamespace(device=torch.device("cpu"))
    f.post_vae_load_setup()
    return f


def _qwen_ref(cfg=None, **kw):
    cfg = cfg or O.QwenVaeConfig(base_dim=16)
    sd = {k: torch.zeros(s) for k, s in O.key_shapes(cfg).items()}
    sd["decoder.conv_in.weight"] = torch.zeros(1)
    return _RefVAE(cfg.as_dict(), sd, **kw)


def test_shim_routes_single_frame_qwen_batches_to_the_b200_encoder():
    from simpletuner_b200.vae.qwen_image import QwenImageVAE
    f = _family(_qwen_ref())
    assert isinstance(f._b200_vae, QwenImageVAE)
    f._b200_vae.encode = lambda s: "b200"
    assert f.encode_with_vae(f.vae, torch.zeros(1, 3, 1, 64, 64)) == "b200"
    assert f.encode_with_vae(f.vae, torch.zeros(1, 3, 2, 64, 64)) == "reference"       # video
    assert f.encode_with_vae(f.vae, torch.zeros(1, 3, 1, 60, 64)) == "reference"       # not a multiple of 8
    assert f.encode_with_vae(object(), torch.zeros(1, 3, 1, 64, 64)) == "reference"    # another VAE
    t = _family(_qwen_ref(use_tiling=True))
    t._b200_vae.encode = lambda s: "b200"
    assert t.encode_with_vae(t.vae, torch.zeros(1, 3, 1, 64, 64)) == "reference"       # tiled encode


def test_shim_keeps_autoencoderkl_and_refuses_unsupported_qwen_configs(caplog):
    from simpletuner_b200.vae.autoencoder import AutoencoderKL
    from simpletuner_b200.vae.qwen_image import QwenImageVAE
    kl = AutoencoderKL(block_out_channels=(32, 32), norm_num_groups=8)
    f = _family(_RefVAE({"block_out_channels": [32, 32], "norm_num_groups": 8, "latent_channels": 16},
                        kl.state_dict(), use_tiling=True))
    assert isinstance(f._b200_vae, AutoencoderKL) and not isinstance(f._b200_vae, QwenImageVAE)
    f._b200_vae.encode = lambda s: "b200"
    assert f.encode_with_vae(f.vae, torch.zeros(1, 3, 64, 64)) == "b200"                # unchanged routing
    cfg = O.QwenVaeConfig(base_dim=16, attn_scales=(1.0,))
    with caplog.at_level(logging.WARNING, logger="simpletuner_b200.shim"):
        g = _family(_qwen_ref(cfg))
    assert g._b200_vae is None and "VAE encode not used" in caplog.text
    assert g.encode_with_vae(g.vae, torch.zeros(1, 3, 1, 64, 64)) == "reference"


@pytest.mark.parametrize("C", [8, 96, 384])
@pytest.mark.parametrize("bias", [False, True])
def test_rmsnorm_replay_matches_the_eager_bf16_chain(C, bias):
    """On rows whose sum of squares is exact in fp32 (small integers times powers of two) the norm does not depend on
    the summation order, so the replay must match torch's eager bf16 chain bit for bit."""
    from tests.qwen_vae_checks import channel_rmsnorm_norms, channel_rmsnorm_replay
    g = torch.Generator().manual_seed(C)
    R = 64
    x = (torch.randint(-7, 8, (R, C), generator=g).double() * torch.pow(2.0, torch.arange(R) % 7 - 3).view(R, 1)).bfloat16()
    x[0] = 0
    gm = (1 + 0.1 * torch.randn(C, generator=g)).bfloat16()
    bv = (0.1 * torch.randn(C, generator=g)).bfloat16() if bias else None
    n_lo, n_hi = channel_rmsnorm_norms(x)
    y = channel_rmsnorm_replay(x, gm, bv, n_lo)
    eager = F.normalize(x, dim=-1) * C ** 0.5 * gm + (bv if bias else 0.0)
    assert torch.equal(y.view(torch.int16), eager.view(torch.int16))
    assert torch.equal(F.silu(y).view(torch.int16), F.silu(eager).view(torch.int16))


def test_channel_normalisation_replay_matches_post_vae_encode_transform_sample():
    """The reference's chain (qwen_image/model.py:1744-1768), restated: latents_std is cast to bf16 before the
    reciprocal, which is then a bf16 op; the kernel's inputs (QwenImageVAE.latent_norm) are built the same way."""
    from simpletuner_b200.vae.qwen_image import QwenImageVAE
    cfg = O.QwenVaeConfig(base_dim=16)
    g = torch.Generator().manual_seed(2)
    z = torch.randn(2, 16, 1, 6, 10, generator=g).bfloat16()
    lm = torch.tensor(cfg.latents_mean).view(1, 16, 1, 1).to("cpu", z.dtype)
    ls = 1.0 / torch.tensor(cfg.latents_std).view(1, 16, 1, 1).to("cpu", z.dtype)
    eager = (z.squeeze(2) - lm) * ls
    vae = QwenImageVAE(**cfg.as_dict())
    mean_c, inv_c = vae.latent_norm()
    replay = ((z.squeeze(2).float() - mean_c.float().view(1, 16, 1, 1)).bfloat16().float()
              * inv_c.float().view(1, 16, 1, 1)).bfloat16()
    assert torch.equal(replay.view(torch.int16), eager.view(torch.int16))
