"""CPU: Flux masked training (`flux_attention_masked_training`, SURVEY.md quirk Q2) — the masked oracle against the
reference's own processor (tests/golden/flux_attn_mask_golden.pt), the config rule that decides when the H100 path runs
it, the per-key `attn_mask` forms the SDPA override accepts, and the C ABI of the attention bias fields."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

from oracle import flux_oracle as O
from simpletuner_b200 import _lib
from simpletuner_b200.flux.model import Flux, check_masked_training, default_config
from simpletuner_b200.flux.transformer import FluxTransformer2DModel
from simpletuner_b200.shim.attention_backend import key_bias_from_mask
from tests import flux_mask_oracle as MO

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden" / "flux_attn_mask_golden.pt"


def _golden():
    return torch.load(GOLDEN, weights_only=False)


def _oracle_attention(g, case, mask):
    cfg = O.FluxConfig(num_attention_heads=g["H"], attention_head_dim=g["HD"])
    with MO.masked(mask):
        return O.flux_attention(case["P"], cfg, "", case["x"], case["enc"], (g["cos"], g["sin"]), None, 1.0)


@pytest.mark.parametrize("joint", [True, False], ids=["double_block", "single_block"])
def test_masked_oracle_matches_the_reference_processor(joint):
    g = _golden()
    case = next(c for c in g["cases"] if c["joint"] == joint)
    S = g["S_txt"] + g["S_img"]
    assert torch.equal(MO.key_bias(case["mask"], S), (case["expanded"] > 0).float())
    out = _oracle_attention(g, case, case["mask"])
    if joint:
        assert float((out[0] - case["out_img"]).abs().max()) <= 1e-5
        assert float((out[1] - case["out_txt"]).abs().max()) <= 1e-5
    else:
        assert case["mask"].shape[1] < g["S_txt"]           # the expansion pads a short mask with ones
        assert float((out - case["out"]).abs().max()) <= 1e-5
    # the mask matters: without it the same call differs
    plain = _oracle_attention(g, case, None)
    assert float(((plain[0] if joint else plain) - (out[0] if joint else out)).abs().max()) > 1e-3


def test_all_ones_mask_equals_no_mask():
    g = _golden()
    case = g["cases"][0]
    ones = torch.ones_like(case["mask"])
    a = _oracle_attention(g, case, ones)
    b = _oracle_attention(g, case, None)
    for x, y in zip(a, b):
        assert float((x - y).abs().max()) <= 1e-6


# ---- the config rule ------------------------------------------------------------------------------------------------
def _cfg(**over):
    kw = dict(lora_rank=4, model_type="lora", lora_type="standard", flux_attention_masked_training=True)
    kw.update(over)
    return default_config(**kw)


def test_masked_training_runs_for_the_default_processor():
    for over in (dict(attention_mechanism="diffusers"), dict(attention_mechanism="diffusers", fuse_qkv_projections=False)):
        c = _cfg(**over)
        Flux.validate_config(c)
        assert check_masked_training(c) is True
    assert check_masked_training(default_config()) is False


@pytest.mark.parametrize("over,needle", [
    (dict(), "attention_mechanism"),
    (dict(attention_mechanism="flash_attn"), "flash_attn"),
    (dict(attention_mechanism="flash-attn-3"), "flash-attn-3"),
    (dict(attention_mechanism="sageattention"), "sageattention"),
    (dict(attention_mechanism="diffusers", fuse_qkv_projections=True), "fuse_qkv_projections"),
])
def test_masked_training_raises_where_the_reference_masks_differently(over, needle):
    c = _cfg(**over)
    for check in (lambda: Flux.validate_config(c), lambda: check_masked_training(c)):
        with pytest.raises(NotImplementedError, match="flux_attention_masked_training") as e:
            check()
        assert needle in str(e.value)
    w = Flux(c, transformer=FluxTransformer2DModel(num_layers=1, num_single_layers=1, num_attention_heads=2,
                                                   joint_attention_dim=64, pooled_projection_dim=32),
             device=torch.device("cpu"))
    with pytest.raises(NotImplementedError, match="flux_attention_masked_training"):
        w.prepare_batch({"latent_batch": torch.zeros(1, 16, 4, 4), "encoder_attention_mask": torch.ones(1, 8)}, {})


def test_a_batch_without_its_mask_raises():
    w = Flux(_cfg(attention_mechanism="diffusers"),
             transformer=FluxTransformer2DModel(num_layers=1, num_single_layers=1, num_attention_heads=2,
                                                joint_attention_dim=64, pooled_projection_dim=32),
             device=torch.device("cpu"))
    with pytest.raises(NotImplementedError, match="flux_attention_masked_training.*encoder_attention_mask"):
        w.prepare_batch({"latent_batch": torch.zeros(1, 16, 4, 4)}, {})


def test_flash_processors_are_refused_while_masked_training_is_on():
    class FluxFusedFlashAttnProcessor3:
        pass

    class FluxAttnProcessor2_0:
        pass

    m = FluxTransformer2DModel(num_layers=1, num_single_layers=1, num_attention_heads=2, joint_attention_dim=64,
                               pooled_projection_dim=32)
    m.set_attn_processor(FluxFusedFlashAttnProcessor3())
    Flux(_cfg(attention_mechanism="diffusers"), transformer=m, device=torch.device("cpu"))
    m.set_attn_processor(FluxAttnProcessor2_0())
    with pytest.raises(NotImplementedError, match="key-padding"):
        m.set_attn_processor(FluxFusedFlashAttnProcessor3())


# ---- the SDPA override's mask forms (shape and strides only) ----------------------------------------------------------
B, H, SQ, SK = 3, 4, 10, 12
BF = torch.bfloat16


@pytest.mark.parametrize("make", [
    lambda: torch.ones(B, 1, 1, SK, dtype=BF),
    lambda: torch.ones(1, 1, 1, SK, dtype=BF),
    lambda: torch.ones(B, 1, 1, SK, dtype=BF).expand(B, H, SQ, SK),     # heads / queries of stride 0
    lambda: torch.ones(1, SK, dtype=BF).expand(B, SK)[:, None, None, :],
    lambda: torch.ones(SK, dtype=BF),
    lambda: torch.ones(1, 1, SK, dtype=BF),
    lambda: torch.ones(B, 2 * SK, dtype=BF)[:, :SK][:, None, None, :],  # batch rows 2 Sk apart
], ids=["B11Sk", "111Sk", "expanded", "batch_stride0", "1d", "3d", "strided_rows"])
def test_sdpa_accepts_per_key_masks(make):
    m = make()
    kb = key_bias_from_mask(m, B, H, SQ, SK, BF)
    assert kb.dim() == 2 and kb.shape[1] == SK and kb.shape[0] in (1, B) and kb.stride(1) == 1
    assert kb.data_ptr() == m.data_ptr()                                 # a view: nothing is copied or read


@pytest.mark.parametrize("make,dtype", [
    (lambda: torch.zeros(200, 200, dtype=BF), BF),                      # [Sq, Sk]: varies per query
    (lambda: torch.ones(B, 1, SQ, SK, dtype=BF), BF),
    (lambda: torch.ones(B, H, 1, SK, dtype=BF), BF),                     # per head
    (lambda: torch.ones(B, 1, 1, SK, dtype=torch.bool), BF),             # boolean mask
    (lambda: torch.ones(B, 1, 1, SK, dtype=torch.float32), BF),          # not the query dtype
    (lambda: torch.ones(2, 1, 1, SK, dtype=BF), BF),                     # batch neither B nor 1
    (lambda: torch.ones(B, 1, 1, SK + 1, dtype=BF), BF),
    (lambda: torch.ones(B, 1, 1, 2 * SK, dtype=BF)[..., ::2], BF),       # keys not contiguous
    (lambda: torch.ones(1, B, 1, 1, SK, dtype=BF), BF),
], ids=["SqSk", "per_query", "per_head", "bool", "fp32", "batch2", "wrong_Sk", "key_stride", "5d"])
def test_sdpa_refuses_other_masks(make, dtype):
    m = make()
    sq = 200 if m.shape[-2:] == (200, 200) else SQ
    sk = 200 if m.shape[-2:] == (200, 200) else SK
    with pytest.raises(NotImplementedError):
        key_bias_from_mask(m, B, H, sq, sk, dtype)


# ---- C ABI -------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_attention_args_ctypes_offsets_match_the_header(tmp_path):
    structs = {"stb_attn_fwd_args": _lib.AttnFwdArgs, "stb_attn_bwd_args": _lib.AttnBwdArgs}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT / "include" / "stb200.h"}"', "int main(void) {"]
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        for name, _ in cls._fields_:
            lines.append(f'  printf("{cname} {name} %zu\\n", offsetof({cname}, {name}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "offsets.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "offsets"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True, capture_output=True)
    got = {}
    for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines():
        cname, field, off = line.split()
        got[(cname, field)] = int(off)
    for cname, cls in structs.items():
        assert got[(cname, "sizeof")] == C.sizeof(cls), cname
        for name, _ in cls._fields_:
            assert got[(cname, name)] == getattr(cls, name).offset, (cname, name)
    assert ("stb_attn_fwd_args", "bias_b") in got and ("stb_attn_bwd_args", "bias") in got
