"""GPU (-m gpu): Flux Kontext training on the H100 path.  The packing kernel writes into the joint token buffer bit-exactly
(tests/golden/flux_kontext_golden.pt holds the reference's own `build_kontext_inputs` output); the Kontext step matches the
fp32 oracle (tests/flux_kontext_oracle.py) with tests/flux_parity.py's criteria; a Kontext run without conditioning is the
plain step bit for bit; seeded Kontext runs repeat bit for bit."""
from pathlib import Path

import pytest
import torch

from tests import flux_kontext_oracle as KO
from tests import flux_parity as FP

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "flux_kontext_golden.pt"
GRAD_REL_L2 = 0.05      # per LoRA gradient tensor: |g - g_ref| / |g_ref|, next to the cosine bound


def _assert(tag, res):
    FP.record(tag, res)
    print(f"[kontext] {tag}", res)
    assert res["timesteps_match"], res
    assert res["loss_rel_err"] <= FP.LOSS_RTOL, res
    assert res["pred_cos"] >= FP.PRED_COS, res
    assert res["grad_cos_min"] >= FP.GRAD_COS, res
    assert res["grad_rel_l2_max"] <= GRAD_REL_L2, res


def test_pack_into_the_joint_buffer_is_bit_exact():
    from oracle import flux_oracle as O
    from simpletuner_b200 import ops

    g = torch.Generator().manual_seed(5)
    for case in torch.load(GOLDEN, weights_only=False)["pack"]:
        B, C = case["B"], case["C"]
        scene = torch.randn(B, C, 6, 10, generator=g).bfloat16().cuda()
        noise = torch.randn(B, C, 6, 10, generator=g).bfloat16().cuda()
        sig = torch.rand(B, generator=g).cuda()
        S_scene, S_c = 15, case["packed"].shape[1]
        joint = torch.full((B, S_scene + S_c + 3, 4 * C), float("nan"), device="cuda", dtype=torch.bfloat16)
        noisy, _ = ops.flow_prep_pack(scene, noise, sig, out=joint[:, :S_scene])
        off = S_scene
        for lat in case["latents"]:
            n = (lat.shape[2] // 2) * (lat.shape[3] // 2)
            _, v = ops.flow_prep_pack(lat.cuda(), None, None, out=joint[:, off:off + n])
            assert v.data_ptr() == joint[:, off:].data_ptr()
            off += n
        assert torch.equal(joint[:, S_scene:off].cpu(), case["packed"]), case["sizes"]
        assert torch.isnan(joint[:, off:].float()).all()                      # nothing written past the range
        # the noisy scene tokens: the old call's bits, and the eager bf16 chain of the reference
        noisy0, packed0 = ops.flow_prep_pack(scene, noise, sig)
        assert torch.equal(noisy, noisy0) and torch.equal(joint[:, :S_scene], packed0)
        ref = O.flow_noisy_latents(scene.cpu(), noise.cpu(), sig.cpu())
        assert torch.equal(noisy.cpu(), ref) and torch.equal(packed0.cpu(), O.pack_latents(ref, B, C, 6, 10))


@pytest.mark.parametrize("hd,sizes", [
    (128, [(16, 16)]),                          # a reference the size of the edit
    (64, [(12, 20)]),                           # non-square, another size
    (128, [(16, 16), (8, 12)]),                 # combined, 2 references
    (64, [(10, 14), (16, 8), (6, 6)]),          # combined, 3 references
], ids=["same_size", "nonsquare", "combined2", "combined3"])
def test_kontext_step_parity(hd, sizes):
    cfg = FP.small_config(hd=hd)
    _assert(f"kontext[hd={hd},{sizes}]", KO.run_kontext_parity(sizes, cfg=cfg))


def test_kontext_step_parity_with_lora_dropout_replayed():
    res = KO.run_kontext_parity([(12, 20)], cfg=FP.small_config(layers=1, single=1), dropout=0.1)
    _assert("kontext_dropout", res)


def test_kontext_step_parity_with_gradient_checkpointing():
    _assert("kontext_checkpoint", KO.run_kontext_parity([(16, 16), (8, 12)], checkpoint=True))


def test_kontext_step_parity_with_masked_training():
    from tests import flux_mask_oracle as MO
    _assert("kontext_masked", KO.run_kontext_parity([(12, 20)], mask=MO.length_mask([9, 32], 32)))


def test_kontext_step_parity_with_lokr():
    from tests.test_flux_lokr_gpu import LYCORIS_CFG
    _assert("kontext_lokr", KO.run_kontext_parity([(16, 16)], lokr=dict(LYCORIS_CFG)))


def test_kontext_full_width_one_double_one_single_block():
    """Flux.1-dev width (D 3072, 24 x 128, T5 4096, pooled 768): a 1024^2 edit with a 1024^2 reference, S = 512 + 8192."""
    from oracle import flux_oracle as O
    cfg = O.FluxConfig(in_channels=64, num_layers=1, num_single_layers=1, attention_head_dim=128, num_attention_heads=24,
                       joint_attention_dim=4096, pooled_projection_dim=768, guidance_embeds=True, axes_dims_rope=(16, 56, 56))
    _assert("kontext_D3072_S512+4096+4096", KO.run_kontext_parity([(128, 128)], cfg=cfg, B=1, Hh=128, Ww=128, S_txt=512,
                                                                  seed=11))


def _step(flavour, conds, seed=0):
    """One Kontext-configured (or plain) step on a fixed model: (prediction, loss, LoRA gradients)."""
    from oracle import flux_oracle as O
    cfg = FP.small_config(layers=1, single=1)
    P = {k: v.bfloat16().float() for k, v in O.init_flux_params(cfg, seed=seed).items()}
    L = {k: v.bfloat16().float() for k, v in O.init_lora_params(cfg, 16, seed=seed + 1, b_std=0.02).items()}
    w = FP.build_cuda_model(cfg, P, L, 16)
    w.config.model_flavour = flavour
    batch = FP.make_batch(2, 16, 16, 32, cfg, seed=seed + 2)
    if conds is not None:
        batch["conditioning_latents"] = conds
    torch.manual_seed(1234)
    torch.cuda.manual_seed(1234)
    prepared = w.prepare_batch(batch, {"global_step": 0, "args": {"conditioning_multidataset_sampling": "combined"}})
    out = w.model_predict(prepared)
    loss = w.loss(prepared, out)
    loss.backward()
    grads = [lin.lora_A["default"].weight.grad.clone() for lin in w._denoiser().lora_linears().values()] + \
            [lin.lora_B["default"].weight.grad.clone() for lin in w._denoiser().lora_linears().values()]
    return out["model_prediction"].detach().clone(), loss.detach().clone(), grads


def test_kontext_batch_without_conditioning_is_the_plain_step():
    a = _step("kontext", None)
    b = _step("dev", None)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(x, y) for x, y in zip(a[2], b[2]))


def test_seeded_kontext_runs_are_bit_identical():
    conds = KO.make_conds(2, [(16, 16), (8, 12)], 7)
    a = _step("kontext", [c.clone() for c in conds])
    b = _step("kontext", [c.clone() for c in conds])
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(x, y) for x, y in zip(a[2], b[2]))
    plain = _step("dev", None)
    assert not torch.equal(a[0], plain[0])         # the references change the prediction
