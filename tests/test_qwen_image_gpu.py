"""GPU (-m gpu): the Qwen-Image LoRA step (prepare_batch -> model_predict -> loss -> backward) against the fp32 oracle
(tests/qwen_image_oracle.py) with the tolerances of tests/flux_parity.py, and bit-exact properties of the step."""
import pytest
import torch

from tests import flux_parity as FP
from tests import qwen_image_oracle as QO

pytestmark = pytest.mark.gpu


def _mask(lengths, S):
    m = torch.zeros(len(lengths), S, dtype=torch.int64)
    for i, n in enumerate(lengths):
        m[i, :n] = 1
    return m


def _ok(res):
    FP.record("qwen_image", res)
    assert res["loss_rel_err"] <= FP.LOSS_RTOL, res
    assert res["pred_cos"] >= FP.PRED_COS, res
    assert res["grad_cos_min"] >= FP.GRAD_COS, res


NON_PREFIX = torch.tensor([[1] * 20 + [0, 1, 0] + [0] * 9, [1] * 32])


@pytest.mark.parametrize("B,mask,targets", [
    (1, None, "default"),
    (1, _mask([19], 32), "attn"),
    (3, _mask([32, 7, 20], 32), "attn+mlp"),
    (2, NON_PREFIX, "attn"),
])
def test_step_parity(B, mask, targets):
    _ok(QO.run_parity(B=B, mask=mask, targets=targets))


def test_step_parity_hd64_non_square_odd_grid():
    cfg = QO.QwenConfig(attention_head_dim=64, num_attention_heads=2, axes_dims_rope=(8, 28, 28))
    _ok(QO.run_parity(cfg, B=2, Hh=18, Ww=14, mask=_mask([5, 32], 32), targets="attn+mlp"))
    _ok(QO.run_parity(B=1, Hh=12, Ww=20, targets="default"))


def test_step_parity_lora_dropout():
    _ok(QO.run_parity(B=2, mask=_mask([12, 32], 32), targets="attn+mlp", dropout=0.1))


def _setup(B=3, mask=None, targets="attn+mlp", five_d=False, cfg=None):
    cfg = cfg or QO.QwenConfig()
    P = {k: v.bfloat16().float() for k, v in QO.init_params(cfg, 0).items()}
    L = {k: v.bfloat16().float() for k, v in QO.init_lora(cfg, 16, QO.TARGETS[targets], 1).items()}
    w = QO.build_cuda(cfg, P, L, 16, QO.TARGETS[targets])
    return w, QO.make_batch(B, 16, 16, 32, cfg, mask, 2, five_d)


def test_checkpointing_padding_values_and_5d_are_bit_identical():
    mask = _mask([32, 9, 20], 32)
    w, batch = _setup(mask=mask)
    _, out0, l0, g0 = QO.run_step(w, batch)
    _, out1, l1, g1 = QO.run_step(w, batch, checkpoint=True)
    assert torch.equal(l0, l1) and all(torch.equal(g0[k], g1[k]) for k in g0)
    # other finite values at padded prompt positions change nothing
    b2 = dict(batch)
    noise = torch.randn(batch["prompt_embeds"].shape, generator=torch.Generator().manual_seed(9)).bfloat16()
    b2["prompt_embeds"] = torch.where(mask[:, :, None] != 0, batch["prompt_embeds"], noise)
    _, out2, l2, g2 = QO.run_step(w, b2)
    assert torch.equal(l0, l2) and all(torch.equal(g0[k], g2[k]) for k in g0)
    assert torch.equal(out0["model_prediction"], out2["model_prediction"])
    # 5-D latents [B, 16, 1, h, w]
    b5 = dict(batch)
    b5["latent_batch"] = batch["latent_batch"].unsqueeze(2)
    _, out5, l5, g5 = QO.run_step(w, b5)
    assert out5["model_prediction"].shape == (3, 16, 1, 16, 16)
    assert torch.equal(l0, l5) and all(torch.equal(g0[k], g5[k]) for k in g0)
    assert torch.equal(out0["model_prediction"], out5["model_prediction"].squeeze(2))
    # an all-ones mask is decided on the host to hide no key: the unbiased kernels run, with the bits of no mask at all
    b_full = dict(batch, encoder_attention_mask=torch.ones_like(mask))
    prep = w.prepare_batch({k: v.clone() for k, v in b_full.items()}, {"global_step": 0})
    assert prep["_qwen_masked_keys"] is False
    b_none = {k: v for k, v in batch.items() if k != "encoder_attention_mask"}
    _, out6, l6, g6 = QO.run_step(w, b_full)
    _, out7, l7, g7 = QO.run_step(w, b_none)
    assert torch.equal(l6, l7) and all(torch.equal(g6[k], g7[k]) for k in g6)
    assert torch.equal(out6["model_prediction"], out7["model_prediction"])


def test_attention_kwargs_scale_multiplies_the_lora_scaling():
    """reference :1255-1263: attention_kwargs["scale"] scales every adapter for the call; scale 0.5 gives the bits of
    lora_B halved (both fold the same exact power-of-two factor into the rank-r up-projection)."""
    w, batch = _setup(B=2, targets="attn")
    m = w._denoiser()
    prep = w.prepare_batch({k: v.clone() for k, v in batch.items()}, {"global_step": 0})
    kw = dict(hidden_states=prep["_packed_noisy_latents"], encoder_hidden_states=prep["encoder_hidden_states"],
              timestep=prep["timesteps"].float() / 1000, img_shapes=[(1, 8, 8)] * 2, return_dict=False)
    with torch.no_grad():
        scaled = m(attention_kwargs={"scale": 0.5}, **kw)[0]
        plain = m(**kw)[0]
        for lin in m.lora_linears().values():
            lin.lora_B["default"].weight.mul_(0.5)
        halved = m(**kw)[0]
    assert torch.equal(scaled, halved) and not torch.equal(scaled, plain)


def test_huber_loss_parity():
    _ok(QO.run_parity(B=2, mask=_mask([20, 32], 32), targets="attn", loss_type="huber"))


def test_eager_train_step_with_flat_grad_sync():
    from simpletuner_b200.training.dist import FlatGradSync
    from simpletuner_b200.training.step import TrainStep
    w, batch = _setup(B=2, mask=_mask([32, 11], 32), targets="attn+mlp")
    m = w._denoiser()
    params = m.trainable_parameters()
    base = {n: p.detach().clone() for n, p in m.named_parameters() if not p.requires_grad}
    before = {n: p.detach().clone() for n, p in m.named_parameters() if p.requires_grad}
    step = TrainStep(w, torch.optim.AdamW(params, lr=1e-3), max_grad_norm=1.0, grad_sync=FlatGradSync(params))
    losses = [step({k: v.clone() for k, v in batch.items()}) for _ in range(2)]
    torch.cuda.synchronize()
    assert all(bool(torch.isfinite(l)) for l in losses)
    # every adapter moves except those of the last block's text queries and text outputs, which feed nothing
    last = f"transformer_blocks.{len(m.transformer_blocks) - 1}."
    dead = tuple(last + t for t in ("attn.add_q_proj", "attn.to_add_out", "txt_mlp"))
    for n, p in m.named_parameters():
        if p.requires_grad:
            assert torch.equal(before[n], p) == n.startswith(dead), n
    assert all(torch.equal(base[n], p) for n, p in m.named_parameters() if not p.requires_grad)


def test_shared_storage_on_the_device_and_plans_allocate_no_weights():
    from simpletuner_b200 import ops
    w, _ = _setup(B=1)
    m = w._denoiser()
    D = m.inner_dim
    for blk in m.transformer_blocks:
        for name, (q, k, v) in blk.attn.streams().items():
            assert q.weight.is_cuda and k.weight.data_ptr() - q.weight.data_ptr() == D * D * 2
            assert v.weight.data_ptr() - k.weight.data_ptr() == D * D * 2
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    for blk in m.transformer_blocks:
        pl = blk.plans()
        assert pl["img_attn"].w_qkv.data_ptr() == blk.attn.to_q.weight.data_ptr()
        assert isinstance(pl["img_attn"].w_qkv_t, ops.WT) and isinstance(pl["txt_mlp"].w2_t, ops.WT)
    assert torch.cuda.memory_allocated() - before < 1 << 20
    m.to("cpu")
    m.to("cuda")
    a = m.transformer_blocks[0].attn
    assert a.to_k.weight.data_ptr() - a.to_q.weight.data_ptr() == D * D * 2


def test_fullwidth_two_blocks():
    """D = 3072 (24 heads x 128), 4096 image tokens (128 x 128 latents), 512 text tokens, ragged padding."""
    cfg = QO.QwenConfig(num_layers=2, num_attention_heads=24, joint_attention_dim=3584)
    res = QO.run_parity(cfg, B=2, Hh=128, Ww=128, S_txt=512, mask=_mask([512, 300], 512), targets="default", rank=16)
    _ok(res)
