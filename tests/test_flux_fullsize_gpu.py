"""GPU (-m gpu): BASELINE full-size checks (Flux.1-dev geometry: 19+38 blocks, D=3072, 4096+512 tokens, B=4) through
size-independent properties — the CPU oracle cannot finish this size in test time (≈20 min/sample on 128 cores).

  * LoRA with B = 0 leaves the prediction bit-identical to the adapter-free model, and gives dA == 0 exactly
    (dA = (dY B)^T x) while dB != 0;
  * batch-permutation equivariance of the whole train-step forward, bit-exact (tiles never straddle samples);
  * run-to-run determinism of prediction and loss (no atomics on the activation path);
  * pack -> unpack round trip of the kernel-side patchify index math at [4,16,128,128].
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def full():
    import bench

    torch.manual_seed(0)
    dev = torch.device("cuda", 0)
    w = bench.build_model(dev, None, rank=16, seed=0)
    # an 80 GB card does not hold the B = 4 backward at this size with every activation saved: keep them only at block
    # boundaries (the reference's default gradient_checkpointing=true); the forward values are unchanged
    w._denoiser().enable_gradient_checkpointing()
    batch = bench.synth_batch(4, dev, seed=7)
    return w, batch


def _predict(w, batch, seed):
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)
    prep = w.prepare_batch({k: v.clone() for k, v in batch.items()}, {"global_step": 0})
    prep["_raw_timesteps"] = prep["timesteps"].clone()  # model_predict overwrites `timesteps` with t / 1000
    out = w.model_predict(prep)
    return prep, out


def test_fullsize_properties(full):
    w, batch = full
    m = w._denoiser()
    # ---- determinism
    with torch.no_grad():
        prep1, out1 = _predict(w, batch, 11)
        prep2, out2 = _predict(w, batch, 11)
    assert torch.equal(out1["model_prediction"], out2["model_prediction"])
    assert torch.equal(prep1["noisy_latents"], prep2["noisy_latents"])
    l1 = w.loss(prep1, out1)
    l2 = w.loss(prep2, out2)
    # the loss kernel reduces per-block partial sums with fp32 atomics: equal up to summation order
    assert torch.isfinite(l1) and abs(float(l1) - float(l2)) <= 1e-6 * abs(float(l1))
    # ---- pack / unpack round trip at full latent size
    from simpletuner_b200.flux.functional import pack_latents, unpack_latents
    assert torch.equal(prep1["_packed_noisy_latents"], pack_latents(prep1["noisy_latents"], 4, 16, 128, 128))
    assert torch.equal(unpack_latents(prep1["_packed_noisy_latents"], 1024, 1024, 16), prep1["noisy_latents"])
    # ---- batch-permutation equivariance (same noise / sigmas, permuted with the samples)
    perm = torch.tensor([2, 0, 3, 1], device="cuda")
    with torch.no_grad():
        pp = dict(prep1)
        for k in ("latents", "noise", "input_noise", "noisy_latents", "_packed_noisy_latents", "encoder_hidden_states", "sigmas"):
            pp[k] = prep1[k][perm].contiguous()
        pp["timesteps"] = prep1["_raw_timesteps"][perm]
        pp["added_cond_kwargs"] = {"text_embeds": prep1["added_cond_kwargs"]["text_embeds"][perm].contiguous()}
        outp = w.model_predict(pp)
    assert torch.equal(outp["model_prediction"], out1["model_prediction"][perm])
    # ---- LoRA B = 0  ==>  identical to the adapter-free model, dA == 0, dB != 0
    saved = {n: lin.lora_B["default"].weight.detach().clone() for n, lin in m.lora_linears().items()}
    with torch.no_grad():
        for lin in m.lora_linears().values():
            lin.lora_B["default"].weight.zero_()
    prep3, out3 = _predict(w, batch, 11)
    loss3 = w.loss(prep3, out3)
    loss3.backward()
    with torch.no_grad():
        m.disable_lora()
        prep4, out4 = _predict(w, batch, 11)
        m.enable_lora()
    assert torch.equal(out3["model_prediction"], out4["model_prediction"])
    n_b_nonzero = 0
    for lin in m.lora_linears().values():
        ga, gb = lin.lora_A["default"].weight.grad, lin.lora_B["default"].weight.grad
        assert ga is not None and gb is not None
        assert float(ga.abs().max()) == 0.0
        assert torch.isfinite(gb).all()
        n_b_nonzero += int(float(gb.abs().max()) > 0)
        lin.lora_A["default"].weight.grad = None
        lin.lora_B["default"].weight.grad = None
    assert n_b_nonzero == len(m.lora_linears())
    with torch.no_grad():
        for n, lin in m.lora_linears().items():
            lin.lora_B["default"].weight.copy_(saved[n])
