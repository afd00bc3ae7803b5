"""GPU (-m gpu): the full Qwen-Image geometry (60 blocks, D = 3072, joint dim 3584; 20.4 B parameters) with random
weights, a 1024^2 LoRA step with gradient checkpointing on every block.  The CPU oracle cannot run this size, so the checks
are size-independent properties (as tests/test_flux_fullsize_gpu.py): finite loss and gradients, no second copy of any
frozen weight, B = 0 LoRA identity, batch-permutation equivariance and determinism.  Peak memory is printed."""
import time

import pytest
import torch

from tests import qwen_image_oracle as QO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def full():
    from simpletuner_b200.qwen_image.model import QwenImage, default_config
    from simpletuner_b200.qwen_image.transformer import QwenImageTransformer2DModel
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.device("cuda"):
        m = QwenImageTransformer2DModel()
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("norm_q.weight") or n.endswith("norm_k.weight") or "norm_added" in n or n == "txt_norm.weight":
                p.fill_(1.0)
            else:
                p.normal_(0, 0.02 if n.endswith("weight") else 0.01, generator=g)
    param_bytes = sum(p.numel() * p.element_size() for p in m.parameters())
    w = QwenImage(default_config(lora_rank=16), transformer=m, device=torch.device("cuda"))
    w.add_lora_adapter()
    with torch.no_grad():
        for lin in m.lora_linears().values():
            lin.lora_B["default"].weight.normal_(0, 0.02, generator=g)
    m.enable_gradient_checkpointing()
    for blk in m.transformer_blocks:
        blk.plans()
    torch.cuda.synchronize()
    resident = torch.cuda.memory_allocated() - base
    return w, m, param_bytes, resident


def _batch(B, seed):
    cfg = QO.QwenConfig(num_layers=60, num_attention_heads=24, joint_attention_dim=3584)
    mask = torch.zeros(B, 512, dtype=torch.int64)
    for i in range(B):
        mask[i, :256 + 64 * i] = 1
    return QO.make_batch(B, 128, 128, 512, cfg, mask if B > 1 else None, seed)


def test_fullsize_step_fits_with_no_weight_copy(full):
    w, m, param_bytes, resident = full
    lora_bytes = sum(p.numel() * p.element_size() for p in m.trainable_parameters())
    # everything allocated besides the parameters and the adapters: the plans add no weight-sized tensor
    assert resident - param_bytes - lora_bytes < 1 << 30, (resident, param_bytes)
    batch = _batch(1, 3)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    _, out, loss, grads = QO.run_step(w, batch, checkpoint=True)
    ms = (time.perf_counter() - t0) * 1e3
    peak = torch.cuda.max_memory_allocated()
    import subprocess
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(f"\nqwen_image fullsize B=1 1024^2: loss {float(loss):.5f}, first step {ms:.0f} ms, peak allocated "
          f"{peak / 2**30:.2f} GiB, parameters {param_bytes / 2**30:.2f} GiB, card "
          f"{smi[torch.cuda.current_device()] if smi else torch.cuda.get_device_name()}")
    assert torch.isfinite(loss) and all(torch.isfinite(g).all() for g in grads.values())
    assert peak < torch.cuda.get_device_properties(0).total_memory


def test_fullsize_properties(full):
    w, m, _, _ = full
    batch = _batch(2, 5)
    with torch.no_grad():
        torch.manual_seed(11)
        torch.cuda.manual_seed(11)
        prep = w.prepare_batch({k: v.clone() for k, v in batch.items()}, {"global_step": 0})
        o1 = w.model_predict(prep)["model_prediction"]
        o2 = w.model_predict(prep)["model_prediction"]
        assert torch.equal(o1, o2)
        perm = torch.tensor([1, 0], device="cuda")
        pp = dict(prep)
        for k in ("latents", "noise", "noisy_latents", "_packed_noisy_latents", "encoder_hidden_states", "timesteps",
                  "encoder_attention_mask"):
            pp[k] = prep[k][perm].contiguous()
        assert torch.equal(w.model_predict(pp)["model_prediction"], o1[perm])
        saved = {n: l.lora_B["default"].weight.detach().clone() for n, l in m.lora_linears().items()}
        for l in m.lora_linears().values():
            l.lora_B["default"].weight.zero_()
        z = w.model_predict(prep)["model_prediction"]
        m.disable_lora()
        base = w.model_predict(prep)["model_prediction"]
        m.enable_lora()
        assert torch.equal(z, base)
        for n, l in m.lora_linears().items():
            l.lora_B["default"].weight.copy_(saved[n])
