"""GPU (-m gpu): one Chroma 1 LoRA step at full size (19 + 38 blocks, D = 3072, approximator width 5120) at 1024^2 with
a 512-token T5 prompt of which 100 tokens are kept, random weights.  The CPU oracle cannot run this size, so the checks are
size-independent properties: the modulation rows have the shape the blocks read, the loss and every LoRA gradient are
finite, and the step is deterministic.  Peak memory is printed."""
import pytest
import torch

from tests import chroma_oracle as CO

pytestmark = pytest.mark.gpu


def test_full_size_step():
    from simpletuner_b200.chroma.model import Chroma, default_config
    from simpletuner_b200.chroma.transformer import ChromaTransformer2DModel
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    with torch.device("cuda"):
        m = ChromaTransformer2DModel()
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "norm" in n:
                p.fill_(1.0)
            elif n.startswith("distilled_guidance_layer") and n.endswith("weight"):
                p.normal_(0, p.shape[1] ** -0.5, generator=g)
            else:
                p.normal_(0, 0.02 if n.endswith("weight") else 0.01, generator=g)
    w = Chroma(default_config(lora_rank=16, flux_lora_target="all"), transformer=m, device=torch.device("cuda"))
    w.add_lora_adapter()
    with torch.no_grad():
        for lin in m.lora_linears().values():
            lin.lora_B["default"].weight.normal_(0, 0.02, generator=g)
    assert m.mod_rows == 344
    cfg = CO.ChromaConfig(joint_attention_dim=4096)
    batch = CO.make_batch(1, 128, 128, CO.ragged_mask(1, 512, (100,)), cfg)
    results = [CO.run_step(w, batch, checkpoint=True) for _ in range(2)]
    (_, out, loss, grads), (_, _, loss2, grads2) = results
    assert out["model_prediction"].shape == (1, 16, 128, 128)
    assert bool(torch.isfinite(loss)) and all(bool(torch.isfinite(v).all()) for v in grads.values())
    assert any(bool(v.any()) for k, v in grads.items() if "lora_A" in k)
    assert torch.equal(loss, loss2) and all(torch.equal(grads[k], grads2[k]) for k in grads)
    print(f"chroma full size: loss {float(loss):.5f}, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
