"""GPU (-m gpu): the weight-gradient and token-reduction kernels at the shapes the PixArt-Sigma full fine-tune schedule
hands them (PixArt-Sigma 600M: D 1152, 16 heads padded 72 -> 128, 1024^2 latents = 4096 tokens, 300-token captions, batch
4), against the fp64 reference of tests/kernel_checks.py: error and exact-input modes, as the existing GEMM-family cases."""
import pytest

from tests import flux_parity as FP
from tests.kernel_checks import check_colsum2, check_gemm, check_wgrad_full

pytestmark = pytest.mark.gpu

CASES = {
    # PatchEmbed: a 16-feature x operand (4 channels x 2 x 2 patch), dW [1152, 16]
    "wgrad_full_patch_k16": dict(B=4, S=4096, N=1152, K=16),
    # caption k | v on the padded layout and the caption projection: 300 tokens per sample, not a multiple of 64
    "wgrad_full_caption_kv_s300": dict(B=4, S=300, N=4096, K=1152),
    "wgrad_full_caption_proj_s300": dict(B=4, S=300, N=1152, K=4096),
    # self-attention q | k | v on the padded layout, and the kept rows of proj_out
    "wgrad_full_padded_qkv": dict(B=1, S=4096, N=6144, K=1152),
    "wgrad_full_proj_out_kept_rows": dict(B=4, S=4096, N=16, K=1152),
}


@pytest.mark.parametrize("exact", [False, True], ids=["fp64_ref", "exact"])
@pytest.mark.parametrize("name", list(CASES))
def test_wgrad_full_pixart_shapes(name, exact):
    r = FP.record("kernel:" + name, check_wgrad_full(**CASES[name], exact=exact))
    print(r)
    assert r["ok"], r


@pytest.mark.parametrize("exact", [False, True], ids=["fp64_ref", "exact"])
@pytest.mark.parametrize("D", [1152, 4096])
def test_colsum2_caption_tokens(D, exact):
    r = FP.record(f"kernel:colsum2_s300_d{D}", check_colsum2(B=4, S=300, D=D, exact=exact))
    print(r)
    assert r["ok"], r


@pytest.mark.parametrize("exact", [False, True], ids=["fp64_ref", "exact"])
def test_gemm_patch_embed_k16(exact):
    """The PatchEmbed forward GEMM over the 16 patch features with the positional table added in the epilogue."""
    from simpletuner_b200 import ops
    r = FP.record("kernel:gemm_patch_k16", check_gemm(4096, 1152, 16, B=2, bias=True, epi=ops.EPI_ADD_RES, exact=exact))
    print(r)
    assert r["ok"], r
