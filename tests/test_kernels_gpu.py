"""GPU (-m gpu): every libstb200 kernel against plain PyTorch fp32 math on the same tensors, through the C ABI."""
import pytest

from tests.kernel_checks import CHECKS

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(CHECKS))
def test_kernel(name):
    r = CHECKS[name]()
    assert r["ok"], r

