"""CPU: the C-ABI library loads, exports every symbol include/stb200.h declares, and the product path
refuses to run without a CUDA device (no silent CPU fallback)."""
import re
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


def _declared():
    txt = (ROOT / "include" / "stb200.h").read_text()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(stb_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    from simpletuner_b200 import _lib

    if _lib.needs_build():
        _lib.build()
    handle = _lib.lib()
    names = _declared()
    assert len(names) >= 14
    for n in names:
        assert hasattr(handle, n), f"libstb200.so does not export {n}"
    # and the ctypes table covers the header exactly
    assert sorted(_lib.SYMBOLS) == names
    assert handle.stb_version() == 100


# entry points that launch nothing: version, error text, launch counters, workspace size, optimizer chunk size
_BOOKKEEPING = {"stb_version", "stb_last_error", "stb_launch_count", "stb_reset_launch_count", "stb_skinny_tn_workspace",
                "stb_adamw_bf16_chunk"}
# GPU tests outside the kernel_checks registry that compare a wrapper with a reference
_GPU_TEST_FILES = ("test_lora_dropout_gpu.py", "test_text_encoders.py")


def _wrappers():
    """{stb_* symbol: names of the top-level functions / classes of the Python layer whose body calls it}"""
    import ast

    found = {}
    for rel in ("simpletuner_b200/ops.py", "simpletuner_b200/training/optim.py"):
        for node in ast.parse((ROOT / rel).read_text()).body:
            if isinstance(node, (ast.FunctionDef, ast.ClassDef)):
                for sub in ast.walk(node):
                    if isinstance(sub, ast.Attribute) and sub.attr.startswith("stb_"):
                        found.setdefault(sub.attr, set()).add(node.name)
    return found


def test_every_kernel_entry_point_has_a_gpu_check():
    """Each kernel entry point of include/stb200.h is reached by a wrapper that tests/kernel_checks.py or a named GPU test
    calls, so a new kernel cannot land without an element-wise check."""
    wrappers = _wrappers()
    tests = ROOT / "tests"
    texts = [(tests / "kernel_checks.py").read_text()] + [(tests / f).read_text() for f in _GPU_TEST_FILES]
    unchecked = {}
    for sym in sorted(set(_declared()) - _BOOKKEEPING):
        names = wrappers.get(sym)
        assert names, f"{sym} is declared in include/stb200.h but no Python wrapper calls it"
        if not any(re.search(rf"\b{n}\s*\(", t) for n in names for t in texts):
            unchecked[sym] = sorted(names)
    assert not unchecked, f"entry points whose wrappers no GPU check calls: {unchecked}"


def test_product_path_fails_loudly_without_cuda():
    from simpletuner_b200 import _lib, ops

    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    a = torch.zeros(128, 64, dtype=torch.bfloat16)
    w = torch.zeros(64, 64, dtype=torch.bfloat16)
    with pytest.raises(_lib.StbError):
        ops.gemm([a], [w])
    from simpletuner_b200.flux.transformer import FluxTransformer2DModel

    m = FluxTransformer2DModel(num_layers=1, num_single_layers=1, num_attention_heads=1, joint_attention_dim=64,
                               pooled_projection_dim=32, in_channels=16)
    with pytest.raises(_lib.StbError):
        m(hidden_states=torch.zeros(1, 4, 16), encoder_hidden_states=torch.zeros(1, 4, 64),
          pooled_projections=torch.zeros(1, 32), timestep=torch.zeros(1), img_ids=torch.zeros(4, 3),
          txt_ids=torch.zeros(4, 3), return_dict=False)


def test_no_oracle_import_in_product():
    bad = []
    for p in (ROOT / "simpletuner_b200").rglob("*.py"):
        s = p.read_text()
        if re.search(r"^\s*(from|import)\s+oracle\b", s, flags=re.M):
            bad.append(str(p))
    assert not bad, f"product code must not import the oracle: {bad}"
