"""CPU: the ctypes mirrors of stb_attn_fwd_args / stb_attn_bwd_args (simpletuner_b200/_lib.py) against the C layout of
include/stb200.h, field by field (offsetof and sizeof from the host C compiler)."""
import shutil
import subprocess
from pathlib import Path

import ctypes as C
import pytest

from simpletuner_b200 import _lib

ROOT = Path(__file__).resolve().parent.parent


@pytest.mark.parametrize("cname,py", [("stb_attn_fwd_args", _lib.AttnFwdArgs), ("stb_attn_bwd_args", _lib.AttnBwdArgs)])
def test_attention_args_match_the_header(cname, py, tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    names = [f[0] for f in py._fields_]
    src = tmp_path / "layout.c"
    body = "".join(f'  printf("{n} %zu\\n", offsetof({cname}, {n}));\n' for n in names)
    src.write_text(f'#include <stddef.h>\n#include <stdio.h>\n#include "stb200.h"\nint main(void) {{\n{body}'
                   f'  printf("sizeof %zu\\n", sizeof({cname}));\n  return 0;\n}}\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    want = {n: str(getattr(py, n).offset) for n in names}
    want["sizeof"] = str(C.sizeof(py))
    assert got == want
