"""ctypes binding of libstb200.so (C ABI declared in include/stb200.h).

The shared library is built in-tree by :func:`build` (nvcc, sm_90a only) and loaded lazily by
:func:`lib`.  There is no fallback: if the library is missing or the device is not sm_90 (H100) the
product path raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading
from pathlib import Path

_HERE = Path(__file__).resolve().parent
CSRC = _HERE / "csrc"
LIB_DIR = _HERE / "_C"
LIB_PATH = Path(os.environ["STB200_LIB"]) if os.environ.get("STB200_LIB") else LIB_DIR / "libstb200.so"  # override: experiments only
INCLUDE = _HERE.parent / "include" / "stb200.h"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--shared", "-Xcompiler", "-fPIC",
]


def _sources():
    return sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cuh")) + [INCLUDE]


def needs_build() -> bool:
    if not LIB_PATH.exists():
        return True
    t = LIB_PATH.stat().st_mtime
    return any(s.stat().st_mtime > t for s in _sources())


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile csrc/api.cu (which includes every kernel header) into _C/libstb200.so."""
    if not force and not needs_build():
        return LIB_PATH
    LIB_DIR.mkdir(exist_ok=True)
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc, *NVCC_FLAGS, "-o", str(LIB_PATH), str(CSRC / "api.cu")]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{proc.stdout}\n{proc.stderr}")
    if verbose:
        print(proc.stderr)
    return LIB_PATH


class GemmSeg(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("a_batch_stride", C.c_longlong), ("a_row_stride", C.c_longlong),
        ("w", C.c_void_p), ("w_row_stride", C.c_longlong), ("K", C.c_int), ("w_kn", C.c_int),
    ]


class GemmArgs(C.Structure):
    _fields_ = [
        ("num_batches", C.c_int), ("rows_per_batch", C.c_int), ("N", C.c_int), ("nseg", C.c_int),
        ("seg", GemmSeg * 3),
        ("d", C.c_void_p), ("d_batch_stride", C.c_longlong), ("d_row_stride", C.c_longlong),
        ("bias", C.c_void_p),
        ("epi", C.c_int), ("nan_to_num", C.c_int),
        ("gate", C.c_void_p), ("gate_batch_stride", C.c_longlong),
        ("res", C.c_void_p), ("res_batch_stride", C.c_longlong), ("res_row_stride", C.c_longlong),
        ("aux", C.c_void_p), ("aux_batch_stride", C.c_longlong), ("aux_row_stride", C.c_longlong),
        ("tile_mt", C.c_int), ("tile_bn", C.c_int),
    ]


class AttnFwdArgs(C.Structure):
    _fields_ = [
        ("B", C.c_int), ("H", C.c_int), ("Sq", C.c_int), ("Sk", C.c_int), ("HD", C.c_int),
        ("scale", C.c_float),
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p),
        ("q_b", C.c_longlong), ("q_s", C.c_longlong), ("q_h", C.c_longlong),
        ("k_b", C.c_longlong), ("k_s", C.c_longlong), ("k_h", C.c_longlong),
        ("v_b", C.c_longlong), ("v_s", C.c_longlong), ("v_h", C.c_longlong),
        ("o", C.c_void_p),
        ("o_b", C.c_longlong), ("o_s", C.c_longlong), ("o_h", C.c_longlong),
        ("lse", C.c_void_p),
        ("bias", C.c_void_p), ("bias_h", C.c_longlong), ("bias_q", C.c_longlong),
        ("bias_b", C.c_longlong),
        ("kv_live", C.c_void_p), ("kv_live_b", C.c_longlong),
    ]


class AttnBwdArgs(C.Structure):
    _fields_ = [
        ("B", C.c_int), ("H", C.c_int), ("Sq", C.c_int), ("Sk", C.c_int), ("HD", C.c_int),
        ("scale", C.c_float),
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("o", C.c_void_p), ("d_o", C.c_void_p),
        ("q_b", C.c_longlong), ("q_s", C.c_longlong), ("q_h", C.c_longlong),
        ("k_b", C.c_longlong), ("k_s", C.c_longlong), ("k_h", C.c_longlong),
        ("v_b", C.c_longlong), ("v_s", C.c_longlong), ("v_h", C.c_longlong),
        ("o_b", C.c_longlong), ("o_s", C.c_longlong), ("o_h", C.c_longlong),
        ("do_b", C.c_longlong), ("do_s", C.c_longlong), ("do_h", C.c_longlong),
        ("lse", C.c_void_p), ("delta", C.c_void_p),
        ("dq", C.c_void_p), ("dk", C.c_void_p), ("dv", C.c_void_p),
        ("dq_b", C.c_longlong), ("dq_s", C.c_longlong), ("dq_h", C.c_longlong),
        ("dk_b", C.c_longlong), ("dk_s", C.c_longlong), ("dk_h", C.c_longlong),
        ("dv_b", C.c_longlong), ("dv_s", C.c_longlong), ("dv_h", C.c_longlong),
        ("bias", C.c_void_p), ("bias_b", C.c_longlong),
        ("kv_live", C.c_void_p), ("kv_live_b", C.c_longlong),
    ]


# every symbol include/stb200.h declares: name -> (restype, argtypes)
_LL, _I, _F, _P = C.c_longlong, C.c_int, C.c_float, C.c_void_p
SYMBOLS = {
    "stb_last_error": (C.c_char_p, []),
    "stb_version": (_I, []),
    "stb_launch_count": (_LL, []),
    "stb_reset_launch_count": (None, []),
    "stb_gemm_bf16": (_I, [C.POINTER(GemmArgs), _P]),
    "stb_attn_fwd": (_I, [C.POINTER(AttnFwdArgs), _P]),
    "stb_attn_bwd": (_I, [C.POINTER(AttnBwdArgs), _P]),
    "stb_ln_modulate_fwd": (_I, [_P, _LL, _LL, _P, _P, _LL, _P, _LL, _LL, _I, _I, _I, _F, _P]),
    "stb_ln_modulate_bwd": (_I, [_P, _LL, _LL, _P, _LL, _LL, _P, _LL, _P, _LL, _LL, _P, _LL, _LL, _I, _I, _I, _F, _P]),
    "stb_qk_rmsnorm_rope_fwd": (_I, [_P, _LL, _LL, _I, _P, _P, _P, _P, _I, _P, _P, _P, _P, _LL, _LL, _I, _I, _I, _I, _F, _P]),
    "stb_qk_rmsnorm_rope_bwd": (_I, [_P, _P, _LL, _LL, _P, _LL, _LL, _I, _P, _P, _P, _P, _I, _P, _P, _P, _LL, _LL, _I, _I, _I, _I, _F, _P, _P]),
    "stb_flow_prep_pack": (_I, [_P, _P, _P, _P, _P, _LL, _I, _I, _I, _I, _P]),
    "stb_flow_mse_loss": (_I, [_P, _P, _P, _P, _P, _F, _I, _I, _I, _I, _I, _I, _P, _P]),
    "stb_ddpm_prep_pack": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "stb_target_mse_loss": (_I, [_P, _P, _P, _P, _P, _F, _I, _I, _I, _I, _I, _I, _P, _P]),
    "stb_adamw_bf16_multi": (_I, [_P, _P, _P, _P, _P, _I, _I, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, _P, _P, _LL, C.c_ulonglong, C.c_double, _P, C.c_double, _P]),
    "stb_adamw_bf16_chunk": (_I, []),
    "stb_gate_mul": (_I, [_P, _LL, _LL, _P, _LL, _P, _LL, _LL, _I, _I, _I, _P]),
    "stb_lokr_rebuild": (_I, [_P, _LL, _P, _P, C.c_float, _P, _LL, _P, _LL, _I, _I, _I, _I, _P]),
    "stb_lokr_factor_grads": (_I, [_P, _LL, _P, _P, C.c_float, _P, _P, _I, _I, _I, _I, _P]),
    "stb_rmsnorm_fwd": (_I, [_P, _LL, _LL, _P, _P, _LL, _LL, _I, _I, _I, C.c_float, _P]),
    "stb_gelu_tanh": (_I, [_P, _LL, _LL, _P, _LL, _LL, _P, _LL, _LL, _I, _I, _I, _I, _P]),
    "stb_dropout_expand": (_I, [_P, _LL, _LL, _P, _I, _I, _I, _I, _F, C.c_uint, C.c_uint, _P]),
    "stb_dropout_accum": (_I, [_P, _P, _LL, _LL, _I, _I, _I, _I, _F, C.c_uint, C.c_uint, _P]),
    "stb_wgrad_full": (_I, [_P, _LL, _LL, _P, _LL, _LL, _P, _LL, _I, _I, _I, _I, _F, _I, _P]),
    "stb_colsum2": (_I, [_P, _LL, _LL, _P, _LL, _LL, _P, _P, _I, _I, _I, _P]),
    "stb_skinny_tn": (_I, [_P, _LL, _LL, _P, _LL, _LL, _P, _I, _I, _I, _I, _F, _P, _LL, _P]),
    "stb_skinny_tn_workspace": (_LL, [_I, _I, _I, _I]),
    "stb_conv3x3_nhwc": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "stb_conv_in_3ch": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "stb_groupnorm_nhwc": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _I, _P]),
    "stb_softmax_rows": (_I, [_P, _LL, _I, _I, _F, _P]),
    "stb_gaussian_sample_scale": (_I, [_P, _P, _P, _I, _I, _I, _F, _F, _I, _P]),
    "stb_gaussian_sample_channel_norm": (_I, [_P, _P, _P, _I, _I, _I, _P, _P, _P]),
    "stb_channel_rmsnorm_nhwc": (_I, [_P, _P, _P, _P, _LL, _I, _F, _I, _P]),
}

_lock = threading.Lock()
_lib = None


class StbError(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load the prebuilt libstb200.so (never builds: `build()` / `__graft_entry__.build()` does that) and bind every
    symbol include/stb200.h declares; raises StbError when the library is missing — there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not LIB_PATH.exists():
            raise StbError(
                f"{LIB_PATH} is missing — run `python -c 'import __graft_entry__ as g; g.build()'`. "
                "simpletuner_b200 has no CPU / eager fallback."
            )
        handle = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(handle, name)  # AttributeError if the .so does not export it
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(code: int) -> None:
    if code != 0:
        msg = lib().stb_last_error()
        raise StbError(f"libstb200 error {code}: {msg.decode() if msg else '?'}")
