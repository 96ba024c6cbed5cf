"""ctypes binding of librf_b200.so (the C ABI declared in include/rf_b200.h).

There is deliberately no fallback: if the shared library is missing or was not built for this
machine, importing a compute entry point raises.  `python __graft_entry__.py build` (or
`make -C reflectionflow_b200/csrc`) produces the library in-tree.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
# RF_B200_LIB: load another build of the same library (kernel A/B experiments across builds)
LIB_PATH = os.environ.get("RF_B200_LIB") or os.path.join(_HERE, "librf_b200.so")

_lib = None


class RFError(RuntimeError):
    pass


def _declare(lib):
    vp, ci, cf = c_void_p, c_int, c_float
    lib.rf_last_error.restype = c_char_p
    lib.rf_last_error.argtypes = []
    lib.rf_abi_version.restype = ci
    lib.rf_launch_count.restype = c_int64
    lib.rf_profile_start.restype = ci
    lib.rf_profile_stop.restype = ci
    lib.rf_profile_stop.argtypes = [c_char_p, ci]
    lib.rf_op_linear.restype = ci
    lib.rf_op_linear.argtypes = [ci, ci, ci, ci, vp, ci, vp, vp, vp, ci, vp, ci, vp, ci, vp, vp, vp,
                                 vp, vp, vp]
    lib.rf_op_linear_lora_workspace_bytes.restype = ctypes.c_size_t
    lib.rf_op_linear_lora_workspace_bytes.argtypes = [ci]
    lib.rf_op_linear_lora.restype = ci
    lib.rf_op_linear_lora.argtypes = [ci, ci, ci, ci, vp, ci, vp, vp, vp, ci, vp, ci, vp, vp, ci, vp, vp, vp,
                                      vp, vp, vp, vp]
    lib.rf_op_attention.restype = ci
    lib.rf_op_attention.argtypes = [vp, vp, vp, ci, vp, ci, ci, ci, ci, ci, ci, cf, vp]
    lib.rf_op_ln_modulate.restype = ci
    lib.rf_op_ln_modulate.argtypes = [vp, ci, vp, ci, ci, ci, vp, vp, ci, ci, vp]
    lib.rf_op_gemv.restype = ci
    lib.rf_op_gemv.argtypes = [vp, ci, ci, vp, vp, vp, ci, ci, ci, ci, vp]
    lib.rf_op_timestep_embed.restype = ci
    lib.rf_op_timestep_embed.argtypes = [vp, cf, vp, ci, vp]
    lib.rf_op_euler_step.restype = ci
    lib.rf_op_euler_step.argtypes = [vp, vp, vp, vp, ci, vp]
    lib.rf_op_resize_u8.restype = ci
    lib.rf_op_resize_u8.argtypes = [vp, ci, ci, vp, vp, ci, ci, vp, vp, ci, vp, vp, ci, vp]
    lib.rf_dbg_force_gemm_v1.restype = None
    lib.rf_dbg_force_gemm_v1.argtypes = [ci]
    if hasattr(lib, "rf_vae_create"):
        lib.rf_vae_create.restype = ci
        lib.rf_vae_create.argtypes = [POINTER(vp)]
        lib.rf_vae_destroy.restype = None
        lib.rf_vae_destroy.argtypes = [vp]
        lib.rf_vae_load_weight.restype = ci
        lib.rf_vae_load_weight.argtypes = [vp, c_char_p, vp, c_int64]
        lib.rf_vae_missing_weights.restype = ci
        lib.rf_vae_missing_weights.argtypes = [vp]
        lib.rf_vae_decode.restype = ci
        lib.rf_vae_decode.argtypes = [vp, vp, ci, ci, cf, cf, vp, vp, vp]
        lib.rf_vae_encode.restype = ci
        lib.rf_vae_encode.argtypes = [vp, vp, vp, ci, ci, vp, cf, cf, vp, vp]
    lib.rf_text_create.restype = ci
    lib.rf_text_create.argtypes = [vp, POINTER(vp)]
    lib.rf_text_destroy.restype = None
    lib.rf_text_destroy.argtypes = [vp]
    lib.rf_text_load_weight.restype = ci
    lib.rf_text_load_weight.argtypes = [vp, c_char_p, vp, c_int64]
    lib.rf_text_missing_weights.restype = ci
    lib.rf_text_missing_weights.argtypes = [vp, c_char_p]
    lib.rf_t5_encode.restype = ci
    lib.rf_t5_encode.argtypes = [vp, vp, ci, ci, vp, vp, vp]
    lib.rf_clip_encode.restype = ci
    lib.rf_clip_encode.argtypes = [vp, vp, vp, ci, ci, vp, vp, vp]
    if hasattr(lib, "rf_dit_create"):
        lib.rf_dit_create.restype = ci
        lib.rf_dit_create.argtypes = [vp, POINTER(vp)]
        lib.rf_dit_destroy.restype = None
        lib.rf_dit_destroy.argtypes = [vp]
        lib.rf_dit_load_weight.restype = ci
        lib.rf_dit_load_weight.argtypes = [vp, c_char_p, vp, c_int64]
        lib.rf_dit_set_lora.restype = ci
        lib.rf_dit_set_lora.argtypes = [vp, c_char_p, vp, vp, ci, ci, ci, cf]
        lib.rf_dit_missing_weights.restype = ci
        lib.rf_dit_missing_weights.argtypes = [vp]
        lib.rf_dit_prepare.restype = ci
        lib.rf_dit_prepare.argtypes = [vp, ci, ci, ci, ci, vp, vp, vp, ci, cf, vp]
        lib.rf_dit_forward.restype = ci
        lib.rf_dit_forward.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp]
        lib.rf_dit_denoise.restype = ci
        lib.rf_dit_denoise.argtypes = [vp, vp, vp, vp, vp, vp, ci, cf, vp, vp]


def load():
    """Return the loaded CDLL; raise RFError if the native library is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RFError(
                f"{LIB_PATH} not found: build it with `python __graft_entry__.py build` "
                "(nvcc, sm_90a). There is no CPU or PyTorch fallback for the DiT hot path.")
        lib = ctypes.CDLL(LIB_PATH)
        _declare(lib)
        _lib = lib
    return _lib


def check(rc: int, what: str = "rf call"):
    if rc != 0:
        msg = load().rf_last_error()
        raise RFError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")


def profile_start():
    check(load().rf_profile_start(), "rf_profile_start")


def profile_stop() -> dict:
    import json
    buf = ctypes.create_string_buffer(1 << 16)
    check(load().rf_profile_stop(buf, len(buf)), "rf_profile_stop")
    return json.loads(buf.value.decode())


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    if t is None:
        return None
    return c_void_p(t.data_ptr())


def cur_stream():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)
