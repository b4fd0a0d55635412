"""ctypes binding of ``libgen3c_b200.so`` (the C ABI declared in ``include/gen3c_b200.h``).

The product path has no CPU fallback: if the shared library is missing, or a call returns a
non-zero status, an exception is raised.  PyTorch is only used by callers for device memory and
streams; nothing here takes or returns torch types.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "lib" / "libgen3c_b200.so"


class G3CError(RuntimeError):
    pass


class DitConfig(C.Structure):
    _fields_ = [
        ("model_channels", C.c_int),
        ("num_blocks", C.c_int),
        ("num_heads", C.c_int),
        ("ffn_dim", C.c_int),
        ("context_dim", C.c_int),
        ("adaln_lora_dim", C.c_int),
        ("in_channels", C.c_int),
        ("out_channels", C.c_int),
        ("concat_padding_mask", C.c_int),
        ("max_frames", C.c_int),
        ("max_h", C.c_int),
        ("max_w", C.c_int),
        ("rope_h_ratio", C.c_float),
        ("rope_w_ratio", C.c_float),
        ("rope_t_ratio", C.c_float),
        ("base_fps", C.c_int),
    ]


class StepArgs(C.Structure):
    _fields_ = [
        ("xt", C.c_void_p),
        ("gt_latent", C.c_void_p),
        ("aug_noise", C.c_void_p),
        ("indicator", C.c_void_p),
        ("cond_mask", C.c_void_p),
        ("pose_cond", C.c_void_p),
        ("padding_mask", C.c_void_p),
        ("ctx_cond", C.c_void_p),
        ("ctx_uncond", C.c_void_p),
        ("sigma", C.c_float),
        ("sigma_next", C.c_float),
        ("sigma_data", C.c_float),
        ("sigma_aug", C.c_float),
        ("guidance", C.c_float),
        ("xt_next", C.c_void_p),
        ("cond_mask_uncond", C.c_void_p),
        ("net_output", C.c_void_p),
    ]


_P = C.c_void_p
_I = C.c_int
_F = C.c_float

# name -> (restype, argtypes); every symbol include/gen3c_b200.h declares
SIGNATURES = {
    "g3c_last_error": (C.c_char_p, []),
    "g3c_version": (_I, []),
    "g3c_device_info": (_I, [C.POINTER(_I), C.POINTER(_I), C.POINTER(_I)]),
    "g3c_render_create": (_I, [_I, _I, _I, C.POINTER(_P)]),
    "g3c_render_destroy": (_I, [_P]),
    "g3c_render_set_deterministic": (_I, [_P, _I]),
    "g3c_forward_warp": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P]),
    "g3c_render_cache": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P]),
    "g3c_bilinear_splatting": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P]),
    "g3c_splat_indices": (_I, [_P, _I, _I, _I, _P, _P]),
    "g3c_unproject_points": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P]),
    "g3c_reliable_depth_mask": (_I, [_P, _I, _I, _I, _I, _F, _F, _P, _P]),
    "g3c_align_depth_nonrigid": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _F, _F, _P, _P]),
    "g3c_foreground_occlusion": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P]),
    "g3c_render_cache_occlusion": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _I, _I, _P]),
    "g3c_gemm_bf16": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _I, _P]),
    "g3c_gemm_norm_rope_bf16": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _F, _P]),
    "g3c_quantize_rows_fp8": (_I, [_P, _I, _I, _I, _P, _I, _P, _P]),
    "g3c_gemm_fp8": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _I, _P]),
    "g3c_gemm_norm_rope_fp8": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _F, _P]),
    "g3c_ln_modulate_fp8": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _F, _P]),
    "g3c_attn_fwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _F, _P]),
    "g3c_attn_fwd_sbhd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _F, _P]),
    "g3c_attn_fwd_sbhd_lse": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _F, _P]),
    "g3c_attn_bwd_sbhd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P] + [_I] * 12 + [_F, _P]),
    "g3c_attn_set_trace": (_I, [_P]),
    "g3c_ln_modulate": (_I, [_P, _P, _P, _P, _P, _I, _I, _F, _P]),
    "g3c_rmsnorm_rope": (_I, [_P, _I, _I, _I, _P, _P, _F, _P]),
    "g3c_dit_create": (_I, [C.POINTER(DitConfig), C.POINTER(_P)]),
    "g3c_dit_destroy": (_I, [_P]),
    "g3c_dit_load": (_I, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), _I, _I]),
    "g3c_nccl_unique_id": (_I, [_P]),
    "g3c_dit_enable_cp": (_I, [_P, _P, _I, _I]),
    "g3c_dit_cp_export": (_I, [_P, _P]),
    "g3c_dit_cp_import": (_I, [_P, _P, _I]),
    "g3c_dit_cp_mode": (_I, [_P]),
    "g3c_dit_disable_cp": (_I, [_P]),
    "g3c_dit_set_linear_fp8": (_I, [_P, _I]),
    "g3c_dit_enable_cfg_parallel": (_I, [_P, _I]),
    "g3c_dit_cfg_export": (_I, [_P, _P]),
    "g3c_dit_cfg_import": (_I, [_P, _P]),
    "g3c_dit_set_shape": (_I, [_P, _I, _I, _I, _I, _F]),
    "g3c_dit_forward": (_I, [_P, _P, _P, _P, _P, _F, _P, _P, _P]),
    "g3c_denoise_step": (_I, [_P, C.POINTER(StepArgs), _P]),
    "g3c_dit_profile": (_I, [_P, _I]),
    "g3c_dit_profile_read": (_I, [_P, C.POINTER(_F), C.POINTER(_I), _I]),
    "g3c_dit_profile_wait_ms": (_I, [_P, C.POINTER(_F)]),
    "g3c_dit_workspace_bytes": (C.c_int64, [_P]),
    "g3c_dit_last_launch_count": (_I, [_P]),
    "g3c_dit_read_tables": (_I, [_P, _I, _P, _P, _P]),
    "g3c_dit_read_modulation": (_I, [_P, _F, _P, _P, _P]),
    "g3c_dit_read_step": (_I, [_P, _P, _P, _P, _P, _P]),
    "g3c_attn_fwd_gated": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _F, _P, C.c_uint32, _I, _P, _P]),
    "g3c_dit_cp_region": (_I, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "g3c_dit_cp_attach": (_I, [_P, C.POINTER(_P), _I]),
    "g3c_dit_cfg_region": (_I, [_P, C.POINTER(_P), C.POINTER(C.c_int64)]),
    "g3c_dit_cfg_attach": (_I, [_P, _P]),
}

_lib = None


def load() -> C.CDLL:
    """Load the shared library (once).  Raises G3CError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("GEN3C_B200_LIB", str(LIB_PATH))
    if not os.path.exists(path):
        raise G3CError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback)"
        )
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library diverge
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().g3c_last_error().decode("utf-8", "replace")
        raise G3CError(f"{what} failed with status {rc}: {msg}")


def ptr(t) -> int | None:
    """Device pointer of a torch tensor (must be contiguous), or None."""
    if t is None:
        return None
    if not t.is_contiguous():
        raise G3CError("tensor passed to the C ABI must be contiguous")
    return t.data_ptr()


def stream_ptr() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream
