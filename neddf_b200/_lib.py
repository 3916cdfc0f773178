"""ctypes binding of libneddf_b200.so (the C ABI declared in include/neddf_b200.h).

There is no CPU or PyTorch fallback: if the shared library is missing or a call fails, the
product raises.  Build it with ``python __graft_entry__.py`` (nvcc, sm_90a).
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# NEDDF_B200_LIB selects another build of the same ABI (e.g. a tuning variant)
LIB_PATH = os.environ.get("NEDDF_B200_LIB") or os.path.join(_HERE, "libneddf_b200.so")

MAX_SKIPS = 8
N_PENALTY = 6
ACT_IDS = {"tanhExp": 0, "ReLU": 1, "LeakyReLU": 2}
SAMPLING_IDS = {"point": 0, "cone": 1}
ENGINE_IDS = {"auto": 0, "fp32": 1, "tc": 2, "tc2": 3}
OUT_FULL, OUT_EVAL = 0, 1
UV_DTYPES = {torch.int64: 0, torch.int32: 1, torch.int16: 2, torch.float32: 3}
# reference insertion order of the penalty dict (neddf/network/neddf.py:259-300)
PENALTY_KEYS = ("constraints_aux_grad", "constraints_dDdt", "range_distance", "range_aux_grad",
                "range_color", "constraints_color")


class FieldConfig(C.Structure):
    _fields_ = [
        ("embed_pos_rank", C.c_int32), ("embed_dir_rank", C.c_int32),
        ("ddf_layer_count", C.c_int32), ("ddf_layer_width", C.c_int32),
        ("col_layer_count", C.c_int32), ("col_layer_width", C.c_int32),
        ("activation_type", C.c_int32), ("density_activation_type", C.c_int32),
        ("d_near", C.c_float), ("n_skips", C.c_int32), ("skips", C.c_int32 * MAX_SKIPS),
        ("penalty_weight", C.c_float * N_PENALTY),
    ]


class NerfConfig(C.Structure):
    _fields_ = [
        ("embed_pos_rank", C.c_int32), ("embed_dir_rank", C.c_int32), ("layer_count", C.c_int32),
        ("layer_width", C.c_int32), ("activation_type", C.c_int32), ("density_activation_type", C.c_int32),
        ("n_skips", C.c_int32), ("skips", C.c_int32 * MAX_SKIPS),
    ]


class NeusConfig(C.Structure):
    _fields_ = [
        ("embed_pos_rank", C.c_int32), ("embed_dir_rank", C.c_int32), ("sdf_layer_count", C.c_int32),
        ("sdf_layer_width", C.c_int32), ("col_layer_count", C.c_int32), ("col_layer_width", C.c_int32),
        ("activation_type", C.c_int32), ("n_skips", C.c_int32), ("skips", C.c_int32 * MAX_SKIPS),
    ]


class FieldState(C.Structure):
    _fields_ = [("aux_grad_scale", C.c_float), ("distance_range_max", C.c_float), ("lowpass_alpha", C.c_float),
                ("penalty_weight", C.c_float * N_PENALTY)]


_P = C.c_void_p
_I32, _I64, _F, _D = C.c_int32, C.c_int64, C.c_float, C.c_double
_FP = C.POINTER(C.c_float)

_SIGNATURES = {
    "neddf_abi_version": (C.c_int32, []),
    "neddf_last_error": (C.c_char_p, []),
    "neddf_launch_count": (C.c_int64, []),
    "neddf_field_layer_shapes": (_I32, [C.POINTER(FieldConfig), C.POINTER(C.c_int32), _I32]),
    "neddf_field_create": (_I32, [C.POINTER(FieldConfig), C.POINTER(_P)]),
    "neddf_field_destroy": (_I32, [_P]),
    "neddf_field_resolve_engine": (_I32, [_P, _I32]),
    "neddf_field_status": (_I32, [_P, C.POINTER(C.c_int32), _P]),
    "neddf_field_set_weights": (_I32, [_P, C.POINTER(_P), C.POINTER(_P), _I32, _P]),
    "neddf_make_rays": (_I32, [_P, _I32, _I64, _FP, _FP, _FP, _P, _P, _P]),
    "neddf_make_image_rays": (_I32, [_I32, _I32, _I32, _I64, _I64, _FP, _FP, _FP, _P, _P, _P]),
    "neddf_coarse_dists": (_I32, [_P, _I64, _I32, _F, _F, _P, _P]),
    "neddf_make_samples": (_I32, [_P, _P, _P, _I64, _I32, _I32, _F, _P, _P, _P, _P]),
    "neddf_field_forward": (_I32, [_P, C.POINTER(FieldState), _P, _P, _P, _I64, _P, _P, _P, _P, _P, _I32, _I32, _P]),
    "neddf_field_forward_rays": (_I32, [_P, C.POINTER(FieldState), _P, _P, _P, _I64, _I32, _I32, _F,
                                        _P, _P, _P, _P, _P, _I32, _I32, _P]),
    "neddf_render_loss": (_I32, [_P] * 8 + [_I64] + [_P] * 8 + [_P]),
    "neddf_field_adam_step": (_I32, [_P, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), C.POINTER(_I64), _I32,
                                     _F, _D, _D, _F, _F, _I64, _P]),
    "neddf_wgrad_workspace_bytes": (_I64, []),
    "neddf_wgrad": (_I32, [_P, _I64, _I32, _I32, _P, _I64, _I64, _P, _I64, _I32, _P, _P]),
    "neddf_colsum_value_rows": (_I32, [_P, _I64, _I64, _P, _P, _P]),
    "neddf_field_forward_rays_segment": (_I32, [_P, C.POINTER(FieldState), _P, _P, _P, _I64, _I32, _I32, _F, _I32, _I32,
                                                _P, _P, _P, _P, _I32, _P]),
    "neddf_terminate_rays": (_I32, [_P, _P, _I64, _I32, _I32, _I32, _P, _P, _P, _F, _P, _P, _P, _P]),
    "neddf_field_forward_train": (_I32, [_P, C.POINTER(FieldState), _P, _P, _P, _I64, _I32, _I32, _F, _P, _P, _P, _P,
                                         _I32, _P]),
    "neddf_field_backward": (_I32, [_P, C.POINTER(FieldState), _P, _P, _P, _I64, _I32, _I32, _F, _P, _P, _P, _P,
                                    _P, _P, _P, _P, _P, _P, _P]),
    "neddf_field_forward_train_samples": (_I32, [_P, C.POINTER(FieldState), _P, _P, _P, _I64, _P, _P, _P, _P, _P, _P,
                                                 _I32, _P]),
    "neddf_field_backward_samples": (_I32, [_P, C.POINTER(FieldState), _P, _P, _P, _I64, _P, _P, _P, _P, _P, _P, _P,
                                            _P, _P, _P, _P]),
    "neddf_composite": (_I32, [_P, _P, _P, _P, _I64, _I32, _F, _P, _P, _P, _P, _P, _P, _P]),
    "neddf_composite_backward": (_I32, [_P, _P, _P, _I64, _I32, _F, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "neddf_sample_pdf": (_I32, [_P, _P, _P, _I64, _I32, _I32, _I32, _P, _P, _P, _P, _P]),
    "neddf_invert_cdf": (_I32, [_P, _P, _P, _I64, _I32, _I32, _P, _P, _P]),
    "neddf_tc_selftest": (_I32, [_P, _P, _I32, _I32, _I32, _P, _P]),
    "neddf_nerf_layer_shapes": (_I32, [C.POINTER(NerfConfig), C.POINTER(C.c_int32), _I32]),
    "neddf_nerf_create": (_I32, [C.POINTER(NerfConfig), C.POINTER(_P)]),
    "neddf_nerf_destroy": (None, [_P]),
    "neddf_nerf_set_weights": (_I32, [_P, C.POINTER(_P), C.POINTER(_P), _I32, _P]),
    "neddf_nerf_forward": (_I32, [_P, _FP, _P, _P, _P, _I64, _P, _P, _P]),
    "neddf_nerf_forward_rays": (_I32, [_P, _FP, _P, _P, _P, _I64, _I32, _I32, _F, _P, _P, _P]),
    "neddf_nerf_forward_rays_segment": (_I32, [_P, _FP, _P, _P, _P, _I64, _I32, _I32, _F, _I32, _I32, _P, _P, _P, _P, _P]),
    "neddf_nerf_train_create": (_I32, [C.POINTER(NerfConfig), C.POINTER(_P)]),
    "neddf_nerf_train_destroy": (None, [_P]),
    "neddf_nerf_train_set_weights": (_I32, [_P, C.POINTER(_P), C.POINTER(_P), _I32, _P]),
    "neddf_nerf_train_backward": (_I32, [_P, _FP, _P, _P, _P, _I64] + [_P] * 9 + [_P]),
    "neddf_nerf_train_backward_rays": (_I32, [_P, _FP, _P, _P, _P, _I64, _I32, _I32, _F] + [_P] * 9 + [_P]),
    "neddf_neus_layer_shapes": (_I32, [C.POINTER(NeusConfig), C.POINTER(C.c_int32), _I32]),
    "neddf_neus_create": (_I32, [C.POINTER(NeusConfig), C.POINTER(_P)]),
    "neddf_neus_destroy": (None, [_P]),
    "neddf_neus_set_weights": (_I32, [_P, C.POINTER(_P), C.POINTER(_P), _I32, _P, _P]),
    "neddf_neus_forward": (_I32, [_P, _P, _P, _I64, _P, _P, _P, _P, _P]),
    "neddf_neus_forward_rays": (_I32, [_P, _P, _P, _P, _I64, _I32, _I32, _F, _P, _P, _P, _P, _P]),
    "neddf_neus_forward_rays_segment": (_I32, [_P, _P, _P, _P, _I64, _I32, _I32, _F, _I32, _I32, _P, _P, _P, _P, _P]),
    "neddf_neus_train_create": (_I32, [C.POINTER(NeusConfig), C.POINTER(_P)]),
    "neddf_neus_train_destroy": (None, [_P]),
    "neddf_neus_train_set_weights": (_I32, [_P, C.POINTER(_P), C.POINTER(_P), _I32, _P, _P]),
    "neddf_neus_train_backward": (_I32, [_P, _P, _P, _I64, _P, _P, _P, _P, C.POINTER(_P), _P]),
    "neddf_neus_train_backward_rays": (_I32, [_P, _P, _P, _P, _I64, _I32, _I32, _F, _P, _P, _P, _P, C.POINTER(_P), _P]),
    "neddf_mc_workspace_bytes": (_I64, [_I32, _I32, _I32]),
    "neddf_mc_count": (_I32, [_P, _I32, _I32, _I32, _F, _P, _P, _P]),
    "neddf_mc_emit": (_I32, [_P, _I32, _I32, _I32, _F, _P, _P, _P, _P]),
    "neddf_mc_normals": (_I32, [_P, _I32, _I32, _I32, _F, _P, _P, _P, _P, _P]),
    "neddf_mcb_points": (_I32, [_P, _I32, _I64, _I64, _P, _P]),
    "neddf_mcb_bricks_workspace_bytes": (_I64, [_I32]),
    "neddf_mcb_bricks": (_I32, [_P, _I32, _F, _F, _P, _P, _P, _P, _P]),
    "neddf_mcb_workspace_bytes": (_I64, [_I32, _I64]),
    "neddf_mcb_count": (_I32, [_P, _I32, _F, _P, _P, _I64, _P, _P, _P]),
    "neddf_mcb_emit_workspace_bytes": (_I64, [_I64, _I64]),
    "neddf_mcb_emit": (_I32, [_P, _I32, _F, _P, _P, _I64, _P, _I64, _I64, _P, _P, _P, _P]),
    "neddf_mcb_normals": (_I32, [_P, _I32, _P, _P, _I64, _P, _I64, _I64, _P, _P, _P, _P, _P]),
    "neddf_trace_init": (_I32, [_P, _P, _I64, _F] + [_P] * 8 + [_P]),
    "neddf_trace_step": (_I32, [_P, _P, _I64, _P, _P, _F, _F, _I32] + [_P] * 9 + [_P]),
    "neddf_trace_hits": (_I32, [_P, _P, _I64, _P, _P, _P, _P, _P, _P, _P]),
    "neddf_trace_fd_points": (_I32, [_P, _P, _I64, _P, _P, _P]),
    "neddf_trace_fd_normals": (_I32, [_P, _P, _P, _I64, _P, _P]),
}

# csrc/surface.cu (include/neddf_b200.h NEDDF_TRACE_*)
TRACE_MARCH, TRACE_BISECT, TRACE_HIT, TRACE_MISS = 0, 1, 16, 17
TRACE_EPS, TRACE_FD_H, TRACE_BISECTIONS = 1e-4, 1e-4, 8

_lib = None


def exported_symbols():
    return sorted(_SIGNATURES)


def lib():
    """Load (once) and return the CDLL; raises if the CUDA library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"neddf_b200: {LIB_PATH} is missing - build it with `python __graft_entry__.py` "
                "(nvcc, sm_90a). There is no CPU / PyTorch fallback for the render hot path.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the ABI lost a symbol
            fn.restype = res
            fn.argtypes = args
        if handle.neddf_abi_version() != 3:
            raise RuntimeError("neddf_b200: ABI version mismatch between Python host and libneddf_b200.so")
        _lib = handle
    return _lib


def check(rc: int, what: str = "") -> int:
    if rc < 0:
        msg = lib().neddf_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"neddf_b200 {what} failed (code {rc}): {msg}")
    return rc


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr(device=None):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def fbuf(values):
    arr = (C.c_float * len(values))(*[float(v) for v in values])
    return arr


def require_cuda_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(f"neddf_b200: `{name}` must be a CUDA tensor (the hot path has no CPU implementation)")
    if t.dtype != torch.float32:
        t = t.to(torch.float32)
    return t.contiguous()
