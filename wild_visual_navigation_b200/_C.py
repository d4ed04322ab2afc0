"""ctypes binding of libwvn_b200.so (the C ABI declared in include/wvn_b200.h).

PyTorch is used here only for device memory and streams: every call passes raw
``tensor.data_ptr()`` values plus the current CUDA stream.  There is no CPU fallback — a
missing library or a non-sm_90 device raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, byref, c_char_p, c_float, c_int, c_longlong, c_size_t, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("WVN_B200_LIB", os.path.join(_HERE, "libwvn_b200.so"))  # override: instrumented builds


class WvnError(RuntimeError):
    pass


# wvn_vit_create_ffn's ffn: the block's FFN (WVN_VIT_FFN_MLP / WVN_VIT_FFN_SWIGLU)
VIT_FFN_MLP, VIT_FFN_SWIGLU = 0, 1


class VitConfig(Structure):
    _fields_ = [
        ("image_size", c_int), ("patch_size", c_int), ("dim", c_int), ("depth", c_int), ("heads", c_int),
        ("mlp_dim", c_int), ("max_batch", c_int), ("chunk", c_int), ("ln_eps", c_float), ("head_out", c_int),
        ("registers", c_int),
    ]


class GemmExArgs(Structure):
    """wvn_gemm_ex_args: the arguments of the testing entry wvn_gemm_bf16_ex (every GEMM epilogue)."""
    _fields_ = [
        ("m", c_int), ("n", c_int), ("k", c_int), ("epi", c_int), ("act", c_int), ("block_n", c_int),
        ("a", c_void_p), ("lda", c_longlong), ("w", c_void_p), ("bias", c_void_p), ("out", c_void_p), ("ldo", c_longlong),
        ("pos", c_void_p), ("tokens_in", c_int), ("npad", c_int), ("dim", c_int), ("heads", c_int),
        ("q_out", c_void_p), ("k_out", c_void_p), ("vt_out", c_void_p),
        ("feat", c_int), ("trav_col", c_int), ("x", c_void_p), ("ldx", c_longlong), ("trav", c_void_p),
        ("conf", c_void_p), ("loss_reco", c_void_p), ("cg_mean", c_void_p), ("cg_std", c_void_p),
        ("cg_std_factor", c_float), ("reverse_m", c_int), ("registers", c_int), ("residual", c_void_p), ("ldr", c_longlong),
    ]


class ResnetConfig(Structure):
    _fields_ = [("image_size", c_int), ("depth", c_int), ("max_batch", c_int)]


class EffnetConfig(Structure):
    _fields_ = [("image_size", c_int), ("max_batch", c_int)]


class TrainConfig(Structure):
    _fields_ = [
        ("w_trav", c_float), ("w_reco", c_float), ("std_factor", c_float), ("anomaly_balanced", c_int),
        ("lr", c_float), ("beta1", c_float), ("beta2", c_float), ("eps", c_float),
    ]


class FlowBuffers(Structure):
    """wvn_flow_buffers: the LinearRnvp buffers the flow kernels read (coupling masks, permutations)."""
    _fields_ = [("mask0", c_void_p), ("mask1", c_void_p), ("p1", c_void_p), ("invp1", c_void_p), ("p3", c_void_p),
                ("invp3", c_void_p)]


_lib = None

# name -> (restype, argtypes); every symbol of include/wvn_b200.h
_P, _I, _L, _F, _S = c_void_p, c_int, c_longlong, c_float, c_size_t
SIGNATURES = {
    "wvn_last_error": (c_char_p, []),
    "wvn_check_device": (_I, []),
    "wvn_version": (_I, []),
    "wvn_launch_count": (_L, []),
    "wvn_profile_enable": (None, [_I]),
    "wvn_profile_collect": (_I, [_P, _P]),
    "wvn_gemm_bf16": (_I, [_P, _L, _P, _P, _P, _L, _I, _I, _I, _I, _I, _I, _P]),
    "wvn_gemm_bf16_ex": (_I, [POINTER(GemmExArgs), _P]),
    "wvn_attention_bf16": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _P]),
    "wvn_layernorm": (_I, [_P, _P, _P, _P, _L, _I, _F, _P]),
    "wvn_image_to_patches": (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P]),
    "wvn_init_token_rows": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "wvn_layernorm_ex": (_I, [_P, _P, _P, _P, _P, _L, _I, _F, _I, _I, _I, _I, _P]),
    "wvn_attention_f32_debug": (_I, [_P, _P, _I, _I, _I, _I, _I, _F, _P]),
    "wvn_vit_create": (_I, [POINTER(VitConfig), POINTER(_P)]),
    "wvn_vit_create_ffn": (_I, [POINTER(VitConfig), _I, POINTER(_P)]),
    "wvn_swiglu_packed_rows": (_I, [_L, _P]),
    "wvn_vit_destroy": (None, [_P]),
    "wvn_vit_set_weight": (_I, [_P, c_char_p, _P, _L]),
    "wvn_vit_forward": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "wvn_vit_forward_u8": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "wvn_vit_forward_tta": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "wvn_vit_stego_head": (_I, [_P, _I, _P, _P]),
    "wvn_vit_npad": (_I, [_P]),
    "wvn_resnet_create": (_I, [POINTER(ResnetConfig), POINTER(_P)]),
    "wvn_resnet_destroy": (None, [_P]),
    "wvn_resnet_workspace_bytes": (_S, [_P]),
    "wvn_resnet_set_weight": (_I, [_P, c_char_p, _P, _L]),
    "wvn_resnet_forward": (_I, [_P, _P, _I, _P, _P]),
    "wvn_im2col_bf16_nhwc": (_I, [_P, _I, _I, _I, _I, _I, _I, _I, _P, _L, _P]),
    "wvn_im2col_image": (_I, [_P, _I, _I, _I, _I, _I, _I, _P, _L, _P]),
    "wvn_maxpool3s2_bf16_nhwc": (_I, [_P, _I, _I, _I, _I, _P, _P]),
    "wvn_segment_pool_pyramid": (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    "wvn_segment_pool_levels": (_I, [_P, _I, _I, _I, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P]),
    "wvn_effnet_create": (_I, [POINTER(EffnetConfig), POINTER(_P)]),
    "wvn_effnet_destroy": (None, [_P]),
    "wvn_effnet_workspace_bytes": (_S, [_P]),
    "wvn_effnet_set_weight": (_I, [_P, c_char_p, _P, _L]),
    "wvn_effnet_forward": (_I, [_P, _P, _I, _P, _P]),
    "wvn_depthwise_silu_bf16_nhwc": (_I, [_P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    "wvn_depthwise_pool_blocks": (_I, [_I, _I]),
    "wvn_se_gates": (_I, [_P, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P, _P, _P]),
    "wvn_channel_scale_bf16_nhwc": (_I, [_P, _I, _L, _I, _P, _P]),
    "wvn_upsample_dense": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "wvn_logits_argmax": (_I, [_P, _L, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "wvn_flip_average": (_I, [_P, _I, _I, _I, _L, _P]),
    "wvn_stego_kmeans_workspace_bytes": (_S, [_I, _I, _I]),
    "wvn_stego_kmeans": (_I, [_P, _L, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "wvn_crf_create": (_I, [_I, _I, _I, _I, POINTER(_P)]),
    "wvn_crf_destroy": (None, [_P]),
    "wvn_crf_workspace_bytes": (_S, [_P]),
    "wvn_crf_run": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P, _L, _I, _I, _I, _I, _I, _I, _F, _P, _P, _P]),
    "wvn_crf_build": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "wvn_crf_filter": (_I, [_P, _I, _P, _I, _P, _P]),
    "wvn_crf_export": (_I, [_P, _I, _P, _P, _P, _P, _P, _P]),
    "wvn_segment_workspace_bytes": (_S, [_I, _I, _I, _I]),
    "wvn_segment_reduce": (_I, [_P, _I, _I, _I, _I, _P, _I, _I, _I, _P, _P, _P, _P, _I, _P, _P]),
    "wvn_segment_relabel": (_I, [_P, _I, _L, _I, _P, _P, _P]),
    "wvn_segment_maps": (_I, [_P, _I, _I, _L, _P, _P, _I, _P, _P, _P, _P]),
    "wvn_supervision_pool": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P]),
    "wvn_slic_tables": (None, [_P, _P, _P]),
    "wvn_slic_geometry": (_I, [_I, _I, _I, _P, _P, _P]),
    "wvn_slic_workspace_bytes": (_S, [_I, _I, _I, _I]),
    "wvn_slic": (_I, [_P, _I, _I, _I, _I, _F, _I, _P, _P, _P, _P, _P, _P]),
    "wvn_project_and_render": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "wvn_mission_propagate_workspace_bytes": (_S, [_I, _I]),
    "wvn_mission_propagate": (_I, [_P, _P, _I, _P, _P, _P, _I, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P]),
    "wvn_mlp_infer_create": (_I, [_I, _I, _I, _I, POINTER(_P)]),
    "wvn_mlp_infer_destroy": (None, [_P]),
    "wvn_mlp_infer_reserve": (_I, [_P, _I]),
    "wvn_mlp_infer_set_params": (_I, [_P, _P, _P]),
    "wvn_mlp_infer_pixels": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P, _F, _P, _P, _P]),
    "wvn_mlp_infer_pixels_vit": (_I, [_P, _P, _I, _I, _I, _P, _P, _F, _P, _P, _P]),
    "wvn_mlp_infer_rows": (_I, [_P, _P, _L, _P, _P, _F, _P, _P, _P]),
    "wvn_mlp_infer_rows_padded": (_I, [_P, _P, _I, _I, _P, _P, _P, _F, _P, _P, _P]),
    "wvn_mlp_infer_create_double": (_I, [_I, _I, _I, _I, POINTER(_P)]),
    "wvn_mlp_param_count": (_S, [_I, _I, _I]),
    "wvn_mlp_train_workspace_bytes": (_S, [_I, _I, _I, _I]),
    "wvn_mlp_train_scalars_bytes": (_S, []),
    "wvn_mlp_train_forward_stats": (_I, [_I, _I, _I, _P, _P, _P, _P, _I, _I, _P, _P, _P]),
    "wvn_mlp_train_backward": (_I, [_I, _I, _I, _P, _P, _P, _P, _I, _I, _L, POINTER(TrainConfig), _P, _P, _P, _P, _P, _P, _P]),
    "wvn_mlp_train_apply": (_I, [_I, _I, _I, _P, _P, _P, _P, _P, _L, POINTER(TrainConfig), _P, _P]),
    "wvn_mlp_train_read_metrics": (_I, [_P, _P, _P]),
    "wvn_mlp_forward_f32": (_I, [_I, _I, _I, _P, _P, _I, _P, _P, _P, _P]),
    "wvn_trainer_destroy": (None, [_P]),
    "wvn_trainer_set_confidence": (_I, [_P, _I, _P, _P, _P, _P, _F, _F]),
    "wvn_trainer_copy_confidence": (_I, [_P, _P, _P]),
    "wvn_trainer_init_comm": (_I, [_P, _P, _I, _I]),
    "wvn_trainer_stats": (_P, [_P, POINTER(_I)]),
    "wvn_mlp_trainer_scalars_bytes": (_S, []),
    "wvn_mlp_trainer_create": (_I, [_I, _I, _I, _I, POINTER(TrainConfig), _P, _P, POINTER(_P)]),
    "wvn_comm_unique_id": (_I, [_P]),
    "wvn_mlp_train_step": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "wvn_double_mlp_param_count": (_S, [_I, _I, _I]),
    "wvn_double_mlp_forward_f32": (_I, [_I, _I, _I, _P, _P, _I, _P, _P, _P, _P]),
    "wvn_double_mlp_trainer_create": (_I, [_I, _I, _I, _I, POINTER(TrainConfig), _P, POINTER(_P)]),
    "wvn_double_mlp_train_step_padded": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "wvn_gcn_param_count": (_S, [_I, _I, _I]),
    "wvn_gcn_trainer_create": (_I, [_I, _I, _I, _I, _I, POINTER(TrainConfig), _P, POINTER(_P)]),
    "wvn_gcn_train_step_padded": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _I,
                                       _P]),
    "wvn_gcn_infer_rows": (_I, [_P, _P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _F, _P, _P, _P, _P]),
    "wvn_flow_param_count": (_S, [_I, _I]),
    "wvn_flow_trainer_create": (_I, [_I, _I, _I, POINTER(TrainConfig), _P, POINTER(_P)]),
    "wvn_flow_infer_create": (_I, [_I, _I, _I, _I, POINTER(_P)]),
    "wvn_flow_infer_destroy": (None, [_P]),
    "wvn_flow_infer_set_params": (_I, [_P, _P, _P]),
    "wvn_flow_infer_rows": (_I, [_P, _P, POINTER(FlowBuffers), _P, _I, _P, _P, _P, _P, _P, _F, _P, _P]),
    "wvn_flow_infer_rows_padded": (_I, [_P, _P, POINTER(FlowBuffers), _P, _I, _I, _P, _P, _P, _F, _P, _P]),
    "wvn_flow_infer_pixels": (_I, [_P, POINTER(FlowBuffers), _P, _I, _I, _I, _I, _I, _P, _P, _F, _P, _P, _P]),
    "wvn_flow_train_step": (_I, [_P, _P, _P, _P, _P, POINTER(FlowBuffers), _P, _I, _P, _P, _P, _P, _P, _I, _P]),
    "wvn_flow_train_step_padded": (_I, [_P, _P, _P, _P, _P, POINTER(FlowBuffers), _P, _I, _I, _P, _P, _P, _P, _P, _P, _I,
                                        _P]),
}


def lib() -> ctypes.CDLL:
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise WvnError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C wild_visual_navigation_b200/csrc` (there is no CPU fallback)"
        )
    l = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(l, name)  # AttributeError if the library lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = l
    return l


def check(status: int) -> None:
    if status != 0:
        msg = lib().wvn_last_error()
        raise WvnError(f"libwvn_b200 error {status}: {msg.decode() if msg else '?'}")


def require_device() -> None:
    """Fail loudly unless a compute-capability-9.0 GPU is the current device."""
    if not torch.cuda.is_available():
        raise WvnError("wild_visual_navigation_b200 needs a CUDA (sm_90a) device; no CPU fallback exists")
    check(lib().wvn_check_device())


def ptr(t) -> c_void_p:
    if t is None:
        return c_void_p(0)
    assert t.is_cuda and t.is_contiguous(), "expected a contiguous CUDA tensor"
    return c_void_p(t.data_ptr())


def stream() -> c_void_p:
    return c_void_p(torch.cuda.current_stream().cuda_stream)
