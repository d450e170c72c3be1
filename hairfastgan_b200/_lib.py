"""ctypes binding of libhairfast_sm90.so (include/hairfast_b200.h).

There is NO fallback: if the shared library is missing the import fails loudly, and every call
checks the status code and raises RuntimeError with hf_last_error() -- the same error type the
reference's pybind ops raise through TORCH_CHECK (op/fused_bias_act.cpp:7, op/upfirdn2d.cpp:8).
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "csrc", "libhairfast_sm90.so")

HF_BF16, HF_F16 = 0, 1
HF_MAX_STYLED, HF_MAX_TORGB = 17, 9

c_float_p = C.c_void_p   # device pointers travel as integers


class hf_conv_desc(C.Structure):
    _fields_ = [("cin", C.c_int), ("cout", C.c_int), ("ksize", C.c_int), ("upsample", C.c_int),
                ("dtype", C.c_int)]


class hf_conv_io(C.Structure):
    _fields_ = [("batch", C.c_int), ("height", C.c_int), ("width", C.c_int),
                ("x", C.c_void_p), ("x_batch_broadcast", C.c_int),
                ("style", C.c_void_p), ("style_dim", C.c_int), ("style_stride", C.c_int64),
                ("mod_weight", C.c_void_p), ("mod_bias", C.c_void_p), ("demodulate", C.c_int),
                ("noise", C.c_void_p), ("noise_batch", C.c_int), ("noise_weight", C.c_void_p),
                ("act_bias", C.c_void_p), ("act", C.c_int), ("y", C.c_void_p), ("workspace", C.c_void_p)]


class hf_conv2d_desc(C.Structure):
    _fields_ = [("cin", C.c_int), ("cout", C.c_int), ("cin_pad", C.c_int), ("ksize", C.c_int), ("stride", C.c_int),
                ("groups", C.c_int), ("dtype", C.c_int), ("prepadded", C.c_int), ("transposed", C.c_int)]


class hf_conv2d_io(C.Structure):
    _fields_ = [("batch", C.c_int), ("height", C.c_int), ("width", C.c_int), ("x16", C.c_void_p),
                ("shift", C.c_void_p), ("act", C.c_int), ("slope", C.c_void_p), ("slope0", C.c_float),
                ("residual16", C.c_void_p), ("y16", C.c_void_p), ("y16b_scale", C.c_void_p),
                ("y16b_shift", C.c_void_p), ("y16b", C.c_void_p), ("y32_nchw", C.c_void_p),
                ("act_after_residual", C.c_int)]


class hf_sean_ace_tables(C.Structure):
    _fields_ = [("fc_w", C.c_void_p), ("fc_b", C.c_void_p), ("tw", C.c_void_p), ("table", C.c_void_p), ("n2", C.c_int)]


class hf_mod_desc(C.Structure):
    _fields_ = [("layers", C.c_int), ("inp", C.c_int), ("middle", C.c_int), ("stacks", C.c_int), ("dtype", C.c_int)]


class hf_mod_rows(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("batch_stride", C.c_longlong), ("row_stride", C.c_longlong)]


class hf_gen_config(C.Structure):
    _fields_ = [("size", C.c_int), ("style_dim", C.c_int), ("channel_multiplier", C.c_int), ("dtype", C.c_int)]


class hf_gen_weights(C.Structure):
    _fields_ = [("const_input", C.c_void_p),
                ("conv_weight", C.c_void_p * HF_MAX_STYLED),
                ("conv_mod_weight", C.c_void_p * HF_MAX_STYLED),
                ("conv_mod_bias", C.c_void_p * HF_MAX_STYLED),
                ("conv_blur_kernel", C.c_void_p * HF_MAX_STYLED),
                ("conv_noise_weight", C.c_void_p * HF_MAX_STYLED),
                ("conv_act_bias", C.c_void_p * HF_MAX_STYLED),
                ("rgb_weight", C.c_void_p * HF_MAX_TORGB),
                ("rgb_mod_weight", C.c_void_p * HF_MAX_TORGB),
                ("rgb_mod_bias", C.c_void_p * HF_MAX_TORGB),
                ("rgb_bias", C.c_void_p * HF_MAX_TORGB),
                ("rgb_up_kernel", C.c_void_p * HF_MAX_TORGB)]


class hf_gen_io(C.Structure):
    _fields_ = [("batch", C.c_int), ("latent", C.c_void_p),
                ("noise", C.c_void_p * HF_MAX_STYLED), ("noise_batch", C.c_int * HF_MAX_STYLED),
                ("start_layer", C.c_int), ("end_layer", C.c_int),
                ("layer_in", C.c_void_p), ("skip_in", C.c_void_p),
                ("out_feature", C.c_void_p), ("out_rgb", C.c_void_p),
                ("feature_in", C.c_void_p * HF_MAX_STYLED), ("feature_alpha", C.c_float),
                ("features_out", C.c_void_p * (HF_MAX_STYLED + 1))]


# every symbol include/hairfast_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "hf_version": (C.c_int, []),
    "hf_last_error": (C.c_char_p, []),
    "hf_set_device": (C.c_int, [C.c_int]),
    "hf_sm_count": (C.c_int, []),
    "hf_last_launch_count": (C.c_int, []),
    "hf_total_launch_count": (C.c_longlong, []),
    "hf_upfirdn2d_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int] * 13 + [C.c_void_p]),
    "hf_bias_act_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_int,
                                  C.c_float, C.c_float, C.c_void_p]),
    "hf_conv_packed_bytes": (C.c_size_t, [C.POINTER(hf_conv_desc)]),
    "hf_conv_pack": (C.c_int, [C.POINTER(hf_conv_desc), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "hf_conv_workspace_bytes": (C.c_size_t, [C.POINTER(hf_conv_desc), C.c_int, C.c_int, C.c_int]),
    "hf_conv_plan_query": (C.c_int, [C.POINTER(hf_conv_desc), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "hf_conv_forward": (C.c_int, [C.POINTER(hf_conv_desc), C.c_void_p, C.POINTER(hf_conv_io), C.c_void_p]),
    "hf_conv_time_kernel": (C.c_int, [C.POINTER(hf_conv_desc), C.c_void_p, C.POINTER(hf_conv_io), C.c_int,
                                      C.POINTER(C.c_float), C.c_void_p]),
    "hf_torgb_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                   C.c_int, C.c_void_p, C.c_void_p]),
    "hf_conv2d_packed_bytes": (C.c_size_t, [C.POINTER(hf_conv2d_desc)]),
    "hf_conv2d_pack": (C.c_int, [C.POINTER(hf_conv2d_desc), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "hf_conv2d_forward": (C.c_int, [C.POINTER(hf_conv2d_desc), C.c_void_p, C.POINTER(hf_conv2d_io), C.c_void_p]),
    "hf_conv2d_plan_query": (C.c_int, [C.POINTER(hf_conv2d_desc), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "hf_nchw_to_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_int, C.c_void_p]),
    "hf_nhwc16_to_nchw": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "hf_channel_reduce_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "hf_instance_norm_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "hf_instance_norm_lrelu_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float,
                                                C.c_int, C.c_void_p]),
    "hf_reflect_pad1_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p]),
    "hf_channel_mean_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p]),
    "hf_se_gate_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                    C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "hf_scale_add_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "hf_upsample_add_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "hf_adaptive_avgpool_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_int, C.c_int, C.c_void_p]),
    "hf_stem3x3_nhwc16": (C.c_int, [C.c_void_p] * 8 + [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "hf_stem7x7s2_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p]),
    "hf_maxpool3x3s2_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p]),
    "hf_pooled_fc_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "hf_gate_add_up_nhwc16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                        C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "hf_bilinear_upsample_nchw_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                C.c_int, C.c_int, C.c_void_p]),
    "hf_bicubic_downsample_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_int, C.c_void_p]),
    "hf_dilate_erode_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                      C.c_int, C.c_void_p]),
    "hf_bilinear_argmax_nchw_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                              C.c_int, C.c_int, C.c_void_p]),
    "hf_align_masks_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "hf_fspace_blend_f32": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_float),
                                      C.POINTER(C.c_float), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_int, C.c_void_p]),
    "hf_sean_labels": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "hf_sean_onehot_conv": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                      C.c_int, C.c_void_p]),
    "hf_sean_style_tables": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(hf_sean_ace_tables), C.c_int, C.c_void_p,
                                       C.c_void_p]),
    "hf_sean_ace_apply": (C.c_int, [C.c_void_p] * 8 + [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "hf_sean_class_means": (C.c_int, [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p]),
    "hf_sean_conv_img": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p]),
    "hf_shape_labels": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "hf_shape_onehot_s2": (C.c_int, [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "hf_shape_gemm": (C.c_int, [C.c_int] + [C.c_void_p] * 6 + [C.c_int] * 5 + [C.c_void_p]),
    "hf_shape_gemm_workspace_bytes": (C.c_size_t, [C.c_int] * 5),
    "hf_shape_gemm_plan": (C.c_int, [C.c_int] * 6 + [C.POINTER(C.c_int)]),
    "hf_shape_layer_norm_lrelu": (C.c_int, [C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p]),
    "hf_shape_layer_norm_workspace_bytes": (C.c_size_t, [C.c_longlong]),
    "hf_shape_logits_argmax": (C.c_int, [C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_void_p]),
    "hf_mod_workspace_bytes": (C.c_size_t, [C.POINTER(hf_mod_desc), C.c_int]),
    "hf_mod_gemm_plan": (C.c_int, [C.POINTER(hf_mod_desc), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "hf_mod_embed16": (C.c_int, [C.POINTER(hf_mod_desc), C.c_int, C.POINTER(hf_mod_rows), C.c_void_p, C.c_void_p]),
    "hf_mod_gemm": (C.c_int, [C.POINTER(hf_mod_desc), C.c_int, C.c_int] + [C.c_void_p] * 6),
    "hf_mod_hidden": (C.c_int, [C.POINTER(hf_mod_desc), C.c_int] + [C.c_void_p] * 8),
    "hf_mod_chain": (C.c_int, [C.POINTER(hf_mod_desc), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.POINTER(hf_mod_rows), C.POINTER(hf_mod_rows), C.c_void_p, C.c_void_p, C.c_void_p]),
    "hf_align_lanczos_taps": (C.c_int, [C.c_int, C.c_int]),
    "hf_align_lanczos_coeffs": (C.c_int, [C.c_int, C.c_int, C.c_void_p]),
    "hf_align_resample_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "hf_align_resample_u8": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "hf_align_pad_blend_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "hf_align_pad_blend_u8": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_void_p,
                                        C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "hf_align_gaussian_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                        C.c_void_p]),
    "hf_align_median_workspace_bytes": (C.c_size_t, []),
    "hf_align_median_f32": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]),
    "hf_align_quad_u8": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.c_void_p,
                                   C.c_int, C.c_int, C.c_void_p]),
    "hf_generator_packed_bytes":(C.c_size_t, [C.POINTER(hf_gen_config)]),
    "hf_generator_workspace_bytes": (C.c_size_t, [C.POINTER(hf_gen_config), C.c_int]),
    "hf_generator_pack": (C.c_int, [C.POINTER(hf_gen_config), C.POINTER(hf_gen_weights), C.c_void_p, C.c_void_p]),
    "hf_generator_forward": (C.c_int, [C.POINTER(hf_gen_config), C.c_void_p, C.POINTER(hf_gen_io), C.c_void_p,
                                       C.POINTER(C.c_int), C.c_void_p]),
}

_lib = None


def lib():
    """Load the shared library (once).  Raises if it has not been built -- no fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -m hairfastgan_b200.build` "
                "(hairfastgan_b200 has no CPU / PyTorch fallback)")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(handle, name)     # AttributeError if a declared symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(status: int, what: str = "") -> None:
    if status != 0:
        msg = lib().hf_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"hairfast_b200 {what} failed ({status}): {msg}")


_device_set = {}


def use_device(index: int) -> None:
    """Point the library at the CUDA device of the tensors about to be passed in."""
    import threading
    key = threading.get_ident()
    if _device_set.get(key) != index:
        check(lib().hf_set_device(index), "hf_set_device")
        _device_set[key] = index


def stream_ptr() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream
