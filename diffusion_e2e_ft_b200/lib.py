"""ctypes binding of libb200_e2eft.so (C ABI in include/b200_e2eft.h).

There is deliberately no fallback: if the shared library is missing (and cannot be built) or a
call fails, a RuntimeError is raised — the engine never routes through PyTorch/CPU arithmetic.
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_longlong, c_void_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200_e2eft.so")

_lib = None
ABI_VERSION = 17       # bumped with every signature change of include/b200_e2eft.h

_P = c_void_p
_LL = c_longlong
_SIGS = {
    "b200_last_error_string": (c_char_p, []),
    "b200_abi_version": (c_int, []),
    "b200_debug_force_block_n": (None, [c_int]),
    "b200_debug_set_flags": (None, [c_int]),
    "b200_debug_set_swap": (None, [c_int]),
    "b200_debug_set_halo": (None, [c_int]),
    "b200_debug_last_path": (c_int, []),
    "b200_debug_last_launch": (c_int, [POINTER(c_int), c_int]),
    "b200_geglu_block_n": (c_int, [c_int]),
    "b200_linear": (c_int, [_P, _LL, _LL, _P, _LL, _LL, c_int, c_int, c_int, c_int, _P, c_int, _P, _LL, _LL,
                            _P, _LL, _LL, c_int, c_int, c_float, _P, c_int, _P, c_int, c_int, c_int, _LL, _P]),
    "b200_conv2d_nhwc": (c_int, [_P, c_int, c_int, c_int, c_int, _P, c_int, _P, c_int, c_int,
                                 POINTER(c_int), POINTER(c_int), c_int, c_int, c_int, c_int, c_int, c_int,
                                 _P, _P, _LL, _P, _P, c_int, c_int, c_int, _P, _P, _P]),
    "b200_conv3x3_small_cout": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, _P]),
    "b200_im2col3x3_nchw": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, _P, c_int, _P]),
    "b200_group_norm_stats": (c_int, [_P, c_int, _P, c_int, c_int, c_int, c_int, c_int, _P, _P]),
    "b200_group_norm_apply": (c_int, [_P, c_int, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, c_float,
                                      c_int, _P, _P, _P]),
    "b200_group_norm_apply_cs": (c_int, [_P, c_int, _P, _P, c_int, _P, c_int, c_int, c_int, c_int, _P, _P, c_float,
                                         c_int, _P, _P, _P]),
    "b200_layer_norm": (c_int, [_P, c_int, _LL, c_int, _P, _P, c_float, _P, _P]),
    "b200_attention": (c_int, [_P, _LL, _LL, _P, _LL, _LL, _P, _LL, _LL, _P, _LL, _LL, c_int, c_int, c_int, c_int,
                               c_int, c_int, c_float, _P, _P]),
    "b200_attention_d64": (c_int, [_P, _LL, _LL, _P, _LL, _LL, _P, _LL, _LL, _P, _LL, _LL, c_int, c_int, c_int,
                                   c_int, c_int, c_float, _P, _P]),
    "b200_attention_d512": (c_int, [_P, _LL, _LL, _P, _LL, _LL, _P, _LL, _LL, _P, _LL, _LL, c_int, c_int, c_int,
                                    c_float, _P]),
    "b200_rowdot_heads_d": (c_int, [_P, _LL, _LL, _P, _LL, _LL, c_int, c_int, c_int, c_int, _P, _P]),
    "b200_rowdot_heads": (c_int, [_P, _LL, _LL, _P, _LL, _LL, c_int, c_int, c_int, _P, _P]),
    "b200_softmax_rows": (c_int, [_P, _LL, _P, _LL, _LL, c_int, c_float, _P]),
    "b200_softmax_groups": (c_int, [_P, c_int, _LL, c_int, c_int, _P, c_int, _P]),
    "b200_upsample_nearest_nhwc": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P]),
    "b200_timestep_embedding": (c_int, [_P, c_int, c_int, _P, _P]),
    "b200_embed_tokens": (c_int, [_P, _P, _P, c_int, _LL, c_int, c_int, c_int, _P, _P]),
    "b200_pointwise_nchw": (c_int, [_P, c_float, _P, c_float, c_int, _P, _P, c_int, c_int, c_int, _LL, _P, _P]),
    "b200_decode_post": (c_int, [_P, c_int, _LL, c_int, c_float, _P, _P]),
    "b200_ddim_step": (c_int, [_P, c_int, _LL, _P, _LL, c_int, c_int, _LL, c_int, c_float, c_float, _P, _P, _P, c_int,
                               _LL, _P]),
    "b200_ssi_loss": (c_int, [_P, _P, _P, c_int, _LL, _P, _P, _P]),
    "b200_angular_loss": (c_int, [_P, _P, _P, c_int, _LL, _P, _P, _P]),
    "b200_sumsq": (c_int, [_P, _LL, _P, _P]),
    "b200_adamw_step": (c_int, [_P, _P, _P, _P, _LL, c_float, c_float, c_float, c_float, c_float, c_int, _P,
                                c_float, _P]),
    "b200_gather_planar": (c_int, [_P, c_int, _LL, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P,
                                   _LL, _P]),
    "b200_col_sum": (c_int, [_P, c_int, _LL, c_int, _LL, _P, _P]),
    "b200_group_norm_mean_rstd": (c_int, [_P, _P, c_int, _P, c_int, c_int, c_int, c_int, c_float, _P, _P]),
    "b200_group_norm_bwd_sums": (c_int, [_P, c_int, c_int, c_int, c_int, _P, c_int, c_int, c_int, _P, _P, _P, c_int,
                                         _P, _P]),
    "b200_group_norm_bwd_apply": (c_int, [_P, c_int, c_int, c_int, c_int, _P, c_int, c_int, c_int, _P, _P, _P, c_int,
                                          _P, _P, _P, c_int, _P]),
    "b200_layer_norm_bwd": (c_int, [_P, c_int, _LL, c_int, _P, _P, c_float, _P, _P, c_int, _P, _P, _P]),
    "b200_softmax_bwd_rows": (c_int, [_P, _LL, _P, _LL, _P, _LL, c_int, c_float, _P]),
    "b200_act_bwd": (c_int, [_P, _P, _LL, c_int, _P, _P]),
    "b200_geglu_bwd": (c_int, [_P, _P, _LL, _P, _LL, c_int, _P, _P, _LL, _P]),
    "b200_ssi_loss_bwd": (c_int, [_P, _P, _P, c_int, _LL, _P, _P, _P, _P]),
    "b200_angular_loss_bwd": (c_int, [_P, _P, _P, c_int, _LL, _P, _P, _P, _P]),
    "b200_decode_post_bwd": (c_int, [_P, _P, c_int, _LL, c_int, _P, _P]),
    "b200_adamw_step_scaled": (c_int, [_P, _P, _P, _P, _LL, c_float, c_float, c_float, c_float, c_float, c_int, _P,
                                       c_float, c_float, _P]),
    "b200_adamw_step_state": (c_int, [_P, _P, _P, _P, _LL, c_float, c_float, c_float, c_float, c_float, _P, c_float,
                                      c_float, _P, c_int, c_float, c_float, c_float, _P]),
    "b200_adamw_step_state_groups": (c_int, [_P, _P, _P, _P, _LL, _P, _P, c_int, _P, _P, c_int, c_float, c_float,
                                             c_float, _P, c_float, c_float, _P, c_int, c_float, c_float, c_float, _P]),
    "b200_upsample_nearest_bwd": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P]),
    "b200_ensemble_normals": (c_int, [_P, c_int, _LL, _P, _P, _P, _P]),
    "b200_ensemble_depths_objective": (c_int, [_P, _P, _P, c_int, _LL, c_int, _P, _P, _P]),
    "b200_ensemble_depths_reduce": (c_int, [_P, _P, _P, c_int, _LL, c_int, _P, _P, _P, _P]),
    "b200_minmax_rows": (c_int, [_P, c_int, _LL, _P, _P, _P]),
    "b200_minmax_normalise": (c_int, [_P, _LL, _P, _P, _P]),
    "b200_rgb_normalise": (c_int, [_P, c_int, _LL, c_int, _P, _P]),
    "b200_resize_bilinear_aa": (c_int, [_P, _LL, c_int, c_int, c_int, c_int, _P, _P, _P]),
    "b200_resize_bicubic_aa": (c_int, [_P, _LL, c_int, c_int, c_int, c_int, _P, _P, _P]),
    "b200_resize_nearest": (c_int, [_P, _LL, c_int, c_int, c_int, c_int, _P, _P]),
    "b200_resize_nearest_exact": (c_int, [_P, _LL, c_int, c_int, c_int, c_int, _P, _P]),
    "b200_colorize_depth": (c_int, [_P, _LL, _P, c_int, _P, _P]),
    "b200_colorize_normals": (c_int, [_P, _LL, _P, _P]),
    "b200_diffusion_inputs": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, _LL, c_int, _P, _P, _P]),
    "b200_masked_latent_mse": (c_int, [_P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P]),
    "b200_masked_latent_mse_bwd": (c_int, [_P, c_int, _P, _P, _P, _P, c_int, c_int, _LL, _P, _P]),
    "b200_ema_update": (c_int, [_P, _P, _LL, c_float, _P]),
    "b200_cast_f32_to_f16": (c_int, [_P, _P, _LL, _P]),
    "b200_nhwc_to_nchw_f32": (c_int, [_P, c_int, c_int, c_int, _LL, _P, _P]),
    "b200_eval_align_depth": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_float, c_int, _P, _P, _P]),
    "b200_eval_depth_metrics": (c_int, [_P, _P, _P, c_int, _LL, _P, c_int, c_int, c_float, c_float, _P, _P, _P, _P]),
    "b200_eval_normal_error": (c_int, [_P, POINTER(c_longlong), _P, POINTER(c_longlong), _P, c_int, c_int, c_int, _P,
                                       _P, _LL, _P, _P, _P, _P, _P]),
    "b200_eval_kth_smallest": (c_int, [_P, _P, _LL, _LL, _P, _P, _P]),
    "b200_data_hypersim_source": (c_int, [_P, _P, _P, c_int, c_int, c_int, POINTER(c_double), _P, _P, _P]),
    "b200_data_resize_u8": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, _P, c_int, _P, _P,
                                    _P, _P]),
    "b200_data_depth_gather": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P]),
    "b200_data_depth_range": (c_int, [_P, c_int, _LL, c_float, c_float, _P, _P, _P]),
    "b200_data_finalise": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, c_int, c_float, c_float,
                                   _P, _P, _P, _P, _P, _P, _P, _P]),
    "b200_data_vkitti_normals": (c_int, [_P, c_int, c_int, c_int, c_float, c_float, c_float, c_float, _P, _P]),
    "b200_debug_pow_e32_neg": (c_int, [_P, _LL, c_int, _P, _P, _P]),
    "b200_data_hypersim_workspace_bytes": (_LL, [c_int, c_int, c_int]),
    "b200_data_hypersim_frames": (c_int, [_P, c_int, _P, c_int, _P, c_int, c_int, c_int, c_double, c_double, _P, _P, _P,
                                          _P, _P, _LL, _P]),
    "b200_debug_hypersim_pow": (c_int, [_P, _LL, c_int, _P, _P, _P, _P]),
}
EXPORTS = tuple(_SIGS)


def load(build_if_missing=True):
    """Load (building in-tree with nvcc when absent) the C-ABI library.  Raises on failure."""
    global _lib
    if _lib is not None:
        return _lib
    from . import build as _build
    if not os.path.exists(LIB_PATH) and not build_if_missing:
        raise RuntimeError(f"{LIB_PATH} is missing — run `python -m diffusion_e2e_ft_b200.build`")
    if build_if_missing and os.path.exists(_build.NVCC):
        _build.build()                 # no-op when the source digest matches the stamp: a stale .so is never loaded
    elif not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing and nvcc is not available to build it")
    lib = ctypes.CDLL(LIB_PATH)
    lib.b200_abi_version.restype = c_int
    if lib.b200_abi_version() != ABI_VERSION:
        raise RuntimeError(f"{LIB_PATH} exports ABI {lib.b200_abi_version()}, this package binds ABI {ABI_VERSION}: "
                           "rebuild with `python -m diffusion_e2e_ft_b200.build --force`")
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().b200_last_error_string()
        raise RuntimeError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
