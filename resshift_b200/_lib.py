"""ctypes binding of ``librs_b200.so`` (C ABI in include/resshift_b200.h).

There is no CPU or PyTorch fallback: if the CUDA library is missing, importing this module
fails loudly, and every compute entry point needs a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("RESSHIFT_B200_LIB", _HERE / "lib" / "librs_b200.so"))

RS_MAX_LEVELS = 8


class RsError(RuntimeError):
    pass


class UNetConfigC(C.Structure):
    """Mirror of ``rs_unet_config``."""
    _fields_ = [
        ("image_size", C.c_int32), ("in_channels", C.c_int32), ("model_channels", C.c_int32),
        ("out_channels", C.c_int32), ("n_levels", C.c_int32),
        ("channel_mult", C.c_int32 * RS_MAX_LEVELS), ("num_res_blocks", C.c_int32 * RS_MAX_LEVELS),
        ("n_attn", C.c_int32), ("attention_resolutions", C.c_int32 * RS_MAX_LEVELS),
        ("swin_depth", C.c_int32), ("swin_embed_dim", C.c_int32), ("swin_heads", C.c_int32),
        ("window_size", C.c_int32), ("mlp_ratio", C.c_float), ("cond_mask", C.c_int32), ("lq_size", C.c_int32),
    ]


class UNetOptionsC(C.Structure):
    """Mirror of ``rs_unet_options``."""
    _fields_ = [("use_scale_shift_norm", C.c_int32), ("resblock_updown", C.c_int32), ("conv_resample", C.c_int32),
                ("patch_norm", C.c_int32)]


class UNetModelConfigC(C.Structure):
    """Mirror of ``rs_unetmodel_config``."""
    _fields_ = [
        ("image_size", C.c_int32), ("in_channels", C.c_int32), ("model_channels", C.c_int32),
        ("out_channels", C.c_int32), ("n_levels", C.c_int32),
        ("channel_mult", C.c_int32 * RS_MAX_LEVELS), ("num_res_blocks", C.c_int32 * RS_MAX_LEVELS),
        ("n_attn", C.c_int32), ("attention_resolutions", C.c_int32 * RS_MAX_LEVELS),
        ("num_heads", C.c_int32), ("num_head_channels", C.c_int32), ("use_new_attention_order", C.c_int32),
    ]


class UNetConvConfigC(C.Structure):
    """Mirror of ``rs_unetconv_config``."""
    _fields_ = [
        ("in_channels", C.c_int32), ("model_channels", C.c_int32), ("out_channels", C.c_int32), ("n_levels", C.c_int32),
        ("channel_mult", C.c_int32 * RS_MAX_LEVELS), ("num_res_blocks", C.c_int32 * RS_MAX_LEVELS),
        ("cond_lq", C.c_int32), ("dims", C.c_int32),
    ]


class VQConfigC(C.Structure):
    """Mirror of ``rs_vq_config``."""
    _fields_ = [
        ("embed_dim", C.c_int32), ("n_embed", C.c_int32), ("z_channels", C.c_int32), ("in_channels", C.c_int32),
        ("out_ch", C.c_int32), ("ch", C.c_int32), ("n_levels", C.c_int32),
        ("ch_mult", C.c_int32 * RS_MAX_LEVELS), ("num_res_blocks", C.c_int32 * RS_MAX_LEVELS),
    ]


class VQOptionsC(C.Structure):
    """Mirror of ``rs_vq_options``."""
    _fields_ = [
        ("enc_attn", C.c_int32 * RS_MAX_LEVELS), ("dec_attn", C.c_int32 * RS_MAX_LEVELS), ("mid_attn", C.c_int32),
        ("resamp_with_conv", C.c_int32), ("tanh_out", C.c_int32),
    ]


class ConvArgsC(C.Structure):
    """Mirror of ``rs_conv_args``."""
    _fields_ = [
        ("x", C.c_void_p), ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32), ("ld", C.c_int32),
        ("w_packed", C.c_void_p), ("ipad", C.c_int32), ("bias", C.c_void_p), ("bias_sN", C.c_int32),
        ("cout", C.c_int32), ("ksize", C.c_int32), ("stride", C.c_int32), ("pad_lo", C.c_int32),
        ("residual", C.c_void_p), ("res_ld", C.c_int32), ("out", C.c_void_p), ("out_ld", C.c_int32),
        ("out_f32_nchw", C.c_void_p), ("act", C.c_int32), ("bn", C.c_int32), ("msub", C.c_int32),
        ("part", C.c_void_p * 2), ("cstride", C.c_int32 * 2), ("coff", C.c_int32 * 2),
        ("gstat", C.c_void_p), ("splitk_scratch", C.c_void_p),
        ("silu_out", C.c_void_p), ("silu_ld", C.c_int32), ("film", C.c_void_p), ("film_sN", C.c_int32),
    ]


# GroupNorm statistics routes (RS_GN_*)
GN_GSTAT, GN_CONV_PAIRS, GN_WINDOW_PAIRS, GN_FINALIZE, GN_STATS_PAIRS, GN_STATS_GSTAT = range(6)


class GnArgsC(C.Structure):
    """Mirror of ``rs_gn_args``."""
    _fields_ = [
        ("x", C.c_void_p), ("x_ld", C.c_int32), ("y", C.c_void_p), ("y_ld", C.c_int32),
        ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
        ("gamma", C.c_void_p), ("beta", C.c_void_p), ("film", C.c_void_p), ("film_sN", C.c_longlong),
        ("silu", C.c_int32), ("eps", C.c_float), ("route", C.c_int32),
        ("part", C.c_void_p), ("slots", C.c_int32), ("gstat", C.c_void_p), ("counter", C.c_void_p),
    ]


class PSampleArgsC(C.Structure):
    """Mirror of ``rs_p_sample_args``."""
    _fields_ = [
        ("x_t", C.c_void_p), ("x0", C.c_void_p), ("noise", C.c_void_p), ("x_next", C.c_void_p),
        ("coef1", C.c_void_p), ("coef2", C.c_void_p), ("stdv", C.c_void_p), ("in_scale", C.c_void_p),
        ("T", C.c_int32), ("t", C.c_int32), ("N", C.c_int32), ("C", C.c_int32), ("HW", C.c_int32),
        ("next_in", C.c_void_p), ("next_cpad", C.c_int32), ("counters", C.c_void_p), ("n_counters", C.c_int32),
    ]


class PSamplePredArgsC(C.Structure):
    """Mirror of ``rs_p_sample_pred_args``."""
    _fields_ = [
        ("out", C.c_void_p), ("x_t", C.c_void_p), ("y", C.c_void_p), ("noise", C.c_void_p), ("x_next", C.c_void_p),
        ("coef1", C.c_void_p), ("coef2", C.c_void_p), ("stdv", C.c_void_p), ("in_scale", C.c_void_p),
        ("eps_coef", C.c_void_p), ("eta", C.c_void_p), ("one_minus_eta", C.c_void_p),
        ("T", C.c_int32), ("t", C.c_int32), ("N", C.c_int32), ("C", C.c_int32), ("HW", C.c_int32),
        ("mean_type", C.c_int32), ("next_in", C.c_void_p), ("next_cpad", C.c_int32), ("x0_out", C.c_void_p),
    ]


class SamplerOptionsC(C.Structure):
    """Mirror of ``rs_sampler_options``."""
    _fields_ = [("mean_type", C.c_int32), ("normalize_input", C.c_int32), ("latent_flag", C.c_int32)]


class DdpmOptionsC(C.Structure):
    """Mirror of ``rs_ddpm_options``."""
    _fields_ = [("kind", C.c_int32), ("mean_type", C.c_int32), ("var_type", C.c_int32), ("clip", C.c_int32),
                ("eta", C.c_double)]


class DdpmStepArgsC(C.Structure):
    """Mirror of ``rs_ddpm_step_args``."""
    _fields_ = [
        ("out", C.c_void_p), ("x_t", C.c_void_p), ("noise", C.c_void_p), ("x_next", C.c_void_p),
        ("sqrt_recip_acp", C.c_void_p), ("sqrt_recipm1_acp", C.c_void_p), ("coef1", C.c_void_p), ("coef2", C.c_void_p),
        ("log_var", C.c_void_p), ("acp", C.c_void_p), ("acp_prev", C.c_void_p),
        ("T", C.c_int32), ("t", C.c_int32), ("N", C.c_int32), ("C", C.c_int32), ("HW", C.c_int32),
        ("kind", C.c_int32), ("mean_type", C.c_int32), ("clip", C.c_int32), ("eta", C.c_float),
        ("next_in", C.c_void_p), ("next_cpad", C.c_int32), ("counters", C.c_void_p), ("n_counters", C.c_int32),
        ("x0_out", C.c_void_p), ("out_sN", C.c_int64), ("var_type", C.c_int32), ("log_betas", C.c_void_p),
    ]


class DdimReverseOptionsC(C.Structure):
    """Mirror of ``rs_ddim_reverse_options``."""
    _fields_ = [("mean_type", C.c_int32), ("clip", C.c_int32)]


class DdimReverseStepArgsC(C.Structure):
    """Mirror of ``rs_ddim_reverse_step_args``."""
    _fields_ = [
        ("out", C.c_void_p), ("x_t", C.c_void_p), ("x_next", C.c_void_p),
        ("sqrt_recip_acp", C.c_void_p), ("sqrt_recipm1_acp", C.c_void_p), ("acp_next", C.c_void_p),
        ("T", C.c_int32), ("t", C.c_int32), ("N", C.c_int32), ("C", C.c_int32), ("HW", C.c_int32),
        ("mean_type", C.c_int32), ("clip", C.c_int32),
        ("next_in", C.c_void_p), ("next_cpad", C.c_int32), ("counters", C.c_void_p), ("n_counters", C.c_int32),
        ("x0_out", C.c_void_p), ("out_sN", C.c_int64),
    ]


# rs_ddpm_kind, rs_ddpm_var_type, and the rows of rs_ddpm_sampler_create's float64 tables (rs_ddpm_table_row)
DDPM_KINDS = {"ancestral": 0, "ddim": 1}
DDPM_VAR_TYPES = {"fixed_large": 0, "fixed_small": 1, "learned_range": 3, "learned": 4}     # 2 is unassigned
DDPM_TABLE_ROWS = ("sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1",
                   "posterior_mean_coef2", "log_variance_fixed_large", "posterior_log_variance_clipped",
                   "alphas_cumprod", "alphas_cumprod_prev")
# rs_ddim_reverse_sampler_create's rows: the same, then RS_DDPM_ACP_NEXT
DDIM_REVERSE_TABLE_ROWS = DDPM_TABLE_ROWS + ("alphas_cumprod_next",)
# rs_ddpm_sampler_create's rows with RS_VAR_LEARNED_RANGE: the same, then RS_DDPM_LOG_BETAS (its max_log)
DDPM_LEARNED_RANGE_TABLE_ROWS = DDPM_TABLE_ROWS + ("log_betas",)

# rs_mean_type, by the reference's predict_type names (models/script_util.py:35-44)
MEAN_TYPES = {"xstart": 0, "epsilon": 1, "epsilon_scale": 2, "residual": 3}


class PackInputArgsC(C.Structure):
    """Mirror of ``rs_pack_input_args``."""
    _fields_ = [
        ("x", C.c_void_p), ("Cx", C.c_int32), ("scale_tab", C.c_void_p), ("scale_n", C.c_int32), ("scale_idx", C.c_int32),
        ("lq_nchw", C.c_void_p), ("Cl", C.c_int32), ("mask_nchw", C.c_void_p), ("lq_nhwc", C.c_void_p), ("lq_ld", C.c_int32),
        ("out", C.c_void_p), ("Cpad", C.c_int32), ("N", C.c_int32), ("HW", C.c_int32), ("lq_unshuffle", C.c_int32),
        ("W", C.c_int32), ("counters", C.c_void_p), ("n_counters", C.c_int32),
    ]


# every symbol include/resshift_b200.h declares: (restype, argtypes)
_P = C.c_void_p
_SIGNATURES = {
    "rs_version": (C.c_int, []),
    "rs_last_error": (C.c_char_p, []),
    "rs_unet_create": (C.c_int, [C.POINTER(UNetConfigC), C.POINTER(_P)]),
    "rs_unet_create_ex": (C.c_int, [C.POINTER(UNetConfigC), C.POINTER(UNetOptionsC), C.POINTER(_P)]),
    "rs_unetmodel_create": (C.c_int, [C.POINTER(UNetModelConfigC), C.POINTER(UNetOptionsC), C.POINTER(_P)]),
    "rs_unetconv_create": (C.c_int, [C.POINTER(UNetConvConfigC), C.POINTER(UNetOptionsC), C.POINTER(_P)]),
    "rs_unet_destroy": (None, [_P]),
    "rs_unet_param_count": (C.c_int, [_P]),
    "rs_unet_param_info": (C.c_int, [_P, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                     C.POINTER(C.c_int32)]),
    "rs_unet_arena_bytes": (C.c_size_t, [_P]),
    "rs_unet_set_arena": (C.c_int, [_P, _P]),
    "rs_unet_load_param": (C.c_int, [_P, C.c_char_p, _P, _P]),
    "rs_plan_create": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "rs_plan_destroy": (None, [_P]),
    "rs_plan_workspace_bytes": (C.c_size_t, [_P]),
    "rs_plan_bind": (C.c_int, [_P, _P]),
    "rs_plan_num_launches": (C.c_int, [_P]),
    "rs_plan_forward": (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    "rs_plan_profile": (C.c_int, [_P, _P, _P, _P, _P, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int32), _P]),
    "rs_plan_profile_ops": (C.c_int, [_P, _P, _P, _P, _P, C.POINTER(C.c_double), C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_int32), _P]),
    "rs_plan_probe": (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), _P]),
    "rs_sampler_create": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.c_double, C.POINTER(C.c_int32), C.POINTER(_P)]),
    "rs_sampler_create_ex": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.c_double, C.POINTER(C.c_int32),
                                       C.POINTER(SamplerOptionsC), C.POINTER(_P)]),
    "rs_sampler_destroy": (None, [_P]),
    "rs_sampler_run": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, _P]),
    "rs_sampler_run_host": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_size_t, C.c_int, _P]),
    "rs_sampler_staging_bytes": (C.c_size_t, [_P]),
    "rs_sampler_set_taps": (C.c_int, [_P, _P, _P]),
    "rs_ddpm_sampler_create": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int32),
                                         C.POINTER(DdpmOptionsC), C.POINTER(_P)]),
    "rs_op_ddpm_step": (C.c_int, [C.POINTER(DdpmStepArgsC), _P]),
    "rs_ddim_reverse_sampler_create": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int32),
                                                 C.POINTER(DdimReverseOptionsC), C.POINTER(_P)]),
    "rs_op_ddim_reverse_step": (C.c_int, [C.POINTER(DdimReverseStepArgsC), _P]),
    "rs_p_sample": (C.c_int, [_P, _P, _P, _P, C.c_float, C.c_float, C.c_float, C.c_int, C.c_longlong, _P]),
    "rs_op_p_sample_ex": (C.c_int, [C.POINTER(PSampleArgsC), _P]),
    "rs_op_p_sample_pred": (C.c_int, [C.POINTER(PSamplePredArgsC), _P]),
    "rs_op_pack_input": (C.c_int, [C.POINTER(PackInputArgsC), _P]),
    "rs_op_pack_image": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, C.c_int, _P]),
    "rs_plan_embedding": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, _P, _P]),
    "rs_sampler_tables": (C.c_int, [_P, C.POINTER(C.c_float)]),
    "rs_schedule_tables": (C.c_int, [C.c_int, C.POINTER(C.c_double), C.c_double, C.POINTER(C.c_int32), C.POINTER(C.c_float)]),
    "rs_schedule_tables_ex": (C.c_int, [C.c_int, C.POINTER(C.c_double), C.c_double, C.POINTER(C.c_int32),
                                        C.POINTER(SamplerOptionsC), C.POINTER(C.c_float)]),
    "rs_op_pointwise_conv": (C.c_int, [_P, _P, C.c_int, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "rs_op_kl_posterior": (C.c_int, [_P, _P, C.c_int, _P, C.c_int, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P]),
    "rs_op_pack_conv_weight": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "rs_op_conv2d": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int,
                               C.c_int, _P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P]),
    "rs_op_conv2d_stats": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int,
                                     C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int, C.c_int,
                                     C.POINTER(C.c_int32), _P, _P, C.c_int, _P]),
    "rs_op_conv2d_splitk": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int,
                                      C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P,
                                      C.POINTER(C.c_int32), _P, _P, _P]),
    "rs_op_conv2d_ex": (C.c_int, [C.POINTER(ConvArgsC), C.POINTER(C.c_int32), _P]),
    "rs_op_conv2d_timeline": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int,
                                        C.c_int, _P, C.c_int, C.c_int, C.c_int, _P, C.POINTER(C.c_int32), _P, _P]),
    "rs_op_groupnorm": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, C.c_longlong, C.c_int,
                                  _P, C.c_int, _P, _P]),
    "rs_op_groupnorm_scratch_floats": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "rs_op_groupnorm_apply": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, C.c_longlong, C.c_int,
                                        _P, C.c_int, _P, _P]),
    "rs_op_groupnorm_finalize": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _P, _P]),
    "rs_op_groupnorm_ex": (C.c_int, [C.POINTER(GnArgsC), C.POINTER(C.c_int32), _P]),
    "rs_op_groupnorm_apply_pairs": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, C.c_longlong,
                                              C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "rs_op_expand_relpos": (C.c_int, [_P, _P, C.c_int, _P]),
    "rs_op_expand_relpos_ex": (C.c_int, [_P, _P, C.c_int, C.c_int, _P]),
    "rs_op_vq_attention": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "rs_op_vq_attention_rows": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "rs_op_unet_attention": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "rs_op_softmax_rows":(C.c_int, [_P, C.c_int, C.c_int, C.c_longlong, C.c_float, _P]),
    "rs_op_window_attention": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "rs_op_window_attention_ex": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "rs_op_window_attention_cfg": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P,
                                             C.c_int, C.c_int, C.POINTER(C.c_int32), _P]),
    "rs_op_swin_attn": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P, _P, _P,
                                  _P, _P, _P, _P, _P]),
    "rs_op_swin_attn_ex": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P,
                                     _P, _P, _P, _P, C.c_int, C.POINTER(C.c_int32), _P]),
    "rs_op_mlp": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P]),
    "rs_op_mlp_ex": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P,
                               C.POINTER(_P), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), _P]),
    "rs_debug_tile_config": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32)]),
    "rs_op_upsample2x": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "rs_op_upsample2x_ex": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "rs_op_avgpool2x2": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "rs_vq_create": (C.c_int, [C.POINTER(VQConfigC), C.POINTER(_P)]),
    "rs_vq_create_ex": (C.c_int, [C.POINTER(VQConfigC), C.POINTER(VQOptionsC), C.POINTER(_P)]),
    "rs_kl_create_ex": (C.c_int, [C.POINTER(VQConfigC), C.POINTER(VQOptionsC), C.POINTER(_P)]),
    "rs_vq_run_between": (C.c_int, [_P, C.c_int, _P]),
    "rs_vq_attention_count": (C.c_int, [_P, C.POINTER(C.c_int32)]),
    "rs_vq_set_attention_rows_at": (C.c_int, [_P, C.c_int, C.c_int, C.c_int]),
    "rs_vq_attention_output_at": (C.c_int, [_P, C.c_int, C.POINTER(_P), C.POINTER(C.c_longlong), C.POINTER(C.c_longlong),
                                            C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "rs_vq_plan_create": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "rs_vq_encode": (C.c_int, [_P, _P, _P, _P]),
    "rs_vq_decode": (C.c_int, [_P, _P, _P, _P, C.c_int, _P]),
    "rs_vq_encode_begin": (C.c_int, [_P, _P, _P]),
    "rs_vq_encode_end": (C.c_int, [_P, _P, _P]),
    "rs_vq_decode_begin": (C.c_int, [_P, _P, _P, C.c_int, _P]),
    "rs_vq_decode_end": (C.c_int, [_P, _P, _P]),
    "rs_vq_set_attention_rows": (C.c_int, [_P, C.c_int, C.c_int]),
    "rs_vq_attention_output": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_longlong), C.POINTER(C.c_longlong),
                                         C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "rs_vq_profile_ops": (C.c_int, [_P, C.POINTER(C.c_double), C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_int32), _P]),
    "rs_vq_decode_code": (C.c_int, [_P, _P, _P, _P]),
    "rs_kl_create": (C.c_int, [C.POINTER(VQConfigC), C.POINTER(_P)]),
    "rs_kl_encode": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "rs_kl_decode": (C.c_int, [_P, _P, _P, _P]),
    "rs_kl_encode_begin": (C.c_int, [_P, _P, _P]),
    "rs_kl_encode_end": (C.c_int, [_P, _P, _P, _P, _P]),
    "rs_kl_decode_begin": (C.c_int, [_P, _P, _P]),
    "rs_kl_decode_end": (C.c_int, [_P, _P, _P]),
    "rs_op_bicubic_upsample": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "rs_op_ingest_u8": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "rs_op_emit_u8": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P]),
    "rs_op_tile_gather": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P]),
}


def _load():
    if not LIB_PATH.exists():
        raise ImportError(
            f"resshift_b200: CUDA library {LIB_PATH} not found. Build it with "
            f"`python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)            # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(rc: int) -> None:
    if rc != 0:
        msg = lib.rs_last_error()
        raise RsError(f"librs_b200 error {rc}: {msg.decode(errors='replace') if msg else '?'}")


def declared_symbols():
    return sorted(_SIGNATURES)


def ptr(t) -> int:
    """Device (or host) address of a torch tensor, or None."""
    return None if t is None else t.data_ptr()


def current_stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


def probe(plan_handle, batch: int, block: str, device):
    """rs_plan_probe: the named tensor of a bound plan's last run as a new fp32 NCHW tensor [batch, C, H, W]."""
    import torch
    c, hh, ww = C.c_int32(), C.c_int32(), C.c_int32()
    check(lib.rs_plan_probe(plan_handle, block.encode(), None, C.byref(c), C.byref(hh), C.byref(ww), None))
    out = torch.empty(batch, c.value, hh.value, ww.value, dtype=torch.float32, device=device)
    check(lib.rs_plan_probe(plan_handle, block.encode(), out.data_ptr(), C.byref(c), C.byref(hh), C.byref(ww), current_stream()))
    return out


def make_config(cfg) -> UNetConfigC:
    c = UNetConfigC()
    c.image_size, c.in_channels, c.model_channels, c.out_channels = cfg.image_size, cfg.in_channels, cfg.model_channels, cfg.out_channels
    c.n_levels = len(cfg.channel_mult)
    for i, v in enumerate(cfg.channel_mult):
        c.channel_mult[i] = int(v)
    for i, v in enumerate(cfg.num_res_blocks):
        c.num_res_blocks[i] = int(v)
    c.n_attn = len(cfg.attention_resolutions)
    for i, v in enumerate(cfg.attention_resolutions):
        c.attention_resolutions[i] = int(v)
    c.swin_depth, c.swin_embed_dim, c.swin_heads = cfg.swin_depth, cfg.swin_embed_dim, cfg.swin_heads
    c.window_size, c.mlp_ratio = cfg.window_size, float(cfg.mlp_ratio)
    c.cond_mask, c.lq_size = int(cfg.cond_mask), cfg.lq_size
    return c


def make_options(cfg) -> UNetOptionsC:
    o = UNetOptionsC()
    o.use_scale_shift_norm, o.resblock_updown = int(cfg.use_scale_shift_norm), int(cfg.resblock_updown)
    o.conv_resample, o.patch_norm = int(cfg.conv_resample), int(getattr(cfg, "patch_norm", False))
    return o


def make_unetmodel_config(cfg) -> UNetModelConfigC:
    c = UNetModelConfigC()
    c.image_size, c.in_channels, c.model_channels, c.out_channels = cfg.image_size, cfg.in_channels, cfg.model_channels, cfg.out_channels
    c.n_levels = len(cfg.channel_mult)
    for i, v in enumerate(cfg.channel_mult):
        c.channel_mult[i] = int(v)
    for i, v in enumerate(cfg.num_res_blocks):
        c.num_res_blocks[i] = int(v)
    c.n_attn = len(cfg.attention_resolutions)
    for i, v in enumerate(cfg.attention_resolutions):
        c.attention_resolutions[i] = int(v)
    c.num_heads, c.num_head_channels = cfg.num_heads, cfg.num_head_channels
    c.use_new_attention_order = int(cfg.use_new_attention_order)
    return c


def make_unetconv_config(cfg) -> UNetConvConfigC:
    c = UNetConvConfigC()
    c.in_channels, c.model_channels, c.out_channels = cfg.in_channels, cfg.model_channels, cfg.out_channels
    c.n_levels = len(cfg.channel_mult)
    for i, v in enumerate(cfg.channel_mult):
        c.channel_mult[i] = int(v)
    for i, v in enumerate(cfg.num_res_blocks):
        c.num_res_blocks[i] = int(v)
    c.cond_lq, c.dims = int(cfg.cond_lq), int(cfg.dims)
    return c


def make_vq_config(cfg) -> VQConfigC:
    c = VQConfigC()
    c.embed_dim, c.n_embed, c.z_channels = cfg.embed_dim, cfg.n_embed, cfg.z_channels
    c.in_channels, c.out_ch, c.ch = cfg.in_channels, cfg.out_ch, cfg.ch
    c.n_levels = len(cfg.ch_mult)
    for i, v in enumerate(cfg.ch_mult):
        c.ch_mult[i] = int(v)
    for i, v in enumerate(cfg.num_res_blocks):
        c.num_res_blocks[i] = int(v)
    return c


def make_vq_options(cfg) -> VQOptionsC:
    """``rs_vq_options`` of a VQConfig: its attention levels (encoder and decoder apart), mid attention, resampling, tanh."""
    o = VQOptionsC()
    for i, (e, d) in enumerate(zip(cfg.enc_attn, cfg.dec_attn)):
        o.enc_attn[i], o.dec_attn[i] = int(e), int(d)
    o.mid_attn, o.resamp_with_conv, o.tanh_out = int(cfg.has_attn), int(cfg.resamp_with_conv), int(cfg.tanh_out)
    return o
