"""ctypes binding of ``libddpo_b200.so`` (the C ABI declared in ``include/ddpo_b200.h``).

The library is the product: there is no Python/CPU fallback.  If the shared object is
missing, or a call returns a non-zero status, this module raises immediately.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DDPO_B200_LIB: developer override used for A/B timing of kernel variants (another build of the same C ABI)
LIB_PATH = os.environ.get("DDPO_B200_LIB") or os.path.join(_HERE, "libddpo_b200.so")

vp, i32, i64, f32, u32p, f32p = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_void_p, C.c_void_p


class DdimCommon(C.Structure):
    _fields_ = [("eps_uncond", vp), ("eps_cond", vp), ("sample", vp), ("alphas_cumprod", vp), ("timesteps", vp),
                ("timestep_stride", i32), ("final_alpha_cumprod", f32), ("step_ratio", i32),
                ("guidance_scale", f32), ("eta", f32), ("batch", i32), ("n", i32), ("workspace", vp),
                ("prediction_type", i32)]


class IGemmArgs(C.Structure):
    _fields_ = [("a0", vp), ("a1", vp), ("c0", i32), ("c1", i32), ("lda0", i32), ("lda1", i32),
                ("is_conv", i32), ("batch", i32), ("h", i32), ("w", i32), ("conv_stride", i32), ("taps", i32),
                ("m", i32), ("n", i32), ("wt", vp), ("bias", vp), ("rowvec", vp), ("rows_per_sample", i32),
                ("rowvec_ld", i32), ("residual", vp), ("ld_res", i32), ("out_f32", vp), ("out_bf16", vp),
                ("ld_out", i32), ("geglu", i32), ("accumulate_out", i32), ("bn_override", i32), ("aux_bf16", vp),
                ("conv_pad", i32), ("gn_stats", vp), ("bm_override", i32)]


class GroupNormArgs(C.Structure):
    _fields_ = [("x0", vp), ("x1", vp), ("c0", i32), ("c1", i32), ("ld0", i32), ("ld1", i32), ("batch", i32),
                ("hw", i32), ("scale", vp), ("bias", vp), ("eps", f32), ("silu", i32), ("y_bf16", vp),
                ("y_f32", vp), ("raw_bf16", vp), ("workspace", vp), ("stats_only_skip", i32), ("stats0", vp), ("stats1", vp),
                ("dy_bf16", i32)]


class AttentionArgs(C.Structure):
    _fields_ = [("q", vp), ("k", vp), ("v", vp), ("out", vp), ("lse", vp), ("batch", i32), ("heads", i32),
                ("nq", i32), ("nk", i32), ("head_dim", i32), ("ldq", i32), ("ldk", i32), ("ldv", i32), ("ldo", i32),
                ("causal", i32)]


class WgradArgs(C.Structure):
    _fields_ = [("dy", vp), ("ldy", i32), ("n", i32), ("x0", vp), ("x1", vp), ("c0", i32), ("c1", i32),
                ("ldx0", i32), ("ldx1", i32), ("is_conv", i32), ("batch", i32), ("h", i32), ("w", i32),
                ("conv_stride", i32), ("taps", i32), ("m", i32), ("dw", vp), ("workspace", vp),
                ("workspace_floats", i64), ("bn_override", i32), ("splits_override", i32)]


class AttentionBwdArgs(C.Structure):
    _fields_ = [("q", vp), ("k", vp), ("v", vp), ("out", vp), ("dout", vp), ("lse", vp), ("delta", vp),
                ("dq", vp), ("dk", vp), ("dv", vp), ("batch", i32), ("heads", i32), ("nq", i32), ("nk", i32),
                ("head_dim", i32), ("ldq", i32), ("ldk", i32), ("ldv", i32), ("ldo", i32), ("lddo", i32),
                ("lddq", i32), ("lddk", i32), ("lddv", i32)]


# name -> (restype, argtypes).  Every symbol declared in include/ddpo_b200.h is listed here;
# tests/test_abi.py checks header <-> binding <-> .so agreement.
SIGNATURES = {
    "ddpo_last_error": (C.c_char_p, []),
    "ddpo_device_sm_count": (i32, []),
    "ddpo_abi_version": (i32, []),
    "ddpo_threefry_split_host": (i32, [vp, i32, vp]),
    "ddpo_prng_key_host": (i32, [C.c_uint64, vp]),
    "ddpo_threefry_normal": (i32, [vp, vp, i64, vp]),
    "ddpo_ddim_step_sample": (i32, [C.POINTER(DdimCommon), vp, vp, vp, vp]),
    "ddpo_ddim_logprob_fwd": (i32, [C.POINTER(DdimCommon), vp, vp, vp]),
    "ddpo_ddim_logprob_bwd": (i32, [C.POINTER(DdimCommon), vp, vp, vp, vp, vp]),
    "ddpo_ppo_loss": (i32, [vp, vp, vp, i32, i32, f32, vp, vp, vp]),
    "ddpo_igemm": (i32, [C.POINTER(IGemmArgs), vp]),
    "ddpo_igemm_plan": (i32, [i32, i32, i32, i32, i32, i32, vp]),
    "ddpo_groupnorm_workspace_floats": (i64, [i32, i32, i32]),
    "ddpo_groupnorm_fwd": (i32, [C.POINTER(GroupNormArgs), vp]),
    "ddpo_groupnorm_bwd": (i32, [C.POINTER(GroupNormArgs), vp, vp, vp, i32, i32, i32, vp, vp, vp]),
    "ddpo_layernorm_fwd": (i32, [vp, vp, vp, vp, vp, i32, i32, f32, vp]),
    "ddpo_layernorm_bwd_workspace_floats": (i64, [i32, i32]),
    "ddpo_layernorm_bwd": (i32, [vp, vp, vp, vp, vp, i32, vp, vp, vp, i32, i32, i32, vp]),
    "ddpo_prep_weight": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    "ddpo_prep_weight_dgrad": (i32, [vp, vp, i32, i32, i32, i32, i32, vp]),
    "ddpo_permute_geglu_bias": (i32, [vp, vp, i32, i32, vp]),
    "ddpo_cast_bf16": (i32, [vp, vp, i64, vp]),
    "ddpo_upsample2x_bf16": (i32, [vp, vp, i32, i32, i32, i32, vp]),
    "ddpo_upsample2x_bwd": (i32, [vp, vp, i32, i32, i32, i32, i32, vp]),
    "ddpo_vae_image_to_nchw": (i32, [vp, vp, i32, i32, i32, vp]),
    "ddpo_image_to_uint8": (i32, [vp, vp, C.c_longlong, vp]),
    "ddpo_vae_encoder_head": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ddpo_conv_in": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp]),
    "ddpo_conv_out": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]),
    "ddpo_timestep_sincos": (i32, [vp, i32, vp, i32, i32, vp]),
    "ddpo_dense_small": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]),
    "ddpo_dense_small_grouped": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ddpo_attention_fwd": (i32, [C.POINTER(AttentionArgs), vp]),
    "ddpo_wgrad_workspace_floats": (i64, [C.POINTER(WgradArgs)]),
    "ddpo_wgrad": (i32, [C.POINTER(WgradArgs), vp]),
    "ddpo_wgrad_plan": (i32, [i32, i32, i32, i32, i32, i32, i32, vp]),
    "ddpo_attention_bwd": (i32, [C.POINTER(AttentionBwdArgs), vp]),
    "ddpo_colsum_workspace_floats": (i64, [i32, i32, i32]),
    "ddpo_colsum_cast": (i32, [vp, i32, vp, vp, i32, i32, vp, i32, i32, vp]),
    "ddpo_colsum_bf16": (i32, [vp, i32, vp, i32, vp, i32, i32, vp]),
    "ddpo_geglu_bwd": (i32, [vp, vp, vp, i64, i32, i32, i32, vp]),
    "ddpo_conv_out_bwd_workspace_floats": (i64, [i32]),
    "ddpo_conv_out_bwd": (i32, [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ddpo_conv_in_wgrad_workspace_floats": (i64, [i32, i32]),
    "ddpo_conv_in_wgrad": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]),
    "ddpo_dense_small_bwd": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    "ddpo_dilate2x_bf16": (i32, [vp, vp, i32, i32, i32, i32, vp]),
    "ddpo_copy2d": (i32, [vp, i32, vp, i32, i64, i32, i32, vp]),
    "ddpo_embed_tokens": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ddpo_act_bf16": (i32, [vp, vp, i64, i32, vp]),
    "ddpo_layernorm_f32": (i32, [vp, vp, vp, vp, i32, i32, f32, vp]),
    "ddpo_patchify_bf16": (i32, [vp, vp, i32, i32, i32, i32, vp]),
    "ddpo_vit_tokens": (i32, [vp, vp, vp, vp, i32, i32, i32, vp]),
    "ddpo_l2norm_rows": (i32, [vp, vp, i32, i32, vp]),
    "ddpo_vae_post_quant": (i32, [vp, vp, vp, f32, i32, i32, i32, i32, vp, vp]),
    "ddpo_softmax_rows": (i32, [vp, i64, f32, vp, i64, i32, i32, vp]),
    "ddpo_vae_conv_out": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "ddpo_threefry_randint_host": (i32, [vp, i32, i32, i32, vp]),
    "ddpo_rwr_workspace_floats": (i64, [i32]),
    "ddpo_rwr_noisy_latents": (i32, [vp, vp, vp, vp, vp, f32, i32, i32, i32, i32, vp, vp, vp, vp]),
    "ddpo_rwr_mse_loss": (i32, [vp, vp, vp, vp, f32, i32, i32, vp, vp, vp, vp, vp, vp]),
    "ddpo_gather_rows": (i32, [vp, vp, vp, i32, i64, vp]),
    "ddpo_optim_workspace_bytes": (i64, []),
    "ddpo_grad_sumsq": (i32, [vp, i64, vp, vp, vp]),
    "ddpo_clip_adamw": (i32, [vp, vp, vp, vp, i64, vp, f32, f32, f32, f32, f32, f32, f32, i32, vp, vp]),
    "ddpo_adafactor_plan": (i32, [i32, vp, vp, vp, i64, i32, vp, i64, vp, vp]),
    "ddpo_clip_adafactor": (i32, [vp, vp, vp, i64, i64, vp, vp, vp, i64, vp, f32, f32, f32, f32, i32, vp, vp]),
    "ddpo_resample_u8": (i32, [vp, i32, i32, i32, i32, i32, i32, vp, vp, i32, vp, vp]),
    "ddpo_clip_normalize_u8": (i32, [vp, i32, i32, i32, i32, i32, i32, vp, vp]),
    "ddpo_pair_stats_u8": (i32, [vp, i32, i32, i32, i32, vp, vp]),
    "ddpo_feature_angles": (i32, [vp, i32, i32, i32, vp, vp]),
    "ddpo_scaled_cosine": (i32, [vp, vp, i32, i32, f32, vp, vp]),
    "ddpo_lora_merge": (i32, [vp, i32, i32, vp, vp, i32, f32, vp, i32, i32, vp, i32, i32, vp, vp]),
    "ddpo_lora_grad_workspace_floats": (i64, [i32, i32, i32, i32, i32]),
    "ddpo_lora_grad": (i32, [vp, i32, vp, i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, vp, i64, vp]),
}

_lib = None


class DdpoError(RuntimeError):
    pass


def lib():
    """Load (once) and return the shared library.  Fails loudly when it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DdpoError(
                f"{LIB_PATH} is missing: build it with `python -m ddpo_b200.build` "
                "(ddpo_b200 has no CPU / PyTorch fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the .so does not export it
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(status, what=""):
    if status != 0:
        msg = lib().ddpo_last_error()
        raise DdpoError(f"{what} failed with status {status}: {msg.decode() if msg else ''}")
