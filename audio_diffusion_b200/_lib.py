"""ctypes binding of libb200ad.so (C ABI declared in include/b200ad.h).

The product path has no CPU fallback: if the shared library is missing, or a compute call is made
without a CUDA device, this module raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200AD_LIB: development override used for kernel A/B builds (csrc/Makefile EXTRA=...); the product loads libb200ad.so
LIB_PATH = os.environ.get("B200AD_LIB") or os.path.join(_HERE, "libb200ad.so")

MAX_BLOCKS = 8


class UNetConfigC(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int), ("out_channels", C.c_int), ("layers_per_block", C.c_int), ("num_blocks", C.c_int),
        ("block_out_channels", C.c_int * MAX_BLOCKS), ("down_attn", C.c_int * MAX_BLOCKS),
        ("up_attn", C.c_int * MAX_BLOCKS), ("norm_num_groups", C.c_int), ("norm_eps", C.c_float),
        ("attention_head_dim", C.c_int), ("cross_attention_dim", C.c_int), ("down_cross", C.c_int * MAX_BLOCKS),
        ("up_cross", C.c_int * MAX_BLOCKS),
    ]


class VAEConfigC(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int), ("out_channels", C.c_int), ("latent_channels", C.c_int), ("layers_per_block", C.c_int),
        ("num_blocks", C.c_int), ("block_out_channels", C.c_int * MAX_BLOCKS), ("norm_num_groups", C.c_int),
        ("norm_eps", C.c_float),
    ]


class OptimHParamsC(C.Structure):
    _fields_ = [("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("weight_decay", C.c_float), ("max_grad_norm", C.c_float), ("ema_decay", C.c_float), ("step", C.c_int)]


class StepCoefC(C.Structure):
    _fields_ = [("sqrt_1m_at", C.c_float), ("inv_sqrt_at", C.c_float), ("clip", C.c_float), ("c_x0", C.c_float),
                ("c_xt", C.c_float), ("c_eps", C.c_float), ("c_z", C.c_float), ("do_clip", C.c_int)]


class MultistepCoefC(C.Structure):
    """b200ad_multistep_coef: a step's coefficients plus those of the two earlier data predictions (history buffers)."""
    _fields_ = [("step", StepCoefC), ("c_h1", C.c_float), ("c_h2", C.c_float)]


class MelConfigC(C.Structure):
    _fields_ = [("x_res", C.c_int), ("y_res", C.c_int), ("sample_rate", C.c_int), ("n_fft", C.c_int),
                ("hop_length", C.c_int), ("top_db", C.c_int), ("n_iter", C.c_int)]


# every symbol include/b200ad.h declares: name -> (restype, argtypes)
_VP, _SZ, _I = C.c_void_p, C.c_size_t, C.c_int
SYMBOLS = {
    "b200ad_last_error": (C.c_char_p, []),
    "b200ad_version": (_I, []),
    "b200ad_unet_create": (_I, [C.POINTER(UNetConfigC), C.POINTER(_VP)]),
    "b200ad_unet_destroy": (None, [_VP]),
    "b200ad_unet_num_params": (_I, [_VP]),
    "b200ad_unet_param_name": (C.c_char_p, [_VP, _I]),
    "b200ad_unet_param_shape": (_I, [_VP, _I, C.POINTER(C.c_int64)]),
    "b200ad_unet_packed_bytes": (_SZ, [_VP]),
    "b200ad_unet_workspace_bytes": (_SZ, [_VP, _I, _I, _I]),
    "b200ad_unet_set_params": (_I, [_VP, C.POINTER(_VP), _VP, _SZ, _VP]),
    "b200ad_unet_bind_workspace": (_I, [_VP, _VP, _SZ, _I, _I, _I, _VP]),
    "b200ad_unet_forward": (_I, [_VP, _VP, _VP, _VP, _VP]),
    "b200ad_unet_set_encoding": (_I, [_VP, _VP, _I]),
    "b200ad_unet_set_encoder_len": (_I, [_VP, _I]),
    "b200ad_unet_forward_step": (_I, [_VP, _VP, _VP, _VP, C.POINTER(StepCoefC), _VP, _VP, _VP]),
    "b200ad_unet_forward_step_dev": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "b200ad_step_scalars_upload": (_I, [C.POINTER(StepCoefC), C.c_float, _VP, _VP, C.c_int, _VP]),
    "b200ad_unet_forward_multistep": (_I, [_VP, _VP, _VP, _VP, C.POINTER(MultistepCoefC), _VP, _VP, _VP, _VP, _VP]),
    "b200ad_unet_forward_multistep_dev": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "b200ad_multistep_scalars_upload": (_I, [C.POINTER(MultistepCoefC), C.c_float, _VP, _VP, C.c_int, _VP]),
    "b200ad_unet_profile_step": (_I, [_VP, _VP, _VP, _VP, C.POINTER(StepCoefC), _VP, C.POINTER(C.c_float),
                                      C.POINTER(_I), C.POINTER(C.c_double), _I, _VP]),
    "b200ad_unet_debug_tensor": (_I, [_VP, C.c_char_p, _VP, C.POINTER(_I), _VP]),
    "b200ad_unet_last_launch_count": (_I, [_VP]),
    "b200ad_unet_conv_plan": (_I, [_VP, _I, _I, _I, _I, C.POINTER(_I), _I]),
    "b200ad_unet_set_training": (_I, [_VP, _I]),
    "b200ad_unet_set_checkpointing": (_I, [_VP, _I]),
    "b200ad_unet_set_param_grads": (_I, [_VP, _I]),
    "b200ad_unet_training_bytes": (_SZ, [_VP, _I, _I, _I, _I]),
    "b200ad_unet_grad_floats": (_SZ, [_VP]),
    "b200ad_unet_grad_offset": (_SZ, [_VP, _I]),
    "b200ad_unet_backward_bytes": (_SZ, [_VP]),
    "b200ad_unet_bind_backward": (_I, [_VP, _VP, _SZ, _VP, _VP]),
    "b200ad_unet_backward": (_I, [_VP, _VP, _VP, _I, _VP]),
    "b200ad_unet_backward_input": (_I, [_VP, _VP, _VP, _VP, _I, _VP]),
    "b200ad_unet_backward_launch_count": (_I, [_VP]),
    "b200ad_unet_debug_grad": (_I, [_VP, C.c_char_p, _I, _VP, C.POINTER(_I), _VP]),
    "b200ad_vae_set_training": (_I, [_VP, _I]),
    "b200ad_vae_set_checkpointing": (_I, [_VP, _I]),
    "b200ad_vae_set_param_grads": (_I, [_VP, _I]),
    "b200ad_vae_training_bytes": (_SZ, [_VP, _I, _I, _I]),
    "b200ad_vae_grad_floats": (_SZ, [_VP]),
    "b200ad_vae_grad_offset": (_SZ, [_VP, _I]),
    "b200ad_vae_backward_bytes": (_SZ, [_VP]),
    "b200ad_vae_bind_backward": (_I, [_VP, _VP, _SZ, _VP, _VP]),
    "b200ad_vae_decoder_backward": (_I, [_VP, _VP, _VP, _I, _VP]),
    "b200ad_vae_encoder_backward": (_I, [_VP, _VP, _VP, _I, _VP]),
    "b200ad_vae_encoder_backward_input": (_I, [_VP, _VP, _VP, _VP, _I, _VP]),
    "b200ad_vae_backward_launch_count": (_I, [_VP]),
    "b200ad_vae_debug_grad": (_I, [_VP, C.c_char_p, _I, _VP, C.POINTER(_I), _VP]),
    "b200ad_vae_create": (_I, [C.POINTER(VAEConfigC), C.POINTER(_VP)]),
    "b200ad_vae_destroy": (None, [_VP]),
    "b200ad_vae_num_params": (_I, [_VP]),
    "b200ad_vae_param_name": (C.c_char_p, [_VP, _I]),
    "b200ad_vae_param_shape": (_I, [_VP, _I, C.POINTER(C.c_int64)]),
    "b200ad_vae_packed_bytes": (_SZ, [_VP]),
    "b200ad_vae_workspace_bytes": (_SZ, [_VP, _I, _I, _I]),
    "b200ad_vae_set_params": (_I, [_VP, C.POINTER(_VP), _VP, _SZ, _VP]),
    "b200ad_vae_bind_workspace": (_I, [_VP, _VP, _SZ, _I, _I, _I, _VP]),
    "b200ad_vae_encode": (_I, [_VP, _VP, _VP, _VP, _VP, _VP]),
    "b200ad_vae_decode": (_I, [_VP, _VP, _VP, _VP]),
    "b200ad_vae_debug_tensor": (_I, [_VP, C.c_char_p, _VP, C.POINTER(_I), _VP]),
    "b200ad_vae_last_launch_count": (_I, [_VP]),
    "b200ad_optim_create": (_I, [_I, C.POINTER(C.c_int64), C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP),
                                C.POINTER(_VP), C.POINTER(_VP)]),
    "b200ad_optim_destroy": (None, [_VP]),
    "b200ad_optim_step": (_I, [_VP, C.POINTER(_VP), C.POINTER(OptimHParamsC), _VP, _VP]),
    "b200ad_mse_loss_grad": (_I, [_VP, _VP, _SZ, _VP, _VP, _VP, _VP]),
    "b200ad_conv2d_scratch_bytes": (_SZ, [_I] * 7),
    "b200ad_conv2d": (_I, [_VP] * 7 + [_I] * 7 + [_VP, _SZ, _VP]),
    "b200ad_conv2d_dgrad": (_I, [_VP, _VP, _VP] + [_I] * 6 + [_VP, _SZ, _VP]),
    "b200ad_conv2d_wgrad_scratch_bytes": (_SZ, [_I] * 5),
    "b200ad_conv2d_wgrad": (_I, [_VP, _VP, _VP] + [_I] * 6 + [_VP, _SZ, _VP]),
    "b200ad_gn_conv2d": (_I, [_VP, _VP, _VP, _I, C.c_float, _I, _VP, _VP, _VP] + [_I] * 6 + [_VP, _SZ, _VP]),
    "b200ad_group_norm": (_I, [_VP] * 4 + [_I] * 5 + [C.c_float, _I, _VP, _SZ, _VP]),
    "b200ad_mha_scratch_bytes": (_SZ, [_I] * 5),
    "b200ad_mha_forward_backward": (_I, [_VP] * 8 + [_I] * 5 + [_VP, _SZ, _VP]),
    "b200ad_xattn_scratch_bytes": (_SZ, [_I] * 6),
    "b200ad_xattn_forward_backward": (_I, [_VP] * 8 + [_I] * 6 + [_VP, _SZ, _VP]),
    "b200ad_mel_scratch_bytes": (_SZ, [C.POINTER(MelConfigC), _I]),
    "b200ad_mel_encode": (_I, [C.POINTER(MelConfigC), _VP, _VP, _VP, _I, _VP, _SZ, _VP]),
    "b200ad_mel_encode_ref": (_I, [C.POINTER(MelConfigC), _VP, _VP, _VP, _I, _VP, _VP, _VP, _SZ, _VP]),
    "b200ad_mel_decode": (_I, [C.POINTER(MelConfigC), _VP, _VP, _VP, _I, C.c_uint64, _VP, _SZ, _VP]),
    "b200ad_sample_to_u8": (_I, [_VP, _VP, _SZ, _VP]),
}

_lib = None


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback for the audio_diffusion_b200 hot path)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


class B200ADError(RuntimeError):
    pass


def check(status: int) -> None:
    if status != 0:
        raise B200ADError(lib().b200ad_last_error().decode())


def require_cuda():
    import torch

    if not torch.cuda.is_available():
        raise B200ADError("audio_diffusion_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")


def stream_ptr():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
