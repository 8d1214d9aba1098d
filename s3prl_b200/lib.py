"""ctypes binding of the C ABI declared in include/s3prl_b200.h.

PyTorch is used only as the owner of device memory and streams: every call below passes raw
``data_ptr()`` addresses and the current ``cudaStream_t`` to the shared library. There is no CPU
fallback: on a host without a CUDA device, anything that computes raises ``S3BError``.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import Optional

import os

# S3B_LIB_PATH: A/B runs of another build of the same C ABI on one box (tools/ab_step.sh); never a CPU fallback
_LIB_PATH = Path(os.environ.get("S3B_LIB_PATH") or Path(__file__).resolve().parent / "_lib" / "libs3prl_b200.so")

EXPORTED_SYMBOLS = [
    "s3b_version",
    "s3b_last_error",
    "s3b_device_count",
    "s3b_model_create",
    "s3b_model_set_tensor",
    "s3b_model_finalize",
    "s3b_model_destroy",
    "s3b_apc_model_create",
    "s3b_decoar_model_create",
    "s3b_npc_model_create",
    "s3b_cpc_model_create",
    "s3b_ssast_model_create",
    "s3b_mae_ast_model_create",
    "s3b_num_frames",
    "s3b_valid_frames",
    "s3b_num_outputs",
    "s3b_default_lanes",
    "s3b_forward",
    "s3b_forward_host",
    "s3b_forward_ex",
    "s3b_forward_host_ex",
    "s3b_wavlm_buckets",
    "s3b_peer_create",
    "s3b_peer_connect",
    "s3b_peer_slot",
    "s3b_peer_push",
    "s3b_peer_wait",
    "s3b_peer_destroy",
    "s3b_profile_enable",
    "s3b_profile_read",
    "s3b_profile_read_ex",
    "s3b_launch_count",
    "s3b_weighted_sum",
    "s3b_weighted_sum_backward",
    "s3b_linear_f32",
    "s3b_linear_ex",
    "s3b_qkv_f32",
    "s3b_qkv_hd_f32",
    "s3b_conv_gemm_f32",
    "s3b_posconv_f32",
    "s3b_layernorm_f32",
    "s3b_gemm_bench",
    "s3b_attention_f32",
    "s3b_attention_ex",
    "s3b_wavlm_gate_f32",
    "s3b_frontend_f32",
    "s3b_conformer_conv_f32",
    "s3b_decoar2_features_f32",
    "s3b_apc_features_f32",
    "s3b_fbank_cmvn_planes",
    "s3b_gru_f32",
    "s3b_gru_max_active_clusters",
    "s3b_lstm_f32",
    "s3b_lstm_fits",
    "s3b_npc_conv_f32",
    "s3b_cpc_conv_f32",
    "s3b_cpc_lstm_f32",
    "s3b_cpc_lstm_max_active_clusters",
    "s3b_layernorm_rope_f32",
    "s3b_layernorm_eps_f32",
    "s3b_layernorm_eps_planes_f32",
    "s3b_ssast_fbank_f32",
    "s3b_ssast_embed_f32",
    "s3b_ssast_fold_f32",
    "s3b_ssast_patch_planes",
    "s3b_mae_ast_fbank_f32",
    "s3b_mae_ast_fbank_planes",
    "s3b_mae_ast_embed_f32",
    "s3b_fbank",
    "s3b_fbank_ex",
    "s3b_fbank_num_frames",
    "s3b_trimmed_lengths",
    "s3b_melspec",
    "s3b_melspec_ex",
]


class S3BError(RuntimeError):
    pass


class S3BConfig(C.Structure):
    """Mirror of ``struct s3b_config``."""

    _fields_ = [
        ("family", C.c_int32),
        ("extractor_layer_norm", C.c_int32),
        ("conv_bias", C.c_int32),
        ("layer_norm_first", C.c_int32),
        ("normalize_wav", C.c_int32),
        ("num_layers", C.c_int32),
        ("embed_dim", C.c_int32),
        ("ffn_dim", C.c_int32),
        ("num_heads", C.c_int32),
        ("pos_conv_kernel", C.c_int32),
        ("pos_conv_groups", C.c_int32),
        ("relative_position", C.c_int32),
        ("num_buckets", C.c_int32),
        ("max_distance", C.c_int32),
        ("gru_rel_pos", C.c_int32),
        ("no_feature_layer_norm", C.c_int32),
        ("pred_heads", C.c_int32),
        ("pos_conv_depth", C.c_int32),
        ("conformer", C.c_int32),
        ("depthwise_kernel", C.c_int32),
        ("frontend", C.c_int32),
        ("reserved", C.c_int32 * 2),
    ]

    # the header's `proj_hidden0` is the first of the two ints this mirror has always named `reserved`
    @property
    def proj_hidden0(self) -> int:
        return self.reserved[0]

    @proj_hidden0.setter
    def proj_hidden0(self, v: int) -> None:
        self.reserved[0] = v


class S3BApcConfig(C.Structure):
    """Mirror of ``struct s3b_apc_config``."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("num_layers", C.c_int32),
        ("hidden", C.c_int32),
        ("residual", C.c_int32),
        ("reserved", C.c_int32 * 4),
    ]

    def __init__(self, **kw):
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BApcConfig)


class S3BDecoarConfig(C.Structure):
    """Mirror of ``struct s3b_decoar_config``."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("num_layers", C.c_int32),
        ("hidden", C.c_int32),
        ("all_layers", C.c_int32),
        ("reserved", C.c_int32 * 4),
    ]

    def __init__(self, **kw):
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BDecoarConfig)


class S3BNpcConfig(C.Structure):
    """Mirror of ``struct s3b_npc_config`` (act: 0 = relu, 1 = tanh)."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("n_blocks", C.c_int32),
        ("hidden", C.c_int32),
        ("kernel_size", C.c_int32),
        ("mask_size", C.c_int32),
        ("residual", C.c_int32),
        ("batch_norm", C.c_int32),
        ("act", C.c_int32),
        ("reserved", C.c_int32 * 4),
    ]

    def __init__(self, **kw):
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BNpcConfig)


class S3BCpcConfig(C.Structure):
    """Mirror of ``struct s3b_cpc_config``."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("hidden", C.c_int32),
        ("num_layers", C.c_int32),
        ("reserved", C.c_int32 * 4),
    ]

    def __init__(self, **kw):
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BCpcConfig)


class S3BSsastConfig(C.Structure):
    """Mirror of ``struct s3b_ssast_config``."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("patch", C.c_int32),
        ("window_samples", C.c_int32),
        ("embed_dim", C.c_int32),
        ("num_heads", C.c_int32),
        ("num_layers", C.c_int32),
        ("reserved", C.c_int32 * 4),
    ]

    def __init__(self, **kw):
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BSsastConfig)


class S3BMaeAstConfig(C.Structure):
    """Mirror of ``struct s3b_mae_ast_config``."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("patch", C.c_int32),
        ("embed_dim", C.c_int32),
        ("num_heads", C.c_int32),
        ("ffn_dim", C.c_int32),
        ("num_layers", C.c_int32),
        ("layer_norm_first", C.c_int32),
        ("sine_pos", C.c_int32),
        ("max_tokens", C.c_int32),
        ("reserved", C.c_int32 * 4),
    ]

    def __init__(self, **kw):
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BMaeAstConfig)


class S3BForwardOpts(C.Structure):
    """Mirror of ``struct s3b_forward_opts``."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("lanes", C.c_int32),
        ("layer_stride", C.c_int64),
        ("ffn_out", C.c_void_p),
        ("ffn_layer_stride", C.c_int64),
        ("last_residual", C.c_void_p),
        ("reserved", C.c_int64 * 4),
    ]

    def __init__(self, **kw):
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BForwardOpts)


class S3BAttentionOpts(C.Structure):
    """Mirror of ``struct s3b_attention_opts``."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("ctx_format", C.c_int32),
        ("rel_emb", C.c_void_p),
        ("num_buckets", C.c_int32),
        ("max_distance", C.c_int32),
        ("gate", C.c_void_p),
        ("table_frames", C.c_int32),
        ("head_dim", C.c_int32),
        ("reserved", C.c_int64 * 2),
    ]

    def __init__(self, **kw):
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BAttentionOpts)


class S3BLinearOpts(C.Structure):
    """Mirror of ``struct s3b_linear_opts`` (scheme and out_fmt default to -1: the library's scheme, fp32 output)."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("scheme", C.c_int32),
        ("tile_n", C.c_int32),
        ("out_fmt", C.c_int32),
        ("row_mask", C.c_void_p),
        ("out_pre", C.c_void_p),
        ("lda", C.c_int64),
        ("a_off", C.c_int64),
        ("scheme_used", C.c_int32),
        ("tile_n_used", C.c_int32),
        ("reserved", C.c_int64 * 2),
    ]

    def __init__(self, **kw):
        kw.setdefault("scheme", -1)
        kw.setdefault("out_fmt", -1)
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BLinearOpts)


class S3BSpectralOpts(C.Structure):
    """Mirror of ``struct s3b_spectral_opts`` (cmvn defaults to 1, as s3b_fbank / s3b_melspec)."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("cmvn", C.c_int32),
        ("reserved", C.c_int64 * 3),
    ]

    def __init__(self, **kw):
        kw.setdefault("cmvn", 1)
        super().__init__(**kw)
        self.struct_size = C.sizeof(S3BSpectralOpts)


FAMILY_HUBERT, FAMILY_WAV2VEC2, FAMILY_WAVLM, FAMILY_DISTILLER = 0, 1, 2, 3
FRONTEND_CONV, FRONTEND_DECOAR2 = 0, 1

_lib: Optional[C.CDLL] = None


def lib_path() -> Path:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load the shared library (building is `__graft_entry__.build()` / `python -m s3prl_b200.build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise S3BError(
            f"{_LIB_PATH} is missing: build it with `python s3prl_b200/build.py` (needs nvcc). "
            "s3prl_b200 has no CPU fallback."
        )
    lib = C.CDLL(str(_LIB_PATH))
    vp, i32, i64, f32p = C.c_void_p, C.c_int32, C.c_int64, C.c_void_p
    lib.s3b_version.restype = C.c_int
    lib.s3b_last_error.restype = C.c_char_p
    lib.s3b_device_count.restype = C.c_int
    lib.s3b_model_create.argtypes = [C.POINTER(S3BConfig), C.POINTER(vp)]
    lib.s3b_model_set_tensor.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32]
    lib.s3b_apc_model_create.argtypes = [C.POINTER(S3BApcConfig), C.POINTER(vp)]
    lib.s3b_decoar_model_create.argtypes = [C.POINTER(S3BDecoarConfig), C.POINTER(vp)]
    lib.s3b_npc_model_create.argtypes = [C.POINTER(S3BNpcConfig), C.POINTER(vp)]
    lib.s3b_cpc_model_create.argtypes = [C.POINTER(S3BCpcConfig), C.POINTER(vp)]
    lib.s3b_ssast_model_create.argtypes = [C.POINTER(S3BSsastConfig), C.POINTER(vp)]
    lib.s3b_mae_ast_model_create.argtypes = [C.POINTER(S3BMaeAstConfig), C.POINTER(vp)]
    lib.s3b_model_finalize.argtypes = [vp]
    lib.s3b_model_destroy.argtypes = [vp]
    lib.s3b_model_destroy.restype = None
    lib.s3b_num_frames.argtypes = [vp, i64]
    lib.s3b_num_frames.restype = i64
    lib.s3b_num_outputs.argtypes = [vp]
    lib.s3b_num_outputs.restype = i32
    lib.s3b_default_lanes.argtypes = [vp, i32, i64]
    lib.s3b_default_lanes.restype = i32
    lib.s3b_valid_frames.argtypes = [vp, C.POINTER(i64), i32, i64, C.POINTER(i32)]
    lib.s3b_forward.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i64, f32p, vp]
    lib.s3b_forward_host.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i64, f32p]
    lib.s3b_forward_ex.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i64, f32p, vp, C.POINTER(S3BForwardOpts)]
    lib.s3b_forward_host_ex.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i64, f32p, f32p]
    lib.s3b_wavlm_buckets.argtypes = [i32, i32, C.POINTER(i32), i32, C.POINTER(i32)]
    lib.s3b_peer_create.argtypes = [i32, i32, i64, i32, C.POINTER(vp), vp]
    lib.s3b_peer_connect.argtypes = [vp, vp]
    lib.s3b_peer_slot.argtypes = [vp, C.c_uint32]
    lib.s3b_peer_slot.restype = vp
    lib.s3b_peer_push.argtypes = [vp, f32p, i32, i64, f32p, C.c_uint32, vp]
    lib.s3b_peer_wait.argtypes = [vp, C.c_uint32, vp]
    lib.s3b_peer_destroy.argtypes = [vp]
    lib.s3b_peer_destroy.restype = None
    lib.s3b_profile_enable.argtypes = [vp, i32]
    lib.s3b_profile_read.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(i64), i32]
    lib.s3b_profile_read_ex.argtypes = [vp, i32, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(i64), i32]
    lib.s3b_launch_count.argtypes = [vp]
    lib.s3b_launch_count.restype = i64
    lib.s3b_weighted_sum.argtypes = [f32p, i32, i64, f32p, f32p, vp]
    lib.s3b_weighted_sum_backward.argtypes = [f32p, i32, i64, f32p, f32p, vp]
    lib.s3b_linear_f32.argtypes = [f32p, f32p, f32p, f32p, i64, i32, i32, i32, f32p, vp]
    lib.s3b_linear_ex.argtypes = [f32p, f32p, f32p, f32p, i64, i32, i32, i32, C.POINTER(S3BLinearOpts), f32p, vp]
    lib.s3b_qkv_f32.argtypes = [f32p, f32p, f32p, i32, i32, i32, i32, f32p, f32p, f32p, vp]
    lib.s3b_qkv_hd_f32.argtypes = [f32p, f32p, f32p, i32, i32, i32, i32, i32, f32p, f32p, f32p, vp]
    lib.s3b_conv_gemm_f32.argtypes = [f32p, f32p, f32p, i32, i64, i32, i32, i32, i32, f32p, vp]
    lib.s3b_posconv_f32.argtypes = [f32p, f32p, f32p, i32, i32, i32, i32, i32, i32, i32, f32p, f32p, i32, f32p, vp]
    lib.s3b_gemm_bench.argtypes = [i64, i32, i32, i32, i32, i32, C.POINTER(C.c_float)]
    lib.s3b_layernorm_f32.argtypes = [f32p, i64, i32, f32p, f32p, i32, f32p, vp]
    lib.s3b_attention_f32.argtypes = [f32p, f32p, f32p, C.POINTER(i32), i32, i32, i32, f32p, vp]
    lib.s3b_attention_ex.argtypes = [f32p, f32p, f32p, C.POINTER(i32), i32, i32, i32, C.POINTER(S3BAttentionOpts),
                                     f32p, vp]
    lib.s3b_wavlm_gate_f32.argtypes = [f32p, i32, i32, i32, f32p, f32p, f32p, i32, f32p, vp]
    lib.s3b_frontend_f32.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, i64, i32, f32p, f32p, f32p, f32p, i32, i32,
                                     f32p, f32p, vp]
    lib.s3b_conformer_conv_f32.argtypes = [f32p, i32, i32, i32, i32, f32p, f32p, f32p, f32p, f32p, i32, f32p, vp]
    lib.s3b_decoar2_features_f32.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, i32, f32p, vp]
    lib.s3b_apc_features_f32.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, i32, f32p, vp]
    lib.s3b_fbank_cmvn_planes.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, i32, i32, f32p, vp, vp]
    lib.s3b_gru_max_active_clusters.argtypes = [C.POINTER(i32)]
    lib.s3b_gru_f32.argtypes = [f32p, f32p, f32p, f32p, C.POINTER(i32), i32, i32, i32, i32, f32p, f32p, vp]
    lib.s3b_lstm_fits.argtypes = [C.POINTER(i32)]
    lib.s3b_cpc_conv_f32.argtypes = [f32p, i32, i32, i32, f32p, f32p, f32p, f32p, i32, f32p, vp]
    lib.s3b_cpc_lstm_f32.argtypes = [f32p, f32p, i32, i32, i32, f32p, f32p, vp]
    lib.s3b_cpc_lstm_max_active_clusters.argtypes = [C.POINTER(i32)]
    lib.s3b_npc_conv_f32.argtypes = [f32p, i32, i32, i32, f32p, i32, i32, f32p, f32p, i32, i32, i32, f32p, f32p, vp]
    lib.s3b_lstm_f32.argtypes = [f32p, f32p, f32p, C.POINTER(i32), i32, i32, i32, i32, f32p, f32p, vp]
    lib.s3b_layernorm_rope_f32.argtypes = [f32p, i64, i32, i32, f32p, f32p, C.POINTER(C.c_float), i32, f32p, f32p, vp]
    lib.s3b_layernorm_eps_f32.argtypes = [f32p, i64, i32, f32p, f32p, i32, C.c_float, f32p, vp]
    lib.s3b_layernorm_eps_planes_f32.argtypes = [f32p, i64, i32, f32p, f32p, C.c_float, i32, f32p, vp]
    lib.s3b_ssast_fbank_f32.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, i64, i32, f32p, vp]
    lib.s3b_ssast_embed_f32.argtypes = [f32p, i32, i32, i32, f32p, f32p, f32p, f32p, f32p, i32, f32p, f32p, vp]
    lib.s3b_ssast_fold_f32.argtypes = [f32p, i32, i32, i32, i32, i32, f32p, vp]
    lib.s3b_ssast_patch_planes.argtypes = [f32p, i32, i32, i32, i32, vp, vp]
    lib.s3b_mae_ast_fbank_f32.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, i64, i32, C.c_float, C.c_float, i32, f32p,
                                          f32p, vp]
    lib.s3b_mae_ast_fbank_planes.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, i64, i32, C.c_float, C.c_float, i32,
                                             vp, vp]
    lib.s3b_mae_ast_embed_f32.argtypes = [f32p, i32, i32, C.POINTER(i32), f32p, f32p, f32p, i32, f32p, vp]
    lib.s3b_fbank_num_frames.argtypes = [i64]
    lib.s3b_fbank_num_frames.restype = i64
    lib.s3b_fbank.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, f32p, vp]
    lib.s3b_fbank_ex.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, C.POINTER(S3BSpectralOpts), f32p, vp]
    lib.s3b_trimmed_lengths.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, C.POINTER(i64)]
    lib.s3b_melspec.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, i64, i32, C.POINTER(i32), C.POINTER(i32), i32, f32p, vp]
    lib.s3b_melspec_ex.argtypes = [C.POINTER(vp), C.POINTER(i64), i32, i64, i32, C.POINTER(i32), C.POINTER(i32), i32,
                                   C.POINTER(S3BSpectralOpts), f32p, vp]
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != 0:
        msg = load().s3b_last_error()
        raise S3BError(msg.decode() if msg else f"s3prl_b200 call failed with status {status}")


def require_gpu() -> None:
    if load().s3b_device_count() < 1:
        raise S3BError("no CUDA device visible: s3prl_b200 has no CPU fallback")


def current_stream_ptr() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream
