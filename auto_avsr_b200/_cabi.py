"""ctypes binding of libavsr_b200.so (include/avsr_b200.h).  No torch types cross this boundary:
only raw device pointers, ints and sizes.  Importing this module without the built library raises --
there is no CPU or PyTorch fallback for the hot path."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
#: AVSR_B200_LIB selects another build of the SAME library (e.g. the phase-trace build of scripts/build_trace.py);
#: it is still this C ABI and still CUDA-only -- there is no alternative implementation to point it at.
LIB_PATH = os.environ.get("AVSR_B200_LIB") or os.path.join(_HERE, "csrc", "libavsr_b200.so")

OK, E_INVALID, E_CUDA, E_WORKSPACE = 0, 1, 2, 3
PREC_FP32, PREC_TF32, PREC_F16, PREC_BF16 = 0, 1, 2, 16
ABI_VERSION = 12


class AvsrError(RuntimeError):
    pass


class EncoderConfig(C.Structure):
    _fields_ = [("d_model", C.c_int32), ("n_heads", C.c_int32), ("linear_units", C.c_int32),
                ("num_blocks", C.c_int32), ("cnn_kernel", C.c_int32)]


#: field order of AvsrLayerParams (include/avsr_b200.h) -> reference state-dict key suffix
LAYER_FIELDS = [
    ("ffm_w1", "feed_forward_macaron.w_1.weight"), ("ffm_b1", "feed_forward_macaron.w_1.bias"),
    ("ffm_w2", "feed_forward_macaron.w_2.weight"), ("ffm_b2", "feed_forward_macaron.w_2.bias"),
    ("norm_ffm_w", "norm_ff_macaron.weight"), ("norm_ffm_b", "norm_ff_macaron.bias"),
    ("q_w", "self_attn.linear_q.weight"), ("q_b", "self_attn.linear_q.bias"),
    ("k_w", "self_attn.linear_k.weight"), ("k_b", "self_attn.linear_k.bias"),
    ("v_w", "self_attn.linear_v.weight"), ("v_b", "self_attn.linear_v.bias"),
    ("out_w", "self_attn.linear_out.weight"), ("out_b", "self_attn.linear_out.bias"),
    ("pos_w", "self_attn.linear_pos.weight"),
    ("pos_bias_u", "self_attn.pos_bias_u"), ("pos_bias_v", "self_attn.pos_bias_v"),
    ("norm_mha_w", "norm_mha.weight"), ("norm_mha_b", "norm_mha.bias"),
    ("pw1_w", "conv_module.pointwise_cov1.weight"), ("pw1_b", "conv_module.pointwise_cov1.bias"),
    ("dw_w", "conv_module.depthwise_conv.weight"), ("dw_b", "conv_module.depthwise_conv.bias"),
    ("bn_w", "conv_module.norm.weight"), ("bn_b", "conv_module.norm.bias"),
    ("bn_mean", "conv_module.norm.running_mean"), ("bn_var", "conv_module.norm.running_var"),
    ("pw2_w", "conv_module.pointwise_cov2.weight"), ("pw2_b", "conv_module.pointwise_cov2.bias"),
    ("norm_conv_w", "norm_conv.weight"), ("norm_conv_b", "norm_conv.bias"),
    ("ff_w1", "feed_forward.w_1.weight"), ("ff_b1", "feed_forward.w_1.bias"),
    ("ff_w2", "feed_forward.w_2.weight"), ("ff_b2", "feed_forward.w_2.bias"),
    ("norm_ff_w", "norm_ff.weight"), ("norm_ff_b", "norm_ff.bias"),
    ("norm_final_w", "norm_final.weight"), ("norm_final_b", "norm_final.bias"),
]


class LayerParams(C.Structure):
    _fields_ = [(name, C.c_void_p) for name, _ in LAYER_FIELDS]


class DecoderConfig(C.Structure):
    _fields_ = [("d_model", C.c_int32), ("n_heads", C.c_int32), ("linear_units", C.c_int32),
                ("num_blocks", C.c_int32), ("odim", C.c_int32)]


#: field order of AvsrDecoderLayerParams (include/avsr_b200.h) -> reference state-dict key suffix
DECODER_LAYER_FIELDS = [
    ("self_q_w", "self_attn.linear_q.weight"), ("self_q_b", "self_attn.linear_q.bias"),
    ("self_k_w", "self_attn.linear_k.weight"), ("self_k_b", "self_attn.linear_k.bias"),
    ("self_v_w", "self_attn.linear_v.weight"), ("self_v_b", "self_attn.linear_v.bias"),
    ("self_out_w", "self_attn.linear_out.weight"), ("self_out_b", "self_attn.linear_out.bias"),
    ("src_q_w", "src_attn.linear_q.weight"), ("src_q_b", "src_attn.linear_q.bias"),
    ("src_k_w", "src_attn.linear_k.weight"), ("src_k_b", "src_attn.linear_k.bias"),
    ("src_v_w", "src_attn.linear_v.weight"), ("src_v_b", "src_attn.linear_v.bias"),
    ("src_out_w", "src_attn.linear_out.weight"), ("src_out_b", "src_attn.linear_out.bias"),
    ("ff_w1", "feed_forward.w_1.weight"), ("ff_b1", "feed_forward.w_1.bias"),
    ("ff_w2", "feed_forward.w_2.weight"), ("ff_b2", "feed_forward.w_2.bias"),
    ("norm1_w", "norm1.weight"), ("norm1_b", "norm1.bias"),
    ("norm2_w", "norm2.weight"), ("norm2_b", "norm2.bias"),
    ("norm3_w", "norm3.weight"), ("norm3_b", "norm3.bias"),
]


class DecoderLayerParams(C.Structure):
    _fields_ = [(name, C.c_void_p) for name, _ in DECODER_LAYER_FIELDS]


FRONTEND_VIDEO, FRONTEND_AUDIO = 0, 1
FRONTEND_CONVS = 20
FRONTEND_TAPS = 10
#: avsr_linear_operands_split: fp32 partial planes of rows x n, and int tile counters, the caller provides
SPLIT_PLANES = 8
SPLIT_COUNTERS = 4096


class ConvBnParams(C.Structure):
    _fields_ = [("conv_w", C.c_void_p), ("bn_w", C.c_void_p), ("bn_b", C.c_void_p), ("bn_mean", C.c_void_p),
                ("bn_var", C.c_void_p), ("eps", C.c_double)]


#: every symbol include/avsr_b200.h declares: name -> (restype, argtypes)
_P, _I, _Z, _F = C.c_void_p, C.c_int, C.c_size_t, C.c_float
_CFG = C.POINTER(EncoderConfig)
_DCFG = C.POINTER(DecoderConfig)
SIGNATURES = {
    "avsr_abi_version": (_I, []),
    "avsr_last_error": (C.c_char_p, []),
    "avsr_launch_count": (C.c_uint64, []),
    "avsr_prepared_bytes": (_Z, [_CFG]),
    "avsr_prepare_weights": (_I, [_CFG, C.POINTER(LayerParams), _P, _P, _P, _Z, _I, _P]),
    "avsr_workspace_bytes": (_Z, [_CFG, _I, _I]),
    "avsr_encoder_forward": (_I, [_CFG, _P, _P, _P, _I, _I, _P, _P, _Z, _I, _P]),
    "avsr_encoder_forward_checked": (_I, [_CFG, _P, _P, _P, _I, _I, _P, _P, _Z, _I, _P, _P]),
    "avsr_encoder_forward_taps": (_I, [_CFG, _P, _P, _P, _I, _I, _P, _P, _P, _Z, _I, _P]),
    "avsr_plan_create": (_I, [_CFG, _P, _I, _I, _P, _Z, _I, _P, C.POINTER(_P)]),
    "avsr_plan_forward": (_I, [_P, _P, _P, _P, _P]),
    "avsr_plan_destroy": (None, [_P]),
    "avsr_layernorm": (_I, [_P, _P, _P, _P, _I, _I, _P]),
    "avsr_linear_workspace_bytes": (_Z, [_I, _I, _I, _I]),
    "avsr_linear": (_I, [_P, _P, _P, _P, _F, _I, _P, _I, _I, _I, _I, _P, _Z, _P]),
    "avsr_linear_operands": (_I, [_P, _P, _P, _P, _F, _P, _I, _I, _I, _I, _I, _I, _P]),
    "avsr_linear_operands_split": (_I, [_P, _P, _P, _P, _F, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "avsr_attention_workspace_bytes": (_Z, [_I, _I, _I]),
    "avsr_relpos_attention": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _Z, _I, _P]),
    "avsr_dwconv_bn_silu": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _P]),
    "avsr_pointwise_glu_workspace_bytes": (_Z, [_I, _I]),
    "avsr_pointwise_glu": (_I, [_P, _P, _P, _P, _I, _I, _P, _Z, _I, _P]),
    "avsr_rel_sinusoid_table": (_I, [_P, _I, _I, _P]),
    "avsr_log_softmax": (_I, [_P, C.c_long, _P, C.c_long, _P, _I, _I, _P]),
    "avsr_train_workspace_bytes": (_Z, [_I, _I, _I]),
    "avsr_layernorm_bwd": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _P, _Z, _P]),
    "avsr_colsum": (_I, [_P, _P, _I, _I, _P, _Z, _P]),
    "avsr_relu_bwd": (_I, [_P, _P, _P, C.c_long, _P]),
    "avsr_pack_operand": (_I, [_P, _P, _I, _I, C.c_long, _I, _I, _P]),
    "avsr_linear_bwd_workspace_bytes": (_Z, [_I, _I, _I, _I]),
    "avsr_linear_bwd": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _P]),
    "avsr_glu_fwd": (_I, [_P, _P, C.c_long, _I, _P]),
    "avsr_glu_bwd": (_I, [_P, _P, _P, C.c_long, _I, _P]),
    "avsr_dwconv_raw": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _Z, _P]),
    "avsr_dwconv_wgrad": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _P]),
    "avsr_bn_train_workspace_bytes": (_Z, [C.c_long, _I]),
    "avsr_bn_train_stats": (_I, [_P, C.c_long, _I, _P, _P, _Z, _P]),
    "avsr_bn_train_finalize": (_I, [_P, _I, _I, C.c_double, C.c_double, _P, _P, _P, _P, _P]),
    "avsr_bn_train_act_fwd": (_I, [_P, _P, _P, _P, _P, _P, _I, _P, C.c_long, _I, _P]),
    "avsr_bn_train_bwd_sums": (_I, [_P] * 7 + [_I, _P, C.c_long, _I, _P, _Z, _P]),
    "avsr_bn_train_bwd_dx": (_I, [_P] * 7 + [_I, _P, _F, _P, _P, C.c_long, _I, _P]),
    "avsr_relpos_attention_bwd_workspace_bytes": (_Z, [_I, _I, _I]),
    "avsr_relpos_attention_bwd": (_I, [_P] * 14 + [_I, _I, _I, _P, _Z, _P]),
    "avsr_relpos_attention_bwd_tc_workspace_bytes": (_Z, [_I, _I, _I, _I]),
    "avsr_relpos_attention_bwd_tc": (_I, [_P] * 14 + [_I, _I, _I, _I, _P, _Z, _P]),
    "avsr_ctc_loss_state_bytes": (_Z, [_I, _I, _I]),
    "avsr_ctc_loss_fwd": (_I, [_P, C.c_long, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _Z, _P]),
    "avsr_ctc_loss_bwd": (_I, [_P, C.c_long, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P, C.c_long, _P]),
    "avsr_mha_core_fwd": (_I, [_P, C.c_long, _P, C.c_long, _P, C.c_long, _I, _I, _I, _I, _I, _P, _P, _F, _P, _P, _P]),
    "avsr_mha_core_bwd_workspace_bytes": (_Z, [_I, _I, _I]),
    "avsr_mha_core_bwd": (_I, [_P, C.c_long, _P, C.c_long, _P, C.c_long, _I, _I, _I, _I, _I, _P, _P, _F, _P, _P, _P,
                               C.c_long, _P, _P, C.c_long, _P, _Z, _P]),
    "avsr_mha_core_bwd_tc_workspace_bytes": (_Z, [_I, _I, _I, _I, _I]),
    "avsr_mha_core_bwd_tc": (_I, [_P, C.c_long, _P, C.c_long, _P, C.c_long, _I, _I, _I, _I, _I, _P, _P, _F, _P, _P, _P,
                                  _P, C.c_long, _P, _P, C.c_long, _I, _P, _Z, _P]),
    "avsr_label_smoothing_fwd": (_I, [_P, C.c_long, _P, _I, _I, _I, _F, _P, _P, _P]),
    "avsr_label_smoothing_bwd": (_I, [_P, C.c_long, _P, _I, _I, _I, _F, _P, _P, _P, C.c_long, _P]),
    "avsr_embed_fwd": (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    "avsr_embed_bwd_workspace_bytes": (_Z, [_I, _I]),
    "avsr_embed_bwd": (_I, [_P, _P, _I, _I, _I, _P, _P, _Z, _P]),
    "avsr_pack_padded": (_I, [_P, _P, _P, _P, _I, _I, _I, _F, _P]),
    "avsr_unpack_padded": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "avsr_head_prepared_bytes": (_Z, [_CFG, _I, _I]),
    "avsr_prepare_head": (_I, [_CFG, _I, _I, _P, _P, _P, _P, _P, _Z, _I, _P]),
    "avsr_head_workspace_bytes": (_Z, [_CFG, _I, _I, _I, _I]),
    "avsr_features_to_logprobs": (_I, [_CFG, _P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _Z, _I, _P]),
    "avsr_head_plan_workspace_bytes": (_Z, [_CFG, _I, _I, _I, _I]),
    "avsr_head_plan_create": (_I, [_CFG, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _Z, _I, _P, C.POINTER(_P)]),
    "avsr_head_plan_forward": (_I, [_P, _P, _P, _P]),
    "avsr_proj_encoder": (_I, [_CFG, _P, _P, _I, _I, _I, _P, _P, _Z, _I, _P]),
    "avsr_ctc_workspace_bytes": (_Z, [_CFG, _I, _I]),
    "avsr_ctc_logprobs": (_I, [_CFG, _P, _P, _I, _I, _I, _P, _P, _P, _Z, _I, _P]),
    "avsr_decoder_prepared_bytes": (_Z, [_DCFG]),
    "avsr_prepare_decoder": (_I, [_DCFG, C.POINTER(DecoderLayerParams), _P, _P, _P, _P, _P, _P, _Z, _I, _P]),
    "avsr_decoder_session_bytes": (_Z, [_DCFG, _I, _I, _I]),
    "avsr_decoder_begin": (_I, [_DCFG, _P, _P, _I, _I, _I, _P, _Z, _I, _P]),
    "avsr_decoder_step_workspace_bytes": (_Z, [_DCFG, _I, _I, _I]),
    "avsr_decoder_step": (_I, [_DCFG, _P, _P, _Z, _I, _I, _I, _P, _P, _I, _I, _P, _P, _Z, _I, _P]),
    "avsr_ctc_prefix_init": (_I, [_P, _I, _I, _I, _P, _P]),
    "avsr_ctc_prefix_score": (_I, [_P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P]),
    "avsr_ctc_prefix_select": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P]),
    "avsr_decoder_batch_session_bytes": (_Z, [_DCFG, _I, _P, _I, _I]),
    "avsr_decoder_batch_step_workspace_bytes": (_Z, [_DCFG, _I, _I, _I]),
    "avsr_decoder_batch_begin": (_I, [_DCFG, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _I, _P]),
    "avsr_decoder_batch_step": (_I, [_DCFG, _P, _P, _Z, _P, _I, _I, _I, _I, _P, _P, _P, _I, _I, _P, _P, _Z, _I, _P]),
    "avsr_ctc_prefix_batch_init": (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _P]),
    "avsr_ctc_prefix_batch_score": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P]),
    "avsr_frontend_prepared_bytes": (_Z, [_I, _I]),
    "avsr_prepare_frontend": (_I, [_I, C.POINTER(ConvBnParams), _P, _Z, _I, _P]),
    "avsr_frontend_workspace_bytes": (_Z, [_I, _I, _I, _I, _I, _I]),
    "avsr_frontend_forward": (_I, [_I, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _I, _P]),
    "avsr_frontend_forward_taps": (_I, [_I, _P, _P, _I, _I, _I, _I, _P, C.POINTER(_P), _P, _Z, _I, _P]),
    "avsr_frontend_tap_shape": (_I, [_I, _I, _I, _I, _I, _I, C.POINTER(C.c_int)]),
    "avsr_conv_bn_act_workspace_bytes": (_Z, [_I] * 9),
    "avsr_conv_bn_act": (_I, [_P, _P, _P, _P, _P, _I, _P] + [_I] * 8 + [_P, _Z, _I, _P]),
    "avsr_frontend_train_conv_workspace_bytes": (_Z, [_I] * 11),
    "avsr_frontend_train_conv_fwd": (_I, [_P, _P, _P, _P] + [_I] * 10 + [_P, _Z, _I, _P]),
    "avsr_frontend_train_dgrad_workspace_bytes": (_Z, [_I] * 9),
    "avsr_frontend_train_conv_dgrad": (_I, [_P, _P, _P] + [_I] * 8 + [_P, _Z, _I, _P]),
    "avsr_frontend_train_wgrad_workspace_bytes": (_Z, [_I] * 10),
    "avsr_frontend_train_conv_wgrad": (_I, [_P, _P, _P] + [_I] * 10 + [_P, _Z, _I, _P]),
    "avsr_frontend_train_maxpool_fwd": (_I, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "avsr_frontend_train_maxpool_bwd": (_I, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "avsr_frontend_train_mean_rows": (_I, [_P, _P, C.c_long, _I, _I, _P]),
    "avsr_frontend_train_mean_rows_bwd": (_I, [_P, _P, C.c_long, _I, _I, _P]),
}

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(nvcc, sm_90a).  auto_avsr_b200 has no CPU / PyTorch fallback for the encoder hot path.")

lib = C.CDLL(LIB_PATH)
for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)          # AttributeError here == header / library mismatch
    _fn.restype = _res
    _fn.argtypes = _args
if lib.avsr_abi_version() != ABI_VERSION:
    raise ImportError(f"libavsr_b200 ABI {lib.avsr_abi_version()} != binding ABI {ABI_VERSION}")


def check(rc: int) -> None:
    if rc != OK:
        msg = lib.avsr_last_error().decode("utf-8", "replace")
        raise AvsrError(f"libavsr_b200 error {rc}: {msg}")


def launch_count() -> int:
    return int(lib.avsr_launch_count())
