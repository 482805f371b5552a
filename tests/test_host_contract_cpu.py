"""The host-side argument contract of libavsr_b200 without a GPU: every `*_bytes` entry over a grid of configs, shapes
and precisions (bad ones included), and the return code of invalid calls that are refused before any launch (NULL
buffers, bad precision, bad config, n > max_hyps, step >= max_steps, bad batch lengths, buffers one byte too small).

The table is tests/golden/host_contract.json; the library must reproduce it exactly.  The probe runs in a subprocess
with CUDA_VISIBLE_DEVICES="", so no call can reach a device.  The decoder entries of the host replay (tests/emu) must
also answer every decoder probe with the product library's code, size and error text: both compile the same entry
bodies of csrc/decoder_body.cuh.

    python tests/test_host_contract_cpu.py --record      # rewrite the golden table from the current library
"""
import ctypes as C
import json
import os
import shutil
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "host_contract.json")

P32, PTF32, PF16 = 0, 1, 2          # AVSR_PREC_FP32, TF32, F16
PRECS = (0, 1, 2, 7, -1)


def _probe(lib, decoder_only):
    """{probe label: size or [code, error text]} for the probes below, run against `lib`."""
    from auto_avsr_b200 import _cabi as A
    for name, (res, args) in A.SIGNATURES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    buf = C.create_string_buffer(1 << 16)
    p = C.addressof(buf)                       # a real host buffer: the refused calls never read it
    out = {}

    def size(name, *args):
        out[f"{name}{args!r}"] = int(getattr(lib, name)(*[_arg(a) for a in args]))

    def code(label, name, *args):
        rc = int(getattr(lib, name)(*[_arg(a) for a in args]))
        out[f"{label}: {name}"] = [rc, lib.avsr_last_error().decode() if rc else ""]

    def _arg(a):
        if isinstance(a, DCfg):
            return C.byref(A.DecoderConfig(*a))
        if isinstance(a, ECfg):
            return C.byref(A.EncoderConfig(*a))
        if isinstance(a, Lens):
            return (C.c_int32 * len(a))(*a)
        return a

    # ---------------------------------------------------------------- decoder / CTC prefix
    dcfgs = [DCfg((256, 4, 2048, 6, 5000)), DCfg((64, 2, 128, 2, 11)), DCfg((100, 4, 2048, 6, 5000)),
             DCfg((256, 4, 2000, 6, 5000)), DCfg((256, 4, 2048, 17, 5000)), DCfg((256, 4, 2048, 0, 5000)),
             DCfg((256, 4, 2048, 6, 1)), DCfg((256, 3, 2048, 6, 5000)), None]
    for dc in dcfgs:
        size("avsr_decoder_prepared_bytes", dc)
        for T, ms, mh in ((1, 1, 1), (37, 20, 40), (400, 100, 10), (0, 5, 5), (5, 0, 5), (5, 5, 0), (-1, 5, 5)):
            size("avsr_decoder_session_bytes", dc, T, ms, mh)
            size("avsr_decoder_step_workspace_bytes", dc, T, ms, mh)
            size("avsr_decoder_batch_step_workspace_bytes", dc, T, ms, mh)
        for U, lens in ((1, Lens((7,))), (3, Lens((5, 1, 9))), (2, Lens((5, 0))), (0, Lens((5,))), (2, None)):
            for ms, mh in ((8, 30), (0, 4), (4, 0)):
                size("avsr_decoder_batch_session_bytes", dc, U, lens, ms, mh)
    tiny = dcfgs[1]
    layers = (A.DecoderLayerParams * 2)(*[A.DecoderLayerParams(*([p] * len(A.DECODER_LAYER_FIELDS)))] * 2)
    holey = (A.DecoderLayerParams * 2)(*[A.DecoderLayerParams(*([p] * len(A.DECODER_LAYER_FIELDS)))] * 2)
    holey[1].ff_w2 = None
    need = {}
    _c = lambda name, *a: int(getattr(lib, name)(*[_arg(x) for x in a]))  # noqa: E731
    need["prep"] = _c("avsr_decoder_prepared_bytes", tiny)
    need["sess"] = _c("avsr_decoder_session_bytes", tiny, 9, 6, 4)
    need["work"] = _c("avsr_decoder_step_workspace_bytes", tiny, 9, 6, 4)
    need["bsess"] = _c("avsr_decoder_batch_session_bytes", tiny, 2, Lens((9, 4)), 6, 4)
    for lab, args in (("ok-shape too small", (tiny, layers, p, p, p, p, p, p, need["prep"] - 1, P32, None)),
                      ("NULL cfg", (None, layers, p, p, p, p, p, p, need["prep"], P32, None)),
                      ("bad cfg", (dcfgs[2], layers, p, p, p, p, p, p, need["prep"], P32, None)),
                      ("NULL prepared", (tiny, layers, p, p, p, p, p, None, need["prep"], P32, None)),
                      ("NULL layers", (tiny, None, p, p, p, p, p, p, need["prep"], P32, None)),
                      ("NULL layer parameter", (tiny, holey, p, p, p, p, p, p, need["prep"], P32, None)),
                      ("bad precision", (tiny, layers, p, p, p, p, p, p, need["prep"], 7, None))):
        code(lab, "avsr_prepare_decoder", *args)
    for lab, args in (("too small", (tiny, p, p, 9, 6, 4, p, need["sess"] - 1, P32, None)),
                      ("NULL cfg", (None, p, p, 9, 6, 4, p, need["sess"], P32, None)),
                      ("bad cfg", (dcfgs[4], p, p, 9, 6, 4, p, need["sess"], P32, None)),
                      ("NULL memory", (tiny, p, None, 9, 6, 4, p, need["sess"], P32, None)),
                      ("T=0", (tiny, p, p, 0, 6, 4, p, need["sess"], P32, None)),
                      ("max_hyps=0", (tiny, p, p, 9, 6, 0, p, need["sess"], P32, None)),
                      ("bad precision", (tiny, p, p, 9, 6, 4, p, need["sess"], 3, None))):
        code(lab, "avsr_decoder_begin", *args)
    toks = (C.c_int32 * 8)(*range(8))
    for lab, args in (("session too small", (tiny, p, p, need["sess"] - 1, 9, 6, 4, toks, p, 1, 2, p, p, need["work"], P32, None)),
                      ("workspace too small", (tiny, p, p, need["sess"], 9, 6, 4, toks, p, 1, 2, p, p, need["work"] - 1, P32, None)),
                      ("step >= max_steps", (tiny, p, p, need["sess"], 9, 6, 4, toks, p, 6, 2, p, p, need["work"], P32, None)),
                      ("step < 0", (tiny, p, p, need["sess"], 9, 6, 4, toks, p, -1, 2, p, p, need["work"], P32, None)),
                      ("n > max_hyps", (tiny, p, p, need["sess"], 9, 6, 4, toks, p, 1, 5, p, p, need["work"], P32, None)),
                      ("n < 0", (tiny, p, p, need["sess"], 9, 6, 4, toks, p, 1, -1, p, p, need["work"], P32, None)),
                      ("no anc", (tiny, p, p, need["sess"], 9, 6, 4, toks, None, 1, 2, p, p, need["work"], P32, None)),
                      ("NULL logp", (tiny, p, p, need["sess"], 9, 6, 4, toks, p, 1, 2, None, p, need["work"], P32, None)),
                      ("bad precision", (tiny, p, p, need["sess"], 9, 6, 4, toks, p, 1, 2, p, p, need["work"], -1, None)),
                      ("bad cfg", (dcfgs[6], p, p, need["sess"], 9, 6, 4, toks, p, 1, 2, p, p, need["work"], P32, None)),
                      ("n = 0", (tiny, p, p, need["sess"], 9, 6, 4, toks, p, 1, 0, p, p, need["work"], P32, None))):
        code(lab, "avsr_decoder_step", *args)
    L2 = Lens((9, 4))
    for lab, args in (("too small", (tiny, p, p, L2, 2, 9, 6, 4, p, need["bsess"] - 1, P32, None)),
                      ("length > T_max", (tiny, p, p, Lens((9, 10)), 2, 9, 6, 4, p, need["bsess"], P32, None)),
                      ("zero length", (tiny, p, p, Lens((9, 0)), 2, 9, 6, 4, p, need["bsess"], P32, None)),
                      ("U=0", (tiny, p, p, L2, 0, 9, 6, 4, p, need["bsess"], P32, None)),
                      ("NULL lengths", (tiny, p, p, None, 2, 9, 6, 4, p, need["bsess"], P32, None)),
                      ("NULL session", (tiny, p, p, L2, 2, 9, 6, 4, None, need["bsess"], P32, None)),
                      ("bad precision", (tiny, p, p, L2, 2, 9, 6, 4, p, need["bsess"], 5, None)),
                      ("bad cfg", (None, p, p, L2, 2, 9, 6, 4, p, need["bsess"], P32, None))):
        code(lab, "avsr_decoder_batch_begin", *args)
    for lab, args in (("session too small", (tiny, p, p, need["bsess"] - 1, L2, 2, 9, 6, 4, toks, p, p, 1, 2, p, p, need["work"], P32, None)),
                      ("workspace too small", (tiny, p, p, need["bsess"], L2, 2, 9, 6, 4, toks, p, p, 1, 2, p, p, need["work"] - 1, P32, None)),
                      ("step >= max_steps", (tiny, p, p, need["bsess"], L2, 2, 9, 6, 4, toks, p, p, 6, 2, p, p, need["work"], P32, None)),
                      ("n > max_hyps", (tiny, p, p, need["bsess"], L2, 2, 9, 6, 4, toks, p, p, 1, 5, p, p, need["work"], P32, None)),
                      ("no anc", (tiny, p, p, need["bsess"], L2, 2, 9, 6, 4, toks, None, p, 1, 2, p, p, need["work"], P32, None)),
                      ("NULL row_utt", (tiny, p, p, need["bsess"], L2, 2, 9, 6, 4, toks, p, None, 1, 2, p, p, need["work"], P32, None)),
                      ("bad lengths", (tiny, p, p, need["bsess"], Lens((9, 12)), 2, 9, 6, 4, toks, p, p, 1, 2, p, p, need["work"], P32, None)),
                      ("T_max=0", (tiny, p, p, need["bsess"], L2, 2, 0, 6, 4, toks, p, p, 1, 2, p, p, need["work"], P32, None)),
                      ("bad precision", (tiny, p, p, need["bsess"], L2, 2, 9, 6, 4, toks, p, p, 1, 2, p, p, need["work"], 9, None)),
                      ("n = 0", (tiny, p, p, need["bsess"], L2, 2, 9, 6, 4, toks, p, p, 1, 0, p, p, need["work"], P32, None))):
        code(lab, "avsr_decoder_batch_step", *args)
    for lab, args in (("NULL logp", (None, 9, 11, 0, p, None)), ("blank >= O", (p, 9, 11, 11, p, None)),
                      ("T=0", (p, 0, 11, 0, p, None))):
        code(lab, "avsr_ctc_prefix_init", *args)
    for lab, args in (("NULL r", (p, 9, 11, 0, 10, 0, p, p, p, p, 2, 3, p, None, p, None)),
                      ("blank == eos", (p, 9, 11, 0, 0, 0, p, p, p, p, 2, 3, p, p, p, None)),
                      ("S > O", (p, 9, 11, 0, 10, 0, p, p, p, p, 2, 12, p, p, p, None)),
                      ("n = 0", (p, 9, 11, 0, 10, 0, p, p, p, p, 0, 3, p, p, p, None))):
        code(lab, "avsr_ctc_prefix_score", *args)
    for lab, args in (("NULL token", (p, p, p, p, None, 9, 11, 2, 3, 2, p, p, None)),
                      ("n = 0", (p, p, p, p, p, 9, 11, 0, 3, 2, p, p, None)),
                      ("m = 0", (p, p, p, p, p, 9, 11, 2, 3, 0, p, p, None))):
        code(lab, "avsr_ctc_prefix_select", *args)
    for lab, args in (("bad lengths", (p, Lens((9, 0)), 2, 9, 11, 0, p, p, None)),
                      ("NULL lengths_dev", (p, L2, 2, 9, 11, 0, None, p, None)),
                      ("T_max=0", (p, L2, 2, 0, 11, 0, p, p, None))):
        code(lab, "avsr_ctc_prefix_batch_init", *args)
    for lab, args in (("U=0", (p, L2, 0, 9, 11, 0, 10, 0, p, p, p, p, p, 2, 3, p, p, p, None)),
                      ("NULL row_utt", (p, L2, 2, 9, 11, 0, 10, 0, p, p, p, p, None, 2, 3, p, p, p, None)),
                      ("n = 0", (p, L2, 2, 9, 11, 0, 10, 0, p, p, p, p, p, 0, 3, p, p, p, None))):
        code(lab, "avsr_ctc_prefix_batch_score", *args)
    if decoder_only:
        return out

    # ---------------------------------------------------------------- encoder / head / per-op
    ecfgs = [ECfg((768, 12, 3072, 12, 31)), ECfg((256, 4, 1024, 2, 15)), ECfg((768, 12, 3072, 12, 30)),
             ECfg((100, 2, 1024, 2, 15)), ECfg((768, 12, 3000, 12, 31)), ECfg((768, 12, 3072, 0, 31)), None]
    for ec in ecfgs:
        size("avsr_prepared_bytes", ec)
        for B, T in ((0, 5), (1, 0), (1, 1), (3, 37), (4, 400), (-1, 5), (2, -1)):
            size("avsr_workspace_bytes", ec, B, T)
            for idim, odim in ((768, 5000), (512, 41), (0, 41), (512, 0)):
                size("avsr_head_workspace_bytes", ec, B, T, idim, odim)
                size("avsr_head_plan_workspace_bytes", ec, B, T, idim, odim)
        for idim, odim in ((768, 5000), (512, 41), (0, 41), (512, -3)):
            size("avsr_head_prepared_bytes", ec, idim, odim)
        for rows, odim in ((0, 41), (37, 5000), (-1, 41), (5, 0)):
            size("avsr_ctc_workspace_bytes", ec, rows, odim)
    for rows, n, k in ((0, 8, 64), (37, 768, 3072), (5, 0, 64)):
        for prec in PRECS:
            size("avsr_linear_workspace_bytes", rows, n, k, prec)
    for B, T, H in ((1, 1, 12), (3, 37, 12), (0, 5, 4), (2, 5, 0)):
        size("avsr_attention_workspace_bytes", B, T, H)
        size("avsr_relpos_attention_bwd_workspace_bytes", B, T, H)
        size("avsr_mha_core_bwd_workspace_bytes", B, H, T)
        size("avsr_ctc_loss_state_bytes", B, T, H)
    for rows, C_ in ((0, 768), (37, 768), (-1, 64), (5, 0)):
        size("avsr_pointwise_glu_workspace_bytes", rows, C_)
        size("avsr_embed_bwd_workspace_bytes", rows, C_)
    size("avsr_ctc_loss_state_bytes", -1, 3, 3)
    for mod in (0, 1, 2):
        for prec in PRECS:
            size("avsr_frontend_prepared_bytes", mod, prec)
            for B, T, H, W in ((2, 29, 88, 88), (1, 1, 45, 61), (2, 16000, 1, 1), (0, 5, 88, 88), (1, 5, 0, 88),
                               (-1, 5, 88, 88)):
                size("avsr_frontend_workspace_bytes", mod, B, T, H, W, prec)
    for g in ((2, 22, 22, 64, 64, 3, 3, 1), (2, 22, 22, 64, 128, 1, 1, 2), (0, 22, 22, 64, 64, 3, 3, 1),
              (2, 0, 22, 64, 64, 3, 3, 1), (2, 22, 22, 64, 64, 3, 3, 0)):
        for prec in PRECS:
            size("avsr_conv_bn_act_workspace_bytes", *g, prec)

    ec, sc = ecfgs[0], ecfgs[1]
    ws = _c("avsr_workspace_bytes", sc, 2, 9)
    code("too small", "avsr_encoder_forward", sc, p, p, None, 2, 9, p, p, ws - 1, PTF32, None)
    code("NULL prepared", "avsr_encoder_forward", sc, None, p, None, 2, 9, p, p, ws, PTF32, None)
    code("bad precision", "avsr_encoder_forward", sc, p, p, None, 2, 9, p, p, ws, 3, None)
    code("bad cfg", "avsr_encoder_forward", ecfgs[2], p, p, None, 2, 9, p, p, ws, PTF32, None)
    code("B<0", "avsr_encoder_forward", sc, p, p, None, -2, 9, p, p, ws, PTF32, None)
    code("empty batch", "avsr_encoder_forward", sc, None, None, None, 0, 9, None, None, 0, PTF32, None)
    code("NULL counter", "avsr_encoder_forward_checked", sc, p, p, None, 2, 9, p, p, ws, PF16, None, None)
    code("too small", "avsr_encoder_forward_taps", sc, p, p, None, 2, 9, p, p, p, ws - 1, PTF32, None)
    pp = C.c_void_p()
    code("too small", "avsr_plan_create", sc, p, 2, 9, p, ws - 1, PF16, None, C.byref(pp))
    code("NULL plan", "avsr_plan_create", sc, p, 2, 9, p, ws, PF16, None, None)
    code("B=0", "avsr_plan_create", sc, p, 0, 9, p, ws, PF16, None, C.byref(pp))
    code("bad precision", "avsr_plan_create", sc, p, 2, 9, p, ws, 4, None, C.byref(pp))
    code("NULL plan", "avsr_plan_forward", None, p, None, p, None)
    hpw = _c("avsr_head_plan_workspace_bytes", sc, 2, 9, 512, 41)
    code("too small", "avsr_head_plan_create", sc, p, p, 2, 9, 512, 41, p, p, None, p, hpw - 1, PF16, None, C.byref(pp))
    code("NULL outputs", "avsr_head_plan_create", sc, p, p, 2, 9, 512, 41, p, None, None, p, hpw, PF16, None, C.byref(pp))
    code("odim=0", "avsr_head_plan_create", sc, p, p, 2, 9, 512, 0, p, p, None, p, hpw, PF16, None, C.byref(pp))
    code("bad precision", "avsr_head_plan_create", sc, p, p, 2, 9, 512, 41, p, p, None, p, hpw, 8, None, C.byref(pp))
    code("not a head plan", "avsr_head_plan_forward", None, p, None, None)
    elayers = (A.LayerParams * 2)(*[A.LayerParams(*([p] * len(A.LAYER_FIELDS)))] * 2)
    pb = _c("avsr_prepared_bytes", sc)
    code("too small", "avsr_prepare_weights", sc, elayers, p, p, p, pb - 1, PTF32, None)
    code("NULL layers", "avsr_prepare_weights", sc, None, p, p, p, pb, PTF32, None)
    code("bad precision", "avsr_prepare_weights", sc, elayers, p, p, p, pb, 6, None)
    hp = _c("avsr_head_prepared_bytes", sc, 512, 41)
    code("too small", "avsr_prepare_head", sc, 512, 41, p, p, p, p, p, hp - 1, PTF32, None)
    code("half a projection", "avsr_prepare_head", sc, 512, 41, p, None, None, None, p, hp, PTF32, None)
    code("idim % 8", "avsr_prepare_head", sc, 511, 41, p, p, p, p, p, hp, PTF32, None)
    hw = _c("avsr_head_workspace_bytes", sc, 2, 9, 512, 41)
    code("too small", "avsr_features_to_logprobs", sc, p, p, p, None, 2, 9, 512, 41, None, p, None, p, hw - 1, PF16, None)
    code("no outputs", "avsr_features_to_logprobs", sc, p, p, p, None, 2, 9, 512, 41, None, None, None, p, hw, PF16, None)
    code("too small", "avsr_proj_encoder", sc, p, p, 18, 512, 41, p, p, 18 * 512 * 4 - 1, PTF32, None)
    cw = _c("avsr_ctc_workspace_bytes", sc, 18, 41)
    code("too small", "avsr_ctc_logprobs", sc, p, p, 18, 256, 41, p, None, p, cw - 1, PTF32, None)
    lw = _c("avsr_linear_workspace_bytes", 18, 64, 64, PF16)
    code("too small", "avsr_linear", p, p, None, None, C.c_float(1.0), 0, p, 18, 64, 64, PF16, p, lw - 1, None)
    code("no workspace", "avsr_linear", p, p, None, None, C.c_float(1.0), 0, p, 18, 64, 64, PF16, None, lw, None)
    code("bad precision", "avsr_linear", p, p, None, None, C.c_float(1.0), 0, p, 18, 64, 64, 5, p, lw, None)
    code("bad precision", "avsr_linear_operands", p, p, None, None, C.c_float(1.0), p, 18, 64, 64, 0, 0, 5, None)
    aw = _c("avsr_attention_workspace_bytes", 2, 9, 4)
    code("too small", "avsr_relpos_attention", p, p, p, p, p, p, None, p, 2, 9, 4, p, aw - 1, PTF32, None)
    code("bad precision", "avsr_relpos_attention", p, p, p, p, p, p, None, p, 2, 9, 4, p, aw, 3, None)
    code("too small", "avsr_dwconv_bn_silu", p, p, p, p, p, p, p, p, 2, 9, 64, 15, p, 17 * 64 * 4 - 1, None)
    code("even K", "avsr_dwconv_bn_silu", p, p, p, p, p, p, p, p, 2, 9, 64, 14, p, 17 * 64 * 4, None)
    gw = _c("avsr_pointwise_glu_workspace_bytes", 18, 64)
    code("too small", "avsr_pointwise_glu", p, p, p, p, 18, 64, p, gw - 1, PTF32, None)
    code("C % 64", "avsr_pointwise_glu", p, p, p, p, 18, 65, p, gw, PTF32, None)
    bw = _c("avsr_relpos_attention_bwd_workspace_bytes", 2, 9, 4)
    code("too small", "avsr_relpos_attention_bwd", *([p] * 14), 2, 9, 4, p, bw - 1, None)
    code("too small", "avsr_layernorm_bwd", p, p, p, p, p, p, 18, 64, p, 2 * 64 * 4 - 1, None)
    code("too small", "avsr_colsum", p, p, 18, 64, p, 64 * 4 - 1, None)
    code("too small", "avsr_dwconv_raw", p, p, p, p, 2, 9, 64, 15, 0, p, 17 * 64 * 4 - 1, None)
    bnw = _c("avsr_bn_train_workspace_bytes", 18, 64)
    code("NULL input", "avsr_bn_train_stats", None, 18, 64, p, p, bnw, None)
    code("too small", "avsr_bn_train_stats", p, 18, 64, p, p, bnw - 1, None)
    code("too small", "avsr_dwconv_wgrad", p, p, p, p, 2, 9, 64, 15, p, 63, None)
    st = _c("avsr_ctc_loss_state_bytes", 2, 9, 3)
    code("too small", "avsr_ctc_loss_fwd", p, 41, p, p, 2, 9, 3, 41, -1, 1, p, p, st - 1, None)
    code("too small", "avsr_ctc_loss_bwd", p, 41, p, p, 2, 9, 3, 41, p, p, st - 1, p, 41, None)
    code("Lmax too large", "avsr_ctc_loss_fwd", p, 41, p, p, 2, 9, 5000, 41, -1, 1, p, p, st, None)
    mw = _c("avsr_mha_core_bwd_workspace_bytes", 2, 4, 9)
    code("too small", "avsr_mha_core_bwd", p, 256, p, 256, p, 256, 2, 4, 9, 9, 0, None, None, C.c_float(1.0), p, p, p,
         256, p, p, 256, p, mw - 1, None)
    ew = _c("avsr_embed_bwd_workspace_bytes", 18, 41)
    code("too small", "avsr_embed_bwd", p, p, 18, 64, 41, p, p, ew - 1, None)
    convs = (A.ConvBnParams * A.FRONTEND_CONVS)(*[A.ConvBnParams(p, p, p, p, p, 1e-5)] * A.FRONTEND_CONVS)
    for mod in (0, 1):
        fp = _c("avsr_frontend_prepared_bytes", mod, PTF32)
        fw = _c("avsr_frontend_workspace_bytes", mod, 2, 1280, 44, 44, PTF32)
        code(f"modality {mod} too small", "avsr_prepare_frontend", mod, convs, p, fp - 1, PTF32, None)
        code(f"modality {mod} bad precision", "avsr_prepare_frontend", mod, convs, p, fp, 3, None)
        code(f"modality {mod} too small", "avsr_frontend_forward", mod, p, p, 2, 1280, 44, 44, p, p, fw - 1, PTF32, None)
        code(f"modality {mod} bad precision", "avsr_frontend_forward", mod, p, p, 2, 1280, 44, 44, p, p, fw, -1, None)
    code("bad modality", "avsr_frontend_forward", 5, p, p, 2, 1280, 44, 44, p, p, 1 << 30, PTF32, None)
    taps = (C.c_void_p * 10)(*([p] * 10))
    fw = _c("avsr_frontend_workspace_bytes", 0, 2, 7, 44, 44, PF16)
    code("too small", "avsr_frontend_forward_taps", 0, p, p, 2, 7, 44, 44, p, taps, p, fw - 1, PF16, None)
    code("NULL taps", "avsr_frontend_forward_taps", 0, p, p, 2, 7, 44, 44, p, None, p, fw, PF16, None)
    code("bad precision", "avsr_frontend_forward_taps", 1, p, p, 2, 1280, 1, 1, p, taps, p, fw, 4, None)
    dims = (C.c_int * 4)()
    for mod, B, T, H, W in ((0, 2, 29, 88, 88), (0, 1, 1, 1, 1), (0, 2, 3, 45, 61), (1, 2, 16000, 1, 1), (1, 3, 639, 1, 1),
                            (0, 2, 5, 0, 88), (2, 1, 5, 88, 88)):
        for tap in (-1, 0, 1, 2, 5, 9, 10):
            rc = int(lib.avsr_frontend_tap_shape(mod, B, T, H, W, tap, dims))
            out[f"avsr_frontend_tap_shape{(mod, B, T, H, W, tap)!r}"] = f"{rc}: {list(dims) if rc == 0 else ''}"
    kw = _c("avsr_conv_bn_act_workspace_bytes", 2, 22, 22, 64, 64, 3, 3, 1, PF16)
    code("too small", "avsr_conv_bn_act", p, p, p, p, None, 1, p, 2, 22, 22, 64, 64, 3, 3, 1, p, kw - 1, PF16, None)
    code("bad precision", "avsr_conv_bn_act", p, p, p, p, None, 1, p, 2, 22, 22, 64, 64, 3, 3, 1, p, kw, 7, None)
    return out


class DCfg(tuple):
    pass


class ECfg(tuple):
    pass


class Lens(tuple):
    pass


def _run_probe(lib_path, decoder_only=False):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--probe", lib_path] +
                       (["--decoder-only"] if decoder_only else []),
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, f"probe of {lib_path} failed ({r.returncode}):\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    return json.loads(r.stdout.strip().splitlines()[-1])


def _product_lib():
    return os.path.join(ROOT, "auto_avsr_b200", "csrc", "libavsr_b200.so")


def _codes_and_sizes(table):
    """what the golden table fixes: every size and every return code (the error texts are checked against the replay)"""
    return {k: (v[0] if isinstance(v, list) else v) for k, v in table.items()}


def test_host_contract_matches_golden():
    with open(GOLDEN) as f:
        golden = json.load(f)
    got = _codes_and_sizes(_run_probe(_product_lib()))
    assert set(got) == set(golden), sorted(set(got) ^ set(golden))[:20]
    diff = {k: (golden[k], got[k]) for k in golden if golden[k] != got[k]}
    assert not diff, diff


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"),
                    reason="nvcc is needed to build the host replay")
def test_emu_decoder_entries_match_product():
    from emu import build
    emu_path = build.build("decoder_batch")
    prod = _run_probe(_product_lib(), decoder_only=True)
    emu = _run_probe(emu_path, decoder_only=True)
    assert set(prod) == set(emu)
    diff = {k: (prod[k], emu[k]) for k in prod if prod[k] != emu[k]}
    assert not diff, diff


if __name__ == "__main__":
    if "--probe" in sys.argv:
        sys.path.insert(0, ROOT)
        lib = C.CDLL(sys.argv[sys.argv.index("--probe") + 1])
        print(json.dumps(_probe(lib, "--decoder-only" in sys.argv), sort_keys=True))
    elif "--record" in sys.argv:
        table = _codes_and_sizes(_run_probe(_product_lib()))
        with open(GOLDEN, "w") as f:
            json.dump(table, f, indent=0, sort_keys=True)
            f.write("\n")
        print(f"wrote {len(table)} entries to {GOLDEN}")
