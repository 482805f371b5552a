"""The bf16 backward of the decoder and the head without a GPU: the ``backward_precision`` attribute of
TransformerDecoder / CTC / ProjEncoder (validated, no environment fallback), what it routes to every ``LinearFn`` and
attention core of the pass, and the C-ABI entry of the tensor-core attention core backward (avsr_mha_core_bwd_tc):
refusals before any launch and its workspace formula."""
import ctypes as C

import pytest
import torch

import auto_avsr_b200.decoder_train as DT
import auto_avsr_b200.espnet_dropin.ctc as CT
import auto_avsr_b200.train as TR
from auto_avsr_b200 import _cabi
from auto_avsr_b200.espnet_dropin.ctc import CTC, ProjEncoder
from auto_avsr_b200.espnet_dropin.transformer_decoder import TransformerDecoder

PREC_FP32, PREC_TF32, PREC_F16, PREC_BF16 = 0, 1, 2, 16
NL, D, H, ODIM = 2, 128, 2, 11


def _modules():
    return [TransformerDecoder(ODIM, D, H, 256, NL), CTC(ODIM, D, 0.0), ProjEncoder(16, D)]


# ------------------------------------------------------------------------------------------------ the attribute
def test_knob_defaults_and_validation(monkeypatch):
    monkeypatch.delenv("AVSR_B200_BWD_PRECISION", raising=False)
    for m in _modules():
        assert m.backward_precision is None
    assert TR.explicit_backward_precision(None) is None
    assert TR.explicit_backward_precision("bf16") == "bf16"
    for bad in ("f16", "fp16", "tf32", "fp32", "BF16"):
        with pytest.raises(ValueError, match="f16"):
            TR.explicit_backward_precision(bad)
    monkeypatch.setenv("AVSR_B200_BWD_PRECISION", "bf16")
    assert TR.explicit_backward_precision(None) is None      # the environment reaches the encoder only


class _Rec:
    """Records the ``backward`` of every LinearFn / MhaCoreFn application and returns grad-requiring zeros."""

    def __init__(self):
        self.linear, self.core = [], []

    def linear_apply(self, x, w, b, relu, precision, backward=None):
        self.linear.append(backward)
        return torch.zeros(*x.shape[:-1], w.size(0), requires_grad=True)

    def core_apply(self, qsrc, kvsrc, self_attn, n_heads, causal, lengths, keep, keep_scale, backward=None):
        self.core.append(backward)
        return torch.zeros(*qsrc.shape[:-1], n_heads * 64, requires_grad=True)


@pytest.fixture
def rec(monkeypatch):
    r = _Rec()
    monkeypatch.setattr(TR.LinearFn, "apply", r.linear_apply)
    monkeypatch.setattr(DT.MhaCoreFn, "apply", r.core_apply)
    monkeypatch.setattr(DT.LayerNormFn, "apply", lambda x, w, b: x)
    monkeypatch.setattr(DT.EmbedFn, "apply", lambda tok, w: torch.zeros(*tok.shape, w.size(1), requires_grad=True))
    return r


@pytest.mark.parametrize("backward", [None, "bf16"])
def test_decoder_routes_the_knob_to_every_gemm_and_attention_core(rec, backward):
    """decoder_forward with NL layers: 7 NL + 1 LinearFn calls (self q|k|v, self out, source q, source k|v, source out,
    w_1, w_2 per layer; the output layer) and 2 NL attention cores, every one with the given ``backward``."""
    dec = TransformerDecoder(ODIM, D, H, 256, NL).train()
    B, L, T = 2, 5, 7
    out = DT.decoder_forward(dec, torch.zeros(B, L, dtype=torch.long), None, torch.zeros(B, T, D), None, "f16", backward)
    assert tuple(out.shape) == (B, L, ODIM)
    assert rec.linear == [backward] * (7 * NL + 1)
    assert rec.core == [backward] * (2 * NL)


def _fake_cuda(t):
    """``t`` reporting is_cuda: lets the modules' forwards run past their device check on the CPU."""
    class FakeCuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True
    return torch.Tensor._make_subclass(FakeCuda, t, t.requires_grad)


@pytest.mark.parametrize("knob,env", [(None, None), ("bf16", None), (None, "bf16")])
def test_decoder_forward_passes_the_attribute_only(monkeypatch, knob, env):
    """TransformerDecoder.forward hands ``backward_precision`` to decoder_forward; AVSR_B200_BWD_PRECISION does not."""
    if env is None:
        monkeypatch.delenv("AVSR_B200_BWD_PRECISION", raising=False)
    else:
        monkeypatch.setenv("AVSR_B200_BWD_PRECISION", env)
    seen = []
    monkeypatch.setattr(DT, "decoder_forward", lambda dec, tgt, tl, mem, ml, prec, backward: seen.append(backward))
    monkeypatch.setattr(DT, "target_lengths", lambda m, B, L, check: None)
    dec = TransformerDecoder(ODIM, D, H, 256, NL).train()
    dec.backward_precision = knob
    dec(_fake_cuda(torch.zeros(2, 5, dtype=torch.long)), None, _fake_cuda(torch.zeros(2, 7, D)), None)
    assert seen == [knob]
    dec.backward_precision = "f16"
    with pytest.raises(ValueError, match="f16"):
        dec(_fake_cuda(torch.zeros(2, 5, dtype=torch.long)), None, _fake_cuda(torch.zeros(2, 7, D)), None)


@pytest.mark.parametrize("knob,env", [(None, None), ("bf16", None), (None, "bf16")])
def test_head_routes_the_attribute_only(rec, monkeypatch, knob, env):
    """ProjEncoder.forward (train) and CTC.forward (ctc_lo) pass ``backward_precision`` to their LinearFn, and only
    that: the environment variable leaves them at None.  The CTC loss itself is not a GEMM."""
    if env is None:
        monkeypatch.delenv("AVSR_B200_BWD_PRECISION", raising=False)
    else:
        monkeypatch.setenv("AVSR_B200_BWD_PRECISION", env)
    monkeypatch.setattr(CT, "require_cuda", lambda t, what: None)
    monkeypatch.setattr(CT.CtcLossFn, "apply", lambda logits, hl, ys, odim, ign: torch.zeros(logits.size(0)))
    proj, ctc = ProjEncoder(16, D).train(), CTC(ODIM, D, 0.0).train()
    proj.backward_precision = ctc.backward_precision = knob
    proj(torch.zeros(2, 7, 16))
    ctc(_fake_cuda(torch.zeros(2, 7, D)), torch.tensor([7, 5]), torch.ones(2, 3, dtype=torch.long))
    assert rec.linear == [knob, knob]
    for m in (proj, ctc):
        m.backward_precision = "tf32"
    with pytest.raises(ValueError, match="f16"):
        proj(torch.zeros(2, 7, 16))
    with pytest.raises(ValueError, match="f16"):
        ctc(_fake_cuda(torch.zeros(2, 7, D)), torch.tensor([7, 5]), torch.ones(2, 3, dtype=torch.long))


# ------------------------------------------------------------------------------------------------ C ABI
def _align(n):
    return (n + 255) // 256 * 256


@pytest.mark.parametrize("B,H,Lq,Lk", [(1, 1, 1, 1), (5, 12, 81, 81), (5, 12, 81, 400), (3, 4, 61, 1600), (2, 2, 300, 1)])
def test_workspace_formula(B, H, Lq, Lk):
    """Delta (B, H, Lq) fp32; 256 bytes for an empty shape; 0 for a precision other than bf16."""
    f = _cabi.lib.avsr_mha_core_bwd_tc_workspace_bytes
    assert f(B, H, Lq, Lk, PREC_BF16) == _align(B * H * Lq * 4)
    assert f(0, H, Lq, Lk, PREC_BF16) == 256 and f(B, H, 0, Lk, PREC_BF16) == 256
    for p in (PREC_FP32, PREC_TF32, PREC_F16, 7, -1):
        assert f(B, H, Lq, Lk, p) == 0


def test_entry_refusals_before_any_launch():
    lib = _cabi.lib
    buf = C.create_string_buffer(1 << 16)
    p = (C.addressof(buf) + 15) // 16 * 16                       # a 16-byte aligned host address inside the buffer
    B, H, Lq, Lk = 2, 2, 9, 7
    D = H * 64
    ws = lib.avsr_mha_core_bwd_tc_workspace_bytes(B, H, Lq, Lk, PREC_BF16)

    def call(q=p, k=p, v=p, probs=p, ctx=p, dctx=p, dq=p, dk=p, dv=p, ld=(D, D, D, D, D), B=B, prec=PREC_BF16, w=p,
             nbytes=ws):
        ldq, ldk, ldv, lddq, lddkv = ld
        return lib.avsr_mha_core_bwd_tc(q, ldq, k, ldk, v, ldv, B, H, Lq, Lk, 1, None, None, 1.0, probs, ctx, dctx, dq,
                                        lddq, dk, dv, lddkv, prec, w, nbytes, None)

    before = _cabi.launch_count()
    for name in ("q", "k", "v", "probs", "ctx", "dctx", "dq", "dk", "dv", "w"):
        assert call(**{name: None}) == 1, name
        assert b"NULL" in lib.avsr_last_error()
    for prec, text in ((PREC_F16, b"AVSR_PREC_F16"), (PREC_TF32, b"AVSR_PREC_TF32"), (PREC_FP32, b"AVSR_PREC_FP32"),
                       (7, b"precision 7")):
        assert call(prec=prec) == 1
        assert text in lib.avsr_last_error()
    for i in range(5):
        for bad in (D + 2, D - 4):                                   # not a multiple of 4; shorter than H*64
            ld = [D] * 5
            ld[i] = bad
            assert call(ld=tuple(ld)) == 1, (i, bad)
            assert b"row strides" in lib.avsr_last_error()
    assert call(nbytes=ws - 1) == 3
    assert b"too small" in lib.avsr_last_error()
    assert call(B=0, w=None, nbytes=0) == 0                      # the empty batch: nothing to do
    assert _cabi.launch_count() == before
