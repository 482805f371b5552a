"""The opt-in bf16 backward without a GPU: how ``backward_precision`` resolves and what it passes to the library, the
C-ABI entries of the tensor-core attention backward (argument checks, workspace formula), and a host restatement of
the dp kernel's tile -> band -> table-row mapping and fix-up order (csrc/attention_bwd_tc.cu)."""
import ctypes as C
import types

import pytest
import torch

import auto_avsr_b200.train as TR
from auto_avsr_b200 import _cabi
from auto_avsr_b200.espnet_dropin.attention import RelPositionMultiHeadedAttention
from auto_avsr_b200.espnet_dropin.conformer_encoder import ConformerEncoder, ConvolutionModule
from auto_avsr_b200.espnet_dropin.positionwise_feed_forward import PositionwiseFeedForward

PREC_F16, PREC_BF16, PREC_TF32, PREC_FP32 = 2, 16, 1, 0


# ------------------------------------------------------------------------------------------------ knob resolution
def test_resolve_backward_precision(monkeypatch):
    monkeypatch.delenv("AVSR_B200_BWD_PRECISION", raising=False)
    assert TR.resolve_backward_precision(None) is None
    assert TR.resolve_backward_precision("bf16") == "bf16"
    monkeypatch.setenv("AVSR_B200_BWD_PRECISION", "bf16")
    assert TR.resolve_backward_precision(None) == "bf16"
    monkeypatch.setenv("AVSR_B200_BWD_PRECISION", "")
    assert TR.resolve_backward_precision(None) is None
    for bad in ("f16", "fp16", "tf32", "fp32", "BF16"):
        with pytest.raises(ValueError, match="f16"):
            TR.resolve_backward_precision(bad)
    monkeypatch.setenv("AVSR_B200_BWD_PRECISION", "f16")
    with pytest.raises(ValueError):
        TR.resolve_backward_precision(None)


def test_modules_carry_the_knob(monkeypatch):
    monkeypatch.delenv("AVSR_B200_BWD_PRECISION", raising=False)
    mods = [RelPositionMultiHeadedAttention(2, 128, 0.0), PositionwiseFeedForward(128, 256, 0.0),
            ConvolutionModule(128, 31), ConformerEncoder(num_blocks=1)]
    for m in mods:
        assert m.backward_precision is None
        assert TR.module_backward_precision(m) is None
    m = mods[1]
    m.backward_precision = "bf16"
    assert TR.module_backward_precision(m) == "bf16"
    m.backward_precision = "f16"
    with pytest.raises(ValueError):
        TR.module_backward_precision(m)
    m.backward_precision = None
    m._inherited_backward_precision = "bf16"           # what ConformerEncoder.forward(train) passes down
    assert TR.module_backward_precision(m) == "bf16"
    m.backward_precision = "bf16"
    m._inherited_backward_precision = None
    assert TR.module_backward_precision(m) == "bf16"   # a module's own setting wins


def test_encoder_propagates_the_knob(monkeypatch):
    """ConformerEncoder.forward(train) hands its resolved value to every sub-module, on every forward (clearing it
    clears theirs); the CPU input raises afterwards, before any kernel."""
    monkeypatch.delenv("AVSR_B200_BWD_PRECISION", raising=False)
    enc = ConformerEncoder(num_blocks=2).train()
    subs = [m for m in enc.modules() if hasattr(m, "backward_precision") and m is not enc]
    assert len(subs) == 2 * 4                           # attention, two FFNs, conv module per layer
    fake = types.SimpleNamespace(is_cuda=True)        # passes the CUDA check, then fails in the positional encoding

    def run(value, env=None):
        if env is None:
            monkeypatch.delenv("AVSR_B200_BWD_PRECISION", raising=False)
        else:
            monkeypatch.setenv("AVSR_B200_BWD_PRECISION", env)
        enc.backward_precision = value
        with pytest.raises(AttributeError):
            enc(fake, None)
        return {m._inherited_backward_precision for m in subs}

    assert run("bf16") == {"bf16"}
    assert run(None) == {None}
    assert run(None, env="bf16") == {"bf16"}
    enc.backward_precision = "f16"
    with pytest.raises(ValueError, match="f16"):
        enc(fake, None)


def test_decoder_feed_forward_rejects_the_knob():
    """The decoder's feed-forward blocks are PositionwiseFeedForward too; the knob is an encoder option, so setting it
    there raises instead of being ignored."""
    from auto_avsr_b200.decoder_train import decoder_layer_train
    ff = PositionwiseFeedForward(128, 256, 0.0)
    ff.backward_precision = "bf16"
    with pytest.raises(ValueError, match="encoder option"):
        decoder_layer_train(types.SimpleNamespace(feed_forward=ff), None, None, None, None, "f16")


class _Ctx:
    def __init__(self, **kw):
        self.__dict__.update(kw)


class _RecordingLib:
    """Stands in for the library: records the name of every entry looked up and refuses to run it."""

    def __init__(self):
        self.seen = []

    def __getattr__(self, name):
        self.seen.append(name)
        raise AssertionError(f"unexpected library call {name}")


def test_linear_backward_is_one_library_call(monkeypatch):
    """Every backward precision makes one linear_bwd call for both GEMMs (avsr_linear_bwd: the library transposes and
    pads the operands) with the resolved precision: backward=None keeps bwd_precision, "bf16" passes through.  No
    ops.linear call and no other library call (no transpose) comes from Python."""
    calls = []
    monkeypatch.setattr(TR.ops, "linear", lambda *a, **kw: calls.append(("linear",)))
    monkeypatch.setattr(TR, "linear_bwd", lambda dy2, x2, w2, a, b, precision: calls.append((
        "linear_bwd", tuple(dy2.shape), tuple(x2.shape), tuple(w2.shape), a, b, precision)) or
        (torch.zeros(5, 8), torch.zeros(6, 8)))
    monkeypatch.setattr(TR, "colsum", lambda t: torch.zeros(t.shape[1]))
    rec = _RecordingLib()
    monkeypatch.setattr(TR, "lib", rec)
    x, w, dy = torch.zeros(5, 8), torch.zeros(6, 8), torch.zeros(5, 6)
    for prec, backward, want in (("f16", None, "tf32"), ("bf16", None, "tf32"), ("fp32", None, "fp32"),
                                 ("f16", "bf16", "bf16"), ("fp32", "bf16", "bf16")):
        calls.clear()
        ctx = _Ctx(saved_tensors=(x, w, None), relu=False, precision=prec, wshape=w.shape, has_bias=True,
                   backward=backward, needs_input_grad=(True, True, True))
        out = TR.LinearFn.backward(ctx, dy)
        assert len(out) == 6 and out[0].shape == x.shape and out[1].shape == w.shape
        assert calls == [("linear_bwd", (5, 6), (5, 8), (6, 8), True, True, want)]
    assert rec.seen == []


def test_pack_operand_and_linear_bwd_argument_errors_without_gpu():
    lib = _cabi.lib
    buf = C.create_string_buffer(1 << 12)
    p = C.addressof(buf)
    assert lib.avsr_pack_operand(None, p, 4, 4, 64, 1, PREC_BF16, None) == 1
    for prec in (PREC_F16, PREC_TF32, 7, -1):                                   # fp32 and bf16 only
        assert lib.avsr_pack_operand(p, p, 4, 4, 64, 1, prec, None) == 1
    assert lib.avsr_pack_operand(p, p, 65, 4, 64, 1, PREC_BF16, None) == 1     # ld < rows (transposed)
    assert lib.avsr_pack_operand(p, p, 4, 65, 64, 0, PREC_BF16, None) == 1     # ld < cols
    assert lib.avsr_pack_operand(p, p, 65, 4, 64, 1, PREC_FP32, None) == 1
    assert lib.avsr_pack_operand(p, p, 0, 4, 64, 1, PREC_BF16, None) == 0      # empty: nothing launched
    assert lib.avsr_pack_operand(p, p, 0, 4, 64, 1, PREC_FP32, None) == 0
    # workspace: [dY (rows, n padded) unless it is read in place,] W^T (k, n padded), dY^T (n, rows padded),
    # X^T (k, rows padded); K padded to 128 bytes
    ws = lib.avsr_linear_bwd_workspace_bytes(100, 6, 8, PREC_BF16)
    assert ws == _align(100 * 64 * 2) + _align(8 * 64 * 2) + _align(6 * 128 * 2) + _align(8 * 128 * 2)
    for prec in (PREC_FP32, PREC_TF32):
        assert lib.avsr_linear_bwd_workspace_bytes(100, 6, 8, prec) == (
            _align(100 * 32 * 4) + _align(8 * 32 * 4) + _align(6 * 128 * 4) + _align(8 * 128 * 4))
        assert lib.avsr_linear_bwd_workspace_bytes(100, 64, 8, prec) == (     # n % 32 == 0: dY read in place
            _align(8 * 64 * 4) + _align(64 * 128 * 4) + _align(8 * 128 * 4))
    assert lib.avsr_linear_bwd_workspace_bytes(100, 64, 8, PREC_BF16) == (
        _align(100 * 64 * 2) + _align(8 * 64 * 2) + _align(64 * 128 * 2) + _align(8 * 128 * 2))
    for prec in (PREC_F16, 7, -1):
        assert lib.avsr_linear_bwd_workspace_bytes(100, 6, 8, prec) == 0
    assert lib.avsr_linear_bwd(p, p, p, None, None, 100, 6, 8, PREC_BF16, p, ws, None) == 1   # neither output wanted
    assert lib.avsr_linear_bwd(p, None, p, None, p, 100, 6, 8, PREC_BF16, p, ws, None) == 1   # dw without x
    assert lib.avsr_linear_bwd(p, p, p, p, p, 0, 6, 8, PREC_BF16, p, ws, None) == 1
    assert lib.avsr_linear_bwd(p, p, p, p, p, 100, 6, 8, PREC_BF16, p, ws - 1, None) == 3
    assert lib.avsr_linear_bwd(p, p, p, p, p, 100, 6, 8, PREC_F16, p, ws, None) == 1          # gradients overflow f16
    assert b"overflow f16" in lib.avsr_last_error()
    assert lib.avsr_linear_bwd(p, p, p, p, p, 100, 6, 8, 7, p, ws, None) == 1


def test_attention_backward_arguments(monkeypatch):
    seen = []
    monkeypatch.setattr(TR, "relpos_attention_bwd", lambda *a, precision: seen.append(precision) or
                        tuple(torch.zeros(1, 2, 64) for _ in range(4)) + (torch.zeros(3, 64),))
    monkeypatch.setattr(TR, "colsum", lambda t: torch.zeros(t.shape[1]))
    q = torch.zeros(1, 2, 64)
    saved = (q, q, q, torch.zeros(3, 64), torch.zeros(1, 64), torch.zeros(1, 64), q, torch.empty(0))
    for backward, want in ((None, "fp32"), ("bf16", "bf16")):
        ctx = _Ctx(saved_tensors=saved, n_heads=1, masked=False, backward=backward)
        assert len(TR.AttentionCoreFn.backward(ctx, q)) == 10
        assert seen[-1] == want


def test_attention_backward_precision_checked():
    q = torch.zeros(1, 2, 64)
    with pytest.raises(ValueError, match="f16"):
        TR.relpos_attention_bwd(q, q, q, torch.zeros(3, 64), q[0, :1], q[0, :1], None, q, q, 1, precision="f16")


# ------------------------------------------------------------------------------------------------ C ABI
def _align(n):
    return (n + 255) // 256 * 256


def dp_chunks(B, T, H):
    """bw_dp_chunks: utterance chunks of the dp kernel (enough CTAs for 2 per SM on 132 SMs) -> (chunks, per chunk)"""
    nd = 2 * ((T + 63) // 64) - 1
    want = min(max((2 * 132) // (H * nd), 1), B)
    per = -(-B // want)
    return -(-B // per), per


def workspace_formula(B, T, H):
    N, D, R, nd = B * T, H * 64, 2 * T - 1, 2 * ((T + 63) // 64) - 1
    chunks = dp_chunks(B, T, H)[0]
    return (5 * _align(N * D * 2) + _align(R * D * 2) + 2 * _align(B * H * T * 4) +
            _align(H * nd * chunks * 128 * 64 * 4))


@pytest.mark.parametrize("B,T,H", [(1, 1, 1), (2, 9, 2), (4, 400, 12), (1, 1600, 2), (5, 400, 12), (200, 8, 12),
                                   (16, 100, 12)])
def test_workspace_formula(B, T, H):
    assert _cabi.lib.avsr_relpos_attention_bwd_tc_workspace_bytes(B, T, H, PREC_BF16) == workspace_formula(B, T, H)


def test_workspace_edges():
    f = _cabi.lib.avsr_relpos_attention_bwd_tc_workspace_bytes
    assert f(0, 9, 2, PREC_BF16) == 256 and f(2, 0, 2, PREC_BF16) == 256 and f(2, 9, 0, PREC_BF16) == 256
    for p in (PREC_FP32, PREC_TF32, PREC_F16, 7, -1):
        assert f(2, 9, 2, p) == 0


def test_entry_argument_errors_without_gpu():
    lib = _cabi.lib
    buf = C.create_string_buffer(1 << 16)
    p = C.addressof(buf)
    ws = lib.avsr_relpos_attention_bwd_tc_workspace_bytes(2, 9, 4, PREC_BF16)

    def call(args14, B, T, H, prec, w, nbytes):
        return lib.avsr_relpos_attention_bwd_tc(*args14, B, T, H, prec, w, nbytes, None)

    ptrs = [p] * 14
    ptrs[6] = None                                     # lengths may be NULL
    assert call([None] + ptrs[1:], 2, 9, 4, PREC_BF16, p, ws) == 1
    assert b"NULL" in lib.avsr_last_error()
    assert call(ptrs, 2, 9, 4, PREC_BF16, None, ws) == 1
    for prec, name in ((PREC_F16, b"AVSR_PREC_F16"), (PREC_TF32, b"AVSR_PREC_TF32"), (PREC_FP32, b"AVSR_PREC_FP32")):
        assert call(ptrs, 2, 9, 4, prec, p, ws) == 1
        assert name in lib.avsr_last_error()
    assert call(ptrs, 2, 9, 4, PREC_BF16, p, ws - 1) == 3
    assert b"too small" in lib.avsr_last_error()
    assert call(ptrs, 0, 9, 4, PREC_BF16, p, 0) == 0   # nothing to do: nothing launched
    assert call(ptrs, 2, 0, 4, PREC_BF16, p, 0) == 0


# ------------------------------------------------------------------------------------------------ dp mapping
def dp_contributions(T, lengths, H=1):
    """Host restatement of attn_bwd_tc_dp_kernel + attn_bwd_tc_dp_fixup_kernel: for every (b, i, j) with j < len[b],
    the (diagonal index, utterance chunk, band row) the dp kernel accumulates it into, then the table rows the fix-up
    reads each band row for, in the fix-up's order.  Returns {m: [(b, i, j), ...]} in summation order."""
    nT = (T + 63) // 64
    nd = 2 * nT - 1
    chunks, per = dp_chunks(len(lengths), T, H)
    band = {}                                          # (di, z, r) -> [(b, i, j)] in the kernel's order
    for di, z in ((di, z) for di in range(nd) for z in range(chunks)):
        dd = di - (nT - 1)
        for b in range(z * per, min(len(lengths), (z + 1) * per)):
            L = lengths[b]
            for qt in range(max(0, -dd), min(nT, nT - dd)):
                i0, j0 = 64 * qt, 64 * (qt + dd)
                if j0 >= L:
                    continue
                for rr in range(64):
                    for c in range(64):
                        i, j = i0 + rr, j0 + c
                        if i >= T or j >= L:
                            continue           # A = 0: rows past T (infinite lse) and masked keys
                        band.setdefault((di, z, c + 63 - rr), []).append((b, i, j))
    out = {}
    for m in range(2 * T - 1):
        off = m + 64 * nT - T
        assert off >= 0
        hi = off // 64
        order = []
        di = max(hi - 1, 0)
        while di <= hi and di < nd:
            r = off - 64 * di
            if r < 127:
                order.append(di)
                for z in range(chunks):
                    out.setdefault(m, []).extend(band.get((di, z, r), []))
            di += 1
        assert order == sorted(order) and len(order) <= 2
    return out


@pytest.mark.parametrize("T,H", [(1, 1), (63, 1), (64, 12), (65, 1), (400, 12), (1600, 1), (8, 12), (100, 12)])
def test_dp_band_mapping_covers_each_pair_once(T, H):
    """(8, 12) and (100, 12): few diagonals, so the utterances are split into chunks (200 x 8 at 12 heads: 20 chunks)."""
    lengths = {65: [65, 58, 1], 400: [400, 393, 1], 8: [8 - (b % 8) for b in range(200)],
               100: [100 - 3 * b for b in range(16)]}.get(T, [T])
    if T in (8, 100):
        assert dp_chunks(len(lengths), T, H)[0] > 1
    got = dp_contributions(T, lengths, H)
    seen = set()
    for m, pairs in got.items():
        for (b, i, j) in pairs:
            assert j - i + T - 1 == m, (T, m, b, i, j)
            assert (b, i, j) not in seen
            seen.add((b, i, j))
    want = sum(T * L for L in lengths)
    assert len(seen) == want
