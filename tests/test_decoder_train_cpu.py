"""CPU checks of the decoder's training kernels (csrc/decoder_train.cu) without a GPU: the masks, dropout factors,
softmax / backward combination, label-smoothing and embedding math of csrc/decoder_train_body.cuh, compiled into the host
replay of tests/emu (same source, the kernels' schedule as plain loops) and called through the package's ctypes
signatures, against the reference's own MultiHeadedAttention (a given keep-mask patched in as its dropout),
LabelSmoothingLoss and PositionalEncoding in float64.  Also the drop-in contract: install_decoder re-homes the criterion
with the same parameters, and masks / tensors the CUDA path cannot take are refused.  The GPU side is
tests/test_zz_gpu_decoder_train.py."""
import ctypes as C
import importlib.util
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "avsr_b200.h")
REF_T = os.path.join(ROOT, "oracle", "_ref", "espnet", "nets", "pytorch_backend", "transformer")
HAVE_NVCC = os.path.exists("/usr/local/cuda/bin/nvcc")
needs_ref = pytest.mark.skipif(not os.path.isdir(REF_T), reason="oracle/_ref not built")


def _ref_module(name):
    """one reference file of oracle/_ref, loaded by path under a private name (no espnet package on sys.path)"""
    spec = importlib.util.spec_from_file_location("_ref_" + name, os.path.join(REF_T, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def emu():
    if not HAVE_NVCC:
        pytest.skip("nvcc is needed to build the host replay")
    from emu import build
    return build.load("decoder_train")


# ------------------------------------------------------------------ attention core
def emu_mha(lib, q, k, v, H, causal, lengths, keep, scale, dctx):
    B, Lq, D = q.shape
    Lk = k.size(1)
    ctx = torch.empty(B, Lq, D)
    probs = torch.empty(B, H, Lq, Lk)
    ln = None if lengths is None else torch.tensor(lengths, dtype=torch.int32)
    kp = None if keep is None else keep.contiguous()
    lp = None if ln is None else ln.data_ptr()
    kpp = None if kp is None else kp.data_ptr()
    rc = lib.avsr_mha_core_fwd(q.data_ptr(), D, k.data_ptr(), D, v.data_ptr(), D, B, H, Lq, Lk, int(causal), lp, kpp,
                               scale, ctx.data_ptr(), probs.data_ptr(), None)
    assert rc == 0, lib.avsr_last_error()
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    ws = torch.empty(int(lib.avsr_mha_core_bwd_workspace_bytes(B, H, Lq)), dtype=torch.uint8)
    rc = lib.avsr_mha_core_bwd(q.data_ptr(), D, k.data_ptr(), D, v.data_ptr(), D, B, H, Lq, Lk, int(causal), lp, kpp, scale,
                               probs.data_ptr(), dctx.data_ptr(), dq.data_ptr(), D, dk.data_ptr(), dv.data_ptr(), D,
                               ws.data_ptr(), ws.numel(), None)
    assert rc == 0, lib.avsr_last_error()
    return ctx, probs, dq, dk, dv


class _KeepDropout(torch.nn.Module):
    """the reference's attention dropout with a given keep-mask"""

    def __init__(self, keep, scale):
        super().__init__()
        self.keep, self.scale = keep, scale

    def forward(self, x):
        return x if self.keep is None else x * self.keep.double() * self.scale


def ref_mha(q, k, v, H, causal, lengths, keep, scale, dctx):
    """MultiHeadedAttention.forward_attention (attention.py:59-88) in float64 on the given projected q, k, v (linear_out
    = identity) -> ctx, attn, dq, dk, dv."""
    A = _ref_module("attention")
    B, Lq, D = q.shape
    Lk = k.size(1)
    m = A.MultiHeadedAttention(H, D, 0.0).double()
    with torch.no_grad():
        m.linear_out.weight.copy_(torch.eye(D, dtype=torch.float64))
        m.linear_out.bias.zero_()
    m.dropout = _KeepDropout(keep, scale)
    heads = lambda t: t.double().view(B, -1, H, 64).transpose(1, 2).contiguous().requires_grad_(True)   # noqa: E731
    qh, kh, vh = heads(q), heads(k), heads(v)
    kl = torch.tensor(lengths if lengths is not None else [Lk] * B)
    mask = (torch.arange(Lk)[None, None, :] < kl[:, None, None])                        # (B, 1, Lk)
    if causal:
        mask = mask & (torch.arange(Lk)[None, None, :] <= torch.arange(Lq)[None, :, None])
    scores = qh @ kh.transpose(-2, -1) / math.sqrt(64)
    out = m.forward_attention(vh, scores, mask)
    (out * dctx.double()).sum().backward()
    back = lambda t: t.transpose(1, 2).reshape(B, -1, D)                                 # noqa: E731
    return out.detach(), m.attn.detach(), back(qh.grad), back(kh.grad), back(vh.grad)


MHA_CASES = [  # (B, H, Lq, Lk, causal, lengths, p)
    (3, 2, 7, 7, True, [7, 4, 0], 0.0),
    (3, 2, 7, 7, True, [7, 5, 2], 0.1),
    (2, 1, 5, 19, False, [19, 0], 0.0),
    (3, 2, 6, 40, False, [40, 33, 1], 0.1),
    (1, 3, 1, 1, True, None, 0.0),
    (2, 1, 33, 70, False, None, 0.3),
]


@needs_ref
@pytest.mark.parametrize("case", range(len(MHA_CASES)))
def test_mha_core_replay_matches_reference_attention(emu, case):
    B, H, Lq, Lk, causal, lengths, p = MHA_CASES[case]
    g = torch.Generator().manual_seed(10 + case)
    D = H * 64
    q, k, v = (torch.randn(B, L, D, generator=g) for L in (Lq, Lk, Lk))
    dctx = torch.randn(B, Lq, D, generator=g)
    keep = (torch.rand(B, H, Lq, Lk, generator=g) >= p).to(torch.uint8) if p > 0 else None
    scale = 1.0 / (1.0 - p)
    ctx, probs, dq, dk, dv = emu_mha(emu, q, k, v, H, causal, lengths, keep, scale, dctx)
    rctx, rattn, rdq, rdk, rdv = ref_mha(q, k, v, H, causal, lengths, keep, scale, dctx)
    for got, want, tol in ((ctx, rctx, 2e-5), (probs, rattn, 2e-6), (dq, rdq, 2e-5), (dk, rdk, 2e-5), (dv, rdv, 2e-5)):
        err = (got.double() - want).abs().max().item()
        assert err < tol * max(1.0, want.abs().max().item()), (err, tol)
    if lengths is not None and 0 in lengths:
        b = lengths.index(0)
        assert (ctx[b] == 0).all() and (probs[b] == 0).all() and (dq[b] == 0).all() and (dk[b] == 0).all()


# ------------------------------------------------------------------ label smoothing
def emu_ls(lib, x, target, odim, smoothing, ld, dscale):
    rows = x.size(0)
    buf = torch.full((rows, ld), 1e4)                    # padding columns must be ignored
    buf[:, :odim] = x
    tg = target.to(torch.int64).contiguous()
    loss, lse = torch.empty(rows), torch.empty(rows)
    assert lib.avsr_label_smoothing_fwd(buf.data_ptr(), ld, tg.data_ptr(), rows, odim, -1, smoothing, loss.data_ptr(),
                                        lse.data_ptr(), None) == 0
    d = torch.full((rows, ld), 7.0)
    ds = torch.tensor([dscale])
    assert lib.avsr_label_smoothing_bwd(buf.data_ptr(), ld, tg.data_ptr(), rows, odim, -1, smoothing, lse.data_ptr(),
                                        ds.data_ptr(), d.data_ptr(), ld, None) == 0
    return loss, d


@needs_ref
@pytest.mark.parametrize("smoothing", [0.0, 0.1])
@pytest.mark.parametrize("odim,ld,scale", [(37, 40, 3.0), (50, 50, 30.0), (5049, 5056, 4.0)])
def test_label_smoothing_replay_matches_reference_loss(emu, smoothing, odim, ld, scale):
    LS = _ref_module("label_smoothing_loss")
    g = torch.Generator().manual_seed(odim)
    B, L = 3, 5
    x = torch.randn(B, L, odim, generator=g) * scale
    t = torch.randint(0, odim, (B, L), generator=g)
    t[0, 3:] = -1
    t[2, :] = -1                                          # an all-ignored utterance
    crit = LS.LabelSmoothingLoss(odim, -1, smoothing, False)
    xr = x.double().requires_grad_(True)
    ref = crit(xr, t)
    ref.backward()
    rows, d = emu_ls(emu, x.reshape(-1, odim), t.reshape(-1), odim, smoothing, ld, 1.0 / B)
    got = rows.double().sum() / B
    assert abs(got.item() - ref.item()) < 2e-6 * max(1.0, abs(ref.item())) * math.sqrt(odim / 37)
    assert (d[:, odim:] == 0).all()
    ign = (t.reshape(-1) == -1)
    assert (d[ign] == 0).all() and (rows[ign] == 0).all()
    # fp32 log-sum-exp: the softmax carries a relative error of about eps * |logits|, plus the rounding of the replay's
    # sequential sum of exp over odim columns
    tol = 3e-8 * max(1.0, x.abs().max().item()) + 1e-9 * odim
    assert (d[:, :odim].double() - xr.grad.reshape(-1, odim)).abs().max().item() < tol


def test_label_smoothing_bad_target_gives_nan_row_only(emu):
    x = torch.randn(3, 9)
    loss, d = emu_ls(emu, x, torch.tensor([2, 9, -1]), 9, 0.1, 12, 1.0)
    assert torch.isfinite(loss[0]) and torch.isnan(loss[1]) and loss[2] == 0
    assert torch.isfinite(d[0]).all() and torch.isnan(d[1, :9]).all() and (d[1, 9:] == 0).all() and (d[2] == 0).all()


# ------------------------------------------------------------------ embedding
@needs_ref
def test_embedding_replay_matches_reference_positional_encoding(emu):
    E = _ref_module("embedding")
    g = torch.Generator().manual_seed(4)
    odim, D, B, L = 23, 128, 3, 9
    w = torch.randn(odim, D, generator=g)
    tok = torch.randint(0, odim, (B, L), generator=g)
    tok[1, :] = 5                                         # one token at many positions
    tok[2, 4] = odim                                      # out of range: NaN row, no gradient
    x = torch.empty(B, L, D)
    assert emu.avsr_embed_fwd(tok.data_ptr(), w.data_ptr(), B * L, L, D, odim, x.data_ptr(), None) == 0
    pe = E.PositionalEncoding(D, 0.0)
    ok = tok.clamp(max=odim - 1)
    wr = w.double().requires_grad_(True)
    ref = pe(torch.nn.functional.embedding(ok, wr))      # x * sqrt(d) + pe[:L] (embedding.py:80-90) in float64
    bad = torch.zeros(B, L, dtype=torch.bool)
    bad[2, 4] = True
    assert torch.isnan(x[bad]).all() and torch.isfinite(x[~bad]).all()
    assert (x[~bad].double() - ref[~bad]).abs().max().item() < 2e-5 * ref.abs().max().item()
    dx = torch.randn(B, L, D, generator=g)
    (ref * dx.double().masked_fill(bad[..., None], 0.0)).sum().backward()
    dw = torch.empty(odim, D)
    ws = torch.empty(int(emu.avsr_embed_bwd_workspace_bytes(B * L, odim)), dtype=torch.uint8)
    assert emu.avsr_embed_bwd(tok.data_ptr(), dx.data_ptr(), B * L, D, odim, dw.data_ptr(), ws.data_ptr(), ws.numel(), None) == 0
    assert (dw.double() - wr.grad).abs().max().item() < 2e-5 * wr.grad.abs().max().item()
    unused = sorted(set(range(odim)) - set(tok.flatten().tolist()))
    assert unused and (dw[unused] == 0).all()


# ------------------------------------------------------------------ drop-in contract
def test_target_mask_forms_and_refusals():
    from auto_avsr_b200.decoder_train import target_lengths
    B, L = 3, 6
    lens = torch.tensor([6, 4, 0])
    ar = torch.arange(L)
    m = (ar[None, None, :] < lens[:, None, None]) & (ar[None, None, :] <= ar[None, :, None])
    assert target_lengths(m, B, L, check_mask=True).tolist() == [6, 4, 0]
    with pytest.raises(NotImplementedError):
        target_lengths(None, B, L)
    with pytest.raises(NotImplementedError):
        target_lengths(m[:, :1, :], B, L)                 # (B, 1, L): no causal structure
    with pytest.raises(NotImplementedError):
        target_lengths(torch.ones(B, L, L, dtype=torch.bool), B, L, check_mask=True)    # not causal
    holes = m.clone()
    holes[0, :, 2] = False
    with pytest.raises(NotImplementedError):
        target_lengths(holes, B, L, check_mask=True)


def test_decoder_forward_and_loss_refuse_cpu_and_unsupported_options():
    from auto_avsr_b200 import LabelSmoothingLoss, TransformerDecoder
    dec = TransformerDecoder(odim=11, attention_dim=64, attention_heads=1, linear_units=64, num_blocks=1).train()
    ys = torch.tensor([[10, 3, 4]])
    mask = torch.tril(torch.ones(1, 3, 3, dtype=torch.bool))
    with pytest.raises(NotImplementedError):
        dec(ys, mask, torch.zeros(1, 5, 64), None)
    crit = LabelSmoothingLoss(11, -1, 0.1, False)
    assert (crit.size, crit.padding_idx, crit.smoothing, crit.confidence, crit.normalize_length, crit.true_dist) == \
        (11, -1, 0.1, 0.9, False, None)
    assert isinstance(crit.criterion, torch.nn.KLDivLoss) and list(crit.state_dict()) == []
    with pytest.raises(NotImplementedError):
        crit(torch.zeros(1, 3, 11), ys)
    with pytest.raises(NotImplementedError):
        LabelSmoothingLoss(11, -1, 0.1, True)(torch.zeros(1, 3, 11), ys)
    with pytest.raises(NotImplementedError):
        LabelSmoothingLoss(11, -1, 0.1, False, torch.nn.MSELoss())(torch.zeros(1, 3, 11), ys)


@pytest.mark.skipif(not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "espnet")), reason="oracle/_ref not built")
def test_install_decoder_rehomes_the_criterion_and_keeps_parameters():
    code = f"""
import sys
sys.path.insert(0, {ROOT!r})
from oracle import build_ref
ref = build_ref.import_reference_search()
import torch
import auto_avsr_b200
from espnet.nets.pytorch_backend.transformer.label_smoothing_loss import LabelSmoothingLoss as RefLS

class Shell(torch.nn.Module):          # the members of E2E the training / decoding paths touch (e2e_asr_conformer.py:41-59)
    def __init__(self):
        super().__init__()
        self.decoder = ref["TransformerDecoder"](odim=37, attention_dim=128, attention_heads=2, linear_units=256, num_blocks=2,
                                                 dropout_rate=0.2, self_attention_dropout_rate=0.3,
                                                 src_attention_dropout_rate=0.4, positional_dropout_rate=0.15)
        self.ctc = ref["CTC"](37, 128, 0.1, reduce=True)
        self.criterion = RefLS(37, -1, 0.1, False)

m = Shell().train()
keys = list(m.state_dict().keys())
params = {{id(p) for p in m.parameters()}}
auto_avsr_b200.install_decoder(m)
assert type(m.criterion).__module__ == "auto_avsr_b200.espnet_dropin.label_smoothing_loss"
assert (m.criterion.size, m.criterion.padding_idx, m.criterion.smoothing, m.criterion.normalize_length) == (37, -1, 0.1, False)
assert list(m.state_dict().keys()) == keys and params == {{id(p) for p in m.parameters()}}
d = m.decoder
assert d.training and m.criterion.training
assert d.embed[1].dropout.p == 0.15 and d.decoders[1].dropout.p == 0.2 and d.decoders[0].feed_forward.dropout.p == 0.2
assert d.decoders[0].self_attn.dropout.p == 0.3 and d.decoders[1].src_attn.dropout.p == 0.4
print("OK")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr[-2000:]


_CTYPE = {"int": C.c_int, "long": C.c_long, "size_t": C.c_size_t, "float": C.c_float}


def test_decoder_train_signatures_match_the_header():
    from auto_avsr_b200 import _cabi
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for name in ("avsr_mha_core_fwd", "avsr_mha_core_bwd_workspace_bytes", "avsr_mha_core_bwd", "avsr_label_smoothing_fwd",
                 "avsr_label_smoothing_bwd", "avsr_embed_fwd", "avsr_embed_bwd_workspace_bytes", "avsr_embed_bwd"):
        m = re.search(r"(\w+)\s+" + name + r"\s*\(([^)]*)\)", src)
        assert m, name
        ret, params = m.group(1), [p.strip() for p in m.group(2).split(",")]
        want = [C.c_void_p if "*" in p else _CTYPE[p.split()[0]] for p in params]
        res, args = _cabi.SIGNATURES[name]
        assert res == _CTYPE[ret], name
        assert args == want, (name, args, want)


@pytest.mark.skipif(not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "espnet")), reason="oracle/_ref not built")
@pytest.mark.parametrize("name", ["decoder_train_tiny", "decoder_train_full"])
def test_fixtures_reproduce_from_reference_copy(name, golden_dir):
    code = f"""
import sys, numpy as np
sys.path.insert(0, {ROOT!r})
from oracle import make_golden_decoder_train as M
z = np.load({os.path.join(golden_dir, name + ".npz")!r})
got = M.reference({name!r})
assert set(got) == set(z.files), (sorted(got), z.files)
for k, v in got.items():
    assert np.allclose(v, z[k], rtol=1e-6, atol=1e-9), k
print("OK")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr[-2000:]
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    if name == "decoder_train_tiny":                     # one empty label row: its only target is <eos>
        assert (z["ys_pad"] == -1).all(axis=1).sum() == 1
