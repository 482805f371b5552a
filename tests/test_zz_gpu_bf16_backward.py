"""The opt-in bf16 backward of the encoder (``backward_precision="bf16"``): the tensor-core rel-pos attention backward
(csrc/attention_bwd_tc.cu, avsr_relpos_attention_bwd_tc) against float64 restatements computed on the same GPU, its
determinism and range, float64 references with one defect each that must miss it, and the 2-layer / 12-layer encoder
in train() with the knob set.

Errors are max-abs differences over the reference's max-abs; bounds are about 4x what the H100 shows.  bf16 keeps 8
mantissa bits, so the attention bounds are in the 1e-2 class (the fp32 kernels' are 1e-6).  Where it is stated, the
library must also be within 2x of what torch.autocast(bfloat16) makes of the same restatement.

Cost on one H100 (700 W): about 20 s of test time; peak torch.cuda.max_memory_allocated 4.2 GB (the float64
restatements at (4, 400, 12) and (1, 1600, 2)).  Observed attention errors 2e-3 .. 1.2e-2 (bound 3e-2); 2-layer encoder
4.2e-3 (bound 1.7e-2); 12-layer S2 gradients against the default backward 1.7e-2 (bound 6e-2); Linear backward GEMMs
2.3e-3 .. 3.2e-3 (bound 1.2e-2)."""
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, record
from auto_avsr_b200.synthetic import SHAPES, encoder_state_dict

pytestmark = pytest.mark.gpu

D, F, K = 768, 3072, 31


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "needs a CUDA GPU"
    import __graft_entry__ as g
    g.build()
    torch.cuda.reset_peak_memory_stats()
    yield torch.device("cuda:0")
    record("bf16_backward_peak_memory", ("max_memory_allocated GB",), torch.cuda.max_memory_allocated() / 2 ** 30, 8.0)


def gen(seed, dev):
    return torch.Generator(device=dev).manual_seed(seed)


def rel(a, ref):
    if ref.numel() == 0:
        return 0.0
    d = (a.double() - ref.double()).abs().max().item()
    return d / max(ref.double().abs().max().item(), 1e-300) if d > 0 else 0.0


def ref_attention(q, k, v, p, u, vb, lengths, H):
    """attention.py:59-82 / 174-189 with the key mask of attention.py:73-77 (finfo.min, softmax, masked_fill 0), under
    autograd; the query enters as two leaves so that its two gradient parts come out separately (the restatement of
    test_zz_gpu_train_kernels.py)."""
    B, T, Dm = q.shape
    qa, qb = q.clone().requires_grad_(True), q.clone().requires_grad_(True)
    kk, vv, pp, uu, vv_b = (t.clone().requires_grad_(True) for t in (k, v, p, u, vb))
    heads = lambda t: t.view(t.size(0), -1, H, 64).transpose(1, 2)          # noqa: E731
    ac = (heads(qa) + uu[None, :, None]) @ heads(kk).transpose(-1, -2)
    bd_full = (heads(qb) + vv_b[None, :, None]) @ pp.view(2 * T - 1, H, 64).permute(1, 2, 0)
    i = torch.arange(T, device=q.device)
    idx = (i[None, :] - i[:, None] + T - 1).expand(B, H, T, T)
    s = (ac + bd_full.gather(-1, idx)) / 8.0
    if lengths is not None:
        mask = (i[None, :] >= torch.as_tensor(lengths, device=q.device)[:, None])[:, None, None, :]
        s = s.masked_fill(mask, torch.finfo(s.dtype).min)
        a = torch.softmax(s, -1).masked_fill(mask, 0.0)
    else:
        a = torch.softmax(s, -1)
    ctx = (a @ heads(vv)).transpose(1, 2).reshape(B, T, Dm)
    return ctx, (qa, qb, kk, vv, pp, uu, vv_b)


def ref_grads(q, k, v, p, u, vb, lengths, H, dctx):
    ctx, (qa, qb, kk, vv, pp, uu, vv_b) = ref_attention(q, k, v, p, u, vb, lengths, H)
    (ctx * dctx).sum().backward()
    return {"dq": qa.grad + qb.grad, "dk": kk.grad, "dv": vv.grad, "dp": pp.grad, "d pos_bias_u": uu.grad,
            "d pos_bias_v": vv_b.grad, "dq_k": qa.grad, "dq_p": qb.grad}


def manual_grads(q, k, v, p, u, vb, lengths, H, dctx, defect=None):
    """The closed-form backward in float64 (attention_bwd.cu's header), with one optional defect: "skew" (dq_p takes
    the table row one off), "band" (the dp partial of one tile diagonal dropped), "delta" (Delta omitted), "mask" (key
    mask shifted by one)."""
    B, T, Dm = q.shape
    heads = lambda t: t.view(t.size(0), -1, H, 64).transpose(1, 2)          # noqa: E731
    qu, qv = heads(q) + u[None, :, None], heads(q) + vb[None, :, None]
    kh, vh, dc = heads(k), heads(v), heads(dctx)
    ph = p.view(2 * T - 1, H, 64).permute(1, 0, 2)                          # (H, R, 64)
    i = torch.arange(T, device=q.device)
    m = (i[None, :] - i[:, None] + T - 1)                                   # (T, T): row m of (i, j)
    pg = ph[:, m]                                                           # (H, T, T, 64)
    s = (qu @ kh.transpose(-1, -2) + torch.einsum("bhid,hijd->bhij", qv, pg)) / 8.0
    L = torch.as_tensor(lengths if lengths is not None else [T] * B, device=q.device)
    if defect == "mask":
        L = L + 1
    keep = (i[None, :] < L[:, None])[:, None, None, :]
    a = torch.softmax(s.masked_fill(~keep, -float("inf")), -1).nan_to_num(0.0).masked_fill(~keep, 0.0)
    dP = dc @ vh.transpose(-1, -2)
    delta = (a * dP).sum(-1, keepdim=True) if defect != "delta" else 0.0
    g = a * (dP - delta) / 8.0
    dq_k = g @ kh
    mq = m if defect != "skew" else (m + 1).clamp(max=2 * T - 2)
    dq_p = torch.einsum("bhij,hijd->bhid", g, ph[:, mq])
    dk = g.transpose(-1, -2) @ qu
    dv = a.transpose(-1, -2) @ dc
    contrib = torch.einsum("bhij,bhid->hijd", g, qv)                        # (H, T, T, 64), summed into row m(i, j)
    if defect == "band":
        J, I = torch.meshgrid(i // 64, i // 64, indexing="xy")              # (T, T): [i, j] -> (I, J)
        contrib = contrib * ((J - I) != 0).to(contrib.dtype)[None, :, :, None]
    dph = torch.zeros(H, 2 * T - 1, 64, dtype=q.dtype, device=q.device)
    dph.index_add_(1, m.reshape(-1), contrib.reshape(H, T * T, 64))
    back = lambda t: t.transpose(1, 2).reshape(B, T, Dm)                   # noqa: E731
    dp = dph.permute(1, 0, 2).reshape(2 * T - 1, Dm)
    return {"dq": back(dq_k + dq_p), "dk": back(dk), "dv": back(dv), "dp": dp, "dq_k": back(dq_k), "dq_p": back(dq_p)}


def inputs(B, T, H, seed, dev):
    g = gen(seed, dev)
    Dm = H * 64
    q, k, v = (torch.randn(B, T, Dm, device=dev, generator=g) for _ in range(3))
    p = torch.randn(2 * T - 1, Dm, device=dev, generator=g)
    u, vb = (0.5 * torch.randn(H, 64, device=dev, generator=g) for _ in range(2))
    r = torch.randn(B, T, Dm, device=dev, generator=g)
    return q, k, v, p, u, vb, r


def library(q, k, v, p, u, vb, ln, H, r, forward="bf16"):
    """AttentionCoreFn with the bf16 backward -> the nine outputs test_relpos_attention_bwd_vs_fp64 checks."""
    from auto_avsr_b200.train import AttentionCoreFn, relpos_attention_bwd
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v, p, u, vb)]
    out = AttentionCoreFn.apply(*leaves, ln, H, forward, "bf16")
    (out * r).sum().backward()
    parts = relpos_attention_bwd(q, k, v, p, u, vb, ln, out.detach(), r, H, precision="bf16")
    names = ["ctx", "dq", "dk", "dv", "dp", "d pos_bias_u", "d pos_bias_v", "dq_k", "dq_p"]
    return dict(zip(names, [out.detach()] + [t.grad for t in leaves] + list(parts[:2])))


# ------------------------------------------------------------------------------------------------ against float64
ATT_CASES = [(1, 1, 1, None), (2, 9, 2, [0, 9]), (3, 33, 3, [33, 32, 1]), (2, 65, 2, [65, 64]), (1, 130, 12, None),
             (4, 400, 12, [400, 333, 7, 129]), (1, 1600, 2, None), (5, 400, 12, SHAPES["S2r"]),
             (200, 8, 2, [8 - (b % 8) for b in range(200)])]
BF16_TOL = 3e-2
AUTOCAST_CASES = {(4, 400, 12), (1, 1600, 2)}


@pytest.mark.parametrize("B,T,H,lengths", ATT_CASES)
def test_bf16_attention_bwd_vs_fp64(dev, B, T, H, lengths):
    """Query / key tiles of 64 with ragged tails, tables of 2T-1 rows, many tile diagonals, zero-length and one-frame
    utterances, more utterances than SMs.  The forward runs in fp32, so the errors are the backward's."""
    q, k, v, p, u, vb, r = inputs(B, T, H, B * 100000 + T * 100 + H, dev)
    ln = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=dev)
    got = library(q, k, v, p, u, vb, ln, H, r, forward="fp32")
    want = ref_grads(*(t.double() for t in (q, k, v, p, u, vb)), lengths, H, r.double())
    errs = {n: rel(got[n], want[n]) for n in want}
    if T == 1:          # one key: every score gradient is 0 exactly; absolute against the scale of dv
        scale = want["dv"].abs().max().item()
        errs.update({n: (got[n].double() - want[n]).abs().max().item() / scale for n in want if n != "dv"})
    for n, e in errs.items():
        record("bf16_attention_bwd", (B, T, H, str(lengths), n), e, BF16_TOL)
    assert all(torch.isfinite(t).all() for t in got.values())
    if lengths is not None and 0 in lengths:
        z = lengths.index(0)
        assert not got["dq"][z].any() and not got["dk"][z].any() and not got["dv"][z].any()
    bad = {n: e for n, e in errs.items() if not e < BF16_TOL}
    assert not bad, bad
    if (B, T, H) in AUTOCAST_CASES:
        with torch.autocast("cuda", dtype=torch.bfloat16):
            mixed = ref_grads(q, k, v, p, u, vb, lengths, H, r)
        for n in want:
            e_torch = rel(mixed[n].float(), want[n])
            record("bf16_attention_bwd_vs_autocast", (B, T, H, n, "autocast error"), e_torch, BF16_TOL)
            assert errs[n] <= 2 * e_torch, (n, errs[n], e_torch)


def test_bf16_attention_bwd_deterministic(dev):
    """Two calls, and a call on another stream, give the same bits: no atomics, every sum in a fixed order."""
    from auto_avsr_b200.train import relpos_attention_bwd
    B, T, H = 4, 400, 12
    q, k, v, p, u, vb, r = inputs(B, T, H, 7, dev)
    ln = torch.tensor([400, 333, 7, 129], dtype=torch.int32, device=dev)
    out = torch.randn(B, T, H * 64, device=dev, generator=gen(8, dev))
    a = relpos_attention_bwd(q, k, v, p, u, vb, ln, out, r, H, precision="bf16")
    b = relpos_attention_bwd(q, k, v, p, u, vb, ln, out, r, H, precision="bf16")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c = relpos_attention_bwd(q, k, v, p, u, vb, ln, out, r, H, precision="bf16")
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_bf16_attention_bwd_range(dev):
    """dctx x 2^20: gradients pass fp16's 65504 and stay finite, within the scale-1 bound (bf16 has fp32's range)."""
    B, T, H, lengths = 4, 400, 12, [400, 333, 7, 129]
    q, k, v, p, u, vb, r = inputs(B, T, H, 11, dev)
    r = r * 2.0 ** 20
    ln = torch.tensor(lengths, dtype=torch.int32, device=dev)
    got = library(q, k, v, p, u, vb, ln, H, r, forward="fp32")
    want = ref_grads(*(t.double() for t in (q, k, v, p, u, vb)), lengths, H, r.double())
    assert max(got[n].abs().max().item() for n in want) > 65504
    for n in want:
        assert torch.isfinite(got[n]).all(), n
        e = rel(got[n], want[n])
        record("bf16_attention_bwd_range", (n,), e, BF16_TOL)
        assert e < BF16_TOL, (n, e)


@pytest.mark.parametrize("defect,outputs", [("skew", ["dq_p"]), ("band", ["dp"]), ("delta", ["dq", "dk"]),
                                            ("mask", ["dk", "dv"])])
def test_bf16_attention_bwd_negative_controls(dev, defect, outputs):
    """A float64 reference with one defect must miss the library by at least 2x the bound, so the bound has teeth.
    The defect-free closed form must agree with the autograd restatement first."""
    B, T, H, lengths = 2, 130, 2, [130, 100]
    q, k, v, p, u, vb, r = inputs(B, T, H, 5, dev)
    ln = torch.tensor(lengths, dtype=torch.int32, device=dev)
    got = library(q, k, v, p, u, vb, ln, H, r, forward="fp32")
    args = [t.double() for t in (q, k, v, p, u, vb)]
    exact = ref_grads(*args, lengths, H, r.double())
    clean = manual_grads(*args, lengths, H, r.double())
    for n in clean:
        assert rel(clean[n], exact[n]) < 1e-10, n
    bad = manual_grads(*args, lengths, H, r.double(), defect=defect)
    for n in outputs:
        e = rel(got[n], bad[n])
        record("bf16_attention_bwd_negative_control", (defect, n), e, 2 * BF16_TOL)
        assert e >= 2 * BF16_TOL, (defect, n, e)


# ------------------------------------------------------------------------------------------------ bf16 backward GEMMs
@pytest.mark.parametrize("rows,cols", [(5, 6), (111, 768), (799, 768), (1600, 3072)])
def test_pack_operand_matches_torch(dev, rows, cols):
    """avsr_pack_operand: transposed or not, zero-padded to 64 along K, equal to torch's bf16 conversion bit for bit."""
    import ctypes as C
    from auto_avsr_b200._cabi import check, lib
    x = torch.randn(rows, cols, device=dev, generator=gen(rows + cols, dev))
    for transpose in (0, 1):
        src = x.t() if transpose else x
        ld = (src.size(1) + 63) // 64 * 64
        got = torch.full((src.size(0), ld), float("nan"), dtype=torch.bfloat16, device=dev)
        check(lib.avsr_pack_operand(x.data_ptr(), got.data_ptr(), rows, cols, ld, transpose, 16,
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        assert torch.equal(got[:, :src.size(1)], src.to(torch.bfloat16))
        assert not got[:, src.size(1):].any()


@pytest.mark.parametrize("rows,n,k", [(5, 6, 8), (111, 768, 768), (799, 768, 768), (1600, 3072, 768), (1600, 768, 3072)])
def test_bf16_linear_bwd_vs_fp64(dev, rows, n, k):
    """Both GEMMs of a Linear's bf16 backward (avsr_linear_bwd, "bf16") against float64, and each alone."""
    from auto_avsr_b200.train import linear_bwd
    g = gen(rows * n + k, dev)
    dy, x, w = (torch.randn(*s, device=dev, generator=g) for s in ((rows, n), (rows, k), (n, k)))
    dx, dw = linear_bwd(dy, x, w, True, True, "bf16")
    ex, ew = rel(dx, dy.double() @ w.double()), rel(dw, dy.double().t() @ x.double())
    record("bf16_backward_linear", (rows, n, k), max(ex, ew), 1.2e-2)
    assert ex < 1.2e-2 and ew < 1.2e-2, (ex, ew)
    dx1, dw1 = linear_bwd(dy, x, w, True, False, "bf16")
    dx2, dw2 = linear_bwd(dy, x, w, False, True, "bf16")
    assert dw1 is None and dx2 is None and torch.equal(dx1, dx) and torch.equal(dw2, dw)


# ------------------------------------------------------------------------------------------------ the encoder
def rel_np(a, ref):
    ref = torch.as_tensor(np.asarray(ref)).double()
    return (a.double().cpu() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def enc2_run(dev, backward):
    from auto_avsr_b200 import ConformerEncoder
    from oracle import conformer_oracle as O
    z = np.load(os.path.join(GOLDEN, "train_enc2.npz"))
    g = torch.Generator().manual_seed(int(z["seed"]))
    x = torch.randn(3, 37, D, generator=g, dtype=torch.float64).float()
    r = torch.randn(3, 37, D, generator=g, dtype=torch.float64).float()
    lengths = [int(v) for v in z["lengths"]]
    enc = ConformerEncoder(num_blocks=2, dropout_rate=0.0, positional_dropout_rate=0.0, attention_dropout_rate=0.0)
    enc.load_state_dict(encoder_state_dict(int(z["wseed"]), D, 12, F, 2, K), strict=True)
    enc = enc.to(dev).train()
    enc.precision = "f16"
    enc.backward_precision = backward
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)
    xg = x.to(dev).requires_grad_(True)
    y, _ = enc(xg, mask)
    (y * r.to(dev)).sum().backward()
    return z, enc, y.detach(), xg.grad


ENC_TOL = 1.7e-2


def test_bf16_backward_encoder2_vs_golden(dev):
    """The 2-layer encoder with backward_precision="bf16" against the float64 reference encoder: output (bit-equal to
    the default run: the forward is unchanged), input gradient and every parameter gradient's checksums."""
    z, enc, y, dx = enc2_run(dev, "bf16")
    _, _, y0, _ = enc2_run(dev, None)
    assert torch.equal(y, y0)
    e = rel_np(dx, z["dx"])
    record("bf16_backward_enc2", ("dx",), e, ENC_TOL)
    assert e < ENC_TOL, e
    worst = 0.0
    for n, p in enc.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
        cs = z["cs_" + n]
        if cs[1] > 1e-6:                         # (a bias in front of BatchNorm has a mathematically zero gradient)
            gd = p.grad.double().cpu()
            worst = max(worst, abs(gd.abs().sum().item() - cs[1]) / cs[1], abs((gd ** 2).sum().item() - cs[2]) / cs[2])
    record("bf16_backward_enc2", ("worst parameter-gradient checksum",), worst, ENC_TOL)
    assert worst < ENC_TOL, worst


def test_bf16_backward_knob_cleared_matches_never_set(dev):
    """Setting the knob and clearing it again gives the bits of a run that never set it."""
    _, enc0, _, dx0 = enc2_run(dev, None)
    z, enc1, _, _ = enc2_run(dev, "bf16")
    enc1.zero_grad(set_to_none=True)
    enc1.backward_precision = None
    from oracle import conformer_oracle as O
    g = torch.Generator().manual_seed(int(z["seed"]))
    x = torch.randn(3, 37, D, generator=g, dtype=torch.float64).float()
    r = torch.randn(3, 37, D, generator=g, dtype=torch.float64).float()
    mask = O.non_pad_mask([int(v) for v in z["lengths"]]).unsqueeze(1).to(dev)
    enc1.load_state_dict(enc0.state_dict())              # BatchNorm running statistics moved in the bf16 run
    xg = x.to(dev).requires_grad_(True)
    y, _ = enc1(xg, mask)
    (y * r.to(dev)).sum().backward()
    assert torch.equal(xg.grad, dx0)
    for (n, p0), (_, p1) in zip(enc0.named_parameters(), enc1.named_parameters()):
        assert torch.equal(p0.grad, p1.grad), n


S2_TOL = 6e-2


def test_bf16_backward_encoder12_s2(dev):
    """The 12-layer encoder at the S2 bucket (4 x 400 frames), reference dropout rates, batch-statistics BatchNorm:
    loss and every gradient finite, and within S2_TOL of the default backward's gradients relative to each tensor's max."""
    from auto_avsr_b200 import ConformerEncoder
    from auto_avsr_b200.synthetic import encoder_input
    from oracle import conformer_oracle as O
    lengths = SHAPES["S2"]
    sd = encoder_state_dict(3, num_blocks=12)
    xs = encoder_input(lengths, D, 7).to(dev)
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)
    grads = {}
    for backward in (None, "bf16"):
        enc = ConformerEncoder(num_blocks=12).to(dev)
        enc.load_state_dict(sd, strict=True)
        enc.train()
        enc.backward_precision = backward
        torch.manual_seed(0)                      # the same dropout masks in both runs
        xg = xs.clone().requires_grad_(True)
        loss = enc(xg, mask)[0].pow(2).mean()
        loss.backward()
        assert torch.isfinite(loss)
        grads[backward] = {"x": xg.grad, **{n: p.grad for n, p in enc.named_parameters()}}
        del enc
    worst = 0.0
    for n, g0 in grads[None].items():
        g1 = grads["bf16"][n]
        assert g1 is not None and torch.isfinite(g1).all(), n
        # mathematically zero: a bias in front of BatchNorm, and linear_k's bias (it shifts a whole score row)
        if not n.endswith(("depthwise_conv.bias", "linear_k.bias")):
            worst = max(worst, rel(g1, g0))
    record("bf16_backward_enc12_s2", ("worst gradient vs the default backward",), worst, S2_TOL)
    assert worst < S2_TOL, worst
