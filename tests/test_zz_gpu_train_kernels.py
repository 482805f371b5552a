"""The training kernels (csrc/train.cu, csrc/attention_bwd.cu, LinearFn's dgrad / wgrad on the tensor-core GEMM) against
plain float64 restatements computed on the same GPU, at the shapes where their code paths differ: one row per first-stage
CTA and several, the LayerNorm backward's 132-CTA branch, depthwise-conv tap gradients over multi-frame segments and over
more utterances than CTAs, attention backward with many key tiles and long rel-pos tables, padded GEMM operands and both
tile widths.  Then the drop-in ConformerEncoder in train() at the bucket shapes against the reference's own encoder in
float64.

Errors are max-abs differences over the reference's max-abs; bounds are about 4x what the H100 shows
(tests/helpers.py record()).  Every op is called twice and must give the same bits: all reductions have a fixed order."""
import contextlib
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from helpers import record

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(ROOT, "oracle", "_ref")

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "needs a CUDA GPU"
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def gen(seed, dev):
    return torch.Generator(device=dev).manual_seed(seed)


def rel(a, ref):
    """max |a - ref| / max |ref| (0 when both are empty or zero)."""
    if ref.numel() == 0:
        return 0.0
    d = (a.double() - ref.double()).abs().max().item()
    return d / max(ref.double().abs().max().item(), 1e-300) if d > 0 else 0.0


def same_bits(a, b, what):
    for x, y in zip(a, b):
        assert torch.equal(x, y), f"{what}: two calls on the same inputs differ"


def check(test, case, errs, bounds):
    """Record every error first, then assert them all: one failure still leaves the whole case in the log."""
    for k, e in errs.items():
        record(test, (*case, k), e, bounds[k] if isinstance(bounds, dict) else bounds)
    bad = {k: e for k, e in errs.items() if not e < (bounds[k] if isinstance(bounds, dict) else bounds)}
    assert not bad, (case, bad, bounds)


# ------------------------------------------------------------------------------------------------ LayerNorm backward
LN_TOL = 2.5e-6


@pytest.mark.parametrize("d", [4, 128, 768, 1024])
@pytest.mark.parametrize("rows", [0, 1, 7, 8, 9, 111, 1055, 1056, 1057, 1600, 6400])
def test_layernorm_bwd_vs_fp64(dev, rows, d):
    """rows >= 132 * 8 take the 132-CTA branch (each warp walks several rows); one row is constant (variance 0:
    x_hat = 0, rstd = 1e6), its dx is checked against its own scale."""
    from auto_avsr_b200.train import layernorm_bwd
    g = gen(rows * 7 + d, dev)
    x = torch.randn(rows, d, device=dev, generator=g) * 2 + 0.5
    dy = torch.randn(rows, d, device=dev, generator=g)
    gamma = 1 + 0.2 * torch.randn(d, device=dev, generator=g)
    const = rows // 2 if rows >= 2 else None
    if const is not None:
        x[const] = 0.75                         # exactly representable mean: x_hat is exactly 0 in both
    a = layernorm_bwd(x, gamma, dy)
    b = layernorm_bwd(x, gamma, dy)
    same_bits(a, b, "layernorm_bwd")
    dx, dg, db = a
    if rows == 0:
        assert dx.numel() == 0 and torch.equal(dg, torch.zeros_like(dg)) and torch.equal(db, torch.zeros_like(db))
        return
    x64, g64 = x.double().requires_grad_(True), gamma.double().requires_grad_(True)
    b64 = torch.zeros(d, dtype=torch.float64, device=dev, requires_grad=True)
    F.layer_norm(x64, (d,), g64, b64, eps=1e-12).backward(dy.double())
    keep = torch.ones(rows, dtype=torch.bool, device=dev)
    errs = {}
    if const is not None:
        keep[const] = False
        errs["dx const row"] = rel(dx[const], x64.grad[const])
    errs.update({"dx": rel(dx[keep], x64.grad[keep]), "dgamma": rel(dg, g64.grad), "dbeta": rel(db, b64.grad)})
    check("train_kernels_layernorm_bwd", (rows, d), errs, LN_TOL)


# ------------------------------------------------------------------------------------------------ column sums
@pytest.mark.parametrize("cols", [1, 5, 768, 3072, 5056])
@pytest.mark.parametrize("rows", [1, 131, 132, 133, 1600, 20000])
def test_colsum_vs_fp64(dev, rows, cols):
    """132 first-stage CTAs of ceil(rows / 132) rows each: one row per partial up to 132 rows, several beyond."""
    from auto_avsr_b200.train import colsum
    y = torch.randn(rows, cols, device=dev, generator=gen(rows + 3 * cols, dev)) + 0.25
    a, b = colsum(y), colsum(y)
    same_bits([a], [b], "colsum")
    check("train_kernels_colsum", (rows, cols), {"sum": rel(a, y.double().sum(0))}, 2.5e-6)


# ------------------------------------------------------------------------------------------------ fp32 operand packing
@pytest.mark.parametrize("transpose", [1, 0])
@pytest.mark.parametrize("rows,cols", [(1, 1), (5, 3), (33, 5), (37, 768), (111, 41), (799, 768), (1600, 5049)])
def test_pack_operand_fp32_exact_with_zero_padding(dev, rows, cols, transpose):
    """avsr_pack_operand(AVSR_PREC_FP32): (rows, cols) -> (cols, rows padded to 32) transposed, else (rows, cols padded
    to 32): an exact copy, and the padding columns exactly 0 (the GEMMs sum over them) over a NaN-filled buffer."""
    import ctypes as C
    from auto_avsr_b200._cabi import PREC_FP32, check, lib
    x = torch.randn(rows, cols, device=dev, generator=gen(rows * 31 + cols, dev))
    src = x.t() if transpose else x
    ld = (src.size(1) + 31) // 32 * 32

    def pack():
        out = torch.full((src.size(0), ld), float("nan"), device=dev)
        check(lib.avsr_pack_operand(x.data_ptr(), out.data_ptr(), rows, cols, ld, transpose, PREC_FP32,
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        return out

    t = pack()
    assert torch.equal(t[:, :src.size(1)], src)
    assert torch.equal(t[:, src.size(1):], torch.zeros(src.size(0), ld - src.size(1), device=dev))
    same_bits([t], [pack()], "pack_operand")


# ------------------------------------------------------------------------------------------------ ReLU / GLU
# grid_for caps the elementwise grids at 132 * 8 CTAs of 256 threads: sizes past 270336 (x4 for relu's float4) take the
# grid-stride loop, and sizes that are not a multiple of it leave a partial last sweep
@pytest.mark.parametrize("n", [4, 1028, 132 * 8 * 256 * 4 * 3 + 12])
def test_relu_bwd_exact(dev, n):
    from auto_avsr_b200.train import relu_bwd
    g = gen(n, dev)
    y = torch.relu(torch.randn(n, device=dev, generator=g))
    dy = torch.randn(n, device=dev, generator=g)
    dx = relu_bwd(y, dy)
    assert torch.equal(dx, torch.where(y > 0, dy, torch.zeros_like(dy)))
    same_bits([dx], [relu_bwd(y, dy)], "relu_bwd")


@pytest.mark.parametrize("rows,C", [(1, 5), (7, 768), (1057, 768), (1600, 768), (371, 1000)])
def test_glu_fwd_bwd_vs_fp64_with_saturated_gates(dev, rows, C):
    """Gates at +-30 and +-100 (sigmoid saturated to 0 / 1 in fp32: no NaN, no inf) among ordinary ones."""
    from auto_avsr_b200.train import GluFn
    g = gen(rows * 13 + C, dev)
    x = torch.randn(rows, 2 * C, device=dev, generator=g) * 2
    sat = torch.tensor([30.0, -30.0, 100.0, -100.0], device=dev)
    pick = torch.randint(0, 4, (rows, C), device=dev, generator=g)
    gate = torch.where(torch.rand(rows, C, device=dev, generator=g) < 0.25, sat[pick], x[:, C:])
    x[:, C:] = gate
    dy = torch.randn(rows, C, device=dev, generator=g)
    outs = []
    for _ in range(2):
        xa = x.clone().requires_grad_(True)
        y = GluFn.apply(xa)
        y.backward(dy)
        outs.append((y.detach(), xa.grad))
    same_bits(outs[0], outs[1], "glu")
    y, dx = outs[0]
    assert torch.isfinite(y).all() and torch.isfinite(dx).all()
    x64 = x.double().requires_grad_(True)
    y64 = F.glu(x64, dim=-1)
    y64.backward(dy.double())
    check("train_kernels_glu", (rows, C), {"y": rel(y, y64), "dx": rel(dx, x64.grad)}, 1e-6)


# ------------------------------------------------------------------------------------------------ depthwise conv + BN + SiLU
DW_TOL = 4e-6


def dwconv_case(dev, B, T, K, C, ratio, seed):
    g = gen(seed, dev)
    x = torch.randn(B, T, C, device=dev, generator=g)
    w = torch.randn(C, 1, K, device=dev, generator=g) / math.sqrt(K)
    b = 0.1 * torch.randn(C, device=dev, generator=g)
    if ratio:
        # per-channel offset = ratio x the channel's standard deviation over all B*T frames, through the conv bias
        raw = F.conv1d(x.double().transpose(1, 2), w.double(), None, padding=(K - 1) // 2, groups=C)
        sd = raw.transpose(0, 1).reshape(C, -1).std(1, unbiased=False)
        sign = torch.where(torch.rand(C, device=dev, generator=g) < 0.5, -1.0, 1.0).double()
        b = (ratio * sd * sign).float()
    bn_w = 1 + 0.1 * torch.randn(C, device=dev, generator=g)
    bn_b = 0.1 * torch.randn(C, device=dev, generator=g)
    rm = 0.1 * torch.randn(C, device=dev, generator=g)
    rv = 1 + 0.1 * torch.rand(C, device=dev, generator=g)
    r = torch.randn(B, T, C, device=dev, generator=g)
    return x, w, b, bn_w, bn_b, rm, rv, r


# batches the running statistics have seen before the one under test: momentum=None averages with 1 / (this + 1)
DW_TRACKED = 3


def run_dwconv(x, w, b, bn_w, bn_b, rm, rv, r, momentum):
    from auto_avsr_b200.train import DwConvBnSiluFn
    leaves = [t.clone().requires_grad_(True) for t in (x, w, b, bn_w, bn_b)]
    bn = torch.nn.BatchNorm1d(x.size(-1), momentum=momentum, eps=1e-5, device=x.device).train()
    bn.running_mean.copy_(rm)
    bn.running_var.copy_(rv)
    bn.num_batches_tracked.fill_(DW_TRACKED)
    y = DwConvBnSiluFn.apply(*leaves, bn, None)
    (y * r).sum().backward()
    assert int(bn.num_batches_tracked) == DW_TRACKED + 1
    return [y.detach()] + [t.grad for t in leaves] + [bn.running_mean, bn.running_var]


def ref_dwconv(x, w, b, bn_w, bn_b, rm, rv, r, momentum, frozen=False):
    """float64 conv1d(groups=C) + F.batch_norm(training) + silu -> [y, dx, dw, db, dgamma, dbeta, running_mean,
    running_var], rho.  momentum None: the cumulative average, factor 1 / num_batches_tracked.  frozen: the batch
    statistics enter as constants (no gradient through them) -- the scale of the gradients that batch statistics
    cancel.  rho = max over channels of max |conv| / sqrt(var + eps): what one fp32 rounding of the conv output moves
    x_hat by, in units of 2^-24."""
    K, C = w.size(-1), w.size(0)
    leaves = [t.double().requires_grad_(True) for t in (x, w, b, bn_w, bn_b)]
    rm_, rv_ = rm.double(), rv.double()
    conv = F.conv1d(leaves[0].transpose(1, 2), leaves[1], leaves[2], padding=(K - 1) // 2, groups=C)
    cd = conv.detach()
    mu, var = cd.mean((0, 2)), cd.var((0, 2), unbiased=False)
    if frozen:
        h = F.batch_norm(conv, mu, var, leaves[3], leaves[4], training=False, eps=1e-5)
    else:
        factor = momentum if momentum is not None else 1.0 / (DW_TRACKED + 1)
        h = F.batch_norm(conv, rm_, rv_, leaves[3], leaves[4], training=True, momentum=factor, eps=1e-5)
    y = F.silu(h).transpose(1, 2)
    (y * r.double()).sum().backward()
    rho = (cd.abs().amax((0, 2)) / (var + 1e-5).sqrt()).max().item()
    return [y.detach()] + [t.grad for t in leaves] + [rm_, rv_], rho


DW_NAMES = ["y", "dx", "dw", "db", "dgamma", "dbeta", "running_mean", "running_var"]
DW_SHAPES = [(1, 2), (2, 1), (1, 5), (3, 37), (4, 400), (16, 100), (1, 1600), (200, 8)]


def check_dwconv(dev, B, T, K, C, ratio, seed, momentum=0.1):
    args = dwconv_case(dev, B, T, K, C, ratio, seed)
    a, b = run_dwconv(*args, momentum), run_dwconv(*args, momentum)
    same_bits(a, b, "DwConvBnSiluFn")
    ref, rho = ref_dwconv(*args, momentum)
    # Gradients the batch statistics cancel are 0 in exact arithmetic (up to eps): the conv bias gradient (the batch
    # mean removes the bias), the tap gradient at K = 1 (BatchNorm removes the tap's scale), every conv gradient of a
    # 2-frame batch (x_hat = +-1 whatever the values).  Those are measured against the gradient with the statistics held
    # constant instead of against their own rounding noise.
    zero = {"db"} | ({"dw"} if K == 1 else set()) | ({"dx", "dw"} if B * T == 2 else set())
    frozen = ref_dwconv(*args, momentum, frozen=True)[0] if zero else None
    errs = {}
    for i, (n, got, want) in enumerate(zip(DW_NAMES, a, ref)):
        if n in zero:
            errs[n] = (got.double() - want).abs().max().item() / frozen[i].abs().max().item()
        else:
            errs[n] = rel(got, want)
    # Storing the conv output in fp32 alone moves x_hat by rho * 2^-24 against the fp64 reference.  Up to rho = 100
    # (offsets of 30 standard deviations included) that is inside the base bound; beyond it the bound grows by it.
    bound = DW_TOL + (4 * rho * 2.0 ** -24 if rho > 100 else 0.0)
    case = (B, T, K, C, f"ratio {ratio}") + (() if momentum == 0.1 else (f"momentum {momentum}",))
    record("train_kernels_dwconv_bn_silu", (*case, "rho"), rho, 100)
    check("train_kernels_dwconv_bn_silu", case, errs, bound)


@pytest.mark.parametrize("C,momentum", [(64, 0.1), (768, 0.1), (64, None), (768, None)],
                         ids=["64", "768", "64-None", "768-None"])
@pytest.mark.parametrize("K", [1, 7, 31])
@pytest.mark.parametrize("B,T", DW_SHAPES)
def test_dwconv_bn_silu_vs_fp64(dev, B, T, K, C, momentum):
    """conv1d(groups=C) + batch-stat BatchNorm (momentum 0.1 or None = the cumulative average, eps 1e-5, running
    statistics) + SiLU, forward and backward.  (200, 8) has more utterances than CTAs (one CTA per utterance in the
    tap gradient); (4, 400), (16, 100) and (1, 1600) give segments of several frames whose 31-tap halo crosses segment
    boundaries."""
    check_dwconv(dev, B, T, K, C, 0, B * 1000 + T * 10 + K + C, momentum)


@pytest.mark.parametrize("ratio,momentum", [(r, m) for m in (0.1, None) for r in (3, 10, 30, 1000)],
                         ids=[f"{r}{m}" for m in ("", "-None") for r in (3, 10, 30, 1000)])
@pytest.mark.parametrize("B,T", [(3, 37), (4, 400), (1, 1600), (200, 8)])
def test_dwconv_bn_silu_batch_stats_with_channel_offsets(dev, B, T, ratio, momentum):
    """Per-channel means of ratio x the standard deviation (set through the depthwise bias): the batch variance must
    not cancel.  A one-pass sum(v^2)/n - mean^2 in fp32 loses ratio^2 x 2^-24 of it.  A tile mean summed from the raw
    values loses several times the rounding of the values once the mean is tens of standard deviations off."""
    check_dwconv(dev, B, T, 31, 768, ratio, 7 * B + T + ratio, momentum)


# ------------------------------------------------------------------------------------------------ rel-pos attention backward
ATT_CASES = [(1, 1, 1, None), (2, 9, 2, [0, 9]), (3, 33, 3, [33, 32, 1]), (2, 65, 2, [65, 64]), (1, 130, 12, None),
             (4, 400, 12, [400, 333, 7, 129]), (1, 1600, 2, None)]
ATT_TOL = {"fp32": 8e-6, "f16": 4e-3}


def ref_attention(q, k, v, p, u, vb, lengths, H):
    """attention.py:59-82 / 174-189 in float64 with the key mask of attention.py:73-77 (finfo.min, softmax,
    masked_fill 0); the query enters as two leaves so that its two gradient parts come out separately."""
    B, T, D = q.shape
    qa, qb = q.clone().requires_grad_(True), q.clone().requires_grad_(True)
    kk, vv, pp, uu, vv_b = (t.clone().requires_grad_(True) for t in (k, v, p, u, vb))
    heads = lambda t: t.view(t.size(0), -1, H, 64).transpose(1, 2)          # noqa: E731
    ac = (heads(qa) + uu[None, :, None]) @ heads(kk).transpose(-1, -2)                   # (B, H, T, T)
    bd_full = (heads(qb) + vv_b[None, :, None]) @ pp.view(2 * T - 1, H, 64).permute(1, 2, 0)   # (B, H, T, 2T-1)
    i = torch.arange(T, device=q.device)
    idx = (i[None, :] - i[:, None] + T - 1).expand(B, H, T, T)              # table row j - i + T - 1
    s = (ac + bd_full.gather(-1, idx)) / 8.0
    if lengths is not None:
        mask = (i[None, :] >= torch.as_tensor(lengths, device=q.device)[:, None])[:, None, None, :]
        s = s.masked_fill(mask, torch.finfo(s.dtype).min)
        a = torch.softmax(s, -1).masked_fill(mask, 0.0)
    else:
        a = torch.softmax(s, -1)
    ctx = (a @ heads(vv)).transpose(1, 2).reshape(B, T, D)
    return ctx, (qa, qb, kk, vv, pp, uu, vv_b)


@pytest.mark.parametrize("B,T,H,lengths,prec", [(*c, "fp32") for c in ATT_CASES] + [(4, 400, 12, [400, 333, 7, 129], "f16")])
def test_relpos_attention_bwd_vs_fp64(dev, B, T, H, lengths, prec):
    """Key tiles of 32, rel-pos table of 2T-1 rows, the pos kernel's query window and 39-row band, zero-length and
    one-frame utterances.  The forward runs in ``prec`` (fp32: the bound is the backward kernels')."""
    from auto_avsr_b200.train import AttentionCoreFn, relpos_attention_bwd
    D = H * 64
    g = gen(B * 100000 + T * 100 + H, dev)
    q, k, v = (torch.randn(B, T, D, device=dev, generator=g) for _ in range(3))
    p = torch.randn(2 * T - 1, D, device=dev, generator=g)
    u, vb = (0.5 * torch.randn(H, 64, device=dev, generator=g) for _ in range(2))
    r = torch.randn(B, T, D, device=dev, generator=g)
    ln = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=dev)
    runs = []
    for _ in range(2):
        leaves = [t.clone().requires_grad_(True) for t in (q, k, v, p, u, vb)]
        out = AttentionCoreFn.apply(*leaves, ln, H, prec)
        (out * r).sum().backward()
        parts = relpos_attention_bwd(q, k, v, p, u, vb, ln, out.detach(), r, H)
        runs.append([out.detach()] + [t.grad for t in leaves] + list(parts[:2]))
    same_bits(runs[0], runs[1], "attention backward")
    got = runs[0]
    ctx64, (qa, qb, kk, vv, pp, uu, vv_b) = ref_attention(*(t.double() for t in (q, k, v, p, u, vb)), lengths, H)
    (ctx64 * r.double()).sum().backward()
    want = [ctx64.detach(), qa.grad + qb.grad, kk.grad, vv.grad, pp.grad, uu.grad, vv_b.grad, qa.grad, qb.grad]
    names = ["ctx", "dq", "dk", "dv", "dp", "d pos_bias_u", "d pos_bias_v", "dq_k", "dq_p"]
    errs = {n: rel(a, b) for n, a, b in zip(names, got, want)}
    if T == 1:
        # one key: the softmax is 1 whatever the scores, so every score gradient is 0 in exact arithmetic (the fp64
        # reference holds 1e-17 of rounding): absolute, against the scale of dv
        scale = want[3].abs().max().item()
        errs.update({n: (a.double() - b).abs().max().item() / scale for n, a, b in zip(names, got, want)
                     if n not in ("ctx", "dv")})
    if lengths is not None and 0 in lengths:
        z = lengths.index(0)
        assert all(torch.isfinite(t).all() for t in got)
        assert not got[1][z].any() and not got[2][z].any() and not got[3][z].any()   # zero-length: zero, not NaN
    check("train_kernels_attention_bwd", (B, T, H, str(lengths), prec), errs, ATT_TOL[prec])


# ------------------------------------------------------------------------------------------------ LinearFn
LIN_TOL = {"fp32": 1e-5, "tf32": 4e-3}


@contextlib.contextmanager
def tile_env(tile):
    old = os.environ.get("AVSR_B200_TILE")
    if tile is None:
        os.environ.pop("AVSR_B200_TILE", None)
    else:
        os.environ["AVSR_B200_TILE"] = tile
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("AVSR_B200_TILE", None)
        else:
            os.environ["AVSR_B200_TILE"] = old


LIN_SHAPES = [(1, 8, 64), (111, 48, 768), (799, 768, 768), (1600, 3072, 768), (1600, 768, 3072), (1600, 5056, 768)]


def linear_case(dev, rows, n, k):
    g = gen(rows * 7 + n * 3 + k, dev)
    x = torch.randn(rows, k, device=dev, generator=g)
    w = torch.rand(n, k, device=dev, generator=g).sub_(0.5).mul_(2 / math.sqrt(k))
    b = 0.1 * torch.randn(n, device=dev, generator=g)
    dy = torch.randn(rows, n, device=dev, generator=g)
    return x, w, b, dy


@pytest.mark.parametrize("tile", [None, "64", "128"])
@pytest.mark.parametrize("prec", ["fp32", "tf32"])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("rows,n,k", LIN_SHAPES)
def test_linear_fwd_bwd_vs_fp64(dev, rows, n, k, relu, prec, tile):
    """y = act(x W^T + b), dX = dY W, dW = dY^T X, db = colsum dY.  n % 32 != 0 pads dY / W^T, rows % 32 != 0 pads
    the wgrad's K; the tile width of every GEMM is left to the cost model or forced to 64 / 128 columns.  With ReLU the
    reference uses the mask the GPU forward produced (a pre-activation within rounding of 0 may flip: a derivative
    discontinuity, not an arithmetic error)."""
    from auto_avsr_b200.train import LinearFn
    x, w, b, dy = linear_case(dev, rows, n, k)
    runs = []
    with tile_env(tile):
        for _ in range(2):
            leaves = [t.clone().requires_grad_(True) for t in (x, w, b)]
            y = LinearFn.apply(*leaves, relu, prec)
            y.backward(dy)
            runs.append([y.detach()] + [t.grad for t in leaves])
    same_bits(runs[0], runs[1], "LinearFn")
    y, dx, dw, db = runs[0]
    x64, w64 = x.double(), w.double()
    h = x64 @ w64.t() + b.double()
    dh = dy.double()
    if relu:
        mask = (y > 0).double()
        h, dh = h * mask, dh * mask
    want = {"y": h, "dx": dh @ w64, "dw": dh.t() @ x64, "db": dh.sum(0)}
    errs = {"y": rel(y, want["y"]), "dx": rel(dx, want["dx"]), "dw": rel(dw, want["dw"]), "db": rel(db, want["db"])}
    check("train_kernels_linear", (rows, n, k, "relu" if relu else "id", prec, f"tile {tile}"), errs, LIN_TOL[prec])


@pytest.mark.parametrize("tile", [None, "64", "128"])
@pytest.mark.parametrize("prec", ["fp32", "tf32"])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("rows,n,k", LIN_SHAPES)
def test_linear_bwd_bit_identical_to_torch_packed_operands(dev, rows, n, k, relu, prec, tile):
    """LinearFn's default backward (one avsr_linear_bwd call) gives the same bits as the per-op GEMM entry on operands
    laid out with torch ops: W^T, dY^T and X^T zero-padded along K to a multiple of 32, dY's columns zero-padded when
    n % 32 != 0, then ops.linear for dX and for dW; db from colsum.  So the library's packing (TF32 operands unrounded,
    the same K, the same epilogue) leaves every GEMM exactly as the per-op entry runs it."""
    from auto_avsr_b200 import ops
    from auto_avsr_b200.train import LinearFn, colsum
    x, w, b, dy = linear_case(dev, rows, n, k)

    def t_pad(a):
        out = torch.zeros(a.size(1), (a.size(0) + 31) // 32 * 32, device=dev)
        out[:, :a.size(0)] = a.t()
        return out

    with tile_env(tile):
        leaves = [t.clone().requires_grad_(True) for t in (x, w, b)]
        y = LinearFn.apply(*leaves, relu, prec)
        y.backward(dy)
        dh = torch.where(y > 0, dy, torch.zeros_like(dy)) if relu else dy
        wt = t_pad(w)
        dhp = torch.zeros(rows, wt.size(1), device=dev)
        dhp[:, :n] = dh
        want = [ops.linear(dhp, wt, None, precision=prec), ops.linear(t_pad(dh), t_pad(x), None, precision=prec),
                colsum(dh)]
    for name, got, ref in zip(("dx", "dw", "db"), [t.grad for t in leaves], want):
        assert torch.equal(got, ref), (name, (got - ref).abs().max().item())


# ------------------------------------------------------------------------------------------------ encoder vs the reference
PRELUDE = f"""
import sys, numpy as np, torch
sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})
from oracle import build_ref
Ref, make_non_pad_mask = build_ref.import_reference_encoder()
from helpers import record
from auto_avsr_b200 import ConformerEncoder
from auto_avsr_b200.synthetic import encoder_input, encoder_state_dict
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
dev = torch.device("cuda:0")
D, H, FF, K = 768, 12, 3072, 31

def rel(a, b):
    d = (a.double() - b.double()).abs().max().item()
    return d / max(b.double().abs().max().item(), 1e-300) if d > 0 else 0.0

def model(cls, sd, nb):
    m = cls(attention_dim=D, attention_heads=H, linear_units=FF, cnn_module_kernel=K, num_blocks=nb, dropout_rate=0.0,
            positional_dropout_rate=0.0, attention_dropout_rate=0.0)
    m.load_state_dict(sd, strict=True)
    return (m.double() if cls is Ref else m).to(dev).train()

def offset_bias(sd, lengths, nb, xs, layer, ratio, seed):
    # depthwise_conv.bias of `layer` := ratio x the std of that conv's output over all frames (random signs)
    ref = model(Ref, sd, nb)
    conv = ref.encoders[layer].conv_module.depthwise_conv
    got = {{}}
    h = conv.register_forward_hook(lambda m, i, o: got.update(o=o.detach() - m.bias.detach()[None, :, None]))
    mask = make_non_pad_mask(lengths).unsqueeze(-2).to(dev)
    with torch.no_grad():
        ref(xs.double().to(dev), mask)
    h.remove()
    o = got["o"]
    std = o.transpose(0, 1).reshape(o.size(1), -1).std(1, unbiased=False).cpu()
    g = torch.Generator().manual_seed(seed)
    sign = torch.where(torch.rand(o.size(1), generator=g) < 0.5, -1.0, 1.0).double()
    sd = dict(sd)
    sd[f"encoders.{{layer}}.conv_module.depthwise_conv.bias"] = (ratio * std * sign).float()
    return sd

def step(m, x, mask, r):
    m.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_(True)
    y, _ = m(xg, mask)
    (y * r).sum().backward()
    return y.detach(), xg.grad, {{n: p.grad for n, p in m.named_parameters()}}

def run_case(tag, lengths, nb, precs, tol, wseed=11, xseed=12, offset=None, repeat=False):
    sd = encoder_state_dict(wseed, D, H, FF, nb, K)
    xs = encoder_input(lengths, D, xseed)
    if offset is not None:
        sd = offset_bias(sd, lengths, nb, xs, offset[0], offset[1], wseed)
    g = torch.Generator().manual_seed(xseed + 1)
    r = torch.randn(xs.shape, generator=g, dtype=torch.float64)
    mask = make_non_pad_mask(lengths).unsqueeze(-2).to(dev)
    ref = model(Ref, sd, nb)
    y64, dx64, g64 = step(ref, xs.double().to(dev), mask, r.to(dev))
    bufs64 = {{n: b.detach().clone() for n, b in ref.named_buffers()}}
    del ref
    torch.cuda.empty_cache()
    fails = []
    for prec in precs:
        ours = model(ConformerEncoder, sd, nb)
        ours.precision = prec
        y, dx, grads = step(ours, xs.to(dev), mask, r.float().to(dev))
        bufs = {{n: b.detach().clone() for n, b in ours.named_buffers()}}
        errs = {{"y": rel(y, y64), "dx": rel(dx, dx64)}}
        worst, worst_n = 0.0, ""
        for n, p64 in g64.items():
            gp = grads[n]
            assert gp is not None and torch.isfinite(gp).all(), n
            wn = n[:-len(".bias")] + ".weight" if n.endswith(".bias") else None
            if wn in g64 and p64.abs().max().item() < 1e-9 * g64[wn].abs().max().item():
                # mathematically zero (depthwise_conv.bias in front of BatchNorm, linear_k.bias under the softmax):
                # absolute, against the scale of the matching weight's gradient
                e = gp.double().abs().max().item() / g64[wn].abs().max().item()
                key = "zero-grad " + n.split(".", 2)[-1]
                errs[key] = max(errs.get(key, 0.0), e)
                continue
            a, b = gp.double(), p64
            cs = max(abs(a.abs().sum().item() - b.abs().sum().item()) / b.abs().sum().item(),
                     abs((a * a).sum().item() - (b * b).sum().item()) / (b * b).sum().item())
            # element-wise where the gradient is smooth in the forward.  A hidden unit whose pre-activation sits within
            # the rounding of 0 flips its ReLU against float64 and moves its whole row of d w_1 (see
            # tests/test_gpu_backward.py).  At 1600 frames x 3072 units x 2 FFNs per layer a few units do so even in
            # fp32, so w_1 is compared by checksums in every precision (its element-wise error is recorded)
            if ".w_1.weight" in n:
                errs["w_1 checksums"] = max(errs.get("w_1 checksums", 0.0), cs)
                record("train_encoder_vs_reference_fp64", (tag, prec, "w_1 element-wise, not asserted", n), rel(a, b), None)
                continue
            e = max(cs, rel(a, b))
            if e > worst:
                worst, worst_n = e, n
        errs["worst parameter gradient"] = worst
        for n, b in bufs64.items():
            if "running" in n:
                errs["bn " + n.rsplit(".", 1)[-1]] = max(errs.get("bn " + n.rsplit(".", 1)[-1], 0.0), rel(bufs[n], b))
            elif "num_batches_tracked" in n:
                assert int(bufs[n]) == int(b) == int(sd[n]) + 1, (n, int(bufs[n]), int(b), int(sd[n]))
        bound = tol[prec]
        for k, e in errs.items():
            bk = bound[k] if k in bound else bound["grad"]
            record("train_encoder_vs_reference_fp64", (tag, prec, k) + ((worst_n,) if k.startswith("worst") else ()), e, bk)
            if not e < bk:
                fails.append((tag, prec, k, e, bk))
        if repeat:
            y2, dx2, grads2 = step(ours, xs.to(dev), mask, r.float().to(dev))
            assert torch.equal(y, y2) and torch.equal(dx, dx2), "two training steps differ"
            for n in grads:
                assert torch.equal(grads[n], grads2[n]), ("two training steps differ", n)
        del ours
        torch.cuda.empty_cache()
    assert not fails, fails
"""


def run_child(body, timeout=1500):
    r = subprocess.run([sys.executable, "-c", PRELUDE + body + "\nprint('CHILD-OK')\n"], capture_output=True, text=True,
                       timeout=timeout, cwd=ROOT)
    sys.stdout.write(r.stdout[-6000:])
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


# bounds per precision: output, input gradient, parameter gradients (element-wise + checksums; w_1 by checksums), BN
# running statistics, mathematically-zero gradients.  The gradient bounds are far above the kernels' own errors (the
# sweeps above: 1e-6 in fp32) because of the ReLU flips: each flipped unit moves dx of its frame by one term of w_1
# (about 1e-3 of max |dx| here, in fp32 as well), d w_1.bias by one term of its sum (the worst element-wise gradient:
# 2e-2 in fp32, 6e-2 in f16 on the H100) and with dx the LayerNorm in front of that FFN.
ENC_TOL = {
    "fp32": {"y": 4e-6, "dx": 8e-3, "grad": 8e-2, "w_1 checksums": 1.1e-4, "bn running_mean": 5e-7,
             "bn running_var": 5e-7, "zero-grad conv_module.depthwise_conv.bias": 1e-5,
             "zero-grad self_attn.linear_k.bias": 4e-6},
    "f16": {"y": 2e-3, "dx": 3e-2, "grad": 2.3e-1, "w_1 checksums": 3.4e-2, "bn running_mean": 8e-4,
            "bn running_var": 5e-6, "zero-grad conv_module.depthwise_conv.bias": 1.1e-5,
            "zero-grad self_attn.linear_k.bias": 2e-3},
}

ENC_CASES = {
    # name: (lengths, blocks, extra keyword arguments of run_case)
    "S2": ("[400] * 4", 12, "repeat=True"),
    "S2r": ("[400, 350, 300, 250, 300]", 12, ""),
    "S3": ("[100] * 16", 12, ""),
    "S4": ("[1600]", 2, ""),
    "S2r_offset30": ("[400, 350, 300, 250, 300]", 2, "offset=(1, 30.0)"),
}


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "espnet")), reason="oracle/_ref not built")
@pytest.mark.parametrize("name", list(ENC_CASES))
def test_encoder_train_step_vs_reference_fp64(name):
    """The drop-in ConformerEncoder in train() (dropout 0) against the reference's ConformerEncoder in float64 on the
    GPU, same weights and ragged mask, loss (y * r).sum(): output, d xs, every parameter gradient, the BatchNorm running
    statistics and num_batches_tracked; S2 (the benchmarked step) also gives the same bits on a second step.
    S2r_offset30: the second layer's depthwise bias puts every channel's mean at 30x its standard deviation."""
    lengths, nb, extra = ENC_CASES[name]
    run_child(f"run_case({name!r}, {lengths}, {nb}, ('fp32', 'f16'), {ENC_TOL!r}{', ' + extra if extra else ''})")
