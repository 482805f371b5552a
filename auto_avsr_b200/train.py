"""Training slice of the encoder path (SURVEY.md 8f #2, first slice): ``torch.autograd.Function``s whose forward AND
backward run in libavsr_b200 -- LayerNorm, Linear (+ReLU) with dgrad / wgrad as the same wgmma GEMMs on operands the
library transposes and pads (one avsr_linear_bwd call), GLU, the depthwise conv, and the batch-statistics BatchNorm step (``bn_train_forward`` /
``bn_train_backward``) that the conformer conv module and the ResNet front-ends (frontend_train.py) share: per-tile
(count, mean, M2) merged with Chan's formula in fp64, running statistics as torch keeps them.  Gradients land on the
original ``nn.Parameter``s (autograd accumulates what ``backward`` returns), so DDP hooks, ``clip_grad_norm_`` and
AdamW (lightning.py:49, train.py:37-41) see them unchanged.  torch supplies device memory, the autograd tape, dropout
masks and the residual adds; no module falls back to PyTorch arithmetic for its own forward or backward.

The rel-pos attention core has a (correctness-first, fp32 CUDA-core) backward too, so a whole ``EncoderLayer`` /
``ConformerEncoder`` runs ``train()``: the reference's layer schedule with its dropouts (conformer_encoder.py:96-170).
SyncBatchNorm (train.py:31) is honoured: the per-rank (count, mean, M2) are all-gathered and merged in rank order, and
[sum ds, sum ds * x_hat] all-reduced in backward.
Not built: dropout on attention probabilities (the reference trains with 0.0).

Backward GEMMs run with TF32 operands (fp32 range: gradients do not fit fp16's; packed unrounded, the tensor core
truncates) unless ``precision="fp32"``; a "bf16" forward keeps the TF32 backward too.  The encoder modules take an opt-in ``backward_precision="bf16"`` (env
AVSR_B200_BWD_PRECISION): every backward GEMM then gets bf16 operands (fp32's exponent range, an 8-bit mantissa) and the
attention core's backward runs on the tensor cores (avsr_relpos_attention_bwd_tc).  ``TransformerDecoder``,
``ProjEncoder`` and ``CTC`` take the same attribute (decoder_train.py, espnet_dropin/ctc.py), without the environment
fallback."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from . import ops
from ._cabi import check, lib
from .engine import PRECISIONS, _ptr, _stream_handle, require_cuda

_WS = {}


def _workspace(device, nbytes: int) -> torch.Tensor:
    key = (device.index or 0, _stream_handle(device))
    ws = _WS.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = _WS[key] = torch.empty(nbytes + nbytes // 4 + 1024, dtype=torch.uint8, device=device)
    return ws


def _c(t: torch.Tensor) -> torch.Tensor:
    return t.detach().contiguous()


def bwd_precision(precision: str) -> str:
    return "fp32" if precision == "fp32" else "tf32"


BACKWARD_PRECISIONS = (None, "bf16")


def resolve_backward_precision(value: Optional[str]) -> Optional[str]:
    """A module's ``backward_precision``: ``value``, else env AVSR_B200_BWD_PRECISION, else None (the default backward,
    ``bwd_precision``).  "bf16" is the only other choice: an f16 backward is not offered, gradients overflow its range."""
    if value is None:
        value = os.environ.get("AVSR_B200_BWD_PRECISION") or None
    return explicit_backward_precision(value)


def explicit_backward_precision(value: Optional[str]) -> Optional[str]:
    """``value`` checked, without the environment fallback: what the decoder, ``ProjEncoder`` and ``CTC`` use, so that
    only their own attribute turns them to the bf16 backward (AVSR_B200_BWD_PRECISION reaches the encoder only)."""
    if value not in BACKWARD_PRECISIONS:
        raise ValueError(f"backward_precision={value!r}: expected None (default backward) or 'bf16'; f16 is not "
                         "offered (gradients overflow its 65504 range)")
    return value


def module_backward_precision(m) -> Optional[str]:
    """``m.backward_precision`` if set, else what the enclosing ConformerEncoder passed down for this forward."""
    v = getattr(m, "backward_precision", None)
    if v is None:
        v = getattr(m, "_inherited_backward_precision", None)
    return resolve_backward_precision(v)


# ------------------------------------------------------------------------------------------------ raw ops
def layernorm_bwd(x, gamma, dy):
    x, gamma, dy = _c(x), _c(gamma), _c(dy)
    d = x.size(-1)
    rows = x.numel() // d
    dx, dg, db = torch.empty_like(x), torch.empty_like(gamma), torch.empty_like(gamma)
    ws = _workspace(x.device, int(lib.avsr_train_workspace_bytes(rows, d, 1)))
    with torch.cuda.device(x.device):
        check(lib.avsr_layernorm_bwd(x.data_ptr(), gamma.data_ptr(), dy.data_ptr(), dx.data_ptr(), dg.data_ptr(), db.data_ptr(),
                                     rows, d, ws.data_ptr(), ws.numel(), _stream_handle(x.device)))
    return dx, dg, db


def colsum(y):
    y = _c(y)
    cols = y.size(-1)
    rows = y.numel() // cols
    out = torch.empty(cols, dtype=torch.float32, device=y.device)
    ws = _workspace(y.device, 132 * cols * 4 + 1024)
    with torch.cuda.device(y.device):
        check(lib.avsr_colsum(y.data_ptr(), out.data_ptr(), rows, cols, ws.data_ptr(), ws.numel(), _stream_handle(y.device)))
    return out


def linear_bwd(dy2, x2, w2, want_dx: bool, want_dw: bool, precision: str):
    """avsr_linear_bwd: dX = dY W and dW = dY^T X in one call, on "fp32", "tf32" or "bf16" operands (transposed and
    zero-padded along K in one pass each inside the library) -> (dx (rows, k) | None, dw (n, k) | None)."""
    dy2, x2, w2 = _c(dy2), _c(x2), _c(w2)
    rows, n = dy2.shape
    k = w2.size(1)
    prec = PRECISIONS[precision]
    dx = torch.empty(rows, k, dtype=torch.float32, device=dy2.device) if want_dx else None
    dw = torch.empty(n, k, dtype=torch.float32, device=dy2.device) if want_dw else None
    ws = _workspace(dy2.device, int(lib.avsr_linear_bwd_workspace_bytes(rows, n, k, prec)))
    with torch.cuda.device(dy2.device):
        check(lib.avsr_linear_bwd(dy2.data_ptr(), x2.data_ptr(), w2.data_ptr(), _ptr(dx), _ptr(dw), rows, n, k, prec,
                                  ws.data_ptr(), ws.numel(), _stream_handle(dy2.device)))
    return dx, dw


def relu_bwd(y, dy):
    y, dy = _c(y), _c(dy)
    dx = torch.empty_like(dy)
    with torch.cuda.device(y.device):
        check(lib.avsr_relu_bwd(y.data_ptr(), dy.data_ptr(), dx.data_ptr(), y.numel(), _stream_handle(y.device)))
    return dx


# ------------------------------------------------------------------------------------------------ autograd functions
class LayerNormFn(torch.autograd.Function):
    """LayerNorm(d, eps 1e-12) (layer_norm.py:21)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        require_cuda(x, "LayerNorm input")
        ctx.save_for_backward(x, weight)
        return ops.layernorm(x, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dx, dg, db = layernorm_bwd(x, weight, dy)
        return dx, dg, db


class LinearFn(torch.autograd.Function):
    """y = act(x W^T + b), act = identity | ReLU (positionwise_feed_forward.py:28-30, the pointwise convs of
    conformer_encoder.py:31,35).  Backward: dX = dY W and dW = dY^T X in one ``linear_bwd`` call (the same GEMM on
    operands the library transposes and pads), db = column sums of dY."""

    @staticmethod
    def forward(ctx, x, weight, bias, relu: bool, precision: str, backward: Optional[str] = None):
        require_cuda(x, "Linear input")
        w2 = weight.reshape(weight.size(0), -1)          # Conv1d(k=1) weights carry a trailing 1
        y = ops.linear(x, w2, bias, relu=relu, precision=precision)
        ctx.relu, ctx.precision, ctx.wshape = relu, precision, weight.shape
        ctx.backward = backward
        ctx.save_for_backward(x, w2, y if relu else None)
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w2, y = ctx.saved_tensors
        dy = _c(dy)
        if ctx.relu:
            dy = relu_bwd(y, dy)
        n, k = w2.shape
        dy2 = dy.reshape(-1, n)
        dx = dw = db = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            dx, dw = linear_bwd(dy2, x.reshape(-1, k), w2, ctx.needs_input_grad[0], ctx.needs_input_grad[1],
                                ctx.backward or bwd_precision(ctx.precision))
            dx = None if dx is None else dx.reshape(x.shape)
            dw = None if dw is None else dw.reshape(ctx.wshape)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = colsum(dy2)
        return dx, dw, db, None, None, None


class GluFn(torch.autograd.Function):
    """F.glu(x, dim=-1) on (…, 2C) (conformer_encoder.py:32 in channel-last layout)."""

    @staticmethod
    def forward(ctx, x):
        require_cuda(x, "GLU input")
        x = _c(x)
        Cc = x.size(-1) // 2
        rows = x.numel() // (2 * Cc)
        y = torch.empty(*x.shape[:-1], Cc, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(lib.avsr_glu_fwd(x.data_ptr(), y.data_ptr(), rows, Cc, _stream_handle(x.device)))
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dy = _c(dy)
        Cc = x.size(-1) // 2
        rows = x.numel() // (2 * Cc)
        dx = torch.empty_like(x)
        with torch.cuda.device(x.device):
            check(lib.avsr_glu_bwd(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), rows, Cc, _stream_handle(x.device)))
        return dx


def _dwconv_raw(x, w, b, flip: bool):
    B, T, Cc = x.shape
    K = w.size(-1)
    y = torch.empty_like(x)
    ws = _workspace(x.device, (K + 2) * Cc * 4 + 1024)
    with torch.cuda.device(x.device):
        check(lib.avsr_dwconv_raw(x.data_ptr(), w.data_ptr(), _ptr(b), y.data_ptr(), B, T, Cc, K, int(flip), ws.data_ptr(),
                                  ws.numel(), _stream_handle(x.device)))
    return y


def _sync_group(bn):
    """The process group a SyncBatchNorm slot reduces over, or None for a plain BatchNorm / one rank."""
    if not isinstance(bn, torch.nn.SyncBatchNorm):
        return None
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return None
    group = bn.process_group if bn.process_group is not None else dist.group.WORLD
    return None if dist.get_world_size(group) == 1 else group


def bn_train_forward(z, gamma, beta, bn, group, resid=None, act: bool = True, stats=None):
    """BatchNorm in training on z (rows, C) fp32 [+ resid] [-> SiLU] -> (y (rows, C), mean, invstd, count).

    ``stats`` is z's (3, C) fp64 (count, mean, M2) when the caller already has it (the front-end's conv produces it),
    else avsr_bn_train_stats computes it.  Under a SyncBatchNorm ``group`` the ranks' statistics are all-gathered and
    merged in rank order, so ``count`` is the global row count.  ``bn``'s running statistics and num_batches_tracked
    move as torch's _BatchNorm.forward moves them (``momentum=None``: the cumulative average)."""
    rows, C = z.shape
    dev = z.device
    if stats is None:
        stats = torch.empty(3, C, dtype=torch.float64, device=dev)
        ws = _workspace(dev, int(lib.avsr_bn_train_workspace_bytes(rows, C)))
        with torch.cuda.device(dev):
            check(lib.avsr_bn_train_stats(z.data_ptr(), rows, C, stats.data_ptr(), ws.data_ptr(), ws.numel(),
                                          _stream_handle(dev)))
    ranks = 1
    if group is not None:
        import torch.distributed as dist
        parts = [torch.empty_like(stats) for _ in range(dist.get_world_size(group))]
        dist.all_gather(parts, stats, group=group)
        stats, ranks = torch.stack(parts), len(parts)
    count = float(stats.view(ranks, 3, C)[:, 0, 0].sum().item()) if ranks > 1 else float(rows)
    if count <= 1:
        raise ValueError(f"Expected more than 1 value per channel when training, got {int(count)} (BatchNorm)")
    track = bn.track_running_stats and bn.running_mean is not None
    factor = 0.0
    if track:   # torch's _BatchNorm.forward: count this batch, then the averaging factor
        bn.num_batches_tracked.add_(1)
        factor = bn.momentum if bn.momentum is not None else 1.0 / float(bn.num_batches_tracked.item())
    mean = torch.empty(C, dtype=torch.float32, device=dev)
    invstd = torch.empty_like(mean)
    y = torch.empty_like(z)
    with torch.cuda.device(dev):
        check(lib.avsr_bn_train_finalize(stats.data_ptr(), ranks, C, float(bn.eps), float(factor),
                                         _ptr(bn.running_mean if track else None),
                                         _ptr(bn.running_var if track else None), mean.data_ptr(), invstd.data_ptr(),
                                         _stream_handle(dev)))
        check(lib.avsr_bn_train_act_fwd(z.data_ptr(), mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(),
                                        beta.data_ptr(), _ptr(resid), int(act), y.data_ptr(), rows, C,
                                        _stream_handle(dev)))
    return y, mean, invstd, count


def bn_train_backward(z, dy, mean, invstd, gamma, beta, count: float, group, resid=None, act: bool = True,
                      want_dres: bool = False):
    """Backward of ``bn_train_forward`` -> (dz, dres | None, dgamma, dbeta).  d gamma / d beta are this rank's sums (DDP
    averages the parameter gradients); under a ``group`` dz uses the sums all-reduced over the ranks."""
    rows, C = z.shape
    dev = z.device
    sums = torch.empty(2, C, dtype=torch.float32, device=dev)
    ws = _workspace(dev, int(lib.avsr_bn_train_workspace_bytes(rows, C)))
    with torch.cuda.device(dev):
        check(lib.avsr_bn_train_bwd_sums(z.data_ptr(), dy.data_ptr(), mean.data_ptr(), invstd.data_ptr(),
                                         gamma.data_ptr(), beta.data_ptr(), _ptr(resid), int(act), sums.data_ptr(),
                                         rows, C, ws.data_ptr(), ws.numel(), _stream_handle(dev)))
    dbeta, dgamma = sums[0].clone(), sums[1].clone()
    if group is not None:
        import torch.distributed as dist
        dist.all_reduce(sums, group=group)
    dz = torch.empty_like(z)
    dres = torch.empty_like(z) if want_dres else None
    with torch.cuda.device(dev):
        check(lib.avsr_bn_train_bwd_dx(z.data_ptr(), dy.data_ptr(), mean.data_ptr(), invstd.data_ptr(),
                                       gamma.data_ptr(), beta.data_ptr(), _ptr(resid), int(act), sums.data_ptr(),
                                       1.0 / count, dz.data_ptr(), _ptr(dres), rows, C, _stream_handle(dev)))
    return dz, dres, dgamma, dbeta


class DwConvBnSiluFn(torch.autograd.Function):
    """depthwise Conv1d + BatchNorm1d / SyncBatchNorm ``bn`` in training + SiLU on (B, T, C)
    (conformer_encoder.py:33-34): batch statistics over all B*T frames (of all ranks of ``group`` when given), ``bn``'s
    running statistics updated in place.  The conv and its tap gradients run in libavsr_b200 around
    ``bn_train_forward`` / ``bn_train_backward``."""

    @staticmethod
    def forward(ctx, x, w, b, bn_w, bn_b, bn, group):
        require_cuda(x, "conv module input")
        x, w, b, bn_w, bn_b = _c(x), _c(w), _c(b), _c(bn_w), _c(bn_b)
        conv = _dwconv_raw(x, w, b, False)
        y, mean, invstd, count = bn_train_forward(conv.view(-1, x.size(-1)), bn_w, bn_b, bn, group)
        ctx.save_for_backward(x, w, conv, mean, invstd, bn_w, bn_b)
        ctx.group, ctx.count = group, count
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x, w, conv, mean, invstd, bn_w, bn_b = ctx.saved_tensors
        B, T, Cc = x.shape
        K = w.size(-1)
        dconv, _, dg, dbt = bn_train_backward(conv.view(-1, Cc), _c(dy).view(-1, Cc), mean, invstd, bn_w, bn_b,
                                              ctx.count, ctx.group)
        dconv = dconv.view(x.shape)
        dx = _dwconv_raw(dconv, w, None, True)                             # correlation with the flipped taps
        dw, db = torch.empty_like(w), torch.empty(Cc, device=x.device)
        ws = _workspace(x.device, int(lib.avsr_train_workspace_bytes(B * T, Cc, K)))
        with torch.cuda.device(x.device):
            check(lib.avsr_dwconv_wgrad(x.data_ptr(), dconv.data_ptr(), dw.data_ptr(), db.data_ptr(), B, T, Cc, K, ws.data_ptr(),
                                        ws.numel(), _stream_handle(x.device)))
        return dx, dw, db, dg, dbt, None, None


class AttentionCoreFn(torch.autograd.Function):
    """ctx = softmax(((q+u) k^T + rel_shift((q+v) p^T)) / 8, key mask) v  (attention.py:174-189 + :59-82) on projected
    q, k, v (B,T,H*64), p (2T-1,H*64).  Forward = the fused attention kernel of the module's precision; backward =
    avsr_relpos_attention_bwd (fp32, scores recomputed), or with ``backward="bf16"`` avsr_relpos_attention_bwd_tc."""

    @staticmethod
    def forward(ctx_, q, k, v, p, u, vb, lengths, n_heads: int, precision: str, backward: Optional[str] = None):
        require_cuda(q, "attention input")
        out = ops.relpos_attention(q, k, v, p, u, vb, lengths, n_heads, precision=precision)
        ctx_.save_for_backward(q, k, v, p, u, vb, out, lengths if lengths is not None else torch.empty(0, device=q.device))
        ctx_.n_heads, ctx_.masked = n_heads, lengths is not None
        ctx_.backward = backward
        return out

    @staticmethod
    def backward(ctx_, dctx):
        q, k, v, p, u, vb, out, lengths = ctx_.saved_tensors
        D = q.size(-1)
        dq_k, dq_p, dk, dv, dp = relpos_attention_bwd(q, k, v, p, u, vb, lengths if ctx_.masked else None, out, dctx,
                                                      ctx_.n_heads, precision=ctx_.backward or "fp32")
        du = colsum(dq_k.reshape(-1, D)).reshape(u.shape)        # d pos_bias_u = sum over (b, t) of the k part of dq
        dvb = colsum(dq_p.reshape(-1, D)).reshape(vb.shape)
        return dq_k + dq_p, dk, dv, dp, du, dvb, None, None, None, None


def relpos_attention_bwd(q, k, v, p, u, vb, lengths, out, dctx, n_heads: int, precision: str = "fp32"):
    """avsr_relpos_attention_bwd ("fp32") or avsr_relpos_attention_bwd_tc ("bf16") -> (dq_k, dq_p, dk, dv, dp): the two
    parts of dq (through the content scores and through the rel-pos scores), the key / value gradients (B, T, H*64) and
    the pos-table gradient (2T-1, H*64)."""
    if precision not in ("fp32", "bf16"):
        raise ValueError(f"relpos_attention_bwd: precision {precision!r}: 'fp32' or 'bf16'")
    q, k, v, p, u, vb, out, dctx = (_c(t) for t in (q, k, v, p, u, vb, out, dctx))
    B, T, D = q.shape
    dq_k, dq_p, dk, dv = (torch.empty_like(q) for _ in range(4))
    dp = torch.empty_like(p)
    ln = lengths.to(torch.int32).contiguous() if lengths is not None else None
    args = (q.data_ptr(), k.data_ptr(), v.data_ptr(), p.data_ptr(), u.data_ptr(), vb.data_ptr(), _ptr(ln),
            out.data_ptr(), dctx.data_ptr(), dq_k.data_ptr(), dq_p.data_ptr(), dk.data_ptr(), dv.data_ptr(),
            dp.data_ptr(), B, T, n_heads)
    with torch.cuda.device(q.device):
        if precision == "fp32":
            ws = _workspace(q.device, int(lib.avsr_relpos_attention_bwd_workspace_bytes(B, T, n_heads)))
            check(lib.avsr_relpos_attention_bwd(*args, ws.data_ptr(), ws.numel(), _stream_handle(q.device)))
        else:
            prec = PRECISIONS["bf16"]
            ws = _workspace(q.device, int(lib.avsr_relpos_attention_bwd_tc_workspace_bytes(B, T, n_heads, prec)))
            check(lib.avsr_relpos_attention_bwd_tc(*args, prec, ws.data_ptr(), ws.numel(), _stream_handle(q.device)))
    return dq_k, dq_p, dk, dv, dp


def ctc_loss_forward(logits, hlens, ys_pad, odim: int, ignore_id: int = -1, want_grad: bool = False):
    """torch.nn.CTCLoss(reduction="none", zero_infinity=True), blank 0, on log_softmax of ``logits`` (B, Tmax, ld) fp32
    (first ``odim`` columns valid) -> (nll (B), state).  ``state`` is what ``ctc_loss_backward`` needs (beta included
    only when ``want_grad``).  ``hlens`` / ``ys_pad`` (B, Lmax) stay on the device: the label rows are compacted there."""
    require_cuda(logits, "CTC logits")
    B, T, ld = logits.shape
    dev = logits.device
    hl = hlens.to(device=dev, dtype=torch.int32).contiguous()
    ys = ys_pad.to(device=dev, dtype=torch.int64).contiguous()
    L = ys.size(1) if ys.dim() == 2 else 0
    nll = torch.empty(B, dtype=torch.float32, device=dev)
    nbytes = int(lib.avsr_ctc_loss_state_bytes(B, T, L))
    state = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)
    x = _c(logits)
    with torch.cuda.device(dev):
        check(lib.avsr_ctc_loss_fwd(x.data_ptr(), ld, hl.data_ptr(), ys.data_ptr(), B, T, L, odim, ignore_id,
                                    int(want_grad), nll.data_ptr(), state.data_ptr(), state.numel(), _stream_handle(dev)))
    return nll, (hl, ys, state)


def ctc_loss_backward(logits, saved, odim: int, dnll):
    """d sum_b(dnll[b] * nll[b]) / d logits, (B, Tmax, ld) with zero padding columns / frames."""
    hl, ys, state = saved
    x = _c(logits)
    B, T, ld = x.shape
    dnll = dnll.to(torch.float32).contiguous()
    dx = torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib.avsr_ctc_loss_bwd(x.data_ptr(), ld, hl.data_ptr(), ys.data_ptr(), B, T, ys.size(1) if ys.dim() == 2 else 0,
                                    odim, dnll.data_ptr(), state.data_ptr(), state.numel(), dx.data_ptr(), ld,
                                    _stream_handle(x.device)))
    return dx


class CtcLossFn(torch.autograd.Function):
    """nll (B) = CTC negative log-likelihood of each utterance (ctc.py:32-39 without the division by B):
    torch.nn.CTCLoss(reduction="none", zero_infinity=True) on log_softmax(logits).  Forward and backward run in
    libavsr_b200 (alpha, beta and the gradient on the device, no host synchronisation); the backward returns d logits."""

    @staticmethod
    def forward(ctx, logits, hlens, ys_pad, odim: int, ignore_id: int):
        nll, saved = ctc_loss_forward(logits, hlens, ys_pad, odim, ignore_id, want_grad=True)
        ctx.save_for_backward(logits, *saved)
        ctx.odim = odim
        return nll

    @staticmethod
    def backward(ctx, dnll):
        logits, *saved = ctx.saved_tensors
        return ctc_loss_backward(logits, saved, ctx.odim, dnll), None, None, None, None


# ------------------------------------------------------------------------------------------------ module forwards (train)
def feed_forward_train(m, x, precision: str, backward: Optional[str] = None):
    """PositionwiseFeedForward.forward in train mode: w_2(dropout(relu(w_1 x)))."""
    h = LinearFn.apply(x, m.w_1.weight, m.w_1.bias, True, precision, backward)
    h = m.dropout(h)
    return LinearFn.apply(h, m.w_2.weight, m.w_2.bias, False, precision, backward)


def conv_module_train(m, x, precision: str, backward: Optional[str] = None):
    """ConvolutionModule.forward in train mode on (B, T, C): pointwise_cov1 -> GLU -> depthwise + BatchNorm(batch stats)
    + SiLU -> pointwise_cov2.  ``m.norm`` stays a real BatchNorm1d / SyncBatchNorm: its running statistics and
    num_batches_tracked are updated like torch's."""
    bn = m.norm
    if not isinstance(bn, torch.nn.SyncBatchNorm) and type(bn) is not torch.nn.BatchNorm1d:
        raise NotImplementedError(f"conv_module.norm is {type(bn).__name__}: BatchNorm1d / SyncBatchNorm only")
    h = LinearFn.apply(x, m.pointwise_cov1.weight, m.pointwise_cov1.bias, False, precision, backward)
    g = GluFn.apply(h)
    y = DwConvBnSiluFn.apply(g, m.depthwise_conv.weight, m.depthwise_conv.bias, bn.weight, bn.bias, bn, _sync_group(bn))
    return LinearFn.apply(y, m.pointwise_cov2.weight, m.pointwise_cov2.bias, False, precision, backward)


def attention_train(m, x, pos_emb, mask, precision: str, backward: Optional[str] = None):
    """RelPositionMultiHeadedAttention.forward (self-attention) in train mode -> (B, T, d)."""
    from .espnet_dropin.attention import mask_to_lengths
    if m.dropout.p > 0:
        raise NotImplementedError("dropout on the attention probabilities (attention_dropout_rate > 0) is not implemented "
                                  "in the fused kernel; auto_avsr trains with 0.0 (e2e_asr_conformer.py:33-39)")
    B, T, D = x.shape
    q = LinearFn.apply(x, m.linear_q.weight, m.linear_q.bias, False, precision, backward)
    k = LinearFn.apply(x, m.linear_k.weight, m.linear_k.bias, False, precision, backward)
    v = LinearFn.apply(x, m.linear_v.weight, m.linear_v.bias, False, precision, backward)
    p = LinearFn.apply(pos_emb.reshape(2 * T - 1, D), m.linear_pos.weight, None, False, precision, backward)
    lengths = None if mask is None else mask_to_lengths(mask, B, T)
    ctx = AttentionCoreFn.apply(q, k, v, p, m.pos_bias_u, m.pos_bias_v, lengths, m.h, precision, backward)
    return LinearFn.apply(ctx, m.linear_out.weight, m.linear_out.bias, False, precision, backward)
