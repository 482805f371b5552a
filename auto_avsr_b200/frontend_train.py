"""Training of the ResNet front-ends (``Conv3dResNet`` / ``Conv1dResNet`` in ``train()`` with ``library_train``) in
libavsr_b200: one ``torch.autograd.Function`` per conv unit -- conv -> BatchNorm (batch statistics) -> [+ residual] ->
[SiLU] -- and small Functions for the video max-pool and the final mean, in the style of ``train.DwConvBnSiluFn``.
Gradients land on the original ``Parameter``s (20 conv weights, 20 BatchNorm weights and biases), so DDP hooks,
``clip_grad_norm_`` and AdamW see them unchanged.  torch supplies device memory, the autograd tape (which also sums
the two gradients that reach a BasicBlock's input) and the collectives; every unit's forward and backward arithmetic
runs in the library.

BatchNorm is the step the conformer conv module uses too (``train.bn_train_forward`` / ``bn_train_backward``), fed
with the statistics the conv computes: torch's training semantics exactly -- statistics over every position the module
normalises (padded frames and samples included), the biased variance to normalise, the unbiased one for
``running_var``, ``num_batches_tracked`` incremented (``momentum=None`` is the cumulative average), and under
``torch.no_grad()`` the batch statistics are still used and the running statistics still updated.  The statistics are
per-tile (count, mean, M2) merged with Chan's formula in fp64, never a one-pass sum of squares.  ``SyncBatchNorm`` with
a group of more than one rank all-gathers the per-rank (count, mean, M2) and merges them in rank order, and
all-reduces [sum ds, sum ds * x_hat] in backward; d gamma / d beta stay local sums (DDP averages them).

Forward convolutions run in the module's precision; dgrad and wgrad on wgmma with TF32 operands unless
``precision="fp32"`` (gradients do not fit fp16's range), which runs both on CUDA cores in fp32."""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from ._cabi import check, lib
from .engine import PRECISIONS, _ptr, _stream_handle, default_precision
from .train import _c, _sync_group, _workspace, bn_train_backward, bn_train_forward, bwd_precision


class _Spec:
    """Geometry of one conv unit: stem 0 (trunk, x (N, H, W, C_in)), 1 (video stem, x (N, H, W) frames, T per
    utterance) or 2 (audio stem, x (N, W) samples); the output is (N, Ho, Wo, C_out)."""

    def __init__(self, stem: int, N: int, T: int, H: int, W: int, conv: torch.nn.Module):
        w = conv.weight
        self.stem, self.N, self.T, self.H, self.W = stem, N, T, H, W
        self.Cout, self.Cin = w.size(0), w.size(1)
        if stem == 1:
            self.KH = self.KW = self.stride = 0
            self.Ho, self.Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        elif stem == 2:
            self.KH = self.KW = self.stride = 0
            self.Ho, self.Wo = 1, (W - 4) // 4 + 1
        else:
            self.KH, self.KW = (w.size(2), w.size(3)) if w.dim() == 4 else (1, w.size(2))
            self.stride = conv.stride[-1]
            self.Ho = (H + 2 * ((self.KH - 1) // 2) - self.KH) // self.stride + 1
            self.Wo = (W + 2 * ((self.KW - 1) // 2) - self.KW) // self.stride + 1

    def args(self):
        return (self.stem, self.N, self.T, self.H, self.W, self.Cin, self.Cout, self.KH, self.KW, self.stride)

    @property
    def rows(self) -> int:
        return self.N * self.Ho * self.Wo


class ConvBnActFn(torch.autograd.Function):
    """y = [SiLU](BatchNorm_train(conv(x)) [+ resid]) on channels-last fp32 tensors, running statistics updated in place."""

    @staticmethod
    def forward(ctx, x, resid, weight, gamma, beta, bn, spec: _Spec, act: bool, precision: str, group):
        x, weight, gamma, beta = _c(x), _c(weight), _c(gamma), _c(beta)
        resid = _c(resid) if resid is not None else None
        dev, C = x.device, spec.Cout
        p = PRECISIONS[precision]
        z = torch.empty(spec.rows, C, dtype=torch.float32, device=dev)
        stats = torch.empty(3, C, dtype=torch.float64, device=dev)
        ws = _workspace(dev, int(lib.avsr_frontend_train_conv_workspace_bytes(*spec.args(), p)))
        with torch.cuda.device(dev):
            check(lib.avsr_frontend_train_conv_fwd(x.data_ptr(), weight.data_ptr(), z.data_ptr(), stats.data_ptr(),
                                                   *spec.args(), ws.data_ptr(), ws.numel(), p, _stream_handle(dev)))
        y, mean, invstd, count = bn_train_forward(z, gamma, beta, bn, group, resid, act, stats)
        ctx.save_for_backward(x, resid, weight, z, mean, invstd, gamma, beta)
        ctx.spec, ctx.act, ctx.precision, ctx.group, ctx.count = spec, act, precision, group, count
        return y.view(spec.N, spec.Ho, spec.Wo, C)

    @staticmethod
    def backward(ctx, dy):
        x, resid, weight, z, mean, invstd, gamma, beta = ctx.saved_tensors
        spec, dev, C = ctx.spec, x.device, ctx.spec.Cout
        dz, dres, dgamma, dbeta = bn_train_backward(z, _c(dy).view(-1, C), mean, invstd, gamma, beta, ctx.count,
                                                    ctx.group, resid, ctx.act,
                                                    resid is not None and ctx.needs_input_grad[1])
        pb = PRECISIONS[bwd_precision(ctx.precision)]
        dw = torch.empty_like(weight)
        ws = _workspace(dev, int(lib.avsr_frontend_train_wgrad_workspace_bytes(*spec.args())))
        with torch.cuda.device(dev):
            check(lib.avsr_frontend_train_conv_wgrad(x.data_ptr(), dz.data_ptr(), dw.data_ptr(), *spec.args(),
                                                     ws.data_ptr(), ws.numel(), pb, _stream_handle(dev)))
        dx = None
        if ctx.needs_input_grad[0] and spec.stem == 0:
            p = PRECISIONS[bwd_precision(ctx.precision)]
            dx = torch.empty_like(x)
            geo = (spec.N, spec.H, spec.W, spec.Cin, C, spec.KH, spec.KW, spec.stride)
            ws = _workspace(dev, int(lib.avsr_frontend_train_dgrad_workspace_bytes(*geo, p)))
            with torch.cuda.device(dev):
                check(lib.avsr_frontend_train_conv_dgrad(dz.data_ptr(), weight.data_ptr(), dx.data_ptr(), *geo,
                                                         ws.data_ptr(), ws.numel(), p, _stream_handle(dev)))
        if dres is not None:
            dres = dres.view(resid.shape)
        return dx, dres, dw, dgamma, dbeta, None, None, None, None, None


class MaxPoolFn(torch.autograd.Function):
    """MaxPool3d((1,3,3), (1,2,2), (0,1,1)) per frame on (N, H, W, C): the winner of each window is recorded (first maximum
    in scan order, a NaN wins, as torch's CUDA kernel picks it) and the backward routes the gradient to it."""

    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        N, H, W, C = x.shape
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = torch.empty(N, Ho, Wo, C, dtype=torch.float32, device=x.device)
        idx = torch.empty(N, Ho, Wo, C, dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            check(lib.avsr_frontend_train_maxpool_fwd(x.data_ptr(), y.data_ptr(), idx.data_ptr(), N, H, W, C,
                                                      _stream_handle(x.device)))
        ctx.save_for_backward(idx)
        ctx.shape = x.shape
        ctx.mark_non_differentiable(idx)
        return y, idx

    @staticmethod
    def backward(ctx, dy, _didx):
        (idx,) = ctx.saved_tensors
        N, H, W, C = ctx.shape
        dy = _c(dy)
        dx = torch.empty(ctx.shape, dtype=torch.float32, device=dy.device)
        with torch.cuda.device(dy.device):
            check(lib.avsr_frontend_train_maxpool_bwd(dy.data_ptr(), idx.data_ptr(), dx.data_ptr(), N, H, W, C,
                                                      _stream_handle(dy.device)))
        return dx


class MeanRowsFn(torch.autograd.Function):
    """(G * P, C) -> (G, C): the mean of each group of P consecutive rows (AdaptiveAvgPool2d(1) per video frame,
    AvgPool1d(20) for audio)."""

    @staticmethod
    def forward(ctx, x, G: int, P: int):
        x = _c(x)
        C = x.size(-1)
        out = torch.empty(G, C, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(lib.avsr_frontend_train_mean_rows(x.data_ptr(), out.data_ptr(), G, P, C, _stream_handle(x.device)))
        ctx.shape, ctx.G, ctx.P = x.shape, G, P
        return out

    @staticmethod
    def backward(ctx, dout):
        dout = _c(dout)
        dx = torch.empty(ctx.shape, dtype=torch.float32, device=dout.device)
        with torch.cuda.device(dout.device):
            check(lib.avsr_frontend_train_mean_rows_bwd(dout.data_ptr(), dx.data_ptr(), ctx.G, ctx.P, dout.size(-1),
                                                        _stream_handle(dout.device)))
        return dx, None, None


def check_library_train(module, x: torch.Tensor) -> None:
    """The cases the library-train path refuses, before any launch."""
    if not x.is_cuda:
        raise NotImplementedError("front-end library_train: CPU tensors are not supported (no CPU fallback)")
    if x.requires_grad:
        raise NotImplementedError("front-end library_train: the input must not require grad (no input gradient is built)")
    if getattr(module.trunk, "relu_type", "swish") != "swish":
        raise NotImplementedError("front-end library_train: only relu_type='swish' is implemented")
    for conv, bn in module.conv_bn_pairs():
        if not bn.track_running_stats or bn.running_mean is None or not bn.affine:
            raise NotImplementedError("front-end library_train: needs affine BatchNorm with track_running_stats=True")
        if not bn.training:
            raise NotImplementedError("front-end library_train: every BatchNorm must be in train() mode")
        if conv.bias is not None:
            raise NotImplementedError("front-end library_train: needs bias-free convolutions")
        if not conv.weight.is_cuda or conv.weight.device != x.device:
            raise NotImplementedError("front-end library_train: parameters must live on the input's CUDA device")


def _unit(x, resid, pair, spec: _Spec, act: bool, precision: str):
    conv, bn = pair
    return ConvBnActFn.apply(x, resid, conv.weight, bn.weight, bn.bias, bn, spec, act, precision, _sync_group(bn))


def _trunk(x, pairs: List[Tuple[torch.nn.Module, torch.nn.Module]], precision: str):
    """The four layers of BasicBlocks on x (N, H, W, 64) -> (N, h, w, 512)."""
    j = 1
    for layer in range(4):
        for b in range(2):
            ds = layer > 0 and b == 0
            N, H, W, _ = x.shape
            s1 = _Spec(0, N, 1, H, W, pairs[j][0])
            h = _unit(x, None, pairs[j], s1, True, precision)
            r = x
            if ds:
                r = _unit(x, None, pairs[j + 2], _Spec(0, N, 1, H, W, pairs[j + 2][0]), False, precision)
            x = _unit(h, r, pairs[j + 1], _Spec(0, N, 1, s1.Ho, s1.Wo, pairs[j + 1][0]), True, precision)
            j += 3 if ds else 2
    return x


def frontend_train_forward(module, xs_pad: torch.Tensor, precision: Optional[str] = None) -> torch.Tensor:
    """The drop-in's training forward in the library: video (B, T, 1, H, W) -> (B, T, 512); audio (B, samples, 1) ->
    (B, samples // 640, 512)."""
    check_library_train(module, xs_pad)
    precision = precision or module.precision or default_precision()
    pairs = module.conv_bn_pairs()
    if module.modality == "video":
        if xs_pad.dim() != 5 or xs_pad.size(2) != 1:
            raise ValueError(f"video front-end: input must be (B, T, 1, H, W), got {tuple(xs_pad.shape)}")
        B, T, _, H, W = xs_pad.shape
        clip = xs_pad.detach().float().contiguous().view(B * T, H, W)
        stem = _unit(clip, None, pairs[0], _Spec(1, B * T, T, H, W, pairs[0][0]), True, precision)
        x, _ = MaxPoolFn.apply(stem)
        x = _trunk(x, pairs, precision)
        N, h, w, C = x.shape
        return MeanRowsFn.apply(x.view(N * h * w, C), N, h * w).view(B, T, C)
    if xs_pad.dim() != 3 or xs_pad.size(2) != 1:
        raise ValueError(f"audio front-end: input must be (B, samples, 1), got {tuple(xs_pad.shape)}")
    B, L, _ = xs_pad.shape
    Lt = L // 640 * 640
    if Lt == 0:
        raise NotImplementedError("audio front-end library_train: the waveform is shorter than one 640-sample frame")
    wav = xs_pad.detach()[:, :Lt, 0].float().contiguous()
    x = _unit(wav, None, pairs[0], _Spec(2, B, 1, 1, Lt, pairs[0][0]), True, precision)
    x = _trunk(x, pairs, precision)
    N, _, Lo, C = x.shape
    return MeanRowsFn.apply(x.view(N * Lo, C), N * Lo // 20, 20).view(B, Lo // 20, C)
