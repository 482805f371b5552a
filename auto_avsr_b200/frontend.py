"""The ResNet front-ends on prepared weights: ``Conv3dResNet`` (video) and ``Conv1dResNet`` (audio) in eval mode, from the
raw clip or waveform to the (B, T, 512) features ``proj_encoder`` consumes, in one library call
(``avsr_frontend_forward``).

``PreparedFrontend`` owns the library-side copy of the 20 convolutions (weights reordered to channels-last implicit-GEMM
rows in operand storage, BatchNorm as an fp32 scale and shift).  It is rebuilt whenever a conv weight, a BatchNorm
affine parameter or a running statistic changes: the cache key holds each tensor's ``data_ptr``, ``_version`` and shape
(``num_batches_tracked`` included), and each BatchNorm's ``eps``."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence, Tuple

import torch

from ._cabi import FRONTEND_AUDIO, FRONTEND_CONVS, FRONTEND_TAPS, FRONTEND_VIDEO, ConvBnParams, check, lib
from .engine import PRECISIONS, _ptr, _stream_handle, require_cuda

MODALITIES = {"video": FRONTEND_VIDEO, "audio": FRONTEND_AUDIO}


def _fp(tensors) -> tuple:
    return tuple((t.data_ptr(), t._version, tuple(t.shape)) for t in tensors)


class PreparedFrontend:
    def __init__(self):
        self._buf: Dict[tuple, Tuple[tuple, torch.Tensor]] = {}
        self._ws: Dict[tuple, torch.Tensor] = {}

    def prepare(self, modality: str, pairs: Sequence[Tuple[torch.nn.Module, torch.nn.Module]], device,
                precision: str) -> torch.Tensor:
        """``pairs``: the 20 (conv, BatchNorm) modules, the stem first, then each BasicBlock's conv1, conv2 and
        downsample in state-dict order."""
        if len(pairs) != FRONTEND_CONVS:
            raise ValueError(f"front-end: expected {FRONTEND_CONVS} conv/BatchNorm pairs, got {len(pairs)}")
        tensors: List[torch.Tensor] = []
        for conv, bn in pairs:
            if conv.bias is not None or bn.weight is None or bn.running_mean is None:
                raise NotImplementedError("front-end: needs bias-free convs and affine BatchNorm with running statistics")
            tensors += [conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var]
        for t in tensors:
            require_cuda(t, "front-end parameter")
            if t.device != device:
                raise RuntimeError(f"front-end parameter lives on {t.device}, input on {device}")
        key = (device.index or 0, modality, PRECISIONS[precision])
        # BatchNorm's training forward updates running_mean / running_var inside the ATen kernel without bumping their
        # _version; the num_batches_tracked.add_(1) it does next to it does
        counters = [bn.num_batches_tracked for _, bn in pairs if bn.num_batches_tracked is not None]
        fp = _fp(tensors + counters) + tuple(float(bn.eps) for _, bn in pairs)
        hit = self._buf.get(key)
        if hit is not None and hit[0] == fp:
            return hit[1]
        nbytes = int(lib.avsr_frontend_prepared_bytes(MODALITIES[modality], PRECISIONS[precision]))
        buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        keep = [t.detach().contiguous() for t in tensors]
        arr = (ConvBnParams * FRONTEND_CONVS)()
        for i, (_, bn) in enumerate(pairs):
            w, g, b, m, v = keep[5 * i:5 * i + 5]
            arr[i] = ConvBnParams(w.data_ptr(), g.data_ptr(), b.data_ptr(), m.data_ptr(), v.data_ptr(), float(bn.eps))
        with torch.cuda.device(device):
            check(lib.avsr_prepare_frontend(MODALITIES[modality], arr, buf.data_ptr(), nbytes, PRECISIONS[precision],
                                            _stream_handle(device)))
        self._buf[key] = (fp, buf)
        return buf

    def workspace(self, nbytes: int, device) -> torch.Tensor:
        key = (device.index or 0, _stream_handle(device))
        ws = self._ws.get(key)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=device)
            self._ws[key] = ws
        return ws


def _geometry(modality: str, x: torch.Tensor) -> Tuple[int, int, int, int, int]:
    """(B, T_in, H, W, output rows per utterance) of a video (B, T, 1, H, W) or audio (B, samples, 1) input"""
    if modality == "video":
        if x.dim() != 5 or x.size(2) != 1:
            raise ValueError(f"video front-end: input must be (B, T, 1, H, W), got {tuple(x.shape)}")
        B, T, _, H, W = x.shape
        return B, T, H, W, T
    if x.dim() != 3 or x.size(2) != 1:
        raise ValueError(f"audio front-end: input must be (B, samples, 1), got {tuple(x.shape)}")
    B, T, _ = x.shape
    return B, T, 1, 1, T // 640


def frontend_workspace_bytes(modality: str, x: torch.Tensor, precision: str) -> int:
    B, T, H, W, _ = _geometry(modality, x)
    return int(lib.avsr_frontend_workspace_bytes(MODALITIES[modality], B, T, H, W, PRECISIONS[precision]))


def frontend_forward(prep: PreparedFrontend, modality: str, pairs, x: torch.Tensor, precision: str,
                     taps=None, workspace=None) -> torch.Tensor:
    """video x (B, T, 1, H, W) -> (B, T, 512); audio x (B, samples, 1) -> (B, samples // 640, 512).  fp32 CUDA tensors.
    ``taps`` (tests): a list of ``FRONTEND_TAPS`` fp32 CUDA tensors or None, shaped by ``frontend_tap_shape``, that
    receive the stage outputs (``avsr_frontend_forward_taps``); ``workspace``: a uint8 CUDA tensor to run in instead of
    the cached one."""
    require_cuda(x, "front-end input")
    x = x.detach().contiguous()
    B, T, H, W, rows = _geometry(modality, x)
    out = torch.empty(B, rows, 512, dtype=torch.float32, device=x.device)
    buf = prep.prepare(modality, pairs, x.device, precision)
    if out.numel() == 0:
        return out
    m, p = MODALITIES[modality], PRECISIONS[precision]
    nbytes = int(lib.avsr_frontend_workspace_bytes(m, B, T, H, W, p))
    ws = prep.workspace(nbytes, x.device) if workspace is None else workspace
    with torch.cuda.device(x.device):
        if taps is None:
            check(lib.avsr_frontend_forward(m, buf.data_ptr(), x.data_ptr(), B, T, H, W, out.data_ptr(), ws.data_ptr(),
                                            ws.numel(), p, _stream_handle(x.device)))
        else:
            if len(taps) != FRONTEND_TAPS:
                raise ValueError(f"front-end taps: expected {FRONTEND_TAPS} entries, got {len(taps)}")
            for i, t in enumerate(taps):
                if t is not None and (t.dtype != torch.float32 or not t.is_contiguous() or t.device != x.device or
                                      tuple(t.shape) != frontend_tap_shape(modality, B, T, H, W, i)):
                    raise ValueError(f"front-end tap {i}: needs a contiguous fp32 tensor of shape "
                                     f"{frontend_tap_shape(modality, B, T, H, W, i)} on {x.device}")
            arr = (C.c_void_p * FRONTEND_TAPS)(*[None if t is None else t.data_ptr() for t in taps])
            check(lib.avsr_frontend_forward_taps(m, buf.data_ptr(), x.data_ptr(), B, T, H, W, out.data_ptr(), arr,
                                                 ws.data_ptr(), ws.numel(), p, _stream_handle(x.device)))
    return out


def frontend_tap_shape(modality: str, B: int, T: int, H: int, W: int, tap: int) -> Tuple[int, int, int, int]:
    """Shape of stage tap ``tap`` (``avsr_frontend_tap_shape``): (frames, H, W, C) for video, (B, 1, L, C) for audio."""
    dims = (C.c_int * 4)()
    check(lib.avsr_frontend_tap_shape(MODALITIES[modality], B, T, H, W, tap, dims))
    return tuple(int(d) for d in dims)


def conv_bn_act(x: torch.Tensor, weight: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, stride: int = 1,
                residual=None, act: bool = True, precision: str = "f16") -> torch.Tensor:
    """One trunk convolution on channels-last fp32 tensors: x (N, H, W, C_in), weight (C_out, C_in, KH, KW) ->
    [SiLU](conv(x) * scale + shift [+ residual]) as (N, Ho, Wo, C_out), padding (K - 1) / 2, computed in ``precision``
    (``avsr_conv_bn_act``)."""
    for t, what in ((x, "x"), (weight, "weight"), (scale, "scale"), (shift, "shift")):
        require_cuda(t, what)
    x, weight = x.contiguous(), weight.contiguous()
    scale, shift = scale.contiguous(), shift.contiguous()
    N, H, W, Cin = x.shape
    Cout, _, KH, KW = weight.shape
    Ho = (H + 2 * ((KH - 1) // 2) - KH) // stride + 1
    Wo = (W + 2 * ((KW - 1) // 2) - KW) // stride + 1
    if residual is not None:
        require_cuda(residual, "residual")
        residual = residual.contiguous()
    y = torch.empty(N, Ho, Wo, Cout, dtype=torch.float32, device=x.device)
    p = PRECISIONS[precision]
    nbytes = int(lib.avsr_conv_bn_act_workspace_bytes(N, H, W, Cin, Cout, KH, KW, stride, p))
    ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.avsr_conv_bn_act(x.data_ptr(), weight.data_ptr(), scale.data_ptr(), shift.data_ptr(), _ptr(residual),
                                   int(act), y.data_ptr(), N, H, W, Cin, Cout, KH, KW, stride, ws.data_ptr(), ws.numel(),
                                   p, _stream_handle(x.device)))
    return y
