"""Functional restatement of the ResNet front-ends' eval forward, stage by stage.

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.  Nothing in the shipped package imports this file.

Written from the layer definitions (``Conv3dResNet``: Conv3d 1->64 5x7x7 / (1,2,2), BatchNorm, SiLU, MaxPool (1,3,3) /
(1,2,2), a 2-D ResNet-18 trunk per frame, the spatial mean; ``Conv1dResNet``: the waveform cut to whole 640-sample
frames, Conv1d 1->64 k80 s4 p38, BatchNorm, SiLU, a 1-D ResNet-18 trunk, AvgPool1d(20)), not from the modules: it works
on a flat ``{key: tensor}`` state dict with ``torch.nn.functional`` and states eval BatchNorm as
``(h - running_mean) / sqrt(running_var + eps) * weight + bias``.

Every stage is a function from its input to its output, and every activation between stages is channels-last in the
layout ``avsr_frontend_forward_taps`` writes: ``(frames, H, W, C)`` for video, ``(B, 1, L, C)`` for audio.  The stages
are

    tap 0  stem(sd, modality, x)          conv + BN + SiLU (video: before the max-pool)
    tap 1  pool(a) / the stem again       video max-pool; audio has no pool
    tap 2+ block(sd, modality, i, a)      BasicBlock i = 2 * layer + index, layer1.0 .. layer4.1
    out    head_mean(modality, a, B)      (B, T, 512): per-frame spatial mean / AvgPool1d(20)

dtype- and device-generic: the tensors are created on the device and in the dtype of the inputs.  Pinned to the
reference modules by ``tests/test_frontend_stages_cpu.py`` (every tap, and the golden fixtures).
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor

BN_EPS = 1e-5          # torch.nn.BatchNorm{1,2,3}d default
AUDIO_FRAME = 640      # samples per 25 Hz output frame at 16 kHz
AUDIO_POOL = 20        # stem stride 4 x trunk stride 8 = 32 samples per position; 640 / 32 = 20 positions per frame
N_TAPS = 10


def to_channels_last(h: Tensor) -> Tensor:
    """(N, C, H, W) -> (N, H, W, C); (N, C, L) -> (N, 1, L, C)"""
    if h.dim() == 3:
        return h.permute(0, 2, 1).unsqueeze(1).contiguous()
    return h.permute(0, 2, 3, 1).contiguous()


def from_channels_last(a: Tensor, modality: str) -> Tensor:
    """inverse of to_channels_last: video (N, H, W, C) -> (N, C, H, W); audio (N, 1, L, C) -> (N, C, L)"""
    if modality == "audio":
        return a.squeeze(1).permute(0, 2, 1)
    return a.permute(0, 3, 1, 2)


def batch_norm(h: Tensor, sd: Dict[str, Tensor], prefix: str, eps: float = BN_EPS) -> Tensor:
    """eval BatchNorm over dim 1 of (N, C, ...): (h - mean) / sqrt(var + eps) * gamma + beta, in h's dtype"""
    shape = (1, -1) + (1,) * (h.dim() - 2)

    def p(leaf):
        return sd[prefix + leaf].to(h).view(shape)

    return (h - p("running_mean")) / torch.sqrt(p("running_var") + eps) * p("weight") + p("bias")


def silu(h: Tensor) -> Tensor:
    return h * torch.sigmoid(h)


# ---------------------------------------------------------------- stems
def video_stem(sd: Dict[str, Tensor], x: Tensor) -> Tensor:
    """x (B, T, 1, H, W) -> (B*T, Hs, Ws, 64).  The 5-frame temporal taps run inside each utterance's row of the padded
    batch: zero padding of 2 frames at either end of the row, never the neighbouring row."""
    B, T = x.shape[:2]
    h = F.conv3d(x.transpose(1, 2), sd["frontend3D.0.weight"].to(x), stride=(1, 2, 2), padding=(2, 3, 3))
    h = silu(batch_norm(h, sd, "frontend3D.1."))                     # (B, 64, T, Hs, Ws)
    return h.permute(0, 2, 3, 4, 1).reshape(B * T, h.shape[3], h.shape[4], h.shape[1]).contiguous()


def video_pool(a: Tensor) -> Tensor:
    """MaxPool (1,3,3) / (1,2,2) / padding (0,1,1) of every frame: (N, Hs, Ws, C) -> (N, H0, W0, C)"""
    return to_channels_last(F.max_pool2d(a.permute(0, 3, 1, 2), 3, stride=2, padding=1))


def audio_stem(sd: Dict[str, Tensor], x: Tensor) -> Tensor:
    """x (B, samples, 1) -> (B, 1, Ls, 64): only whole 640-sample frames are data; the tail past the last one is cut
    before the convolution (k 80, stride 4, padding 38, so Ls = 160 per frame)."""
    keep = x.shape[1] // AUDIO_FRAME * AUDIO_FRAME
    h = F.conv1d(x[:, :keep, :].transpose(1, 2), sd["trunk.conv1.weight"].to(x), stride=4, padding=38)
    return to_channels_last(silu(batch_norm(h, sd, "trunk.bn1.")))


def stem(sd: Dict[str, Tensor], modality: str, x: Tensor) -> Tensor:
    return video_stem(sd, x) if modality == "video" else audio_stem(sd, x)


def pool(modality: str, a: Tensor) -> Tensor:
    """tap 0 -> tap 1: the video max-pool; the audio stem feeds the trunk directly"""
    return video_pool(a) if modality == "video" else a


# ---------------------------------------------------------------- trunk
def block_name(i: int) -> str:
    """BasicBlock i (0..7) -> its state-dict prefix, trunk.layer1.0. .. trunk.layer4.1."""
    return f"trunk.layer{i // 2 + 1}.{i % 2}."


def conv(h: Tensor, w: Tensor, stride: int) -> Tensor:
    """the trunk's bias-free convs with padding (k - 1) / 2: 2-D for video, 1-D for audio (by the weight's rank)"""
    w = w.to(h)
    pad = (w.shape[-1] - 1) // 2
    return F.conv2d(h, w, stride=stride, padding=pad) if w.dim() == 4 else F.conv1d(h, w, stride=stride, padding=pad)


def block(sd: Dict[str, Tensor], modality: str, i: int, a: Tensor) -> Tensor:
    """BasicBlock i on a channels-last activation: y = SiLU(BN2(conv2 SiLU(BN1(conv1 x))) + r), r = BN(conv1x1 x) in
    the first block of layer2..4 (stride 2), else x."""
    p = block_name(i)
    stride = 2 if i in (2, 4, 6) else 1
    x = from_channels_last(a, modality)
    h = silu(batch_norm(conv(x, sd[p + "conv1.weight"], stride), sd, p + "bn1."))
    h = batch_norm(conv(h, sd[p + "conv2.weight"], 1), sd, p + "bn2.")
    if p + "downsample.0.weight" in sd:
        r = batch_norm(conv(x, sd[p + "downsample.0.weight"], stride), sd, p + "downsample.1.")
    else:
        r = x
    return to_channels_last(silu(h + r))


def head_mean(modality: str, a: Tensor, B: int) -> Tensor:
    """the last tap -> (B, T, 512): video, the mean over each frame's pixels; audio, the mean of each 20 consecutive
    positions (AvgPool1d(20), whose floor drops a partial window)"""
    if modality == "video":
        return a.mean(dim=(1, 2)).reshape(B, -1, a.shape[-1])
    h = F.avg_pool1d(from_channels_last(a, modality), AUDIO_POOL, AUDIO_POOL)
    return h.transpose(1, 2)


# ---------------------------------------------------------------- chained
def next_tap(sd: Dict[str, Tensor], modality: str, k: int, prev: Tensor) -> Tensor:
    """tap k from tap k - 1 (k >= 1): the stage a test isolates by feeding it the library's own tap k - 1"""
    return pool(modality, prev) if k == 1 else block(sd, modality, k - 2, prev)


def taps(sd: Dict[str, Tensor], modality: str, x: Tensor) -> Tuple[List[Tensor], Tensor]:
    """all 10 taps and the (B, T, 512) output, chained from the raw clip / waveform"""
    out = [stem(sd, modality, x)]
    for k in range(1, N_TAPS):
        out.append(next_tap(sd, modality, k, out[-1]))
    return out, head_mean(modality, out[-1], x.shape[0])


def forward(sd: Dict[str, Tensor], modality: str, x: Tensor) -> Tensor:
    return taps(sd, modality, x)[1]
