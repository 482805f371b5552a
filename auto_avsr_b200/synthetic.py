"""Deterministic synthetic encoder weights and inputs (no network, no checkpoints).

Keys and shapes are the reference encoder's state-dict contract
(espnet/nets/pytorch_backend/encoder/conformer_encoder.py:212-262; 40 keys per
layer + ``after_norm.{weight,bias}``, SURVEY.md §8a).  Values are *not* the
reference's default init: LayerNorm/BatchNorm affine, running statistics and all
biases are non-trivial so that a kernel that drops one of them cannot pass parity
(default init leaves them 0/1).

Every tensor is drawn from its own ``torch.Generator`` seeded by (seed, key), so the
same (seed, config) gives the same weights on any host with this torch build; the
golden fixtures under ``tests/golden`` store only the seed.
"""
from __future__ import annotations

import math
import zlib
from collections import OrderedDict
from typing import Dict, Sequence

import torch


def _gen(seed: int, key: str) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((seed * 1000003 + zlib.crc32(key.encode())) % (2 ** 63 - 1))
    return g


def encoder_state_dict(seed: int = 0, d_model: int = 768, n_heads: int = 12, linear_units: int = 3072,
                       num_blocks: int = 12, cnn_kernel: int = 31,
                       dtype: torch.dtype = torch.float32) -> "OrderedDict[str, torch.Tensor]":
    """Synthetic ``ConformerEncoder.state_dict()`` in the reference's key order."""
    dk = d_model // n_heads
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()

    def uni(key, shape, bound):
        sd[key] = (torch.rand(shape, generator=_gen(seed, key), dtype=torch.float64) * 2 - 1).mul_(bound).to(dtype)

    def nrm(key, shape, std, mean=0.0):
        sd[key] = (torch.randn(shape, generator=_gen(seed, key), dtype=torch.float64) * std + mean).to(dtype)

    def pos(key, shape, lo, hi):
        sd[key] = (torch.rand(shape, generator=_gen(seed, key), dtype=torch.float64) * (hi - lo) + lo).to(dtype)

    def linear(pfx, out_f, in_f, bias=True):
        uni(pfx + ".weight", (out_f, in_f), 1.0 / math.sqrt(in_f))
        if bias:
            nrm(pfx + ".bias", (out_f,), 0.1)

    def lnorm(pfx):
        pos(pfx + ".weight", (d_model,), 0.5, 1.5)
        nrm(pfx + ".bias", (d_model,), 0.1)

    for l in range(num_blocks):
        p = f"encoders.{l}."
        # key order == the reference module registration order (conformer_encoder.py:61-94)
        uni(p + "self_attn.pos_bias_u", (n_heads, dk), math.sqrt(6.0 / (n_heads + dk)))
        uni(p + "self_attn.pos_bias_v", (n_heads, dk), math.sqrt(6.0 / (n_heads + dk)))
        linear(p + "self_attn.linear_q", d_model, d_model)
        linear(p + "self_attn.linear_k", d_model, d_model)
        linear(p + "self_attn.linear_v", d_model, d_model)
        linear(p + "self_attn.linear_out", d_model, d_model)
        linear(p + "self_attn.linear_pos", d_model, d_model, bias=False)
        linear(p + "feed_forward.w_1", linear_units, d_model)
        linear(p + "feed_forward.w_2", d_model, linear_units)
        uni(p + "conv_module.pointwise_cov1.weight", (2 * d_model, d_model, 1), 1.0 / math.sqrt(d_model))
        nrm(p + "conv_module.pointwise_cov1.bias", (2 * d_model,), 0.1)
        uni(p + "conv_module.depthwise_conv.weight", (d_model, 1, cnn_kernel), 1.0 / math.sqrt(cnn_kernel))
        nrm(p + "conv_module.depthwise_conv.bias", (d_model,), 0.1)
        pos(p + "conv_module.norm.weight", (d_model,), 0.5, 1.5)
        nrm(p + "conv_module.norm.bias", (d_model,), 0.1)
        nrm(p + "conv_module.norm.running_mean", (d_model,), 0.1)
        pos(p + "conv_module.norm.running_var", (d_model,), 0.5, 1.5)
        sd[p + "conv_module.norm.num_batches_tracked"] = torch.tensor(100 + l, dtype=torch.long)
        uni(p + "conv_module.pointwise_cov2.weight", (d_model, d_model, 1), 1.0 / math.sqrt(d_model))
        nrm(p + "conv_module.pointwise_cov2.bias", (d_model,), 0.1)
        lnorm(p + "norm_ff")
        lnorm(p + "norm_mha")
        linear(p + "feed_forward_macaron.w_1", linear_units, d_model)
        linear(p + "feed_forward_macaron.w_2", d_model, linear_units)
        lnorm(p + "norm_ff_macaron")
        lnorm(p + "norm_conv")
        lnorm(p + "norm_final")
    lnorm("after_norm")
    return sd


def encoder_input(lengths: Sequence[int], d_model: int = 768, seed: int = 1234,
                  dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """(B, Tmax, d) O(1)-scale frames; padded positions keep random values (SURVEY.md D6)."""
    B, T = len(lengths), max(int(v) for v in lengths)
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    return torch.randn(B, T, d_model, generator=g, dtype=torch.float64).to(dtype)


def head_state_dict(seed: int = 0, idim: int = 512, d_model: int = 768, odim: int = 5049,
                    dtype: torch.dtype = torch.float32) -> "OrderedDict[str, torch.Tensor]":
    """Synthetic weights of the two Linear layers either side of the encoder in the reference's ``E2E`` model, under
    the reference's state-dict keys: ``proj_encoder`` (e2e_asr_conformer.py:31) and ``ctc.ctc_lo`` (ctc.py:21)."""
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for key, out_f, in_f in (("proj_encoder", d_model, idim), ("ctc.ctc_lo", odim, d_model)):
        w = (torch.rand((out_f, in_f), generator=_gen(seed, key + ".weight"), dtype=torch.float64) * 2 - 1)
        sd[key + ".weight"] = w.mul_(1.0 / math.sqrt(in_f)).to(dtype)
        sd[key + ".bias"] = (torch.randn((out_f,), generator=_gen(seed, key + ".bias"), dtype=torch.float64) * 0.1).to(dtype)
    return sd


def frontend_features(lengths: Sequence[int], idim: int = 512, seed: int = 4321,
                      dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """(B, Tmax, idim) stand-in for the ResNet front-end's output (the input of ``proj_encoder``)."""
    return encoder_input(lengths, idim, seed, dtype)


def decoder_state_dict(seed: int = 0, odim: int = 5049, d_model: int = 768, n_heads: int = 12, linear_units: int = 3072,
                       num_blocks: int = 6, dtype: torch.dtype = torch.float32) -> "OrderedDict[str, torch.Tensor]":
    """Synthetic ``TransformerDecoder.state_dict()`` in the reference's key order
    (espnet/nets/pytorch_backend/decoder/transformer_decoder.py:159-229; 26 keys per ``DecoderLayer`` + ``embed.0``,
    ``after_norm``, ``output_layer``).  As for the encoder every LayerNorm affine and bias is non-trivial."""
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()

    def uni(key, shape, bound):
        sd[key] = (torch.rand(shape, generator=_gen(seed, key), dtype=torch.float64) * 2 - 1).mul_(bound).to(dtype)

    def nrm(key, shape, std):
        sd[key] = (torch.randn(shape, generator=_gen(seed, key), dtype=torch.float64) * std).to(dtype)

    def linear(pfx, out_f, in_f):
        uni(pfx + ".weight", (out_f, in_f), 1.0 / math.sqrt(in_f))
        nrm(pfx + ".bias", (out_f,), 0.1)

    def lnorm(pfx):
        sd[pfx + ".weight"] = (torch.rand((d_model,), generator=_gen(seed, pfx + ".weight"), dtype=torch.float64) + 0.5).to(dtype)
        nrm(pfx + ".bias", (d_model,), 0.1)

    nrm("embed.0.weight", (odim, d_model), 1.0 / math.sqrt(d_model))      # x sqrt(d) in PositionalEncoding -> O(1) rows
    for l in range(num_blocks):
        p = f"decoders.{l}."
        for att in ("self_attn", "src_attn"):
            for lin in ("linear_q", "linear_k", "linear_v", "linear_out"):
                linear(p + att + "." + lin, d_model, d_model)
        linear(p + "feed_forward.w_1", linear_units, d_model)
        linear(p + "feed_forward.w_2", d_model, linear_units)
        lnorm(p + "norm1")
        lnorm(p + "norm2")
        lnorm(p + "norm3")
    lnorm("after_norm")
    linear("output_layer", odim, d_model)
    return sd


def _frontend_shapes(modality: str):
    """(key, shape) of every tensor of the reference front-end's state dict, in its order: Conv3dResNet registers
    ``trunk`` before ``frontend3D``; Conv1dResNet's stem is ``trunk.conv1`` / ``trunk.bn1``."""
    video = modality == "video"
    if modality not in ("video", "audio"):
        raise ValueError(f"modality must be 'video' or 'audio', got {modality!r}")
    k = (3, 3) if video else (3,)
    one = (1, 1) if video else (1,)
    out = []

    def conv_bn(conv, bn, shape):
        out.append((conv + ".weight", shape))
        for leaf in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked"):
            out.append((f"{bn}.{leaf}", (shape[0],) if leaf != "num_batches_tracked" else ()))

    if not video:
        conv_bn("trunk.conv1", "trunk.bn1", (64, 1, 80))
    cin = 64
    for i, planes in enumerate((64, 128, 256, 512)):
        for b in range(2):
            p = f"trunk.layer{i + 1}.{b}."
            conv_bn(p + "conv1", p + "bn1", (planes, cin) + k)
            conv_bn(p + "conv2", p + "bn2", (planes, planes) + k)
            if i > 0 and b == 0:
                conv_bn(p + "downsample.0", p + "downsample.1", (planes, cin) + one)
            cin = planes
    if video:
        conv_bn("frontend3D.0", "frontend3D.1", (64, 1, 5, 7, 7))
    return out


def frontend_state_dict(seed: int = 0, modality: str = "video",
                        dtype: torch.dtype = torch.float32) -> "OrderedDict[str, torch.Tensor]":
    """Synthetic ``Conv3dResNet`` / ``Conv1dResNet`` state dict under the reference's keys: He-scaled conv weights
    (std sqrt(2 / fan_in)), BatchNorm weight in [0.5, 1.5], bias and running_mean N(0, 0.1), running_var in [0.5, 1.5],
    and a non-zero ``num_batches_tracked``."""
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for key, shape in _frontend_shapes(modality):
        g = _gen(seed, key)
        leaf = key.rsplit(".", 1)[1]
        if leaf == "num_batches_tracked":
            sd[key] = torch.tensor(1000 + len(sd), dtype=torch.long)
        elif len(shape) > 1:
            fan_in = math.prod(shape[1:])
            sd[key] = (torch.randn(shape, generator=g, dtype=torch.float64) * math.sqrt(2.0 / fan_in)).to(dtype)
        elif leaf in ("weight", "running_var"):
            sd[key] = (torch.rand(shape, generator=g, dtype=torch.float64) + 0.5).to(dtype)
        else:
            sd[key] = (torch.randn(shape, generator=g, dtype=torch.float64) * 0.1).to(dtype)
    return sd


def frontend_input(modality: str, B: int, T: int, H: int = 88, W: int = 88, seed: int = 777,
                   dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """Seeded N(0, 1) input of the front-end: video (B, T, 1, H, W) clips, audio (B, T, 1) waveforms of T samples.
    Every frame / sample is drawn, so the padded tail of a shorter utterance holds non-zero data, as it may in a batch."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    shape = (B, T, 1, H, W) if modality == "video" else (B, T, 1)
    return torch.randn(shape, generator=g, dtype=torch.float64).to(dtype)


#: Canonical length sets of SURVEY.md §8 (25 Hz frames).
SHAPES: Dict[str, Sequence[int]] = {
    "S1": [100],
    "S2": [400] * 4,
    "S2r": [400, 350, 300, 250, 300],
    "S3": [100] * 16,
    "S4": [1600],
}
