"""Drop-ins for the reference's ResNet front-ends: ``Conv3dResNet`` (espnet/nets/pytorch_backend/frontend/resnet.py) and
``Conv1dResNet`` (frontend/resnet1d.py), with the same constructor, sub-module tree and state-dict keys.

Every sub-module is a plain ``nn.Conv*`` / ``nn.BatchNorm*``, so Lightning's ``sync_batchnorm`` conversion still
applies.  ``train()``: the sub-modules run as ordinary torch modules (autograd, running-statistics updates), exactly as
in the reference -- or, with ``library_train = True`` and CUDA inputs, forward and backward run in libavsr_b200
(auto_avsr_b200/frontend_train.py) on the same parameters and buffers.  ``eval()``: one ``avsr_frontend_forward`` call on prepared weights (auto_avsr_b200/frontend.py), reading
the BatchNorm constants from whatever ``_BatchNorm`` module sits in each slot.  CPU tensors are refused: there is no CPU
fallback for the eval path.  Only ``relu_type="swish"`` (the one ``E2E`` builds) is implemented."""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import nn

from ..engine import default_precision
from ..frontend import PreparedFrontend, frontend_forward


def _check_relu_type(relu_type: str) -> None:
    if relu_type != "swish":
        raise NotImplementedError(f"front-end relu_type={relu_type!r}: only 'swish' is implemented")


class BasicBlock(nn.Module):
    """conv3x3 -> BN -> SiLU -> conv3x3 -> BN, + (downsampled) input, SiLU; 2-D (video) or 1-D (audio)."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, relu_type="swish", dims=2):
        super().__init__()
        _check_relu_type(relu_type)
        Conv, BN = (nn.Conv2d, nn.BatchNorm2d) if dims == 2 else (nn.Conv1d, nn.BatchNorm1d)
        self.conv1 = Conv(inplanes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn1 = BN(planes)
        self.relu1 = nn.SiLU(inplace=True)
        self.relu2 = nn.SiLU(inplace=True)
        self.conv2 = Conv(planes, planes, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn2 = BN(planes)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        out = self.relu1(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        out += x if self.downsample is None else self.downsample(x)
        return self.relu2(out)


def _make_layers(module: nn.Module, relu_type: str, dims: int) -> None:
    Conv, BN = (nn.Conv2d, nn.BatchNorm2d) if dims == 2 else (nn.Conv1d, nn.BatchNorm1d)
    inplanes = 64
    for i, planes in enumerate((64, 128, 256, 512)):
        stride = 1 if i == 0 else 2
        ds = None
        if stride != 1 or inplanes != planes:
            ds = nn.Sequential(Conv(inplanes, planes, kernel_size=1, stride=stride, bias=False), BN(planes))
        blocks = [BasicBlock(inplanes, planes, stride, ds, relu_type, dims), BasicBlock(planes, planes, 1, None, relu_type, dims)]
        setattr(module, f"layer{i + 1}", nn.Sequential(*blocks))
        inplanes = planes


def _block_pairs(trunk: nn.Module) -> List[Tuple[nn.Module, nn.Module]]:
    pairs = []
    for layer in (trunk.layer1, trunk.layer2, trunk.layer3, trunk.layer4):
        for block in layer:
            pairs += [(block.conv1, block.bn1), (block.conv2, block.bn2)]
            if block.downsample is not None:
                pairs.append((block.downsample[0], block.downsample[1]))
    return pairs


class ResNet(nn.Module):
    def __init__(self, relu_type="swish"):
        super().__init__()
        _check_relu_type(relu_type)
        self.inplanes = 64
        self.relu_type = relu_type
        _make_layers(self, relu_type, 2)
        self.avgpool = nn.AdaptiveAvgPool2d(1)

    def forward(self, x):
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.avgpool(x).view(x.size(0), -1)


class ResNet1D(nn.Module):
    def __init__(self, relu_type="swish", a_upsample_ratio=1):
        super().__init__()
        _check_relu_type(relu_type)
        self.inplanes = 64
        self.relu_type = relu_type
        self.a_upsample_ratio = a_upsample_ratio
        self.conv1 = nn.Conv1d(1, 64, kernel_size=80, stride=4, padding=38, bias=False)
        self.bn1 = nn.BatchNorm1d(64)
        self.relu = nn.SiLU(inplace=True)
        _make_layers(self, relu_type, 1)
        self.avgpool = nn.AvgPool1d(kernel_size=20 // a_upsample_ratio, stride=20 // a_upsample_ratio)

    def forward(self, x):
        x = self.relu(self.bn1(self.conv1(x)))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.avgpool(x)


class _LibraryFrontend(nn.Module):
    modality = ""
    precision: Optional[str] = None
    #: train() forward and backward in the library instead of torch sub-modules (install_frontend(..., library_train=True))
    library_train: bool = False
    _prep: Optional[PreparedFrontend] = None

    def conv_bn_pairs(self) -> List[Tuple[nn.Module, nn.Module]]:
        raise NotImplementedError

    def _library_forward(self, xs_pad):
        if self._prep is None:
            self._prep = PreparedFrontend()
        return frontend_forward(self._prep, self.modality, self.conv_bn_pairs(), xs_pad,
                                self.precision or default_precision())

    def _library_train_forward(self, xs_pad):
        from ..frontend_train import frontend_train_forward
        return frontend_train_forward(self, xs_pad)


class Conv3dResNet(_LibraryFrontend):
    """Video front-end: Conv3d 1->64 (5,7,7) / (1,2,2) -> BN -> SiLU -> MaxPool3d, then a 2-D ResNet-18 trunk per frame
    and a spatial mean: (B, T, 1, H, W) -> (B, T, 512)."""
    modality = "video"

    def __init__(self, backbone_type="resnet", relu_type="swish"):
        super().__init__()
        _check_relu_type(relu_type)
        self.backbone_type = backbone_type
        self.frontend_nout = 64
        self.trunk = ResNet(relu_type=relu_type)
        self.frontend3D = nn.Sequential(
            nn.Conv3d(1, 64, kernel_size=(5, 7, 7), stride=(1, 2, 2), padding=(2, 3, 3), bias=False),
            nn.BatchNorm3d(64),
            nn.SiLU(inplace=True),
            nn.MaxPool3d(kernel_size=(1, 3, 3), stride=(1, 2, 2), padding=(0, 1, 1)),
        )

    def conv_bn_pairs(self):
        return [(self.frontend3D[0], self.frontend3D[1])] + _block_pairs(self.trunk)

    def forward(self, xs_pad):
        if not self.training:
            return self._library_forward(xs_pad)
        if self.library_train:
            return self._library_train_forward(xs_pad)
        xs_pad = xs_pad.transpose(2, 1)
        B = xs_pad.size(0)
        xs_pad = self.frontend3D(xs_pad)
        Tnew = xs_pad.shape[2]
        n, c, t, h, w = xs_pad.shape
        xs_pad = xs_pad.transpose(1, 2).reshape(n * t, c, h, w)
        xs_pad = self.trunk(xs_pad)
        return xs_pad.view(B, Tnew, xs_pad.size(1))


class Conv1dResNet(_LibraryFrontend):
    """Audio front-end: the waveform cut to whole 640-sample frames, Conv1d 1->64 k80 s4 -> BN -> SiLU, a 1-D ResNet-18
    trunk and AvgPool1d(20): (B, samples, 1) -> (B, samples // 640, 512)."""
    modality = "audio"

    def __init__(self, relu_type="swish", a_upsample_ratio=1):
        super().__init__()
        _check_relu_type(relu_type)
        if a_upsample_ratio != 1:
            raise NotImplementedError("front-end a_upsample_ratio != 1 is not implemented")
        self.a_upsample_ratio = a_upsample_ratio
        self.trunk = ResNet1D(relu_type=relu_type, a_upsample_ratio=a_upsample_ratio)

    def conv_bn_pairs(self):
        return [(self.trunk.conv1, self.trunk.bn1)] + _block_pairs(self.trunk)

    def forward(self, xs_pad):
        if not self.training:
            return self._library_forward(xs_pad)
        if self.library_train:
            return self._library_train_forward(xs_pad)
        T = xs_pad.size(1)
        xs_pad = xs_pad[:, : T // 640 * 640, :].transpose(1, 2)
        return self.trunk(xs_pad).transpose(1, 2)
