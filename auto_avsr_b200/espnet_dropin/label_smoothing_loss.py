"""Drop-in for espnet.nets.pytorch_backend.transformer.label_smoothing_loss.LabelSmoothingLoss (reference
label_smoothing_loss.py:13-63): the attention decoder's training loss (e2e_asr_conformer.py:58, :80)."""
import torch
from torch import nn

from ..decoder_train import label_smoothing_loss


class LabelSmoothingLoss(nn.Module):
    """Same constructor and attributes as the reference.  ``forward(x, target)`` computes
    sum over rows with target != padding_idx of KL(smoothed target || softmax(x)) / batch size in libavsr_b200, forward
    and backward, without the reference's host synchronisation.  ``x`` (B, L, size) may be a column view of a wider
    tensor (the decoder's padded output-layer GEMM); it is read in place.  What E2E does not use is refused:
    ``normalize_length=True``, a criterion other than ``KLDivLoss(reduction="none")``, CPU tensors."""

    def __init__(self, size, padding_idx, smoothing, normalize_length=False, criterion=nn.KLDivLoss(reduction="none")):
        super().__init__()
        self.criterion = criterion
        self.padding_idx = padding_idx
        self.confidence = 1.0 - smoothing
        self.smoothing = smoothing
        self.size = size
        self.true_dist = None
        self.normalize_length = normalize_length

    def forward(self, x, target):
        assert x.size(2) == self.size
        if self.normalize_length:
            raise NotImplementedError("LabelSmoothingLoss(normalize_length=True) is not on the CUDA path (E2E uses False)")
        if not (type(self.criterion) is nn.KLDivLoss and self.criterion.reduction == "none" and not self.criterion.log_target):
            raise NotImplementedError("LabelSmoothingLoss: only the default criterion KLDivLoss(reduction='none')")
        if not x.is_cuda:
            raise NotImplementedError("LabelSmoothingLoss runs on CUDA tensors only (no CPU fallback)")
        if x.dtype != torch.float32:
            raise TypeError(f"LabelSmoothingLoss: expected float32 logits, got {x.dtype}")
        return label_smoothing_loss(x, target, self.padding_idx, self.smoothing)
