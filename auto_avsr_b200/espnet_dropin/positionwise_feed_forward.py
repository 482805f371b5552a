"""Drop-in for espnet.nets.pytorch_backend.transformer.positionwise_feed_forward (reference :12-30)."""
from typing import Optional

import torch

from .. import ops
from ..engine import default_precision


class PositionwiseFeedForward(torch.nn.Module):
    """w_2(relu(w_1 x)) -- ReLU as in the reference (SURVEY.md D5).  Both GEMMs run in libavsr_b200 with the
    bias+ReLU and bias(+residual) epilogues fused."""

    def __init__(self, idim, hidden_units, dropout_rate):
        super().__init__()
        self.w_1 = torch.nn.Linear(idim, hidden_units)
        self.w_2 = torch.nn.Linear(hidden_units, idim)
        self.dropout = torch.nn.Dropout(dropout_rate)
        self.precision: Optional[str] = None
        # None (default backward) | "bf16"; see train.py.  An encoder option: a decoder layer's feed-forward raises if
        # it is set (the decoder trains with the default backward)
        self.backward_precision: Optional[str] = None

    def forward(self, x, residual: Optional[torch.Tensor] = None, scale: float = 1.0):
        """``residual``/``scale`` (extension): returns residual + scale * ffn(x) from the second GEMM's epilogue."""
        prec = self.precision or default_precision()
        if self.training:
            # training slice (SURVEY.md 8f #2): autograd Functions whose forward and backward run in libavsr_b200
            from ..train import feed_forward_train, module_backward_precision
            if not x.is_cuda:
                raise RuntimeError("PositionwiseFeedForward: CPU tensor; auto_avsr_b200 has no CPU fallback")
            y = feed_forward_train(self, x, prec, module_backward_precision(self))
            return y if residual is None else residual + scale * y
        h = ops.linear(x, self.w_1.weight, self.w_1.bias, relu=True, precision=prec)
        return ops.linear(h, self.w_2.weight, self.w_2.bias, residual=residual, alpha=scale, precision=prec)
