"""Drop-in for the inference surface of espnet.nets.pytorch_backend.ctc.CTC (reference ctc.py:9-93) and for the
``proj_encoder`` Linear in front of the encoder (e2e_asr_conformer.py:31): SURVEY.md 8f #1, the steps either side of
the encoder hot path."""
from typing import Optional, Tuple

import torch

from ..engine import default_precision, require_cuda
from ..head import PreparedHead, ctc_log_probs, proj_forward


class ProjEncoder(torch.nn.Linear):
    """``torch.nn.Linear(512, 768)`` whose eval forward runs in libavsr_b200 (same parameters, same state-dict keys).
    Training / CPU tensors are refused rather than silently computed elsewhere."""

    precision: Optional[str] = None
    _head: Optional[PreparedHead] = None

    def forward(self, x):
        if self.training:
            raise NotImplementedError("ProjEncoder: inference forward only on the CUDA path (call .eval())")
        require_cuda(x, "ProjEncoder input")
        if self._head is None:
            self._head = PreparedHead(self.out_features, max(1, self.out_features // 64))
        return proj_forward(self._head, self, x, self.precision or default_precision())


class CTC(torch.nn.Module):
    """Same constructor, attributes and state-dict keys (``ctc_lo.weight``, ``ctc_lo.bias``) as the reference's CTC
    module.  ``log_softmax`` / ``softmax`` / ``argmax`` (what CTCPrefixScorer and greedy decoding call) run on the
    GPU: ctc_lo as a tensor-core GEMM, then one row-wise log-sum-exp kernel.  The training loss is row 8f #2."""

    def __init__(self, odim, eprojs, dropout_rate, reduce=True):
        super().__init__()
        self.dropout_rate = dropout_rate
        self.loss = None
        self.ctc_lo = torch.nn.Linear(eprojs, odim)
        self.dropout = torch.nn.Dropout(dropout_rate)
        self.probs = None  # for visualization (reference attribute)
        self.ctc_loss = torch.nn.CTCLoss(reduction="sum" if reduce else "none", zero_infinity=True)
        self.ignore_id = -1
        self.reduce = reduce
        self.precision: Optional[str] = None
        self._head: Optional[PreparedHead] = None

    # ------------------------------------------------------------------ helpers
    def _run(self, hs_pad, want_logp=True, want_argmax=False):
        """ctc_lo GEMM into fp32 logits (weights prepared + padded once per parameter update) followed by one row-wise
        log-softmax / arg-max pass -- libavsr_b200 ``avsr_ctc_logprobs``."""
        if self.training:
            raise NotImplementedError("CTC: inference methods only on the CUDA path (call .eval())")
        require_cuda(hs_pad, "CTC input")
        if self._head is None:
            d = self.ctc_lo.in_features
            self._head = PreparedHead(d, max(1, d // 64))
        return ctc_log_probs(self._head, self.ctc_lo, hs_pad, self.precision or default_precision(), want_logp, want_argmax)

    # ------------------------------------------------------------------ reference surface
    def forward(self, hs_pad, hlens, ys_pad):
        raise NotImplementedError("CTC.forward (the training loss, ctc.py:41-65) is not on the CUDA inference path")

    def loss_fn(self, th_pred, th_target, th_ilen, th_olen):
        raise NotImplementedError("CTC.loss_fn (ctc.py:32-39) is not on the CUDA inference path")

    def log_softmax(self, hs_pad):
        """(B, Tmax, eprojs) -> (B, Tmax, odim) log-probs (ctc.py:77-84)."""
        return self._run(hs_pad)[0]

    def softmax(self, hs_pad):
        """(B, Tmax, eprojs) -> (B, Tmax, odim) probabilities; also kept in ``self.probs`` (ctc.py:67-75)."""
        self.probs = self._run(hs_pad)[0].exp_()
        return self.probs

    def argmax(self, hs_pad):
        """(B, Tmax, eprojs) -> (B, Tmax) greedy token ids (ctc.py:86-93)."""
        return self._run(hs_pad, want_logp=False, want_argmax=True)[1]
