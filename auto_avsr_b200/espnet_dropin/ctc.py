"""Drop-in for espnet.nets.pytorch_backend.ctc.CTC (reference ctc.py:9-93) and for the ``proj_encoder`` Linear in front
of the encoder (e2e_asr_conformer.py:31): SURVEY.md 8f #1, the steps either side of the encoder hot path, and the CTC
loss of the training step (e2e_asr_conformer.py:77)."""
from typing import Optional

import torch
import torch.nn.functional as F

from .. import ops
from ..engine import default_precision, require_cuda
from ..head import PreparedHead, ctc_log_probs, proj_forward
from ..train import CtcLossFn, LinearFn, ctc_loss_forward, explicit_backward_precision


class ProjEncoder(torch.nn.Linear):
    """``torch.nn.Linear(512, 768)`` that runs in libavsr_b200 (same parameters, same state-dict keys).  Eval: on the
    prepared weights.  Train: ``LinearFn`` (forward GEMM in the module's precision, dgrad / wgrad as TF32 GEMMs in one
    ``avsr_linear_bwd`` call, bf16 ones with ``backward_precision="bf16"``), so the input gradient flows back to the
    front-end.  CPU tensors are refused rather than silently computed elsewhere."""

    precision: Optional[str] = None
    #: training backward: None (default) | "bf16"; AVSR_B200_BWD_PRECISION does not apply here
    backward_precision: Optional[str] = None
    _head: Optional[PreparedHead] = None

    def forward(self, x):
        prec = self.precision or default_precision()
        if self.training:
            return LinearFn.apply(x, self.weight, self.bias, False, prec,
                                  explicit_backward_precision(self.backward_precision))
        require_cuda(x, "ProjEncoder input")
        if self._head is None:
            self._head = PreparedHead(self.out_features, max(1, self.out_features // 64))
        return proj_forward(self._head, self, x, prec)


class CTC(torch.nn.Module):
    """Same constructor, attributes and state-dict keys (``ctc_lo.weight``, ``ctc_lo.bias``) as the reference's CTC
    module.  ``forward`` (the training loss) and ``log_softmax`` / ``softmax`` / ``argmax`` (what CTCPrefixScorer and
    greedy decoding call, eval mode) run on the GPU: ctc_lo as a tensor-core GEMM, then the library's row kernels."""

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
        #: backward of the ctc_lo GEMM: None (default) | "bf16"; AVSR_B200_BWD_PRECISION does not apply here
        self.backward_precision: Optional[str] = None
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
        """CTC loss (ctc.py:41-65) -> (loss, ys_hat).  hs_pad (B, Tmax, eprojs), hlens (B), ys_pad (B, Lmax) with
        ``ignore_id`` (-1) entries dropped wherever they sit; loss = CTCLoss(zero_infinity) / B, summed when ``reduce``;
        ys_hat = the (Tmax, B, odim) logits.  ctc_lo is ``LinearFn`` on the weight padded to a multiple of 8 rows (the
        tensor-core GEMM's N; its backward bf16 with ``backward_precision="bf16"``), the loss ``CtcLossFn`` (fp32);
        labels and lengths stay on the device.  Without autograd
        (``torch.no_grad()``, as in Lightning's validation step, or when nothing involved needs a gradient) the loss is
        computed without the beta recursion and nothing is kept for a backward."""
        if not hs_pad.is_cuda:
            raise NotImplementedError("CTC.forward: the CTC loss runs on CUDA tensors only (no CPU fallback)")
        require_cuda(hs_pad, "CTC input")
        prec = self.precision or default_precision()
        backward = explicit_backward_precision(self.backward_precision)
        B = hs_pad.size(0)
        odim = self.ctc_lo.out_features
        w, b = self.ctc_lo.weight, self.ctc_lo.bias
        npad = (odim + 7) // 8 * 8
        if npad != odim:
            w, b = F.pad(w, (0, 0, 0, npad - odim)), F.pad(b, (0, npad - odim))
        x = self.dropout(hs_pad)
        if torch.is_grad_enabled() and (x.requires_grad or w.requires_grad or b.requires_grad):
            logits = LinearFn.apply(x, w, b, False, prec, backward)
            nll = CtcLossFn.apply(logits, hlens, ys_pad, odim, self.ignore_id)
        else:
            with torch.no_grad():
                logits = ops.linear(x, w, b, precision=prec)
                nll, _ = ctc_loss_forward(logits, hlens, ys_pad, odim, self.ignore_id, want_grad=False)
        loss = nll / B
        if self.reduce:
            loss = loss.sum()
        self.loss = loss
        return self.loss, logits[..., :odim].transpose(0, 1)

    def loss_fn(self, th_pred, th_target, th_ilen, th_olen):
        raise NotImplementedError("CTC.loss_fn (ctc.py:32-39) is not on the CUDA path: CTC.forward computes the loss")

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
