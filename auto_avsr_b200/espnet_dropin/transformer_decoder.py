"""Drop-in for the SCORING surface of espnet.nets.pytorch_backend.decoder.transformer_decoder.TransformerDecoder
(reference transformer_decoder.py:143-334): what ``BatchBeamSearch`` calls at every step of the search
(``batch_score`` :302-334, ``score`` :292-299).  SURVEY.md 8f #3.

Same constructor signature, sub-module / parameter names and state-dict keys as the reference (``embed.0.weight``,
``decoders.N.{self_attn,src_attn}.linear_{q,k,v,out}``, ``decoders.N.feed_forward.w_{1,2}``, ``decoders.N.norm{1,2,3}``,
``after_norm``, ``output_layer``; the ``output_norm.`` -> ``after_norm.`` load hook), so a reference checkpoint loads with
``strict=True`` and ``install_decoder(model)`` can re-home an existing ``E2E.decoder``'s parameters.

Scorer state: the reference hands the beam search, per hypothesis, the list of every layer's output over the prefix
and re-projects K/V of the whole prefix -- and of the whole encoder memory -- at every step.  Here the K/V live in the
library's per-utterance session (``auto_avsr_b200.decoder.DecoderEngine``); the state of a hypothesis is just the tuple
(utterance serial, beam slot of prefix position 0, 1, ...), which the beam search's ``select_state`` (``state[i]``)
shuffles for free.  One utterance at a time per decoder module (as the reference's CTCPrefixScorer.impl).

``forward`` -- the teacher-forced pass of the training loss (transformer_decoder.py:229-258) -- runs in libavsr_b200 as
well, forward and backward, in train and eval mode (auto_avsr_b200/decoder_train.py), on the same parameters."""
import os
from typing import Any, List, Optional, Tuple

import torch

from ..engine import default_precision
from . import scorer_interface as _si
from .layer_norm import LayerNorm
from .positionwise_feed_forward import PositionwiseFeedForward
from .repeat import repeat


class MultiHeadedAttention(torch.nn.Module):
    """Parameter container with the reference's names (transformer/attention.py:17-36); the arithmetic runs inside
    ``avsr_decoder_step``."""

    def __init__(self, n_head, n_feat, dropout_rate):
        super().__init__()
        assert n_feat % n_head == 0
        self.d_k = n_feat // n_head
        self.h = n_head
        self.linear_q = torch.nn.Linear(n_feat, n_feat)
        self.linear_k = torch.nn.Linear(n_feat, n_feat)
        self.linear_v = torch.nn.Linear(n_feat, n_feat)
        self.linear_out = torch.nn.Linear(n_feat, n_feat)
        self.attn = None
        self.dropout = torch.nn.Dropout(p=dropout_rate)

    def forward(self, *args, **kwargs):
        raise NotImplementedError("decoder attention runs inside avsr_decoder_step (TransformerDecoder.batch_score)")


class PositionalEncoding(torch.nn.Module):
    """Place-holder for ``embed.1`` (transformer/embedding.py:37-90; it has no parameters or buffers in the state dict);
    ``x * sqrt(d) + pe`` is evaluated by the embedding kernel of ``avsr_decoder_step``."""

    def __init__(self, d_model, dropout_rate, max_len=5000):
        super().__init__()
        self.d_model = d_model
        self.dropout = torch.nn.Dropout(p=dropout_rate)

    def forward(self, x):
        raise NotImplementedError("the positional encoding is applied inside avsr_decoder_step")


class DecoderLayer(torch.nn.Module):
    """Sub-module registration of the reference's DecoderLayer (transformer_decoder.py:36-61)."""

    def __init__(self, size, self_attn, src_attn, feed_forward, dropout_rate, normalize_before=True, concat_after=False):
        super().__init__()
        self.size = size
        self.self_attn = self_attn
        self.src_attn = src_attn
        self.feed_forward = feed_forward
        self.norm1 = LayerNorm(size)
        self.norm2 = LayerNorm(size)
        self.norm3 = LayerNorm(size)
        self.dropout = torch.nn.Dropout(dropout_rate)
        self.normalize_before = normalize_before
        self.concat_after = concat_after

    def forward(self, *args, **kwargs):
        raise NotImplementedError("decoder layers run inside avsr_decoder_step (TransformerDecoder.batch_score)")


def _pre_hook(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
    # transformer_decoder.py:143-156: checkpoints older than espnet 3d422f6 call after_norm "output_norm"
    old, new = prefix + "output_norm.", prefix + "after_norm."
    for k in [k for k in state_dict if k.startswith(old)]:
        state_dict[new + k[len(old):]] = state_dict.pop(k)


class TransformerDecoder(_si.BatchScorerInterface, torch.nn.Module):
    def __init__(self, odim, attention_dim=256, attention_heads=4, linear_units=2048, num_blocks=6, dropout_rate=0.1,
                 positional_dropout_rate=0.1, self_attention_dropout_rate=0.1, src_attention_dropout_rate=0.1,
                 input_layer="embed", use_output_layer=True, pos_enc_class=None, normalize_before=True,
                 concat_after=False, layer_drop_rate=0.0):
        torch.nn.Module.__init__(self)
        if input_layer != "embed" or not use_output_layer or not normalize_before or concat_after:
            raise NotImplementedError("CUDA decoder path: input_layer='embed', use_output_layer, normalize_before and "
                                      "not concat_after (what E2E builds, e2e_asr_conformer.py:41-47)")
        self._register_load_state_dict_pre_hook(_pre_hook)
        self.embed = torch.nn.Sequential(torch.nn.Embedding(odim, attention_dim),
                                         PositionalEncoding(attention_dim, positional_dropout_rate))
        self.normalize_before = normalize_before
        self.decoders = repeat(
            num_blocks,
            lambda lnum: DecoderLayer(attention_dim,
                                      MultiHeadedAttention(attention_heads, attention_dim, self_attention_dropout_rate),
                                      MultiHeadedAttention(attention_heads, attention_dim, src_attention_dropout_rate),
                                      PositionwiseFeedForward(attention_dim, linear_units, dropout_rate),
                                      dropout_rate, normalize_before, concat_after),
            layer_drop_rate)
        self.after_norm = LayerNorm(attention_dim)
        self.output_layer = torch.nn.Linear(attention_dim, odim)
        self.odim = odim
        self._cfg = (odim, attention_dim, attention_heads, linear_units, num_blocks)
        self.precision: Optional[str] = None
        #: training backward: None (TF32 GEMMs, fp32 attention core) | "bf16" (bf16 GEMM operands, tensor-core attention
        #: core).  AVSR_B200_BWD_PRECISION does not apply here: only this attribute selects it.
        self.backward_precision: Optional[str] = None
        #: verify that forward's tgt_mask / memory_mask have the form passed on as lengths (one host sync each)
        self.check_mask = os.environ.get("AVSR_B200_CHECK_MASK", "0") == "1"
        #: beam slots per position the per-utterance session is sized for (>= the beam size of the search)
        self.beam_slots = 64
        #: positions per session; None = memory length + 1 (BeamSearch.forward's maxlen with maxlenratio 0, + the <eos> step)
        self.max_steps: Optional[int] = None
        self._engine = None
        self._utterance = 0         # serial of the utterance the session currently holds
        self._lib = None            # tests inject the host replay here; None = libavsr_b200

    # ---------------------------------------------------------------- engine
    def engine(self):
        if self._engine is None:
            from ..decoder import DecoderEngine
            self._engine = DecoderEngine(*self._cfg, _lib=self._lib)
        return self._engine

    # ---------------------------------------------------------------- reference surface
    def forward(self, tgt, tgt_mask, memory, memory_mask):
        """Teacher-forced pass (transformer_decoder.py:229-258) -> (pred_pad (B, L, odim), tgt_mask), in train and eval
        mode, forward and backward in libavsr_b200 (auto_avsr_b200/decoder_train.py).  tgt (B, L) int64 token ids;
        tgt_mask (B, L, L) = target_mask(tgt, ignore_id) (key prefix AND causal: passed on as key lengths + a causal
        flag); memory (B, T, d) fp32; memory_mask (B, 1, T) prefix mask or None.  GEMMs run in ``precision`` (backward
        GEMMs TF32 unless fp32, or bf16 with ``backward_precision="bf16"``); pred_pad is a column view of the
        output-layer GEMM padded to a multiple of 8 columns."""
        if not (tgt.is_cuda and memory.is_cuda):
            raise NotImplementedError("TransformerDecoder.forward runs on CUDA tensors only (no CPU fallback)")
        from ..decoder_train import decoder_forward, target_lengths
        from ..train import explicit_backward_precision
        from .attention import mask_to_lengths
        backward = explicit_backward_precision(self.backward_precision)
        B, L = tgt.shape
        tgt_lengths = target_lengths(tgt_mask, B, L, self.check_mask)
        mem_lengths = None if memory_mask is None else mask_to_lengths(memory_mask, B, memory.size(1), check=self.check_mask)
        pred = decoder_forward(self, tgt, tgt_lengths, memory, mem_lengths, self.precision or default_precision(),
                               backward)
        return pred, tgt_mask

    def forward_one_step(self, tgt, tgt_mask, memory, memory_mask=None, cache=None):
        raise NotImplementedError("forward_one_step exposes the reference's per-layer output cache, which this path does not "
                                  "keep (K/V live in the library's session); call score / batch_score")

    def score(self, ys, state, x):
        """ScorerInterface.score (transformer_decoder.py:292-299): one hypothesis."""
        logp, states = self.batch_score(ys.unsqueeze(0), [state], x.unsqueeze(0))
        return logp.squeeze(0), states[0]

    def batch_score(self, ys: torch.Tensor, states: List[Any], xs: torch.Tensor) -> Tuple[torch.Tensor, List[Any]]:
        """BatchScorerInterface.batch_score (transformer_decoder.py:302-334).
        ys (n, ylen) int64 prefixes of equal length; states: per hypothesis ``None`` (search start) or the tuple of beam
        slots this method returned for its parent; xs (n, T, d) the encoder output repeated per hypothesis (row 0 is
        read).  -> ((n, odim) log-probabilities, next states)."""
        if self.training:
            raise NotImplementedError("TransformerDecoder: inference scoring only on the CUDA path (call .eval())")
        n, ylen = ys.shape
        eng = self.engine()
        step = ylen - 1
        if states[0] is None:
            if step != 0:
                raise ValueError("a hypothesis without a state must be the bare <sos> prefix")
            eng.begin(self, xs[0], max(self.beam_slots, n), self.max_steps, self.precision or default_precision())
            self._utterance += 1
            anc = None
            prev = [(self._utterance,)] * n
        else:
            # a state is (utterance serial, slot of position 0, slot of position 1, ...): the session holds ONE utterance,
            # so states of an utterance another search has since replaced must not be scored against its K/V
            if any(len(s) != step + 1 for s in states):
                raise ValueError("batch_score: every hypothesis must have the same prefix length")
            if any(s[0] != self._utterance for s in states):
                raise ValueError("batch_score: these hypotheses belong to an utterance whose session was replaced "
                                 "(one utterance at a time per decoder module)")
            anc = torch.tensor([s[1:] for s in states], dtype=torch.int32).t().contiguous().to(ys.device)        # (step, n)
            prev = states
        logp = eng.step(ys[:, -1].to(torch.int32), anc, step)
        return logp, [tuple(prev[i]) + (i,) for i in range(n)]
