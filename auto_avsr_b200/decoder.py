"""Host side of the attention-decoder scoring path and the CTC prefix scorer (SURVEY.md 8f #3) above the C ABI
(``avsr_prepare_decoder`` / ``avsr_decoder_begin`` / ``avsr_decoder_step`` / ``avsr_ctc_prefix_*``).

``DecoderEngine`` owns what the library borrows: the prepared weights (rebuilt when a parameter changes), the
per-utterance session (source-attention K|V of every layer + the self-attention q|k|v slots, addressed
(layer, position, beam slot)) and the step workspace.  ``CtcPrefixEngine`` wraps the three CTC entries.  Both take
device tensors and return device tensors; there is no CPU path (a CPU tensor raises) -- ``_lib`` exists so that the
CPU test-suite can replay the same host logic against tests/emu's host build of the schedule.

Reference being replaced: TransformerDecoder.batch_score / forward_one_step
(espnet/nets/pytorch_backend/decoder/transformer_decoder.py:260-334) and CTCPrefixScoreTH / CTCPrefixScorer
(espnet/nets/ctc_prefix_score.py:9-200, espnet/nets/scorers/ctc.py:9-130)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import torch

from . import _cabi
from ._cabi import DECODER_LAYER_FIELDS, DecoderConfig, DecoderLayerParams
from .engine import PRECISIONS, default_precision

LOGZERO = -10000000000.0


def _check(lib, rc: int) -> None:
    if rc != _cabi.OK:
        raise _cabi.AvsrError(f"libavsr_b200 error {rc}: {lib.avsr_last_error().decode('utf-8', 'replace')}")


class _Ctx:
    """device / stream plumbing shared by the two engines; `lib` is libavsr_b200 unless a test injected the host replay"""

    def __init__(self, _lib=None):
        self.lib = _cabi.lib if _lib is None else _lib
        self.emulated = _lib is not None

    def require(self, t: torch.Tensor, what: str, dtype=torch.float32) -> None:
        if not t.is_cuda and not self.emulated:
            raise RuntimeError(f"{what}: tensor is on {t.device}; the CUDA decoder path has no CPU fallback "
                               "(move the module and its inputs to a CUDA device)")
        if t.dtype != dtype:
            raise TypeError(f"{what}: expected {dtype}, got {t.dtype}")

    def stream(self, device) -> int:
        return 0 if self.emulated else torch.cuda.current_stream(device).cuda_stream

    def guard(self, device):
        import contextlib
        return contextlib.nullcontext() if self.emulated else torch.cuda.device(device)


class DecoderEngine(_Ctx):
    def __init__(self, odim: int, d_model: int = 768, n_heads: int = 12, linear_units: int = 3072, num_blocks: int = 6,
                 _lib=None):
        super().__init__(_lib)
        self.cfg = DecoderConfig(d_model, n_heads, linear_units, num_blocks, odim)
        self._prepared: Dict[tuple, Tuple[tuple, torch.Tensor]] = {}
        self._session: Optional[torch.Tensor] = None
        self._work: Optional[torch.Tensor] = None
        self.geom: Optional[Tuple[int, int, int]] = None       # (T, max_steps, max_hyps) of the running utterance
        self._prep_buf: Optional[torch.Tensor] = None
        self._prec: Optional[int] = None
        self.stats = {"begin": 0, "step": 0, "prepare": 0}

    # ---- weights ------------------------------------------------------------------------------------------------
    def prepare(self, module: torch.nn.Module, device, precision: str) -> torch.Tensor:
        """`module`: anything with the reference TransformerDecoder's parameter names (embed.0, decoders.N.*, after_norm,
        output_layer).  Re-prepared only when a parameter's storage / version changed."""
        sd = dict(module.named_parameters())
        names = ["embed.0.weight", "after_norm.weight", "after_norm.bias", "output_layer.weight", "output_layer.bias"]
        L = self.cfg.num_blocks
        for l in range(L):
            names += [f"decoders.{l}.{suffix}" for _, suffix in DECODER_LAYER_FIELDS]
        params = []
        for k in names:
            p = sd[k]
            self.require(p, f"decoder parameter {k}")
            if p.device != device:
                raise RuntimeError(f"decoder parameter {k} lives on {p.device}, input on {device}")
            params.append(p)
        key = (str(device), PRECISIONS[precision])
        fp = tuple((p.data_ptr(), p._version) for p in params)
        hit = self._prepared.get(key)
        if hit is not None and hit[0] == fp:
            return hit[1]
        keep = {k: p.detach().contiguous() for k, p in zip(names, params)}
        arr = (DecoderLayerParams * L)()
        for l in range(L):
            for field, suffix in DECODER_LAYER_FIELDS:
                setattr(arr[l], field, keep[f"decoders.{l}.{suffix}"].data_ptr())
        nbytes = int(self.lib.avsr_decoder_prepared_bytes(C.byref(self.cfg)))
        if nbytes == 0:
            raise _cabi.AvsrError("bad decoder configuration: " + self.lib.avsr_last_error().decode("utf-8", "replace"))
        buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        with self.guard(device):
            _check(self.lib, self.lib.avsr_prepare_decoder(
                C.byref(self.cfg), arr, keep["embed.0.weight"].data_ptr(), keep["after_norm.weight"].data_ptr(),
                keep["after_norm.bias"].data_ptr(), keep["output_layer.weight"].data_ptr(),
                keep["output_layer.bias"].data_ptr(), buf.data_ptr(), nbytes, PRECISIONS[precision], self.stream(device)))
        self._prepared[key] = (fp, buf)
        self.stats["prepare"] += 1
        return buf

    # ---- one utterance ------------------------------------------------------------------------------------------
    def begin(self, module: torch.nn.Module, memory: torch.Tensor, max_hyps: int, max_steps: Optional[int] = None,
              precision: Optional[str] = None) -> None:
        """Start decoding an utterance: memory (T, d) = the encoder output.  Projects the source-attention K|V of every
        layer once and sizes the session for `max_steps` positions (default T + 1: BeamSearch.forward's maxlen) x
        `max_hyps` beam slots."""
        precision = precision or default_precision()
        self.require(memory, "decoder memory")
        if memory.dim() != 2 or memory.size(1) != self.cfg.d_model:
            raise ValueError(f"memory must be (T, {self.cfg.d_model}), got {tuple(memory.shape)}")
        memory = memory.detach().contiguous()
        dev = memory.device
        T = memory.size(0)
        max_steps = int(max_steps or T + 1)
        self._prep_buf = self.prepare(module, dev, precision)
        self._prec = PRECISIONS[precision]
        need = int(self.lib.avsr_decoder_session_bytes(C.byref(self.cfg), T, max_steps, max_hyps))
        if self._session is None or self._session.numel() < need or self._session.device != dev:
            self._session = torch.empty(need, dtype=torch.uint8, device=dev)
        wneed = int(self.lib.avsr_decoder_step_workspace_bytes(C.byref(self.cfg), T, max_steps, max_hyps))
        if self._work is None or self._work.numel() < wneed or self._work.device != dev:
            self._work = torch.empty(wneed, dtype=torch.uint8, device=dev)
        self.geom = (T, max_steps, max_hyps)
        with self.guard(dev):
            _check(self.lib, self.lib.avsr_decoder_begin(C.byref(self.cfg), self._prep_buf.data_ptr(), memory.data_ptr(), T,
                                                         max_steps, max_hyps, self._session.data_ptr(),
                                                         self._session.numel(), self._prec, self.stream(dev)))
        self.stats["begin"] += 1

    def step(self, tokens: torch.Tensor, anc: Optional[torch.Tensor], step: int) -> torch.Tensor:
        """tokens (n) int32: last token of each hypothesis; anc (step, n) int32: beam slots of the earlier positions of
        each hypothesis' prefix (None at step 0).  Hypothesis i takes beam slot i of position `step`.
        -> (n, odim) next-token log-probabilities."""
        if self.geom is None:
            raise RuntimeError("DecoderEngine.step before begin()")
        T, max_steps, max_hyps = self.geom
        self.require(tokens, "decoder tokens", torch.int32)
        n = tokens.numel()
        if n > max_hyps:
            raise ValueError(f"{n} hypotheses exceed the session's {max_hyps} beam slots")
        if step >= max_steps:
            raise ValueError(f"step {step} exceeds the session's {max_steps} positions")
        dev = tokens.device
        if step > 0:
            if anc is None:
                raise ValueError("step > 0 needs the ancestor table")
            self.require(anc, "decoder ancestors", torch.int32)
            if tuple(anc.shape) != (step, n):
                raise ValueError(f"ancestor table must be ({step}, {n}), got {tuple(anc.shape)}")
            anc = anc.contiguous()
        logp = torch.empty(n, self.cfg.odim, dtype=torch.float32, device=dev)
        with self.guard(dev):
            _check(self.lib, self.lib.avsr_decoder_step(
                C.byref(self.cfg), self._prep_buf.data_ptr(), self._session.data_ptr(), self._session.numel(), T, max_steps,
                max_hyps, tokens.contiguous().data_ptr(), None if step == 0 else anc.data_ptr(), step, n, logp.data_ptr(),
                self._work.data_ptr(), self._work.numel(), self._prec, self.stream(dev)))
        self.stats["step"] += 1
        return logp


class CtcPrefixEngine(_Ctx):
    """CTCPrefixScoreTH for one utterance on the device: `logp` (T, O) log-posteriors stay resident, every call is two
    launches (fill + one thread per (hypothesis, candidate) running the T-step recursion in registers)."""

    def __init__(self, logp: torch.Tensor, blank: int, eos: int, _lib=None):
        super().__init__(_lib)
        self.require(logp, "CTC log-probabilities")
        if logp.dim() != 2:
            raise ValueError(f"logp must be (T, O), got {tuple(logp.shape)}")
        self.logp = logp.detach().contiguous()
        self.T, self.O = self.logp.shape
        self.blank, self.eos = int(blank), int(eos)
        dev = self.logp.device
        self.r0 = torch.empty(self.T, 2, dtype=torch.float32, device=dev)
        with self.guard(dev):
            _check(self.lib, self.lib.avsr_ctc_prefix_init(self.logp.data_ptr(), self.T, self.O, self.blank,
                                                           self.r0.data_ptr(), self.stream(dev)))

    def initial(self, n: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """(r_prev (T, 2, n), s_prev (n)) of n copies of the empty prefix"""
        return self.r0.unsqueeze(2).expand(self.T, 2, n).contiguous(), torch.zeros(n, dtype=torch.float32, device=self.r0.device)

    def score(self, out_len: int, last_ids: torch.Tensor, r_prev: torch.Tensor, s_prev: torch.Tensor, cand: torch.Tensor):
        """-> local (n, O), r (T, 2, n, S), log_psi (n, O).  last_ids (n) int32, cand (n, S) int32."""
        n, S = cand.shape
        dev = cand.device
        self.require(last_ids, "last ids", torch.int32)
        self.require(cand, "candidates", torch.int32)
        self.require(r_prev, "r_prev")
        self.require(s_prev, "s_prev")
        if tuple(r_prev.shape) != (self.T, 2, n) or tuple(s_prev.shape) != (n,):
            raise ValueError(f"state shapes {tuple(r_prev.shape)}, {tuple(s_prev.shape)} do not match n = {n}")
        local = torch.empty(n, self.O, dtype=torch.float32, device=dev)
        log_psi = torch.empty(n, self.O, dtype=torch.float32, device=dev)
        r = torch.empty(self.T, 2, n, S, dtype=torch.float32, device=dev)
        with self.guard(dev):
            _check(self.lib, self.lib.avsr_ctc_prefix_score(
                self.logp.data_ptr(), self.T, self.O, self.blank, self.eos, int(out_len), last_ids.contiguous().data_ptr(),
                r_prev.contiguous().data_ptr(), s_prev.contiguous().data_ptr(), cand.contiguous().data_ptr(), n, S,
                local.data_ptr(), r.data_ptr(), log_psi.data_ptr(), self.stream(dev)))
        return local, r, log_psi

    def select(self, r: torch.Tensor, log_psi: torch.Tensor, cand: torch.Tensor, parent: torch.Tensor, token: torch.Tensor):
        """states of the kept (parent hypothesis, new token) pairs: r_next (T, 2, m), s_next (m)"""
        m = parent.numel()
        n, S = cand.shape
        dev = cand.device
        self.require(parent, "parents", torch.int32)
        self.require(token, "tokens", torch.int32)
        r_next = torch.empty(self.T, 2, m, dtype=torch.float32, device=dev)
        s_next = torch.empty(m, dtype=torch.float32, device=dev)
        with self.guard(dev):
            _check(self.lib, self.lib.avsr_ctc_prefix_select(
                r.data_ptr(), log_psi.data_ptr(), cand.contiguous().data_ptr(), parent.contiguous().data_ptr(),
                token.contiguous().data_ptr(), self.T, self.O, n, S, m, r_next.data_ptr(), s_next.data_ptr(),
                self.stream(dev)))
        return r_next, s_next
