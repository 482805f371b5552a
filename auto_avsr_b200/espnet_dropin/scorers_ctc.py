"""Drop-in for espnet.nets.scorers.ctc.CTCPrefixScorer on its batch path (reference scorers/ctc.py:9-130, the scorer
``E2E.scorers()`` hands to the beam search, e2e_asr_conformer.py:58-59) with CTCPrefixScoreTH
(ctc_prefix_score.py:9-200) behind it.  SURVEY.md 8f #3.

The reference runs the T-frame forward recursion as a Python loop of five tensor ops per frame for every search step,
stacks and slices the per-hypothesis states on the host side of the beam search, and keeps log-posteriors duplicated
as a (2, T, B, O) tensor.  Here the posteriors stay resident once; a step is ``avsr_ctc_prefix_select`` (states of the
kept hypotheses gathered in one launch) + ``avsr_ctc_prefix_score`` (one thread per (hypothesis, candidate) runs the
whole recursion in registers).  ``select_state`` therefore does no work: it returns a reference to the step's batch
state and the (hypothesis, token) pair; the gather happens, batched, at the next ``batch_score_partial``."""
from typing import Any, List, Tuple

import torch

from . import scorer_interface as _si


class _StepState:
    """everything one batch_score_partial call produced: r (T, 2, n, S), log_psi (n, O), cand (n, S)"""
    __slots__ = ("r", "log_psi", "cand")

    def __init__(self, r, log_psi, cand):
        self.r, self.log_psi, self.cand = r, log_psi, cand


class CTCPrefixScorer(_si.BatchPartialScorerInterface):
    def __init__(self, ctc: torch.nn.Module, eos: int):
        self.ctc = ctc
        self.eos = eos
        self.impl = None
        self._lib = None            # tests inject the host replay here; None = libavsr_b200

    # ---------------------------------------------------------------- reference surface (batch path)
    def batch_init_state(self, x: torch.Tensor):
        """scorers/ctc.py:86-97: log-posteriors of the utterance; the initial state is None."""
        from ..decoder import CtcPrefixEngine
        logp = self.ctc.log_softmax(x.unsqueeze(0))                     # (1, T, O)
        self.impl = CtcPrefixEngine(logp[0], 0, self.eos, _lib=self._lib)
        return None

    def select_state(self, state, i, new_id=None):
        """scorers/ctc.py:37-60.  A list of per-hypothesis states (the beam search's bookkeeping) is indexed; the batch
        state of the last step becomes a lazy (step, hypothesis, token) reference."""
        if state is None:
            return None
        if isinstance(state, _StepState):
            return (state, int(i), int(new_id))
        return state[i]

    def batch_score_partial(self, y: torch.Tensor, ids: torch.Tensor, state: List[Any], x: torch.Tensor):
        """scorers/ctc.py:99-130 -> CTCPrefixScoreTH.__call__: y (n, ylen) prefixes, ids (n, S) candidate tokens,
        state: per hypothesis None or what select_state returned.  -> ((n, O) local scores, batch state)."""
        if self.impl is None:
            raise RuntimeError("CTCPrefixScorer.batch_score_partial before batch_init_state")
        n = y.size(0)
        dev = y.device
        if state[0] is None:
            r_prev, s_prev = self.impl.initial(n)
        else:
            step_state = state[0][0]
            if any(s[0] is not step_state for s in state):
                raise ValueError("CTCPrefixScorer: hypotheses of one step must come from the same previous step")
            parent = torch.tensor([s[1] for s in state], dtype=torch.int32).to(dev)
            token = torch.tensor([s[2] for s in state], dtype=torch.int32).to(dev)
            r_prev, s_prev = self.impl.select(step_state.r, step_state.log_psi, step_state.cand, parent, token)
        cand = ids.to(torch.int32).contiguous()
        local, r, log_psi = self.impl.score(y.size(1) - 1, y[:, -1].to(torch.int32), r_prev, s_prev, cand)
        return local, _StepState(r, log_psi, cand)

    # ---------------------------------------------------------------- not on the batch path
    def init_state(self, x):
        raise NotImplementedError("CTCPrefixScorer: the non-batch numpy path (scorers/ctc.py:25-36) is not on the CUDA path; "
                                  "use BatchBeamSearch / DeviceBeamSearch")

    def score_partial(self, y, ids, state, x):
        raise NotImplementedError("CTCPrefixScorer.score_partial: use batch_score_partial")
