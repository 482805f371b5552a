"""The beam loop of the reference's inference path with every per-step tensor kept on the device
(SURVEY.md 8f #3; BASELINE.json configs[4]).

Restates ``BatchBeamSearch`` as ``get_beam_search_decoder`` configures it (lightning.py:126-157): decoder weight
1 - ctc_weight (full scorer and pre-beam key), CTC prefix scorer weight ctc_weight (partial scorer over the
int(1.5 * beam) pre-beam candidates), no LM, length bonus 0 --
``BatchBeamSearch.search`` / ``post_process`` (espnet/nets/batch_beam_search.py:208-349), ``BeamSearch.forward``
(espnet/nets/beam_search.py:330-400) and ``end_detect`` (espnet/nets/e2e_asr_common.py:15-45).

What is different from the reference (and why it is faster on a GPU): the reference rebuilds a Python ``Hypothesis``
(namedtuple of 0-d tensors, a dict of scores, a dict of states) for every surviving hypothesis at every step,
re-batches them with ``pad_sequence`` / ``torch.tensor([...])`` and slices device tensors element by element -- about
a thousand tiny device operations and several host syncs per step at beam 40.  Here a step is: one
``avsr_decoder_step`` (slot-addressed K/V session), one pre-beam top-k, one ``avsr_ctc_prefix_select`` + ``_score``,
one flat top-k over (n x vocab), a handful of batched gathers, and ONE device -> host copy (the ``is <eos>`` flags and
scores of the new beam) for the end detection.  The reference's ``BatchBeamSearch`` itself can also drive the two
drop-in scorers unchanged (tests do both)."""
from __future__ import annotations

import math
from typing import Dict, List, NamedTuple, Optional

import torch

from .decoder import CtcPrefixEngine
from .engine import default_precision


class Hypothesis(NamedTuple):
    """What ``BeamSearch.forward`` returns per ended hypothesis (beam_search.py:19-38); ``states`` is not kept."""
    yseq: torch.Tensor
    score: float = 0.0
    scores: Dict[str, float] = dict()
    states: Dict[str, object] = dict()

    def asdict(self) -> dict:
        return dict(yseq=self.yseq.tolist(), score=float(self.score),
                    scores={k: float(v) for k, v in self.scores.items()}, states={})


def end_detect(ended: List[dict], i: int, M: int = 3, d_end: float = math.log(1 * math.exp(-10))) -> bool:
    """e2e_asr_common.py:15-45: stop when, for the last M lengths, the best ended hypothesis of that length is more than
    |d_end| below the best ended hypothesis overall."""
    if not ended:
        return False
    best = max(h["score"] for h in ended)
    count = 0
    for m in range(M):
        same = [h["score"] for h in ended if len(h["yseq"]) == i - m]
        if same and max(same) - best < d_end:
            count += 1
    return count == M


class DeviceBeamSearch:
    """``DeviceBeamSearch(decoder, ctc, ...)`` with ``decoder`` the drop-in ``TransformerDecoder`` and ``ctc`` a module
    with ``log_softmax`` (the drop-in ``CTC``); same search, same scores and the same n-best order as the reference's
    ``BatchBeamSearch`` built by ``get_beam_search_decoder(model, token_list, ctc_weight=0.1, beam_size=40)``."""

    def __init__(self, decoder, ctc, beam_size: int = 40, vocab_size: Optional[int] = None, sos: Optional[int] = None,
                 eos: Optional[int] = None, ctc_weight: float = 0.1, pre_beam_ratio: float = 1.5, blank: int = 0):
        self.decoder = decoder
        self.ctc = ctc
        self.n_vocab = int(vocab_size or decoder.odim)
        self.sos = self.n_vocab - 1 if sos is None else int(sos)
        self.eos = self.n_vocab - 1 if eos is None else int(eos)
        self.beam_size = int(beam_size)
        self.pre_beam_size = int(pre_beam_ratio * beam_size)
        self.weights = {"decoder": 1.0 - ctc_weight, "ctc": ctc_weight}
        self.blank = blank
        self.use_ctc = ctc is not None and ctc_weight != 0
        self.do_pre_beam = self.use_ctc and self.pre_beam_size < self.n_vocab          # beam_search.py:119-123
        self.stats = {"steps": 0, "utterances": 0}

    def __call__(self, x: torch.Tensor, maxlenratio: float = 0.0, minlenratio: float = 0.0) -> List[Hypothesis]:
        return self.forward(x, maxlenratio, minlenratio)

    @torch.no_grad()
    def forward(self, x: torch.Tensor, maxlenratio: float = 0.0, minlenratio: float = 0.0) -> List[Hypothesis]:
        """x (T, d): encoder output of ONE utterance (lightning.py:73-74).  -> ended hypotheses, best first."""
        T = x.shape[0]
        if maxlenratio == 0:
            maxlen = T
        elif maxlenratio < 0:
            maxlen = -1 * int(maxlenratio)
        else:
            maxlen = max(1, int(maxlenratio * T))
        dev = x.device
        O, beam = self.n_vocab, self.beam_size
        w_dec, w_ctc = self.weights["decoder"], self.weights["ctc"]
        dec = self.decoder
        eng = dec.engine()
        eng.begin(dec, x, max(beam, 1), maxlen + 1, dec.precision or default_precision())
        ctc_eng = None
        if self.use_ctc:
            ctc_eng = CtcPrefixEngine(self.ctc.log_softmax(x.unsqueeze(0))[0], self.blank, self.eos, _lib=eng.lib if eng.emulated else None)
            r_prev, s_prev = ctc_eng.initial(1)
        yseq = torch.full((1, 1), self.sos, dtype=torch.int64, device=dev)
        score = torch.zeros(1, dtype=torch.float32, device=dev)
        dec_sc = torch.zeros(1, dtype=torch.float32, device=dev)
        ctc_sc = torch.zeros(1, dtype=torch.float32, device=dev)
        anc = None
        ended: List[dict] = []
        self.stats["utterances"] += 1
        for i in range(maxlen):
            n = yseq.size(0)
            tokens = yseq[:, -1].to(torch.int32)
            dec_lp = eng.step(tokens, anc, i)                                       # (n, O)
            weighted = w_dec * dec_lp
            if ctc_eng is not None:
                if self.do_pre_beam:
                    cand = torch.topk(dec_lp, self.pre_beam_size, dim=-1)[1].to(torch.int32)
                else:
                    cand = torch.arange(O, dtype=torch.int32, device=dev).repeat(n, 1)
                local, r, log_psi = ctc_eng.score(i, tokens, r_prev, s_prev, cand)
                weighted = weighted + w_ctc * local
            weighted = weighted + score.unsqueeze(1)
            k = min(beam, n * O)
            top_v, top_i = weighted.view(-1).topk(k)                                  # batch_beam, batch_beam_search.py:86-107
            parent = torch.div(top_i, O, rounding_mode="trunc")
            tok = top_i - parent * O
            yseq = torch.cat([yseq[parent], tok.unsqueeze(1)], dim=1)
            score = top_v
            dec_sc = dec_sc[parent] + dec_lp[parent, tok]
            p32, t32 = parent.to(torch.int32), tok.to(torch.int32)
            if ctc_eng is not None:
                ctc_sc = ctc_sc[parent] + local[parent, tok]
                r_prev, s_prev = ctc_eng.select(r, log_psi, cand, p32, t32)
            else:
                ctc_sc = ctc_sc[parent]
            anc = p32.unsqueeze(0) if anc is None else torch.cat([anc[:, parent], p32.unsqueeze(0)], dim=0)
            self.stats["steps"] += 1
            # ---- post_process (batch_beam_search.py:287-349): close every hypothesis at the last position, move the ones
            # that end in <eos> to the ended list (one host copy per step), keep the rest running
            if i == maxlen - 1:
                yseq = torch.cat([yseq, torch.full((yseq.size(0), 1), self.eos, dtype=torch.int64, device=dev)], dim=1)
            host = torch.stack([(yseq[:, -1] == self.eos).float(), score, dec_sc, ctc_sc], dim=0).cpu()
            is_eos = host[0] > 0
            if bool(is_eos.any()):
                ys_host = yseq[is_eos.to(dev)].cpu()
                for row, j in enumerate(torch.nonzero(is_eos).view(-1).tolist()):
                    ended.append(dict(yseq=ys_host[row], score=float(host[1, j]), decoder=float(host[2, j]), ctc=float(host[3, j])))
            if end_detect([dict(yseq=h["yseq"], score=h["score"]) for h in ended], i) and maxlenratio == 0.0:
                break
            keep = ~is_eos
            if not bool(keep.any()):
                break
            if not bool(keep.all()):
                kd = keep.to(dev)
                yseq, score, dec_sc, ctc_sc, anc = yseq[kd], score[kd], dec_sc[kd], ctc_sc[kd], anc[:, kd].contiguous()
                if ctc_eng is not None:
                    r_prev, s_prev = r_prev[:, :, kd].contiguous(), s_prev[kd]
        nbest = sorted(ended, key=lambda h: h["score"], reverse=True)
        if not nbest:                                                                 # beam_search.py:374-384
            return [] if minlenratio < 0.1 else self.forward(x, maxlenratio, max(0.0, minlenratio - 0.1))
        return [Hypothesis(yseq=h["yseq"], score=h["score"], scores={"decoder": h["decoder"], "ctc": h["ctc"]})
                for h in nbest]

    @torch.no_grad()
    def forward_batch(self, xs: torch.Tensor, lengths=None, maxlenratio: float = 0.0,
                      minlenratio: float = 0.0) -> List[List[Hypothesis]]:
        """xs (U, T_max, d): padded encoder outputs of U utterances, lengths (U) their frames (None: all T_max).
        -> per utterance, what ``forward(xs[u, :T_u])`` returns.

        The utterances are searched in lock-step in one decoder session (``DecoderEngine.begin_batch``): one decoder step,
        one CTC scoring call, one top-k and one device -> host copy per step for the whole batch.  Rows stay grouped by
        utterance, in the order ``forward`` keeps them; each utterance has its own maxlen, end detection and n-best, and
        leaves the batch when its search ends."""
        U, T_max = xs.shape[0], xs.shape[1]
        lens = [T_max] * U if lengths is None else [int(t) for t in (lengths.tolist() if torch.is_tensor(lengths) else lengths)]
        if len(lens) != U or not all(1 <= t <= T_max for t in lens):
            raise ValueError(f"lengths {lens} must be {U} values in 1..{T_max}")
        maxlens = []
        for T in lens:                                       # forward's maxlen, per utterance
            if maxlenratio == 0:
                maxlens.append(T)
            elif maxlenratio < 0:
                maxlens.append(-1 * int(maxlenratio))
            else:
                maxlens.append(max(1, int(maxlenratio * T)))
        dev = xs.device
        O, beam = self.n_vocab, self.beam_size
        w_dec, w_ctc = self.weights["decoder"], self.weights["ctc"]
        dec = self.decoder
        eng = dec.engine()
        max_steps, max_hyps = max(maxlens) + 1, U * max(beam, 1)
        need = eng.batch_session_bytes(lens, max_hyps, max_steps)
        if not eng.emulated:
            # session + step workspace + the CTC scorer's per-step buffers (posteriors, r (T_max, 2, n, pre-beam), and
            # the (n, odim) local / log_psi / logp rows); the engine's current buffers are released first if needed
            work = eng.batch_workspace_bytes(T_max, max_hyps, max_steps)
            cand = self.pre_beam_size if self.do_pre_beam else O
            ctc_bytes = 4 * (U * T_max * O + 2 * T_max * 2 * max_hyps * cand + 4 * max_hyps * O) if self.use_ctc else 0
            total = need + work + ctc_bytes
            free = torch.cuda.mem_get_info(dev)[0] + eng.held_bytes(dev)
            if total > free:
                raise RuntimeError(f"forward_batch: {U} utterances (longest {max(lens)} frames, {max_hyps} beam slots, "
                                   f"{max_steps} positions) need {total / 2**30:.2f} GiB (decoder session "
                                   f"{need / 2**30:.2f} GiB), the device has {free / 2**30:.2f} GiB available; decode "
                                   "fewer or shorter utterances per batch")
        eng.begin_batch(dec, xs, lens, max_hyps, max_steps, dec.precision or default_precision())
        ru = torch.arange(U, dtype=torch.int32, device=dev)                     # utterance of each row
        ctc_eng = None
        if self.use_ctc:
            # per utterance, exactly the call forward makes, so every frame's posteriors have forward's bits
            lp = [self.ctc.log_softmax(xs[u, :lens[u]].unsqueeze(0))[0] for u in range(U)]
            logp = torch.zeros(U, T_max, lp[0].size(-1), dtype=torch.float32, device=dev)
            for u in range(U):
                logp[u, :lens[u]] = lp[u]
            ctc_eng = CtcPrefixEngine(logp, self.blank, self.eos, _lib=eng.lib if eng.emulated else None, lengths=lens)
            r_prev, s_prev = ctc_eng.initial(ru)
        yseq = torch.full((U, 1), self.sos, dtype=torch.int64, device=dev)
        score = torch.zeros(U, dtype=torch.float32, device=dev)
        dec_sc = torch.zeros(U, dtype=torch.float32, device=dev)
        ctc_sc = torch.zeros(U, dtype=torch.float32, device=dev)
        anc = None
        ended: List[List[dict]] = [[] for _ in range(U)]
        self.stats["utterances"] += U
        act = list(range(U))                      # utterances still searching, in batch order
        counts = [1] * U                          # their rows (grouped: utterance act[a] holds the next counts[a] rows)
        flat = torch.arange(U, dtype=torch.int64, device=dev)      # row -> a * R + its position within its utterance
        first = flat.clone()                                       # a -> its first row
        for i in range(max(maxlens)):
            A, R = len(act), max(counts)
            tokens = yseq[:, -1].to(torch.int32)
            dec_lp = eng.step(tokens, anc, i, row_utt=ru)                           # (n, O)
            weighted = w_dec * dec_lp
            if ctc_eng is not None:
                if self.do_pre_beam:
                    cand = torch.topk(dec_lp, self.pre_beam_size, dim=-1)[1].to(torch.int32)
                else:
                    cand = torch.arange(O, dtype=torch.int32, device=dev).repeat(yseq.size(0), 1)
                local, r, log_psi = ctc_eng.score(i, tokens, r_prev, s_prev, cand, row_utt=ru)
                weighted = weighted + w_ctc * local
            weighted = weighted + score.unsqueeze(1)
            # per-utterance top-k over its (rows x vocab) scores: rows scattered into (A, R, O), -inf padded
            k = min(beam, R * O)
            if A == 1:
                top_v, top_i = weighted.view(-1).topk(k)                              # forward's call
                top_v, top_i = top_v.unsqueeze(0), top_i.unsqueeze(0)
            else:
                padded = torch.full((A * R, O), float("-inf"), dtype=weighted.dtype, device=dev)
                padded[flat] = weighted
                top_v, top_i = padded.view(A, R * O).topk(k, dim=1)
            parent = torch.div(top_i, O, rounding_mode="trunc")
            tok = top_i - parent * O
            parent = parent + first.unsqueeze(1)
            counts = [min(beam, c * O) for c in counts]
            top_v, parent, tok = top_v.reshape(-1), parent.reshape(-1), tok.reshape(-1)
            if any(c < k for c in counts):           # an utterance with fewer than k (rows x vocab) entries
                sel = torch.tensor([a * k + j for a in range(A) for j in range(counts[a])], device=dev)
                top_v, parent, tok = top_v[sel], parent[sel], tok[sel]
            yseq = torch.cat([yseq[parent], tok.unsqueeze(1)], dim=1)
            score = top_v
            dec_sc = dec_sc[parent] + dec_lp[parent, tok]
            p32, t32 = parent.to(torch.int32), tok.to(torch.int32)
            if ctc_eng is not None:
                ctc_sc = ctc_sc[parent] + local[parent, tok]
                r_prev, s_prev = ctc_eng.select(r, log_psi, cand, p32, t32)
            else:
                ctc_sc = ctc_sc[parent]
            anc = p32.unsqueeze(0) if anc is None else torch.cat([anc[:, parent], p32.unsqueeze(0)], dim=0)
            ru = ru[parent]
            self.stats["steps"] += 1
            # ---- forward's post_process per utterance; one host copy for the batch
            row_u = [u for u, c in zip(act, counts) for _ in range(c)]
            host = torch.stack([(yseq[:, -1] == self.eos).float(), score, dec_sc, ctc_sc], dim=0).cpu().tolist()
            closing = [i == maxlens[u] - 1 for u in row_u]           # forward appends <eos> to every row at maxlen - 1
            done_rows = [j for j in range(len(row_u)) if closing[j] or host[0][j] > 0]
            if done_rows:
                ys_host = yseq[torch.tensor(done_rows, device=dev)].cpu()
                eos_col = torch.tensor([self.eos], dtype=ys_host.dtype)
                for row, j in enumerate(done_rows):
                    y = torch.cat([ys_host[row], eos_col]) if closing[j] else ys_host[row]
                    ended[row_u[j]].append(dict(yseq=y, score=host[1][j], decoder=host[2][j], ctc=host[3][j]))
            ended_set = set(done_rows)
            live = {u: 0 for u in act}
            for j, u in enumerate(row_u):
                live[u] += j not in ended_set
            done = {u for u in act if live[u] == 0 or (maxlenratio == 0.0 and end_detect(ended[u], i))}
            keep = [j for j, u in enumerate(row_u) if j not in ended_set and u not in done]
            if not keep:
                break
            act = [u for u in act if u not in done]
            counts = [live[u] for u in act]
            R = max(counts)
            firsts = [sum(counts[:a]) for a in range(len(act))]
            flat_h = [a * R + j for a in range(len(act)) for j in range(counts[a])]
            idx = torch.tensor(keep + flat_h + firsts, dtype=torch.int64, device=dev)           # one upload per step
            nk = len(keep)
            flat, first = idx[nk:2 * nk], idx[2 * nk:]
            if nk < len(row_u):
                kd = idx[:nk]
                yseq, score, dec_sc, ctc_sc, ru = yseq[kd], score[kd], dec_sc[kd], ctc_sc[kd], ru[kd]
                anc = anc[:, kd].contiguous()
                if ctc_eng is not None:
                    r_prev, s_prev = r_prev[:, :, kd].contiguous(), s_prev[kd]
        out: List[List[Hypothesis]] = []
        for u in range(U):
            nbest = sorted(ended[u], key=lambda h: h["score"], reverse=True)
            out.append([Hypothesis(yseq=h["yseq"], score=h["score"], scores={"decoder": h["decoder"], "ctc": h["ctc"]})
                        for h in nbest])
        empty = [u for u in range(U) if not out[u]]                                  # beam_search.py:374-384
        if empty and minlenratio >= 0.1:
            again = self.forward_batch(xs[empty], [lens[u] for u in empty], maxlenratio, max(0.0, minlenratio - 0.1))
            for u, nb in zip(empty, again):
                out[u] = nb
        return out


def shard_utterances(lengths, world: int) -> List[List[int]]:
    """Which utterances each rank decodes (SURVEY.md 8e: decoding shards by utterance, no exchange on the data path).
    Search cost grows like T * steps ~ T^2, so: longest first onto the least-loaded rank (LPT), ties to the lower rank;
    each rank's list is returned in corpus order.  Deterministic on every rank (no communication)."""
    load = [0] * world
    owner: List[List[int]] = [[] for _ in range(world)]
    for idx in sorted(range(len(lengths)), key=lambda i: (-int(lengths[i]), i)):
        r = min(range(world), key=lambda k: (load[k], k))
        owner[r].append(idx)
        load[r] += int(lengths[idx]) ** 2
    return [sorted(o) for o in owner]


def decode_sharded(search, utterances, rank: int = 0, world: int = 1, gather: bool = True, batch_size: int = 1):
    """Decode a corpus data-parallel: rank r runs `search` (a DeviceBeamSearch, or the reference's BatchBeamSearch over the
    drop-in scorers) on its share of `utterances` (list of (T_i, d) encoder outputs on that rank's device); the only
    exchange is the host-side gather of the n-best lists at the end (``torch.distributed.all_gather_object``).
    batch_size > 1 (DeviceBeamSearch only): the rank sorts its share by length and decodes batches of up to batch_size
    utterances with ``forward_batch`` -- sorting keeps the padded batch session (which grows with the longest utterance
    times the batch) small.
    -> list over the corpus of n-best lists (dicts as ``Hypothesis.asdict()``); with gather=False only this rank's entries
    are filled (others None)."""
    mine = shard_utterances([u.shape[0] for u in utterances], world)[rank]
    out: List[Optional[list]] = [None] * len(utterances)
    if batch_size > 1:
        if not hasattr(search, "forward_batch"):
            raise TypeError("decode_sharded(batch_size > 1) needs a DeviceBeamSearch (forward_batch)")
        order = sorted(mine, key=lambda i: (int(utterances[i].shape[0]), i))
        for b in range(0, len(order), batch_size):
            ids = order[b:b + batch_size]
            lens = [int(utterances[i].shape[0]) for i in ids]
            first = utterances[ids[0]]
            xs = first.new_zeros(len(ids), max(lens), first.shape[1])
            for row, i in enumerate(ids):
                xs[row, :lens[row]] = utterances[i]
            for i, nbest in zip(ids, search.forward_batch(xs, lens)):
                out[i] = [h.asdict() for h in nbest]
    else:
        for i in mine:
            out[i] = [h.asdict() for h in search(utterances[i])]
    if world > 1 and gather:
        import torch.distributed as dist
        if not dist.is_initialized():
            raise RuntimeError("decode_sharded(world > 1, gather=True) needs an initialised torch.distributed process group")
        parts: List[Optional[list]] = [None] * world
        dist.all_gather_object(parts, {i: out[i] for i in mine})
        for part in parts:
            for i, nbest in part.items():
                out[i] = nbest
    return out
