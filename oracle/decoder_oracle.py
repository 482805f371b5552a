"""CPU restatement of the reference's attention-decoder scoring path and of the beam loop that drives it
(SURVEY.md §8f #3; BASELINE.json configs[4]).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.  Nothing in the shipped package imports this file.

What it restates (paths relative to /root/reference):

* ``decoder_logp``      -- ``TransformerDecoder.forward_one_step`` / ``batch_score``
  (espnet/nets/pytorch_backend/decoder/transformer_decoder.py:260-334) with ``DecoderLayer.forward`` (:63-140),
  ``PositionalEncoding`` (transformer/embedding.py:60-90) and ``MultiHeadedAttention`` (transformer/attention.py:38-88),
  written WITHOUT the reference's per-layer output cache: every position of every prefix is recomputed, which is what
  the cache is an optimisation of (causal mask => identical values).
* ``ctc_prefix_scores`` -- ``CTCPrefixScoreTH.__call__`` for one utterance (espnet/nets/ctc_prefix_score.py:72-200,
  Algorithm 2 of Watanabe et al. 2017 vectorised over hypotheses x candidate tokens) and the state selection of
  ``CTCPrefixScorer.select_state`` (espnet/nets/scorers/ctc.py:37-60).
* ``beam_search``       -- ``BatchBeamSearch.search`` / ``post_process`` (espnet/nets/batch_beam_search.py:208-349),
  ``BeamSearch.forward`` (espnet/nets/beam_search.py:330-400) and ``end_detect`` (espnet/nets/e2e_asr_common.py:15-45)
  with the scorer set ``get_beam_search_decoder`` builds (lightning.py:126-157): decoder weight 0.9 (full scorer and
  pre-beam key), CTC weight 0.1 (partial scorer), no LM, length bonus 0.

Pinned against the unmodified reference by ``oracle/make_golden_decoder.py`` -> ``tests/golden/decoder_*.npz``
(checked in ``tests/test_oracle_decoder_golden.py``).
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

Tensor = torch.Tensor
LOGZERO = -10000000000.0      # ctc_prefix_score.py:31


# ------------------------------------------------------------------------------------------------ decoder
def _ln(x: Tensor, w: Tensor, b: Tensor) -> Tensor:
    """LayerNorm(d, eps=1e-12) (transformer/layer_norm.py:21)."""
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-12) * w + b


def _lin(x: Tensor, sd: Dict[str, Tensor], pfx: str) -> Tensor:
    return x @ sd[pfx + ".weight"].to(x.dtype).T + sd[pfx + ".bias"].to(x.dtype)


def positional_table(length: int, d: int, dtype, device=None) -> Tensor:
    """``PositionalEncoding.extend_pe`` (embedding.py:60-80): built in fp32 exactly as the reference does, then cast."""
    pos = torch.arange(0, length, dtype=torch.float32, device=device).unsqueeze(1)
    div = torch.exp(torch.arange(0, d, 2, dtype=torch.float32, device=device) * -(math.log(10000.0) / d))
    pe = torch.zeros(length, d, device=device)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe.to(dtype)


def _mha(q_in: Tensor, kv_in: Tensor, sd: Dict[str, Tensor], pfx: str, H: int, causal: bool) -> Tensor:
    """MultiHeadedAttention.forward (attention.py:59-107): ``causal`` = the subsequent_mask of the decoder's
    self-attention (transformer/mask.py:9-24); the source attention sees every memory frame (memory_mask is None in
    batch_score, transformer_decoder.py:262,302)."""
    n, Lq, d = q_in.shape
    dk = d // H
    q = _lin(q_in, sd, pfx + ".linear_q").view(n, Lq, H, dk).transpose(1, 2)
    k = _lin(kv_in, sd, pfx + ".linear_k").view(n, -1, H, dk).transpose(1, 2)
    v = _lin(kv_in, sd, pfx + ".linear_v").view(n, -1, H, dk).transpose(1, 2)
    s = q @ k.transpose(-1, -2) / math.sqrt(dk)
    if causal:
        s = s.masked_fill(~torch.tril(torch.ones(Lq, Lq, dtype=torch.bool, device=s.device)), float("-inf"))
    p = torch.softmax(s, dim=-1)
    ctx = (p @ v).transpose(1, 2).reshape(n, Lq, d)
    return _lin(ctx, sd, pfx + ".linear_out")


def decoder_hidden(sd: Dict[str, Tensor], ys: Tensor, memory: Tensor, n_heads: int) -> Tensor:
    """Hidden states of all positions, (n, ylen, d): embed -> num_blocks x DecoderLayer (pre-norm, no concat)."""
    num_blocks = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("decoders."))
    dtype = memory.dtype
    d = sd["embed.0.weight"].shape[1]
    n, L = ys.shape
    x = sd["embed.0.weight"].to(dtype)[ys] * math.sqrt(d) + positional_table(L, d, dtype, memory.device)[None]
    mem = memory[None].expand(n, -1, -1) if memory.dim() == 2 else memory
    for l in range(num_blocks):
        p = f"decoders.{l}."
        g = lambda k: sd[p + k].to(dtype)  # noqa: E731
        t = _ln(x, g("norm1.weight"), g("norm1.bias"))
        x = x + _mha(t, t, sd, p + "self_attn", n_heads, causal=True)
        t = _ln(x, g("norm2.weight"), g("norm2.bias"))
        x = x + _mha(t, mem, sd, p + "src_attn", n_heads, causal=False)
        t = _ln(x, g("norm3.weight"), g("norm3.bias"))
        x = x + _lin(torch.relu(_lin(t, sd, p + "feed_forward.w_1")), sd, p + "feed_forward.w_2")
    return x


def decoder_logp(sd: Dict[str, Tensor], ys: Tensor, memory: Tensor, n_heads: int) -> Tensor:
    """Next-token log-probabilities (n, odim) for the prefixes ``ys`` (n, ylen) -- what ``batch_score`` returns."""
    x = decoder_hidden(sd, ys, memory, n_heads)[:, -1]
    y = _ln(x, sd["after_norm.weight"].to(x.dtype), sd["after_norm.bias"].to(x.dtype))
    z = _lin(y, sd, "output_layer")
    zs = z - z.max(dim=-1, keepdim=True).values
    return zs - zs.exp().sum(dim=-1, keepdim=True).log()


# ------------------------------------------------------------------------------------------------ CTC prefix score
def ctc_initial_state(logp: Tensor, blank: int = 0) -> Tuple[Tensor, Tensor]:
    """State of the empty prefix: r^n = logzero, r^b_t = sum_{tau<=t} log p_tau(blank); prefix score 0
    (ctc_prefix_score.py:87-98).  -> r (T, 2, 1), s (1,)."""
    T = logp.shape[0]
    r = torch.full((T, 2, 1), LOGZERO, dtype=logp.dtype, device=logp.device)
    r[:, 1, 0] = torch.cumsum(logp[:, blank], 0)
    return r, torch.zeros(1, dtype=logp.dtype, device=logp.device)


def ctc_prefix_scores(logp: Tensor, out_len: int, last_ids: Sequence[int], r_prev: Tensor, s_prev: Tensor,
                      cand: Tensor, blank: int, eos: int) -> Tuple[Tensor, Tensor, Tensor]:
    """One step of the prefix scorer for n hypotheses of equal length.

    logp (T, O) CTC log-posteriors; out_len = tokens after <sos>; last_ids[n]; r_prev (T, 2, n), s_prev (n) the states
    the hypotheses carry; cand (n, S) candidate token ids.  Returns
      local (n, O)  = log_psi - s_prev  (what batch_score_partial returns: logzero-based off the candidates),
      r (T, 2, n, S) forward variables of every (hypothesis, candidate),
      log_psi (n, O) prefix log-probabilities (the next s_prev of whichever candidate is kept)."""
    T, O = logp.shape
    n, S = cand.shape
    dt = logp.dtype
    xc = logp[:, cand.reshape(-1)].reshape(T, n, S)                 # log p_t(candidate)
    xb = logp[:, blank].reshape(T, 1, 1)
    r_sum = torch.logaddexp(r_prev[:, 0], r_prev[:, 1])             # (T, n)
    same = cand == torch.as_tensor(list(last_ids), device=cand.device).reshape(n, 1)    # candidate repeats the last label
    log_phi = torch.where(same[None], r_prev[:, 1].unsqueeze(2), r_sum.unsqueeze(2))      # (T, n, S)
    rn = torch.full((T, n, S), LOGZERO, dtype=dt, device=logp.device)
    rb = torch.full((T, n, S), LOGZERO, dtype=dt, device=logp.device)
    if out_len == 0:
        rn[0] = xc[0]
    start = max(out_len, 1)
    for t in range(start, T):
        rn[t] = torch.logaddexp(rn[t - 1], log_phi[t - 1]) + xc[t]
        rb[t] = torch.logaddexp(rn[t - 1], rb[t - 1]) + xb[t]
    # log psi = logsumexp( phi_{t-1} + x_t  for t in [start, T),  r^n_{start-1} )
    phi_x = torch.cat([log_phi[:1], log_phi[:-1]], 0) + xc
    psi_c = torch.logsumexp(torch.cat([phi_x[start:], rn[start - 1:start]], 0), dim=0)    # (n, S)
    log_psi = torch.full((n, O), LOGZERO, dtype=dt, device=logp.device)
    log_psi.scatter_(1, cand, psi_c)
    log_psi[:, eos] = r_sum[T - 1]
    log_psi[:, blank] = LOGZERO
    r = torch.stack([rn, rb], dim=1)                                 # (T, 2, n, S)
    return log_psi - s_prev.reshape(n, 1), r, log_psi


# ------------------------------------------------------------------------------------------------ beam loop
def end_detect(ended: List[dict], i: int, M: int = 3, d_end: float = math.log(1 * math.exp(-10))) -> bool:
    """e2e_asr_common.py:15-45."""
    if not ended:
        return False
    best = max(h["score"] for h in ended)
    count = 0
    for m in range(M):
        same = [h["score"] for h in ended if len(h["yseq"]) == i - m]
        if same and max(same) - best < d_end:
            count += 1
    return count == M


def beam_search(score_decoder: Callable[[Tensor], Tensor], ctc_logp: Optional[Tensor], odim: int, beam: int,
                maxlen: int, w_dec: float = 0.9, w_ctc: float = 0.1, pre_beam_ratio: float = 1.5,
                blank: int = 0) -> List[dict]:
    """The search ``ModelModule.test_step`` runs (lightning.py:72; maxlenratio = minlenratio = 0).
    ``score_decoder(ys (n, ylen) int64) -> (n, odim)`` next-token log-probabilities; ``ctc_logp`` (T, odim).
    Returns the ended hypotheses sorted by score: dicts ``yseq`` (list, with <sos> and <eos>), ``score``, ``scores``."""
    sos = eos = odim - 1
    pre = int(pre_beam_ratio * beam)
    do_pre = ctc_logp is not None and w_ctc != 0 and pre < odim
    dt = ctc_logp.dtype if ctc_logp is not None else torch.float32
    run = [dict(yseq=[sos], score=torch.zeros((), dtype=dt), dec=torch.zeros((), dtype=dt), ctc=torch.zeros((), dtype=dt),
                r=None, s=None)]
    if ctc_logp is not None and w_ctc != 0:
        r0, s0 = ctc_initial_state(ctc_logp, blank)
        run[0]["r"], run[0]["s"] = r0[:, :, 0], s0[0]
    ended: List[dict] = []
    for i in range(maxlen):
        n = len(run)
        ys = torch.tensor([h["yseq"] for h in run], dtype=torch.long)
        dec = score_decoder(ys).to(dt)                                        # (n, odim)
        weighted = w_dec * dec
        part = None
        if ctc_logp is not None and w_ctc != 0:
            cand = torch.topk(dec, pre, dim=-1)[1] if do_pre else torch.arange(odim).repeat(n, 1)
            r_prev = torch.stack([h["r"] for h in run], dim=2)
            s_prev = torch.stack([h["s"] for h in run])
            part, r_new, log_psi = ctc_prefix_scores(ctc_logp, len(run[0]["yseq"]) - 1, [h["yseq"][-1] for h in run],
                                                     r_prev, s_prev, cand, blank, eos)
            weighted = weighted + w_ctc * part
        weighted = weighted + torch.stack([h["score"] for h in run]).reshape(n, 1)
        top = weighted.reshape(-1).topk(beam)[1]
        new = []
        for flat in top.tolist():
            p, tok = flat // odim, flat % odim
            h = run[p]
            item = dict(yseq=h["yseq"] + [tok], score=weighted[p, tok], dec=h["dec"] + dec[p, tok], ctc=h["ctc"], r=None, s=None)
            if part is not None:
                item["ctc"] = h["ctc"] + part[p, tok]
                pos = (cand[p] == tok).nonzero()
                item["r"] = r_new[:, :, p, int(pos[0, 0])] if len(pos) else torch.full_like(h["r"], LOGZERO)
                item["s"] = log_psi[p, tok]
            new.append(item)
        if i == maxlen - 1:
            for h in new:
                h["yseq"] = h["yseq"] + [eos]
        run = []
        for h in new:
            (ended if h["yseq"][-1] == eos else run).append(h)
        if end_detect([dict(yseq=h["yseq"], score=float(h["score"])) for h in ended], i):
            break
        if not run:
            break
    out = sorted(ended, key=lambda h: float(h["score"]), reverse=True)
    return [dict(yseq=h["yseq"], score=float(h["score"]), scores=dict(decoder=float(h["dec"]), ctc=float(h["ctc"])))
            for h in out]
