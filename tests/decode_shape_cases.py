"""Bodies of the decoding-path checks at the shapes the beam search runs (tests/test_zzz_gpu_decode_shapes.py on the GPU,
tests/test_decode_shapes_cpu.py on the host replay of tests/emu at reduced sizes; one case alone in its own process:
python tests/decode_shape_cases.py <case> [args...], with AVSR_CASES_DRYRUN=1 for the host replay).

Three groups:
  A  decoder steps deep into a prefix, with a full beam that is re-ordered, forked, shrunk and re-grown at every step,
     against oracle.decoder_oracle.decoder_logp in float64 (full recompute of every prefix: no cache, no ancestor table);
  B  the CTC prefix scorer driven along whole utterances (diffuse and CTC-shaped posteriors, T = 1 ... 1600), against
     oracle.decoder_oracle.ctc_prefix_scores in float64 carried with its own float64 state, with the reference's fp32
     CTCPrefixScoreTH (oracle/_ref) measured against the same float64 numbers beside it;
  C  DeviceBeamSearch.forward at bench.py's decode shape against the reference's BatchBeamSearch in float64.

The float64 yardsticks run on the device of the case.  Every comparison goes through helpers.record.  GPU bounds are
about 4x the errors observed on an NVIDIA H100 80GB HBM3; the host-replay bounds 4x what the replay shows."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from decoder_gpu_cases import TOL_BEST_F16, TOL_NBEST_FP32  # noqa: E402
from helpers import record  # noqa: E402
from oracle import build_ref  # noqa: E402
from oracle import decoder_oracle as DO  # noqa: E402

FULL6 = dict(odim=5049, d=768, H=12, F=3072, L=6)
FULL2 = dict(FULL6, L=2)
TINY = dict(odim=37, d=128, H=2, F=256, L=2)

# ---- A: size tables.  `few` and the single-row steps of _row_counts fall on checked steps 16 and 32.
DEPTH = {
    "A1": dict(cfg=FULL6, T=100, hyps=40, steps=101, checked=(0, 1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 99, 100)),
    "A2": dict(cfg=FULL2, T=400, hyps=40, steps=401, checked=(0, 127, 128, 129, 255, 256, 257, 399, 400)),
    "A3": dict(cfg=FULL2, T=1600, hyps=40, steps=4, checked=(0, 1, 2, 3)),
    "A4": dict(cfg=TINY, T=1, hyps=3, steps=2, checked=(0, 1)),
    "dry": dict(cfg=TINY, T=23, hyps=5, steps=40, checked=(0, 1, 2, 16, 17, 31, 32, 33, 39)),
}
BATCH_DEPTH = {
    "gpu": dict(cfg=FULL6, Ts=(100, 97, 64, 1), hyps=10, steps=66, checked=(63, 64, 65)),
    "dry": dict(cfg=TINY, Ts=(23, 17, 5, 1), hyps=2, steps=20, checked=(15, 16, 17)),
}
# max |logp - float64| over the rows of a checked step.  The error does not grow with depth (fp32: 2.8e-6 at step 0,
# 2.5e-6 ... 4.7e-6 at steps 1 ... 400; DESIGN.md 4b has the table), so one bound per precision serves every step.
TOL_DEPTH = {"fp32": 1.9e-5, "tf32": 5e-3, "f16": 5e-3, "replay": 1.5e-6}

# ---- B: sizes (odim, rows, candidates per row, utterance lengths)
CTC_SIZES = {"gpu": dict(O=5049, n=40, S=60, Ts=(1, 2, 3, 100, 400, 1600)),
             "dry": dict(O=37, n=5, S=8, Ts=(1, 2, 3, 100))}
CTC_BATCH = {"gpu": dict(O=5049, n=40, S=60, Ts=(1, 2, 37, 100, 250, 400, 900, 1600), steps=6),
             "dry": dict(O=37, n=5, S=8, Ts=(1, 2, 3, 100), steps=6)}
# absolute error of `local` (what the beam adds, x 0.1, to a score) at the candidates, by utterance length; lengths
# between the listed ones take the next larger entry
TOL_CTC_LOCAL = {3: 1.7e-5, 100: 2.1e-3, 400: 1.4e-2, 1600: 0.17}
TOL_CTC_LOCAL_REPLAY = {3: 8e-6, 100: 8e-4}
# log_psi, r and the initial state, relative to max(1, |float64 value|).  T serial fp32 logaddexp steps on values that
# reach 1e4 in magnitude: the error grows with T, and the reference's fp32 recursion shows the same numbers.
TOL_CTC_REL = {3: 6e-7, 100: 3e-6, 400: 6.4e-6, 1600: 5e-5}


class Backend:
    """where a case runs: the device library on cuda:0, or (dry) the host replay of tests/emu on the CPU, fp32 only"""

    def __init__(self, dry=None):
        self.dry = os.environ.get("AVSR_CASES_DRYRUN") == "1" if dry is None else dry
        self.dev = torch.device("cpu" if self.dry else "cuda:0")
        self.lib = None
        if self.dry:
            from emu import build
            self.lib = build.load("decoder_batch")

    def sync(self):
        if not self.dry:
            torch.cuda.synchronize()

    def i32(self, values):
        return torch.tensor(values, dtype=torch.int32, device=self.dev)


def _engine(bk, cfg, seed):
    """-> (DecoderEngine, parameter bag on the device, the same weights in float64 for the oracle)"""
    from auto_avsr_b200.decoder import DecoderEngine
    from auto_avsr_b200.synthetic import decoder_state_dict
    from test_decoder_batch_emu_cpu import _Params
    sd = decoder_state_dict(seed, cfg["odim"], cfg["d"], cfg["H"], cfg["F"], cfg["L"])
    eng = DecoderEngine(cfg["odim"], cfg["d"], cfg["H"], cfg["F"], cfg["L"], _lib=bk.lib)
    return eng, _Params(sd).to(bk.dev), {k: v.double().to(bk.dev) for k, v in sd.items()}


# ------------------------------------------------------------------------------------------------ A: the beam schedule
def _row_counts(steps, hyps):
    """rows of every step: 1 at step 0, the full beam for most steps, a drop to a handful (hypotheses ended) every 11
    steps and to a single row every 23, each followed by a step that forks back to the full beam"""
    few = max(2, hyps // 8)
    return [1 if s == 0 or s % 23 == 9 else min(hyps, few) if s % 11 == 5 else hyps for s in range(steps)]


def _plan(counts, odim, seed):
    """per step (tokens, parents): each row's parent drawn among the previous step's rows (so some rows have several
    children and some none), tokens over the whole vocabulary with 0 and odim - 1 forced in"""
    g = torch.Generator().manual_seed(seed)
    plan = [([odim - 1], None)]
    for s in range(1, len(counts)):
        n = counts[s]
        parents = torch.randint(0, counts[s - 1], (n,), generator=g).tolist()
        toks = torch.randint(0, odim, (n,), generator=g).tolist()
        if n >= 2:
            toks[0], toks[-1] = 0, odim - 1
        plan.append((toks, parents))
    return plan


def _permuted(plan, seed):
    """the same hypotheses with the rows of every step in another order -> (plan, per step the old row of each new row)"""
    g = torch.Generator().manual_seed(seed)
    out, perms, inv_prev = [], [], None
    for toks, parents in plan:
        perm = torch.randperm(len(toks), generator=g).tolist()
        out.append(([toks[p] for p in perm], None if parents is None else [inv_prev[parents[p]] for p in perm]))
        inv_prev = [0] * len(perm)
        for j, p in enumerate(perm):
            inv_prev[p] = j
        perms.append(perm)
    return out, perms


def _walk(plan):
    """-> per step (tokens, parents, token prefix of every row, slot chain of every row: its ancestors' rows at positions
    0 .. step - 1, what the ancestor table holds)"""
    prefixes, chains = [[]], [[]]
    for toks, parents in plan:
        if parents is not None:
            prefixes, chains = [prefixes[p] for p in parents], [chains[p] + [p] for p in parents]
        prefixes = [pre + [t] for pre, t in zip(prefixes, toks)]
        yield toks, parents, prefixes, chains


def _anc(bk, chains):
    return bk.i32(chains).T.contiguous() if chains[0] else None


def _drive(bk, eng, plan):
    for step, (toks, _, prefixes, chains) in enumerate(_walk(plan)):
        t, a = bk.i32(toks), _anc(bk, chains)
        yield step, t, a, prefixes, chains, eng.step(t, a, step)


def _memory(T, d, seed):
    return torch.randn(T, d, generator=torch.Generator().manual_seed(seed))


def _begin(bk, name, prec):
    spec = DEPTH[name]
    cfg = spec["cfg"]
    eng, params, sd64 = _engine(bk, cfg, 11)
    mem = _memory(spec["T"], cfg["d"], 12).to(bk.dev)
    eng.begin(params, mem, max_hyps=spec["hyps"], max_steps=spec["steps"], precision=prec)
    plan = _plan(_row_counts(spec["steps"], spec["hyps"]), cfg["odim"], 13)
    return spec, eng, params, sd64, mem, plan


def depth(bk, name, prec):
    """every position 0 .. max_steps - 1 of a session is stepped; at the checked steps all rows against float64"""
    spec, eng, _, sd64, mem, plan = _begin(bk, name, prec)
    bound = TOL_DEPTH["replay" if bk.dry else prec]
    errs = {}
    for step, _, _, prefixes, _, logp in _drive(bk, eng, plan):
        if step not in spec["checked"]:
            continue
        want = DO.decoder_logp(sd64, torch.tensor(prefixes, device=bk.dev), mem.double(), spec["cfg"]["H"])
        assert logp.shape == want.shape and bool(torch.isfinite(logp).all()), step
        assert torch.allclose(logp.exp().sum(-1), torch.ones(len(prefixes), device=bk.dev), atol=1e-4), step
        errs[step] = float((logp.double() - want).abs().max())
        record("decoder_depth_logp", (name, prec, step, len(prefixes)), errs[step], bound)
    assert sorted(errs) == sorted(spec["checked"])
    assert max(errs.values()) < bound, errs


def _self_slots(eng, T, steps, hyps):
    """(L, max_steps, max_hyps, 3d) fp32 view of the session's self-attention slots (layout_dec_session in
    csrc/decoder_body.cuh: 256-byte aligned regions, the source K|V of every layer first)"""
    c = eng.cfg
    off = (c.num_blocks * T * 2 * c.d_model * 4 + 255) // 256 * 256
    nbytes = c.num_blocks * steps * hyps * 3 * c.d_model * 4
    return eng._session[off:off + nbytes].view(torch.float32).view(c.num_blocks, steps, hyps, 3 * c.d_model)


def reads_only_its_chains(bk, name, prec):
    """at each checked step, every self-attention slot that no live row's chain reaches is overwritten with NaN and the
    step repeated: finite and the same bits.  Last, a NaN in a slot a chain does reach must show in that row (the view
    addresses what the step reads)."""
    spec, eng, _, _, _, plan = _begin(bk, name, prec)
    slots = _self_slots(eng, spec["T"], spec["steps"], spec["hyps"])
    poisoned = 0
    for step, toks, anc, _, chains, logp in _drive(bk, eng, plan):
        if step == 0 or step not in spec["checked"]:
            continue
        live = torch.zeros(spec["steps"], spec["hyps"], dtype=torch.bool)
        for chain in chains:
            live[torch.arange(step), torch.tensor(chain)] = True
        slots[:, ~live.to(bk.dev)] = float("nan")
        poisoned += int((~live).sum())
        again = eng.step(toks, anc, step)
        bk.sync()
        assert bool(torch.isfinite(again).all()), step
        assert torch.equal(again, logp), step
    assert poisoned > 0
    slots[:, 0, chains[0][0]] = float("nan")
    assert bool(torch.isnan(eng.step(toks, anc, step)[0]).all())


def row_order(bk, name, prec):
    """the same prefixes with the rows of every step permuted (tokens and ancestor columns alike) give the permuted rows,
    bit for bit (with f16 operands too: a GEMM row does not depend on which of the M rows it is)"""
    spec, eng, params, _, mem, plan = _begin(bk, name, prec)
    base = {s: logp.clone() for s, _, _, _, _, logp in _drive(bk, eng, plan) if s in spec["checked"]}
    eng.begin(params, mem, max_hyps=spec["hyps"], max_steps=spec["steps"], precision=prec)
    shuffled, perms = _permuted(plan, 17)
    worst = 0.0
    for step, _, _, _, _, logp in _drive(bk, eng, shuffled):
        if step in spec["checked"]:
            worst = max(worst, float((logp - base[step][perms[step]]).abs().max()))
    record("decoder_row_order_max_difference", (name, prec), worst, 0.0)
    assert worst == 0.0, worst


def batched_depth(bk, prec):
    """U = 4 utterances decoded together deep into their prefixes, every utterance with its own beam schedule, rows of
    different utterances interleaved: at the checked steps every row has the bits of the same prefix stepped in a
    one-utterance session"""
    spec = BATCH_DEPTH["dry" if bk.dry else "gpu"]
    cfg, Ts, U = spec["cfg"], spec["Ts"], len(spec["Ts"])
    batch, params, _ = _engine(bk, cfg, 11)
    mems = [_memory(T, cfg["d"], 30 + u).to(bk.dev) for u, T in enumerate(Ts)]
    padded = torch.zeros(U, max(Ts), cfg["d"], device=bk.dev)
    for u, m in enumerate(mems):
        padded[u, :Ts[u]] = m
    batch.begin_batch(params, padded, list(Ts), max_hyps=U * spec["hyps"], max_steps=spec["steps"], precision=prec)
    alone, walks = [], []
    for u in range(U):
        e = _engine(bk, cfg, 11)[0]
        e.begin(params, mems[u], max_hyps=spec["hyps"], max_steps=spec["steps"], precision=prec)
        alone.append(e)
        counts = [1] + _row_counts(spec["steps"] + U, spec["hyps"])[1 + u:spec["steps"] + u]      # drops at other steps per utterance
        walks.append(_walk(_plan(counts, cfg["odim"], 40 + u)))
    g = torch.Generator().manual_seed(19)
    slot, chain = {}, {}             # (utterance, its row) -> batched row of the previous step / batched slot chain
    compared = 0
    for step in range(spec["steps"]):
        per = [next(w) for w in walks]
        rows = [(u, k) for u in range(U) for k in range(len(per[u][0]))]
        rows = [rows[j] for j in torch.randperm(len(rows), generator=g).tolist()]
        chain = {(u, k): chain[(u, per[u][1][k])] + [slot[(u, per[u][1][k])]] if step else [] for u, k in rows}
        slot = {rk: j for j, rk in enumerate(rows)}
        got = batch.step(bk.i32([per[u][0][k] for u, k in rows]), _anc(bk, [chain[rk] for rk in rows]), step,
                         row_utt=bk.i32([u for u, _ in rows]))
        for u in range(U):
            want = alone[u].step(bk.i32(per[u][0]), _anc(bk, per[u][3]), step)
            if step in spec["checked"]:
                bk.sync()
                for k in range(want.shape[0]):
                    assert torch.equal(got[slot[(u, k)]], want[k]), (step, u, k)
                    compared += 1
    assert compared >= U * len(spec["checked"])


# ------------------------------------------------------------------------------------------------ B: CTC prefix scorer
def _labels(T, O, steps, g):
    """about T/8 labels with an adjacent repeat every fourth label, then random labels up to steps + 1"""
    L = max(1, T // 8)
    lab = torch.randint(1, O - 1, (max(L, steps + 1),), generator=g).tolist()
    for k in range(1, L, 4):
        lab[k] = lab[k - 1]
    return lab, L


def _posterior(kind, T, O, lab, L, g):
    """(T, O) fp32 log-posteriors.  diffuse: log_softmax(randn * 3).  peaked: `lab[:L]` rendered as a CTC alignment --
    blank at 0.9-0.999 on most frames, each label on one or two frames at 0.5-0.99, the rest spread over the vocabulary"""
    if kind == "diffuse":
        return torch.log_softmax(torch.randn(T, O, generator=g) * 3, -1)
    main = torch.zeros(T, dtype=torch.long)
    for k in range(L):
        t = int((k + 0.5) * T / L)
        main[t] = lab[k]
        if T >= 8 * L and float(torch.rand(1, generator=g)) < 0.5:
            main[t + 1] = lab[k]
    u = torch.rand(T, generator=g, dtype=torch.float64)
    peak = torch.where(main == 0, 0.9 + 0.099 * u, 0.5 + 0.49 * u)
    p = torch.softmax(torch.randn(T, O, generator=g, dtype=torch.float64), -1)
    p.scatter_(1, main[:, None], 0.0)
    p = p / p.sum(-1, keepdim=True) * (1 - peak)[:, None]
    p.scatter_(1, main[:, None], peak[:, None])
    return p.log().float()


def _row_sequences(lab, L, n, steps, O, g):
    """row 0 follows the labels; the others substitute (odd rows) or drop (even rows) one label of it"""
    seqs = [lab[:steps]]
    for i in range(1, n):
        q = i % min(L, steps)
        if i % 2:
            sub = int(torch.randint(1, O - 1, (1,), generator=g))
            seqs.append(lab[:q] + [sub if sub != lab[q] else 1 + sub % (O - 2)] + lab[q + 1:steps])
        else:
            seqs.append(lab[:q] + lab[q + 1:steps + 1])
    return seqs


def _candidates(seqs, s, S, O, g):
    """per row S distinct tokens: its next label, a repeat of its last label, <eos>, blank, random ones; rotated so that
    the next label's column differs from row to row"""
    out = []
    for i, seq in enumerate(seqs):
        c = list(dict.fromkeys([seq[s]] + ([seq[s - 1]] if s else []) + [O - 1, 0]))
        c += [t for t in torch.randperm(O, generator=g).tolist() if t not in c][:S - len(c)]
        k = (i + s) % S
        out.append(c[-k:] + c[:-k] if k else c)
    return out


def _ctc_case(kind, T, O, n, S, seed):
    steps = min(T + 2, 40)
    g = torch.Generator().manual_seed(seed)
    lab, L = _labels(T, O, steps, g)
    logp = _posterior(kind, T, O, lab, L, g)
    seqs = _row_sequences(lab, L, n, steps, O, g)
    return logp, seqs, [_candidates(seqs, s, S, O, g) for s in range(steps)]


def _reference_ctc(logp, T, eos):
    if not build_ref.available():
        return None
    build_ref.import_reference_search()
    from espnet.nets.ctc_prefix_score import CTCPrefixScoreTH
    return CTCPrefixScoreTH(logp.unsqueeze(0).clone(), torch.tensor([T]), 0, eos)


def _live_err(got, want, rows, relative):
    """logzero pattern of `got` = that of the float64 `want` on `rows`; -> worst error over the live entries"""
    got, want = got.double()[rows], want[rows]
    live = want > DO.LOGZERO / 2
    assert bool(((got > DO.LOGZERO / 2) == live).all())
    if not bool(live.any()):
        return 0.0
    d = (got - want).abs()
    return float((d / want.abs().clamp(min=1.0) if relative else d)[live].max())


def _by_length(table, T):
    return table[min(k for k in table if k >= T)]


def ctc_whole(bk, kind, T):
    """score -> select along the label sequence for min(T + 2, 40) steps (past out_len == T for the short utterances)"""
    from auto_avsr_b200.decoder import CtcPrefixEngine
    sz = CTC_SIZES["dry" if bk.dry else "gpu"]
    O, n, S = sz["O"], sz["n"], sz["S"]
    eos = O - 1
    logp, seqs, cands = _ctc_case(kind, T, O, n, S, 100 + T)
    logp = logp.to(bk.dev)
    lp64 = logp.double()
    eng = CtcPrefixEngine(logp, 0, eos, _lib=bk.lib)
    r_prev, s_prev = eng.initial(n)
    r64, s64 = DO.ctc_initial_state(lp64)
    r64, s64 = r64.expand(-1, -1, n).contiguous(), s64.expand(n).contiguous()
    e_init = float(((r_prev[:, 1].double() - r64[:, 1]).abs() / r64[:, 1].abs().clamp(min=1.0)).max())
    assert bool((r_prev[:, 0] == DO.LOGZERO).all())
    ref, ref_state = _reference_ctc(logp, T, eos), None
    rows_all = torch.arange(n, device=bk.dev)
    e_local = e_psi = e_r = e_ref = e_r_ref = 0.0
    tol_local = _by_length(TOL_CTC_LOCAL_REPLAY if bk.dry else TOL_CTC_LOCAL, T)
    tol_rel = _by_length(TOL_CTC_REL, T)
    for s, cand_l in enumerate(cands):
        last = [seq[s - 1] if s else eos for seq in seqs]
        keep = [seq[s] for seq in seqs]
        cand = bk.i32(cand_l)
        local, r, log_psi = eng.score(s, bk.i32(last), r_prev, s_prev, cand)
        for t in (local, r, log_psi):
            assert not bool(torch.isnan(t).any()), (kind, T, s)
        pos = (cand == bk.i32(keep)[:, None]).int().argmax(1)
        if s <= T:          # a prefix of more than T labels is outside what CTCPrefixScoreTH defines
            want, r_new, psi = DO.ctc_prefix_scores(lp64, s, last, r64, s64, cand.long(), 0, eos)
            ok = s64 > DO.LOGZERO / 2                 # rows whose own prefix is possible
            e_local = max(e_local, _live_err(local.gather(1, cand.long()), want.gather(1, cand.long()), ok, False))
            e_psi = max(e_psi, _live_err(log_psi.gather(1, cand.long()), psi.gather(1, cand.long()), ok, True))
            e_r = max(e_r, _live_err(r.permute(2, 0, 1, 3), r_new.permute(2, 0, 1, 3), ok, True))
            if ref is not None:
                ys = [[eos] + seq[:s] for seq in seqs]
                loc_ref, st = ref(ys, ref_state, cand.long())
                e_ref = max(e_ref, _live_err(loc_ref.gather(1, cand.long()), want.gather(1, cand.long()), ok, False))
                e_r_ref = max(e_r_ref, _live_err(st[0].permute(2, 0, 1, 3), r_new.permute(2, 0, 1, 3), ok, True))
                ref_state = (st[0][:, :, rows_all, pos], st[1][rows_all, torch.tensor(keep, device=bk.dev)][:, None], st[2], st[3])
            r64, s64 = r_new[:, :, rows_all, pos], psi[rows_all, torch.tensor(keep, device=bk.dev)]
        r_prev, s_prev = eng.select(r, log_psi, cand, bk.i32(list(range(n))), bk.i32(keep))
        assert torch.equal(r_prev, r[:, :, rows_all, pos]), s
        assert torch.equal(s_prev, log_psi[rows_all, torch.tensor(keep, device=bk.dev)]), s
    record("ctc_whole_local_abs", dict(kind=kind, T=T, reference_fp32=e_ref), e_local, tol_local)
    record("ctc_whole_log_psi_rel", (kind, T), e_psi, tol_rel)
    record("ctc_whole_r_rel", dict(kind=kind, T=T, reference_fp32=e_r_ref), e_r, tol_rel)
    record("ctc_whole_initial_state_rel", (kind, T), e_init, tol_rel)
    assert e_local <= max(tol_local, 2 * e_ref), (e_local, e_ref)
    assert e_r <= max(tol_rel, 2 * e_r_ref), (e_r, e_r_ref)
    assert max(e_psi, e_init) < tol_rel, (e_psi, e_init)


def ctc_batch_whole(bk):
    """U utterances (diffuse and peaked alternating) scored together, n rows each, interleaved: every row has the
    one-utterance scorer's bits; state frames past the utterance's length are logzero"""
    from auto_avsr_b200.decoder import CtcPrefixEngine
    sz = CTC_BATCH["dry" if bk.dry else "gpu"]
    O, n, S, Ts, steps = sz["O"], sz["n"], sz["S"], sz["Ts"], sz["steps"]
    U, eos = len(Ts), O - 1
    cases = []
    for u, T in enumerate(Ts):
        g = torch.Generator().manual_seed(200 + T)
        lab, L = _labels(T, O, steps, g)
        logp = _posterior(("diffuse", "peaked")[u % 2], T, O, lab, L, g)
        seqs = _row_sequences(lab, L, n, steps, O, g)
        cases.append((logp.to(bk.dev), seqs, [_candidates(seqs, s, S, O, g) for s in range(steps)]))
    padded = torch.zeros(U, max(Ts), O, device=bk.dev)
    for u, c in enumerate(cases):
        padded[u, :Ts[u]] = c[0]
    beng = CtcPrefixEngine(padded, 0, eos, _lib=bk.lib, lengths=list(Ts))
    ones = [CtcPrefixEngine(c[0], 0, eos, _lib=bk.lib) for c in cases]
    order = torch.randperm(U * n, generator=torch.Generator().manual_seed(23)).tolist()      # batched row -> (u, k)
    ru = bk.i32([j // n for j in order])
    mine = [torch.tensor([b for b, j in enumerate(order) if j // n == u], device=bk.dev) for u in range(U)]
    r_prev, s_prev = beng.initial(ru)
    singles = [e.initial(n) for e in ones]
    every = bk.i32(list(range(U * n)))
    for s in range(steps):
        pick = lambda f: bk.i32([f(cases[j // n], j % n) for j in order])      # noqa: E731
        last = pick(lambda c, k: c[1][k][s - 1] if s else eos)
        keep = pick(lambda c, k: c[1][k][s])
        cand = pick(lambda c, k: c[2][s][k])
        local, r, log_psi = beng.score(s, last, r_prev, s_prev, cand, row_utt=ru)
        for u, m in enumerate(mine):
            l1, r1, p1 = ones[u].score(s, last[m], singles[u][0], singles[u][1], cand[m])
            bk.sync()
            assert torch.equal(local[m], l1) and torch.equal(log_psi[m], p1), (s, u)
            assert torch.equal(r[:Ts[u], :, m], r1) and bool((r[Ts[u]:, :, m] == DO.LOGZERO).all()), (s, u)
            singles[u] = ones[u].select(r1, p1, cand[m], bk.i32(list(range(n))), keep[m])
        r_prev, s_prev = beng.select(r, log_psi, cand, every, keep)
        for u, m in enumerate(mine):
            assert torch.equal(r_prev[:Ts[u], :, m], singles[u][0]) and torch.equal(s_prev[m], singles[u][1]), (s, u)


# ------------------------------------------------------------------------------------------------ C: the search
def _scaled(got, want):
    """|got - want|, relative above magnitude 100 (scores of a 100-step search run to several hundred)"""
    return abs(got - want) / max(1.0, abs(want) / 100)


def _nbest_error(got, want, tol):
    """same count, same best sequence, the listed sequences in the reference's order -> worst score error.  Two
    neighbours may come out swapped only where their float64 scores are closer than `tol`."""
    assert len(got) == len(want), (len(got), len(want))
    assert got[0]["yseq"] == want[0]["yseq"]
    worst, i = 0.0, 0
    while i < len(want):
        if got[i]["yseq"] == want[i]["yseq"]:
            worst = max(worst, _scaled(got[i]["score"], want[i]["score"]))
            i += 1
            continue
        assert i + 1 < len(want) and got[i]["yseq"] == want[i + 1]["yseq"] and got[i + 1]["yseq"] == want[i]["yseq"], i
        print("SWAPPED", i, i + 1, want[i]["score"], want[i + 1]["score"])
        assert _scaled(want[i]["score"], want[i + 1]["score"]) < tol, (i, want[i]["score"], want[i + 1]["score"])
        worst = max(worst, _scaled(got[i]["score"], want[i + 1]["score"]), _scaled(got[i + 1]["score"], want[i]["score"]))
        i += 2
    return worst


def _as_lists(nbest):
    return [dict(yseq=[int(t) for t in h["yseq"]], score=float(h["score"])) for h in (x.asdict() for x in nbest)]


def search(bk, T):
    """DeviceBeamSearch.forward, beam 40, full-size synthetic decoder and CTC head, over a T-frame memory (T = 100 is the
    shape bench.py's decode_beam_search times) against the reference's unmodified BatchBeamSearch over the reference's
    own decoder and CTCPrefixScorer (oracle/_ref) in float64 on the same device"""
    from auto_avsr_b200 import CTC, TransformerDecoder
    from auto_avsr_b200.beam_search import DeviceBeamSearch
    from auto_avsr_b200.synthetic import decoder_state_dict, encoder_input, head_state_dict
    ref = build_ref.import_reference_search()
    cfg, beam = (TINY, 5) if bk.dry else (FULL6, 40)
    odim, eos = cfg["odim"], cfg["odim"] - 1
    sd = decoder_state_dict(4, odim, cfg["d"], cfg["H"], cfg["F"], cfg["L"])
    hsd = head_state_dict(4, 64, cfg["d"], odim)
    head = {"ctc_lo.weight": hsd["ctc.ctc_lo.weight"], "ctc_lo.bias": hsd["ctc.ctc_lo.bias"]}
    mem = encoder_input([T], cfg["d"], 50 + T)[0].to(bk.dev)

    rdec = ref["TransformerDecoder"](odim=odim, attention_dim=cfg["d"], attention_heads=cfg["H"],
                                     linear_units=cfg["F"], num_blocks=cfg["L"])
    rdec.load_state_dict(sd, strict=True)
    rctc = ref["CTC"](odim, cfg["d"], 0.1, reduce=True)
    rctc.load_state_dict(head, strict=True)
    rdec, rctc = rdec.double().to(bk.dev).eval(), rctc.double().to(bk.dev).eval()
    tokens = [str(i) for i in range(odim)]
    scorers = dict(decoder=rdec, ctc=ref["CTCPrefixScorer"](rctc, eos), lm=None, length_bonus=ref["LengthBonus"](odim))
    rbs = ref["BatchBeamSearch"](beam_size=beam, vocab_size=odim, weights=dict(decoder=0.9, ctc=0.1, lm=0.0, length_bonus=0),
                                 scorers=scorers, sos=eos, eos=eos, token_list=tokens, pre_beam_score_key="decoder")
    with torch.no_grad():
        want = _as_lists(rbs(mem.double()))

    def library(prec):
        dec = TransformerDecoder(odim, cfg["d"], cfg["H"], cfg["F"], cfg["L"])
        dec.load_state_dict(sd, strict=True)
        dec = dec.to(bk.dev).eval()
        dec.precision, dec._lib = prec, bk.lib
        if bk.dry:
            from test_decoder_dropin_cpu import CpuCTC
            ctc = CpuCTC(hsd)
        else:
            ctc = CTC(odim, cfg["d"], 0.1)
            ctc.load_state_dict(head)
            ctc = ctc.to(bk.dev).eval()
            ctc.precision = prec
        return _as_lists(DeviceBeamSearch(dec, ctc, beam_size=beam, vocab_size=odim)(mem))

    got = library("fp32")
    tol = 2.5e-5 if bk.dry else TOL_NBEST_FP32
    err = _nbest_error(got, want, tol)
    record("search_fp32_vs_reference_fp64", dict(T=T, ended=len(want), best_len=len(want[0]["yseq"])), err, tol)
    assert err < tol, err
    if bk.dry:
        return
    got16 = library("f16")
    assert got16 and got16[0]["yseq"][-1] == eos
    if got16[0]["yseq"] == want[0]["yseq"]:
        gap = _scaled(got16[0]["score"], want[0]["score"])
        record("search_f16_best_score", dict(T=T), gap, TOL_BEST_F16)
        assert gap < TOL_BEST_F16, gap


if __name__ == "__main__":
    bk = Backend()
    assert bk.dry or torch.cuda.is_available(), "needs a GPU (or AVSR_CASES_DRYRUN=1)"
    args = [int(a) if a.isdigit() else a for a in sys.argv[2:]]
    globals()[sys.argv[1]](bk, *args)
    bk.sync()
    print("CASE-OK")
