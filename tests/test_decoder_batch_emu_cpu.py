"""CPU checks of the multi-utterance decoding path without a GPU: the batched schedule of csrc/decoder_body.cuh
(begin_batch_body / step_batch_body, the batched source-attention and CTC functors) compiled against the host backend
of tests/emu/decoder_batch_emu.cu, driven through the package's own host code.  The yardstick is the one-utterance
path replayed by the same library: a batched row must have the bits of the same hypothesis decoded alone, and
DeviceBeamSearch.forward_batch must return, per utterance, what forward returns.  The GPU side is
tests/test_zzz_gpu_decoder_batch.py."""
import ctypes as C
import os

import pytest
import torch

from helpers import err_stats, load_decoder_case
from oracle import decoder_oracle as DO

pytestmark = pytest.mark.skipif(not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="nvcc is needed to build the host replay")


@pytest.fixture(scope="module")
def emu():
    from emu import build
    return build.load("decoder_batch")


class _Params(torch.nn.Module):
    def __init__(self, sd):
        super().__init__()
        self._names = {}
        for k, v in sd.items():
            name = k.replace(".", "__")
            self.register_parameter(name, torch.nn.Parameter(v.clone(), requires_grad=False))
            self._names[name] = k

    def named_parameters(self, *a, **kw):
        for name, p in super().named_parameters(*a, **kw):
            yield self._names[name], p


def _engine(cfg, emu):
    from auto_avsr_b200.decoder import DecoderEngine
    return DecoderEngine(cfg["odim"], cfg["d_model"], cfg["n_heads"], cfg["linear_units"], cfg["num_blocks"], _lib=emu)


def _padded(mems):
    T_max = max(m.shape[0] for m in mems)
    xs = torch.zeros(len(mems), T_max, mems[0].shape[1])
    for u, m in enumerate(mems):
        xs[u, :m.shape[0]] = m
    return xs


def _random_mems(lengths, d, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(T, d, generator=g) for T in lengths]


def test_batched_steps_equal_one_utterance_steps_bit_for_bit(emu):
    """U = 4 utterances of 1 / 5 / 23 / 40 frames, 5 steps; every step forks and re-orders each utterance's beam and
    interleaves the rows of different utterances at random.  Each utterance also runs alone in a one-utterance session
    (its rows in their batch order); every batched logp row must equal its one-utterance row bit for bit."""
    c = load_decoder_case("decoder_tiny")
    cfg = c["cfg"]
    params = _Params(c["dec_sd"])
    lengths = [1, 5, 23, 40]
    mems = _random_mems(lengths, cfg["d_model"], 3)
    U, odim, sos = len(lengths), cfg["odim"], cfg["odim"] - 1
    slots = 4
    batch = _engine(cfg, emu)
    batch.begin_batch(params, _padded(mems), lengths, max_hyps=U * slots, max_steps=6, precision="fp32")
    alone = []
    for m in mems:
        e = _engine(cfg, emu)
        e.begin(params, m, max_hyps=slots, max_steps=6, precision="fp32")
        alone.append(e)
    g = torch.Generator().manual_seed(7)
    # a row: (utterance, token, batched slot chain, one-utterance slot chain)
    rows = [(u, sos, [], []) for u in range(U)]
    for step in range(5):
        order = torch.randperm(len(rows), generator=g).tolist()
        rows = [rows[j] for j in order]
        ru = torch.tensor([r[0] for r in rows], dtype=torch.int32)
        toks = torch.tensor([r[1] for r in rows], dtype=torch.int32)
        anc = None if step == 0 else torch.tensor([r[2] for r in rows], dtype=torch.int32).T.contiguous()
        got = batch.step(toks, anc, step, row_utt=ru)
        single_slot = {}
        for u in range(U):
            mine = [j for j, r in enumerate(rows) if r[0] == u]
            a = None if step == 0 else torch.tensor([rows[j][3] for j in mine], dtype=torch.int32).T.contiguous()
            want = alone[u].step(toks[mine], a, step)
            for k, j in enumerate(mine):
                assert torch.equal(got[j], want[k]), (step, u, k)
                single_slot[j] = k
        # next rows: per utterance 1..slots children of random parents, random tokens
        nxt = []
        for u in range(U):
            mine = [j for j, r in enumerate(rows) if r[0] == u]
            for _ in range(int(torch.randint(1, slots + 1, (1,), generator=g))):
                p = mine[int(torch.randint(0, len(mine), (1,), generator=g))]
                t = int(torch.randint(1, odim - 1, (1,), generator=g))
                nxt.append((u, t, rows[p][2] + [p], rows[p][3] + [single_slot[p]]))
        rows = nxt


def test_batched_steps_against_the_oracle(emu):
    """the batched session against a full fp64 recomputation of each prefix over its own utterance's frames"""
    c = load_decoder_case("decoder_tiny")
    cfg = c["cfg"]
    lengths = [3, 17]
    mems = _random_mems(lengths, cfg["d_model"], 5)
    eng = _engine(cfg, emu)
    eng.begin_batch(_Params(c["dec_sd"]), _padded(mems), lengths, max_hyps=4, max_steps=3, precision="fp32")
    sos = cfg["odim"] - 1
    ru = torch.tensor([1, 0, 1], dtype=torch.int32)
    eng.step(torch.tensor([sos] * 3, dtype=torch.int32), None, 0, row_utt=ru)
    logp = eng.step(torch.tensor([4, 9, 11], dtype=torch.int32), torch.tensor([[0, 1, 2]], dtype=torch.int32), 1,
                    row_utt=ru)
    for j, (u, t) in enumerate([(1, 4), (0, 9), (1, 11)]):
        ref = DO.decoder_logp(c["dec_sd"], torch.tensor([[sos, t]]), mems[u].double(), cfg["n_heads"])
        assert err_stats(logp[j:j + 1], ref)[0] < 2e-4, j


def test_batched_ctc_prefix_scores_equal_one_utterance_scores(emu):
    """CTC prefix scoring over U = 4 utterances of 1 / 5 / 23 / 40 frames (random candidates incl. blank, <eos> and the
    last label, rows interleaved): local scores, log_psi and forward variables equal the one-utterance scorer's bit for
    bit; state entries past an utterance's length are logzero; and against the fp64 oracle."""
    from auto_avsr_b200.decoder import CtcPrefixEngine
    g = torch.Generator().manual_seed(13)
    lengths, O, S = [1, 5, 23, 40], 12, 6
    U, T_max, eos = len(lengths), max(lengths), O - 1
    lps = [torch.log_softmax(torch.randn(T, O, generator=g, dtype=torch.float64) * 2, -1) for T in lengths]
    padded = torch.zeros(U, T_max, O)
    for u, lp in enumerate(lps):
        padded[u, :lengths[u]] = lp.float()
    beng = CtcPrefixEngine(padded, 0, eos, _lib=emu, lengths=lengths)
    engs = [CtcPrefixEngine(lp.float(), 0, eos, _lib=emu) for lp in lps]
    ru = torch.tensor([2, 0, 3, 1, 3, 2], dtype=torch.int32)
    n = ru.numel()
    r_prev, s_prev = beng.initial(ru)
    mine = [[j for j in range(n) if int(ru[j]) == u] for u in range(U)]
    singles = [e.initial(len(m)) for e, m in zip(engs, mine)]
    oracle = []
    for u in range(U):
        r64, s64 = DO.ctc_initial_state(lps[u])
        oracle.append((r64.expand(-1, -1, len(mine[u])).clone(), s64.expand(len(mine[u])).clone()))
    last = [eos] * n
    for out_len in range(3):
        cand = torch.stack([torch.randperm(O, generator=g)[:S] for _ in range(n)]).to(torch.int32)
        if out_len:
            cand[0, 0] = last[0]
        local, r, log_psi = beng.score(out_len, torch.tensor(last, dtype=torch.int32), r_prev, s_prev, cand, row_utt=ru)
        keep = []
        for j in range(n):
            ok = [t for t in cand[j].tolist() if t not in (0, eos)]
            keep.append(ok[0])
        for u in range(U):
            m, T = mine[u], lengths[u]
            l1, r1, p1 = engs[u].score(out_len, torch.tensor([last[j] for j in m], dtype=torch.int32), singles[u][0],
                                       singles[u][1], cand[m])
            assert torch.equal(local[m], l1) and torch.equal(log_psi[m], p1), (out_len, u)
            assert torch.equal(r[:T, :, m], r1), (out_len, u)
            assert (r[T:, :, m] == DO.LOGZERO).all()
            want, r_new, psi = DO.ctc_prefix_scores(lps[u], out_len, [last[j] for j in m], oracle[u][0], oracle[u][1],
                                                    cand[m].long(), 0, eos)
            if out_len < T:          # (a prefix longer than T frames has probability logzero: degenerate)
                live = want > DO.LOGZERO / 2
                got = local[m]
                assert ((got > DO.LOGZERO / 2) == live).all()
                assert err_stats(got[live], want[live])[0] < 1e-4, (out_len, u)
            pos = [cand[j].tolist().index(keep[j]) for j in m]
            oracle[u] = (torch.stack([r_new[:, :, k, pos[k]] for k in range(len(m))], dim=2),
                         psi[torch.arange(len(m)), torch.tensor([keep[j] for j in m])])
            singles[u] = engs[u].select(r1, p1, cand[m], torch.arange(len(m), dtype=torch.int32),
                                        torch.tensor([keep[j] for j in m], dtype=torch.int32))
        r_prev, s_prev = beng.select(r, log_psi, cand, torch.arange(n, dtype=torch.int32),
                                     torch.tensor(keep, dtype=torch.int32))
        last = keep
    assert (beng.r0[1:, :, 0] == DO.LOGZERO).all() and (beng.r0[:, 0, :] == DO.LOGZERO).all()


def _search(cfg, sd, hsd, emu, beam, ctc_weight=0.1):
    from auto_avsr_b200 import TransformerDecoder
    from auto_avsr_b200.beam_search import DeviceBeamSearch
    from test_decoder_dropin_cpu import CpuCTC
    dec = TransformerDecoder(cfg["odim"], cfg["d_model"], cfg["n_heads"], cfg["linear_units"], cfg["num_blocks"])
    dec.load_state_dict(sd, strict=True)
    dec.eval()
    dec.precision, dec._lib = "fp32", emu
    return DeviceBeamSearch(dec, CpuCTC(hsd) if ctc_weight else None, beam_size=beam, vocab_size=cfg["odim"],
                            ctc_weight=ctc_weight)


def _same_nbest(batched, alone, floor=None):
    """same n-best per utterance: token sequences, scores and score parts identical.  floor: compare only hypotheses
    scoring above it -- those carrying the CTC's logzero tie exactly in fp32 (-1e9 + O(10)), and the top-k may order
    exact ties differently in a (U, rows x vocab) call than in forward's (rows x vocab) call."""
    assert len(batched) == len(alone)
    for b, a in zip(batched, alone):
        if floor is not None:
            b, a = [h for h in b if h.score > floor], [h for h in a if h.score > floor]
        assert [h.yseq.tolist() for h in b] == [h.yseq.tolist() for h in a]
        assert [(h.score, h.scores) for h in b] == [(h.score, h.scores) for h in a]


def test_forward_batch_equals_forward_per_utterance_and_the_reference(emu):
    """decoder_tiny weights; the fixture's own utterance (23 frames) among others of 1, 5 and 40 frames: forward_batch
    returns per utterance forward's n-best (same token sequences, identical scores), and the fixture utterance's n-best
    is the reference BatchBeamSearch's."""
    from test_decoder_dropin_cpu import _check_nbest
    c = load_decoder_case("decoder_tiny")
    cfg = c["cfg"]
    mems = _random_mems([5, 1, 40], cfg["d_model"], 9)
    mems.insert(2, c["memory"])
    bs = _search(cfg, c["dec_sd"], c["head_sd"], emu, cfg["beam"])
    got = bs.forward_batch(_padded(mems), [m.shape[0] for m in mems])
    _same_nbest(got, [bs.forward(m) for m in mems])
    _check_nbest([h.asdict() for h in got[2]], c["z"], "f32", 2e-3)
    # maxlenratio > 0: per-utterance maxlen, rows closed with <eos> at their own maxlen - 1
    _same_nbest(bs.forward_batch(_padded(mems), [m.shape[0] for m in mems], maxlenratio=0.3),
                [bs.forward(m, maxlenratio=0.3) for m in mems])


@pytest.mark.parametrize("odim,beam,ctc_weight", [(6, 5, 0.1), (9, 1, 0.1), (23, 6, 0.0)])
def test_forward_batch_corner_shapes(emu, odim, beam, ctc_weight):
    """a vocabulary below the beam (fewer candidates than beam slots at step 0; the beam runs dry), beam 1, no CTC"""
    from auto_avsr_b200.synthetic import decoder_state_dict, head_state_dict
    cfg = dict(odim=odim, d_model=64, n_heads=1, linear_units=64, num_blocks=1)
    sd = decoder_state_dict(300 + odim, odim, 64, 1, 64, 1)
    hsd = head_state_dict(300 + odim, 64, 64, odim)
    lengths = [2, 1, 9, 14, 7]
    mems = _random_mems(lengths, 64, odim)
    bs = _search(cfg, sd, hsd, emu, beam, ctc_weight)
    _same_nbest(bs.forward_batch(_padded(mems), lengths), [bs.forward(m) for m in mems], floor=ctc_weight * DO.LOGZERO / 2)


def test_decode_sharded_batches_by_length(emu):
    from auto_avsr_b200.beam_search import decode_sharded
    c = load_decoder_case("decoder_tiny")
    cfg = c["cfg"]
    mems = _random_mems([7, 3, 12, 1, 9], cfg["d_model"], 17)
    bs = _search(cfg, c["dec_sd"], c["head_sd"], emu, cfg["beam"])
    assert decode_sharded(bs, mems, batch_size=2) == decode_sharded(bs, mems)


def test_batch_argument_errors(emu):
    """T_u = 0, T_u > T_max, U = 0, n > max_hyps, short buffers: error codes, no crash; and the Python layer's checks"""
    from auto_avsr_b200 import _cabi
    from auto_avsr_b200._cabi import DecoderConfig
    c = load_decoder_case("decoder_tiny")
    cfg = c["cfg"]
    dc = DecoderConfig(cfg["d_model"], cfg["n_heads"], cfg["linear_units"], cfg["num_blocks"], cfg["odim"])
    lens = lambda *v: (C.c_int32 * len(v))(*v)        # noqa: E731
    assert emu.avsr_decoder_batch_session_bytes(C.byref(dc), 2, lens(3, 0), 4, 8) == 0
    assert emu.avsr_decoder_batch_session_bytes(C.byref(dc), 0, lens(3), 4, 8) == 0
    eng = _engine(cfg, emu)
    params = _Params(c["dec_sd"])
    prep = eng.prepare(params, torch.device("cpu"), "fp32")
    need = emu.avsr_decoder_batch_session_bytes(C.byref(dc), 2, lens(3, 5), 4, 8)
    wneed = emu.avsr_decoder_batch_step_workspace_bytes(C.byref(dc), 5, 4, 8)
    sess, work = torch.empty(need, dtype=torch.uint8), torch.empty(wneed, dtype=torch.uint8)
    mem = torch.zeros(2, 5, cfg["d_model"])
    begin = lambda L, U, T_max, nbytes: emu.avsr_decoder_batch_begin(  # noqa: E731
        C.byref(dc), prep.data_ptr(), mem.data_ptr(), L, U, T_max, 4, 8, sess.data_ptr(), nbytes, _cabi.PREC_FP32, None)
    assert begin(lens(3, 0), 2, 5, need) == _cabi.E_INVALID
    assert begin(lens(3, 6), 2, 5, need) == _cabi.E_INVALID
    assert begin(lens(3), 0, 5, need) == _cabi.E_INVALID
    assert begin(lens(3, 5), 2, 5, need - 1) == _cabi.E_WORKSPACE
    assert begin(lens(3, 5), 2, 5, need) == _cabi.OK
    tok = torch.zeros(9, dtype=torch.int32)
    logp = torch.empty(9, cfg["odim"])
    step = lambda L, n, nbytes, wbytes: emu.avsr_decoder_batch_step(  # noqa: E731
        C.byref(dc), prep.data_ptr(), sess.data_ptr(), nbytes, L, 2, 5, 4, 8, tok.data_ptr(), None, tok.data_ptr(), 0, n,
        logp.data_ptr(), work.data_ptr(), wbytes, _cabi.PREC_FP32, None)
    assert step(lens(3, 5), 9, need, wneed) == _cabi.E_INVALID
    assert step(lens(3, 9), 2, need, wneed) == _cabi.E_INVALID
    assert step(lens(3, 5), 2, need - 1, wneed) == _cabi.E_WORKSPACE
    assert step(lens(3, 5), 2, need, wneed - 1) == _cabi.E_WORKSPACE
    assert step(lens(3, 5), 2, need, wneed) == _cabi.OK
    # Python layer
    with pytest.raises(ValueError, match="lengths|geometry"):
        eng.begin_batch(params, mem, [3, 0], max_hyps=8, precision="fp32")
    with pytest.raises(ValueError, match="lengths"):
        eng.begin_batch(params, mem, [3], max_hyps=8, precision="fp32")
    eng.begin_batch(params, mem, [3, 5], max_hyps=2, max_steps=4, precision="fp32")
    with pytest.raises(ValueError, match="row_utt"):
        eng.step(torch.zeros(2, dtype=torch.int32), None, 0)
    with pytest.raises(ValueError, match="beam slots"):
        eng.step(torch.zeros(3, dtype=torch.int32), None, 0, row_utt=torch.zeros(3, dtype=torch.int32))
    eng.begin(params, mem[0], max_hyps=2, precision="fp32")
    with pytest.raises(ValueError, match="begin_batch"):
        eng.step(torch.zeros(2, dtype=torch.int32), None, 0, row_utt=torch.zeros(2, dtype=torch.int32))


def test_batched_step_launch_count_does_not_depend_on_U(emu):
    c = load_decoder_case("decoder_tiny")
    cfg = c["cfg"]
    params = _Params(c["dec_sd"])
    sos = cfg["odim"] - 1
    counts = []
    for lengths in ([6], [6, 2, 9, 4], [1, 3, 5, 7, 9, 11, 13, 15]):
        eng = _engine(cfg, emu)
        eng.begin_batch(params, _padded(_random_mems(lengths, cfg["d_model"], 1)), lengths, max_hyps=8, precision="fp32")
        ru = torch.arange(8, dtype=torch.int32) % len(lengths)
        before = emu.avsr_launch_count()
        eng.step(torch.full((8,), sos, dtype=torch.int32), None, 0, row_utt=ru)
        counts.append(emu.avsr_launch_count() - before)
    assert counts[0] == counts[1] == counts[2], counts


# ---- the reference on several utterances at once (oracle/make_golden_decoder_batch.py) -----------------------------------
def load_decoder_batch_case(name):
    """decoder_batch_{tiny,full}.npz: config, lengths, regenerated decoder / CTC weights and the (U, T_max, d) memory"""
    import numpy as np
    from helpers import GOLDEN
    from auto_avsr_b200.synthetic import decoder_state_dict, encoder_input, head_state_dict
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = {k[4:]: int(z[k]) for k in z.files if k.startswith("cfg_")}
    lengths = [int(v) for v in z["lengths"]]
    dec_sd = decoder_state_dict(cfg["wseed"], cfg["odim"], cfg["d_model"], cfg["n_heads"], cfg["linear_units"],
                                cfg["num_blocks"])
    head_sd = head_state_dict(cfg["wseed"], 64, cfg["d_model"], cfg["odim"])
    memory = encoder_input(lengths, cfg["d_model"], cfg["xseed"])
    return dict(z=z, cfg=cfg, lengths=lengths, dec_sd=dec_sd, head_sd=head_sd, memory=memory)


def ctc_batch_fixture_error(c, dev, lib=None):
    """CtcPrefixEngine over the fixture's U utterances (padded (U, T_max, O) posteriors + lengths), driven with the
    reference's prefixes, candidates and kept tokens, over rows whose prefix is still possible -> (worst error of the local
    scores at the candidates against the reference's float64 ones, relative above magnitude 50; worst excess of the
    <eos> score's error over twice the reference's own float32 error there -- the <eos> score sums a whole utterance's
    frames, and fp32 rounding of that sum is what the reference's fp32 run shows as well)"""
    from auto_avsr_b200.decoder import CtcPrefixEngine
    z, cfg, lengths = c["z"], c["cfg"], c["lengths"]
    eos, n, U = cfg["odim"] - 1, cfg["n_hyp"], len(lengths)
    w, b = c["head_sd"]["ctc.ctc_lo.weight"].double(), c["head_sd"]["ctc.ctc_lo.bias"].double()
    logp = torch.log_softmax(c["memory"].double() @ w.T + b, -1).float().to(dev)
    eng = CtcPrefixEngine(logp, 0, eos, _lib=lib, lengths=lengths)
    ru = (torch.arange(U * n) // n).to(torch.int32).to(dev)               # the reference's rows: utterance-major
    r_prev, s_prev = eng.initial(ru)
    worst = eos_excess = 0.0
    for step in range(cfg["steps"]):
        pre = torch.from_numpy(z[f"ctc_prefix_{step}"])
        cand = torch.from_numpy(z[f"ctc_cand_{step}"]).to(torch.int32).to(dev)
        local, r, log_psi = eng.score(step, pre[:, -1].to(torch.int32).to(dev), r_prev, s_prev, cand, row_utt=ru)
        ok = (s_prev > DO.LOGZERO / 2).cpu()
        got = torch.gather(local, 1, cand.long()).cpu()[ok]
        want = torch.from_numpy(z[f"ctc_local_f64_{step}"])[ok]
        live = (want > DO.LOGZERO / 2) & (want < -DO.LOGZERO / 2)
        assert (((got <= DO.LOGZERO / 2) | (got >= -DO.LOGZERO / 2)) == ~live).all(), step
        scale = max(1.0, float(want[live].abs().max()) / 50) if live.any() else 1.0
        if live.any():
            worst = max(worst, err_stats(got[live], want[live])[0] / scale)
        want_eos = torch.from_numpy(z[f"ctc_eos_f64_{step}"])[ok]
        ref32 = (torch.from_numpy(z[f"ctc_eos_f32_{step}"])[ok].double() - want_eos).abs()
        eos_excess = max(eos_excess, float(((local[:, eos].cpu()[ok].double() - want_eos).abs() - 2 * ref32).max()))
        r_prev, s_prev = eng.select(r, log_psi, cand, torch.arange(U * n, dtype=torch.int32, device=dev), cand[:, 0].contiguous())
    return worst, eos_excess


def nbest_fixture_error(nbest, z, tag, u):
    """utterance u's n-best against the reference's: same count, same listed token sequences -> max score error, relative
    above magnitude 100 (a 30-step search sums to scores of ~200, where fp32 spacing is 1.5e-5)"""
    assert len(nbest) == int(z[f"nbest_count_{tag}_{u}"]), u
    worst = 0.0
    for i in range(len(z[f"nbest_len_{tag}_{u}"])):
        L = int(z[f"nbest_len_{tag}_{u}"][i])
        h = nbest[i]
        assert h["yseq"] == z[f"nbest_yseq_{tag}_{u}"][i, :L].tolist(), (u, i)
        for got, key in ((h["score"], "score"), (h["scores"]["decoder"], "dec"), (h["scores"]["ctc"], "ctc")):
            want = float(z[f"nbest_{key}_{tag}_{u}"][i])
            worst = max(worst, abs(got - want) / max(1.0, abs(want) / 100))
    return worst


def test_batched_ctc_prefix_scorer_matches_reference_fixture(emu):
    """the reference's CTCPrefixScoreTH with xlens over 1 / 9 / 23 / 40-frame utterances (padded frames carry only
    blank, <eos> reads frame xlens - 1)"""
    err, eos_excess = ctc_batch_fixture_error(load_decoder_batch_case("decoder_batch_tiny"), torch.device("cpu"), emu)
    assert err < 2e-3 and eos_excess < 2e-3, (err, eos_excess)


def test_forward_batch_matches_reference_nbest_of_every_utterance(emu):
    """forward_batch over the fixture's 4 utterances: each one's n-best is the reference BatchBeamSearch's on it alone"""
    c = load_decoder_batch_case("decoder_batch_tiny")
    bs = _search(c["cfg"], c["dec_sd"], c["head_sd"], emu, c["cfg"]["beam"])
    got = bs.forward_batch(c["memory"], c["lengths"])
    for u in range(len(c["lengths"])):
        assert nbest_fixture_error([h.asdict() for h in got[u]], c["z"], "f32", u) < 2e-3, u


def test_forward_batch_minlenratio_retry(emu):
    """maxlen 0 (maxlenratio -0.5) is the one way a search ends without hypotheses: forward retries with minlenratio
    lowered by 0.1 until it is below 0.1 and returns []; forward_batch does the same per utterance"""
    c = load_decoder_case("decoder_tiny")
    mems = _random_mems([4, 9], c["cfg"]["d_model"], 2)
    bs = _search(c["cfg"], c["dec_sd"], c["head_sd"], emu, c["cfg"]["beam"])
    s0 = bs.stats["utterances"]
    assert bs.forward_batch(_padded(mems), [4, 9], maxlenratio=-0.5, minlenratio=0.25) == [[], []]
    assert bs.stats["utterances"] - s0 == 3 * 2                       # minlenratio 0.25, 0.15, 0.05
    assert [bs.forward(m, maxlenratio=-0.5, minlenratio=0.25) for m in mems] == [[], []]
