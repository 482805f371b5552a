"""GPU checks of decoding several utterances in lock-step: avsr_decoder_batch_* (with the grouped source-attention kernel)
and avsr_ctc_prefix_batch_* through DecoderEngine.begin_batch / CtcPrefixEngine, and DeviceBeamSearch.forward_batch.
The yardstick is the one-utterance path on the same GPU: a batched row must have the bits of the same hypothesis
scored alone, and forward_batch must return forward's n-best per utterance."""
import os

import pytest
import torch

import decoder_gpu_cases as cases
from helpers import record
from oracle import decoder_oracle as DO
from test_decoder_batch_emu_cpu import ctc_batch_fixture_error, load_decoder_batch_case, nbest_fixture_error

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def built():
    assert torch.cuda.is_available(), "needs a GPU"
    import __graft_entry__ as g
    g.build()


def _full_search(prec, beam=40):
    from auto_avsr_b200 import CTC, TransformerDecoder
    from auto_avsr_b200.beam_search import DeviceBeamSearch
    from auto_avsr_b200.synthetic import decoder_state_dict, head_state_dict
    dec = TransformerDecoder(odim=5049, attention_dim=768, attention_heads=12, linear_units=3072, num_blocks=6)
    dec.load_state_dict(decoder_state_dict(4), strict=True)
    hsd = head_state_dict(4)
    ctc = CTC(5049, 768, 0.1)
    ctc.load_state_dict({"ctc_lo.weight": hsd["ctc.ctc_lo.weight"], "ctc_lo.bias": hsd["ctc.ctc_lo.bias"]})
    dec, ctc = dec.to(dev).eval(), ctc.to(dev).eval()
    dec.precision = ctc.precision = prec
    return DeviceBeamSearch(dec, ctc, beam_size=beam)


def _padded(mems):
    xs = torch.zeros(len(mems), max(m.shape[0] for m in mems), mems[0].shape[1], device=dev)
    for u, m in enumerate(mems):
        xs[u, :m.shape[0]] = m
    return xs


def _same_nbest(batched, alone):
    assert len(batched) == len(alone)
    for u, (b, a) in enumerate(zip(batched, alone)):
        assert len(b) == len(a) and len(a) >= 1, u
        assert [h.yseq.tolist() for h in b] == [h.yseq.tolist() for h in a], u
        assert [(h.score, h.scores) for h in b] == [(h.score, h.scores) for h in a], u


@pytest.mark.parametrize("prec", ["fp32", "tf32", "f16"])
def test_forward_batch_equals_forward_per_utterance(prec):
    """full-size synthetic weights, U = 6 utterances of 1 / 3 / 40 / 97 / 150 / 400 frames: same token sequences and
    bitwise-equal scores as forward on each utterance"""
    g = torch.Generator().manual_seed(31)
    mems = [torch.randn(T, 768, generator=g).to(dev) for T in (1, 3, 40, 97, 150, 400)]
    bs = _full_search(prec)
    got = bs.forward_batch(_padded(mems), [m.shape[0] for m in mems])
    _same_nbest(got, [bs.forward(m) for m in mems])


@pytest.mark.parametrize("name", ["decoder_batch_tiny", "decoder_batch_full"])
def test_forward_batch_matches_reference_fixture(name):
    """the reference BatchBeamSearch on each utterance of the fixture (tiny: 1 / 9 / 23 / 40 frames, full: 5 / 17 / 30):
    in fp32 every utterance's n-best has the reference's count and listed token sequences, scores within
    TOL_NBEST_FP32 (relative above 100).  In f16 every utterance's n-best is forward's on that utterance, and where the
    f16 search ends on the reference's best token sequence its score is within TOL_BEST_F16 of the fp64 one (over the
    40-frame tiny utterance the f16 operands steer forward itself to another hypothesis)"""
    from auto_avsr_b200.beam_search import DeviceBeamSearch
    c = load_decoder_batch_case(name)
    cfg, z = c["cfg"], c["z"]
    xs = c["memory"].to(dev)
    for prec in ("fp32", "f16"):
        bs = DeviceBeamSearch(cases._decoder(c, prec), cases._ctc(c, prec), beam_size=cfg["beam"], vocab_size=cfg["odim"])
        got = bs.forward_batch(xs, c["lengths"])
        for u in range(len(c["lengths"])):
            nbest = [h.asdict() for h in got[u]]
            if prec == "fp32":
                err = nbest_fixture_error(nbest, z, "f32", u)
                record("forward_batch_fp32", (name, u), err, cases.TOL_NBEST_FP32)
                assert err < cases.TOL_NBEST_FP32, (u, err)
            else:
                assert int(nbest[0]["yseq"][-1]) == cfg["odim"] - 1
                L = int(z[f"nbest_len_f64_{u}"][0])
                if nbest[0]["yseq"] == z[f"nbest_yseq_f64_{u}"][0, :L].tolist():
                    gap = abs(nbest[0]["score"] - float(z[f"nbest_score_f64_{u}"][0]))
                    record("forward_batch_f16_best_score", (name, u), gap, cases.TOL_BEST_F16)
                    assert gap < cases.TOL_BEST_F16, (u, gap)
        if prec == "f16":
            _same_nbest(got, [bs.forward(xs[u, :T]) for u, T in enumerate(c["lengths"])])


@pytest.mark.parametrize("name", ["decoder_batch_tiny", "decoder_batch_full"])
def test_batched_ctc_prefix_scorer_matches_reference_fixture(name):
    """the reference's CTCPrefixScoreTH with xlens: every row of every utterance within TOL_CTC"""
    err, eos_excess = ctc_batch_fixture_error(load_decoder_batch_case(name), dev)
    record("ctc_prefix_batch", name, err, cases.TOL_CTC)
    record("ctc_prefix_batch_eos_excess_over_2x_reference_fp32", name, eos_excess, cases.TOL_CTC)
    assert err < cases.TOL_CTC and eos_excess < cases.TOL_CTC, (err, eos_excess)


def test_batched_ctc_prefix_scorer_equals_one_utterance_scorer():
    """rows of three utterances interleaved: every row has the one-utterance scorer's bits; frames past its utterance's
    length are logzero"""
    from auto_avsr_b200.decoder import CtcPrefixEngine
    g = torch.Generator().manual_seed(8)
    O, S, n = 5049, 60, 4
    lps = [torch.log_softmax(torch.randn(T, O, generator=g) * 3, -1).to(dev) for T in (1, 30, 37)]
    lens = [lp.shape[0] for lp in lps]
    padded = torch.zeros(len(lps), max(lens), O, device=dev)
    for u, lp in enumerate(lps):
        padded[u, :lens[u]] = lp
    beng = CtcPrefixEngine(padded, 0, O - 1, lengths=lens)
    ones = [CtcPrefixEngine(lp, 0, O - 1) for lp in lps]
    ru = torch.arange(len(lps) * n, dtype=torch.int32) % len(lps)
    ru = ru[torch.randperm(ru.numel(), generator=g)].to(dev)
    mine = [(ru == u).nonzero().view(-1) for u in range(len(lps))]
    r_prev, s_prev = beng.initial(ru)
    singles = [e.initial(n) for e in ones]
    last = torch.full((ru.numel(),), O - 1, dtype=torch.int32, device=dev)
    for step in range(3):
        cand = torch.stack([torch.randperm(O - 2, generator=g)[:S] + 1 for _ in range(ru.numel())]).to(torch.int32).to(dev)
        local, r, log_psi = beng.score(step, last, r_prev, s_prev, cand, row_utt=ru)
        for u, m in enumerate(mine):
            l1, r1, p1 = ones[u].score(step, last[m], singles[u][0], singles[u][1], cand[m])
            torch.cuda.synchronize()
            assert torch.equal(local[m], l1) and torch.equal(log_psi[m], p1), (step, u)
            assert torch.equal(r[:lens[u], :, m], r1) and (r[lens[u]:, :, m] == DO.LOGZERO).all(), (step, u)
            singles[u] = ones[u].select(r1, p1, cand[m], torch.arange(n, dtype=torch.int32, device=dev), cand[m, 0].contiguous())
        r_prev, s_prev = beng.select(r, log_psi, cand, torch.arange(ru.numel(), dtype=torch.int32, device=dev),
                                     cand[:, 0].contiguous())
        last = cand[:, 0].contiguous()


def _work_views(eng, n_max, T_max, max_steps):
    """(q2, ctx) fp32 views of the step workspace (layout_dec_work in csrc/decoder_body.cuh: 256-byte aligned slots)"""
    cfg = eng.cfg
    al = lambda b: (b + 255) // 256 * 256      # noqa: E731
    D, H = cfg.d_model, cfg.n_heads
    a = al(n_max * D * 4)
    off_q2 = 2 * a
    off_ctx = 3 * a + al(n_max * H * max(T_max, max_steps) * 4)
    w = eng._work
    q2 = w[off_q2:off_q2 + n_max * D * 4].view(torch.float32).view(n_max, D)
    ctx = w[off_ctx:off_ctx + n_max * D * 4].view(torch.float32).view(n_max, D)
    return q2, ctx


@pytest.mark.parametrize("U,T_max,rows_max,layers", [(32, 1600, 64, 2), (7, 1600, 5, 1), (3, 64, 40, 1), (5, 65, 1, 1),
                                                     (3, 700, 150, 1)])
def test_grouped_source_attention(U, T_max, rows_max, layers):
    """batched steps with ragged lengths up to T_max and 1..rows_max rows per utterance, rows interleaved: every logp row
    equals the one-utterance step bit for bit, the last layer's attention context matches a float64 restatement, and a
    second call repeats the bits"""
    from auto_avsr_b200.decoder import DecoderEngine
    from auto_avsr_b200.synthetic import decoder_state_dict
    from test_decoder_batch_emu_cpu import _Params
    g = torch.Generator().manual_seed(U * 7 + T_max)
    odim, D, H = 97, 768, 12
    params = _Params(decoder_state_dict(6, odim, D, H, 3072, layers)).to(dev)
    lens = torch.randint(1, T_max + 1, (U,), generator=g).tolist()
    lens[0] = T_max
    if U > 2:
        lens[1] = 1
    rows = torch.randint(1, rows_max + 1, (U,), generator=g).tolist()
    rows[0] = rows_max
    mems = [torch.randn(T, D, generator=g).to(dev) for T in lens]
    ru = torch.cat([torch.full((r,), u, dtype=torch.int32) for u, r in enumerate(rows)])
    ru = ru[torch.randperm(ru.numel(), generator=g)].to(dev)
    n = ru.numel()
    toks = torch.randint(0, odim, (n,), generator=g, dtype=torch.int32).to(dev)
    toks2 = torch.randint(0, odim, (n,), generator=g, dtype=torch.int32).to(dev)
    anc = torch.randint(0, n, (1, n), generator=g, dtype=torch.int32).to(dev)
    for u in range(U):                      # each row's step-0 ancestor in its own utterance
        m = (ru == u).nonzero().view(-1)
        anc[0, m] = m[torch.randint(0, m.numel(), (m.numel(),), generator=g).to(dev)].to(torch.int32)
    eng = DecoderEngine(odim, D, H, 3072, layers)
    eng.begin_batch(params, _padded(mems), lens, max_hyps=n, max_steps=2, precision="fp32")
    eng.step(toks, None, 0, row_utt=ru)
    logp = eng.step(toks2, anc, 1, row_utt=ru)
    q2, ctx = (t[:n].clone() for t in _work_views(eng, n, T_max, 2))
    again = eng.step(toks2, anc, 1, row_utt=ru)
    torch.cuda.synchronize()
    assert torch.equal(logp, again)
    # float64 restatement of the last layer's source attention from its query and the session's K|V
    sum_T = sum(lens)
    kv = eng._session[:layers * sum_T * 2 * D * 4].view(torch.float32).view(layers, sum_T, 2 * D)[-1].double()
    offs = [sum(lens[:u]) for u in range(U)]
    worst = 0.0
    for u in range(U):
        m = (ru == u).nonzero().view(-1)
        k = kv[offs[u]:offs[u] + lens[u], :D].view(lens[u], H, 64)
        v = kv[offs[u]:offs[u] + lens[u], D:].view(lens[u], H, 64)
        q = q2[m].double().view(-1, H, 64)
        p = torch.softmax(torch.einsum("rhe,she->rhs", q, k) / 8.0, dim=-1)
        want = torch.einsum("rhs,she->rhe", p, v).reshape(-1, D)
        worst = max(worst, float((ctx[m].double() - want).abs().max() / max(1.0, float(want.abs().max()))))
    record("grouped_src_attention_ctx_vs_fp64", (U, T_max, rows_max), worst, 2e-5)
    assert worst < 2e-5
    # the same rows, utterance by utterance, in one-utterance sessions
    one = DecoderEngine(odim, D, H, 3072, layers)
    pos = torch.empty(n, dtype=torch.long)
    for u in range(U):
        m = (ru == u).nonzero().view(-1)
        pos[m.cpu()] = torch.arange(m.numel())
        one.begin(params, mems[u], max_hyps=m.numel(), max_steps=2, precision="fp32")
        one.step(toks[m], None, 0)
        a1 = pos.to(dev)[anc[0, m].long()].to(torch.int32).view(1, -1)
        want = one.step(toks2[m], a1, 1)
        torch.cuda.synchronize()
        assert torch.equal(logp[m], want), u
    # a step given other lengths than begin stored (here one frame fewer for utterance 0) lays the
    # session out differently: NaN rows, not some other utterance's K/V (last: the misplaced slots overwrite the session)
    lens_ok = eng.batch[0]
    stale = type(lens_ok)(*lens_ok)
    stale[0] -= 1
    eng.batch = (stale,) + eng.batch[1:]
    bad = eng.step(toks2, anc, 1, row_utt=ru)
    torch.cuda.synchronize()
    assert torch.isnan(bad).all()


def test_encoder_chain_ragged_batch():
    """the drop-in encoder's padded output for a ragged batch, lengths from its masks, straight into forward_batch:
    per utterance, the n-best of forward on that utterance's frames"""
    from auto_avsr_b200 import ConformerEncoder
    from auto_avsr_b200.synthetic import encoder_input, encoder_state_dict
    from oracle import conformer_oracle as O
    enc = ConformerEncoder(num_blocks=2)
    enc.load_state_dict(encoder_state_dict(3, num_blocks=2), strict=True)
    enc = enc.to(dev).eval()
    lengths = [40, 17, 29]
    x = encoder_input(lengths, 768, 9).to(dev)
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)
    with torch.no_grad():
        feat, out_mask = enc(x, mask)
    lens = out_mask.view(len(lengths), -1).sum(-1)
    bs = _full_search("f16", beam=10)
    got = bs.forward_batch(feat, lens)
    _same_nbest(got, [bs.forward(feat[u, :int(lens[u])]) for u in range(len(lengths))])


if __name__ == "__main__":
    os.sys.exit(pytest.main([__file__, "-q"]))
