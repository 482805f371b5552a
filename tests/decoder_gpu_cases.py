"""Bodies of the row 8f#3 GPU parity cases (tests/test_zzz_gpu_decoder.py calls them in-process; each can also run alone in
its own process / CUDA context:  python tests/decoder_gpu_cases.py <case> [args...]).

The bounds below are about 4x the errors observed on the GPU (max-abs on log-probabilities of O(5..10) magnitude)."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from helpers import err_stats, load_decoder_case, record  # noqa: E402
from oracle import decoder_oracle as DO  # noqa: E402
from oracle import head_oracle as HO  # noqa: E402

TOL_LOGP = {"fp32": 9e-6, "tf32": 3.2e-3, "f16": 3.2e-3}
TOL_CTC = 1.6e-5
TOL_NBEST_FP32 = 6e-5        # |score - reference fp32 score| over the listed n-best
TOL_BEST_F16 = 6e-3          # |best score (f16 operands) - reference fp64 best score|
# AVSR_CASES_DRYRUN=1: CPU dry run of THESE BODIES on the host replay (tests/emu), so that a typo here is caught by the CPU
# suite and not by the one GPU run; fp32 only, no claim about the device.
DRY = os.environ.get("AVSR_CASES_DRYRUN") == "1"
dev = torch.device("cpu" if DRY else "cuda:0")
LIB = None
if DRY:
    from emu import build as _emu_build
    LIB = _emu_build.load()


def _sync():
    if not DRY:
        torch.cuda.synchronize()


def _decoder(c, prec):
    from auto_avsr_b200 import TransformerDecoder
    cfg = c["cfg"]
    dec = TransformerDecoder(cfg["odim"], cfg["d_model"], cfg["n_heads"], cfg["linear_units"], cfg["num_blocks"])
    dec.load_state_dict(c["dec_sd"], strict=True)
    dec = dec.to(dev).eval()
    dec.precision = "fp32" if DRY else prec
    dec._lib = LIB
    return dec


def _ctc(c, prec):
    from auto_avsr_b200 import CTC
    cfg = c["cfg"]
    if DRY:
        from test_decoder_dropin_cpu import CpuCTC
        return CpuCTC(c["head_sd"])
    ctc = CTC(cfg["odim"], cfg["d_model"], 0.1)
    ctc.load_state_dict({"ctc_lo.weight": c["head_sd"]["ctc.ctc_lo.weight"], "ctc_lo.bias": c["head_sd"]["ctc.ctc_lo.bias"]})
    ctc = ctc.to(dev).eval()
    ctc.precision = prec
    return ctc


def batch_score(name, prec):
    """TransformerDecoder.batch_score driven the way the beam search drives it (states handed back), vs the reference's
    batch_score outputs."""
    c = load_decoder_case(name)
    z, cfg = c["z"], c["cfg"]
    dec = _decoder(c, prec)
    cols = torch.from_numpy(z["cols"])
    mem = c["memory"].to(dev)
    states = [None] * cfg["n_hyp"]
    worst = 0.0
    for step in range(cfg["steps"]):
        ys = c["prefixes"][step].to(dev)
        logp, states = dec.batch_score(ys, states, mem.unsqueeze(0).expand(cfg["n_hyp"], -1, -1))
        _sync()
        mx, _ = err_stats(logp.cpu()[:, cols], torch.from_numpy(z[f"dec_logp_f64_{step}"]))
        worst = max(worst, mx)
        assert torch.allclose(logp.exp().sum(-1).cpu(), torch.ones(cfg["n_hyp"]), atol=1e-4)
        if prec == "fp32":
            assert torch.equal(torch.topk(logp.cpu(), 3, dim=-1)[1], torch.from_numpy(z[f"dec_top_f64_{step}"])[:, :3])
    record("decoder_batch_score", (name, prec), worst, TOL_LOGP[prec])
    assert worst < TOL_LOGP[prec], (name, prec, worst)


def forked_beam(prec):
    c = load_decoder_case("decoder_tiny")
    cfg = c["cfg"]
    dec = _decoder(c, prec)
    eng = dec.engine()
    odim, sos = cfg["odim"], cfg["odim"] - 1
    mem = c["memory"]
    eng.begin(dec, mem.to(dev), max_hyps=5, max_steps=6, precision=prec)
    g = torch.Generator().manual_seed(5)
    prefixes, chains = [[sos]], [[]]
    eng.step(torch.tensor([sos], dtype=torch.int32, device=dev), None, 0)
    worst = 0.0
    for step in range(1, 5):
        n_prev = len(prefixes)
        n = min(5, n_prev + 2)
        parents = torch.randint(0, n_prev, (n,), generator=g).tolist()
        toks = torch.randint(1, odim - 1, (n,), generator=g).tolist()
        prefixes = [prefixes[p] + [t] for p, t in zip(parents, toks)]
        chains = [chains[p] + [p] for p in parents]
        anc = torch.tensor(chains, dtype=torch.int32).T.contiguous().to(dev)
        logp = eng.step(torch.tensor(toks, dtype=torch.int32, device=dev), anc, step)
        ref = DO.decoder_logp(c["dec_sd"], torch.tensor(prefixes), mem.double(), cfg["n_heads"])
        worst = max(worst, err_stats(logp.cpu(), ref)[0])
    record("decoder_forked_beam", prec, worst, TOL_LOGP[prec])
    assert worst < TOL_LOGP[prec], worst


def long_memory(prec):
    """T = 401 > 192: the source K|V projection runs in row chunks"""
    c = load_decoder_case("decoder_tiny")
    cfg = c["cfg"]
    dec = _decoder(c, prec)
    g = torch.Generator().manual_seed(21)
    mem = torch.randn(401, cfg["d_model"], generator=g)
    sos = cfg["odim"] - 1
    logp, _ = dec.batch_score(torch.tensor([[sos], [sos]], device=dev), [None, None], mem.to(dev).unsqueeze(0).expand(2, -1, -1))
    ref = DO.decoder_logp(c["dec_sd"], torch.tensor([[sos], [sos]]), mem.double(), cfg["n_heads"])
    err = err_stats(logp.cpu(), ref)[0]
    record("decoder_long_memory", prec, err, TOL_LOGP[prec])
    assert err < TOL_LOGP[prec], err


def ctc_prefix(name):
    from auto_avsr_b200.decoder import CtcPrefixEngine
    c = load_decoder_case(name)
    z, cfg = c["z"], c["cfg"]
    eos, n = cfg["odim"] - 1, cfg["n_hyp"]
    logp = HO.ctc_log_softmax(c["memory"].float(), c["head_sd"]).to(dev)
    eng = CtcPrefixEngine(logp, 0, eos, _lib=LIB)
    r_prev, s_prev = eng.initial(n)
    worst = 0.0
    for step in range(cfg["steps"]):
        ys = c["prefixes"][step]
        cand = torch.from_numpy(z[f"ctc_cand_{step}"]).to(torch.int32).to(dev)
        local, r, log_psi = eng.score(step, ys[:, -1].to(torch.int32).to(dev), r_prev, s_prev, cand)
        got = torch.gather(local, 1, cand.long()).cpu()
        want = torch.from_numpy(z[f"ctc_local_f64_{step}"])
        live = (want > DO.LOGZERO / 2) & (want < -DO.LOGZERO / 2)
        assert (((got <= DO.LOGZERO / 2) | (got >= -DO.LOGZERO / 2)) == ~live).all()
        worst = max(worst, err_stats(got[live], want[live])[0] / max(1.0, float(want[live].abs().max()) / 50))
        if f"ctc_keep_{step}" in z.files:
            keep = torch.from_numpy(z[f"ctc_keep_{step}"]).to(torch.int32).to(dev)
            r_prev, s_prev = eng.select(r, log_psi, cand, torch.arange(n, dtype=torch.int32, device=dev), keep)
            pos = (cand == keep[:, None]).int().argmax(1)
            assert torch.equal(r_prev, torch.stack([r[:, :, i, int(pos[i])] for i in range(n)], dim=2))
    record("ctc_prefix_scorer", name, worst, TOL_CTC)
    assert worst < TOL_CTC, worst


def _compare_nbest(nbest, z, tag):
    """best hypothesis identical to the reference's; -> max |score - reference score| over the listed n-best"""
    assert nbest, "no hypothesis ended"
    L = int(z[f"nbest_len_{tag}"][0])
    assert nbest[0]["yseq"] == z[f"nbest_yseq_{tag}"][0, :L].tolist()
    k = min(len(nbest), len(z[f"nbest_score_{tag}"]))
    got = torch.tensor([h["score"] for h in nbest[:k]])
    want = torch.from_numpy(z[f"nbest_score_{tag}"][:k]).float()
    return float((got - want).abs().max())


def device_beam_search(name):
    from auto_avsr_b200.beam_search import DeviceBeamSearch
    c = load_decoder_case(name)
    cfg = c["cfg"]
    dec, ctc = _decoder(c, "fp32"), _ctc(c, "fp32")
    bs = DeviceBeamSearch(dec, ctc, beam_size=cfg["beam"], vocab_size=cfg["odim"])
    nbest = [h.asdict() for h in bs(c["memory"].to(dev))]
    err = _compare_nbest(nbest, c["z"], "f32")
    record("device_beam_search_fp32", name, err, TOL_NBEST_FP32)
    assert err < TOL_NBEST_FP32 and len(nbest) == int(c["z"]["nbest_count_f32"])
    # the product precision: <eos>-closed best hypothesis whose score sits within the f16 operand noise of the reference's
    dec16, ctc16 = _decoder(c, "f16"), _ctc(c, "f16")
    nb16 = [h.asdict() for h in DeviceBeamSearch(dec16, ctc16, beam_size=cfg["beam"], vocab_size=cfg["odim"])(c["memory"].to(dev))]
    gap = abs(nb16[0]["score"] - float(c["z"]["nbest_score_f64"][0]))
    record("device_beam_search_f16_best_score", name, gap, TOL_BEST_F16)
    assert gap < TOL_BEST_F16 and int(nb16[0]["yseq"][-1]) == cfg["odim"] - 1


def reference_loop():
    """the UNMODIFIED reference BatchBeamSearch (oracle/_ref) over the drop-in scorers, on the GPU"""
    from oracle import build_ref
    ref = build_ref.import_reference_search()
    from auto_avsr_b200 import CTCPrefixScorer
    from auto_avsr_b200.espnet_dropin import scorer_interface
    assert scorer_interface.rebind()
    c = load_decoder_case("decoder_tiny")
    cfg = c["cfg"]
    dec = _decoder(c, "fp32")
    ctc = CTCPrefixScorer(_ctc(c, "fp32"), cfg["odim"] - 1)
    ctc._lib = LIB
    token_list = [str(i) for i in range(cfg["odim"])]
    scorers = dict(decoder=dec, ctc=ctc, lm=None, length_bonus=ref["LengthBonus"](len(token_list)))
    weights = dict(decoder=0.9, ctc=0.1, lm=0.0, length_bonus=0)
    bs = ref["BatchBeamSearch"](beam_size=cfg["beam"], vocab_size=len(token_list), weights=weights, scorers=scorers,
                                sos=cfg["odim"] - 1, eos=cfg["odim"] - 1, token_list=token_list, pre_beam_score_key="decoder")
    with torch.no_grad():
        nbest = [h.asdict() for h in bs(c["memory"].to(dev))]
    err = _compare_nbest(nbest, c["z"], "f32")
    record("reference_loop_on_dropins", "decoder_tiny", err, TOL_NBEST_FP32)
    assert err < TOL_NBEST_FP32 and len(nbest) == int(c["z"]["nbest_count_f32"]), err


def encoder_chain():
    """lightning.py:69-75 after the front-end, on the drop-ins end to end: encoder(x, None) -> beam search (decoder + CTC prefix
    scorer): every hypothesis is <eos>-closed, scores finite, n-best sorted."""
    from auto_avsr_b200 import CTC, ConformerEncoder, TransformerDecoder
    from auto_avsr_b200.beam_search import DeviceBeamSearch
    from auto_avsr_b200.synthetic import decoder_state_dict, encoder_input, encoder_state_dict, head_state_dict
    enc = ConformerEncoder(num_blocks=2)
    enc.load_state_dict(encoder_state_dict(3, num_blocks=2), strict=True)
    dec = TransformerDecoder(odim=5049, attention_dim=768, attention_heads=12, linear_units=3072, num_blocks=6)
    dec.load_state_dict(decoder_state_dict(4), strict=True)
    hsd = head_state_dict(4)
    ctc = CTC(5049, 768, 0.1)
    ctc.load_state_dict({"ctc_lo.weight": hsd["ctc.ctc_lo.weight"], "ctc_lo.bias": hsd["ctc.ctc_lo.bias"]})
    enc, dec, ctc = enc.to(dev).eval(), dec.to(dev).eval(), ctc.to(dev).eval()
    x = encoder_input([40], 768, 9).to(dev)
    with torch.no_grad():
        feat, _ = enc(x, None)
    nbest = DeviceBeamSearch(dec, ctc, beam_size=10)(feat.squeeze(0))
    assert nbest and all(int(h.yseq[0]) == 5048 and int(h.yseq[-1]) == 5048 for h in nbest)
    scores = [h.score for h in nbest]
    assert all(s == s and abs(s) < 1e6 for s in scores) and scores == sorted(scores, reverse=True)


if __name__ == "__main__":
    assert DRY or torch.cuda.is_available(), "run with gpurun"
    globals()[sys.argv[1]](*sys.argv[2:])
    _sync()
    print("CHILD-OK")
