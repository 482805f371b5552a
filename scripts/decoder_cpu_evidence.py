#!/usr/bin/env python3
"""Observed errors of the row 8f#3 schedule / functors on the CPU (host replay of csrc/decoder_body.cuh, tests/emu) against
the reference-generated fixtures: what the CPU suite asserts, printed."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from emu import build  # noqa: E402
from helpers import err_stats, load_decoder_case  # noqa: E402
from oracle import decoder_oracle as DO  # noqa: E402
from oracle import head_oracle as HO  # noqa: E402
from test_decoder_dropin_cpu import CpuCTC, _dropin_decoder  # noqa: E402
from test_decoder_emu_cpu import _engine  # noqa: E402

from auto_avsr_b200.beam_search import DeviceBeamSearch  # noqa: E402
from auto_avsr_b200.decoder import CtcPrefixEngine  # noqa: E402

emu = build.load()
print("host replay of auto_avsr_b200/csrc/decoder_body.cuh (same schedule + functors, naive fp32 GEMM / LN / log-softmax), fp32")
for name in ("decoder_tiny", "decoder_full"):
    c = load_decoder_case(name)
    z, cfg = c["z"], c["cfg"]
    print(f"\n[{name}] d={cfg['d_model']} heads={cfg['n_heads']} ff={cfg['linear_units']} layers={cfg['num_blocks']} "
          f"odim={cfg['odim']} T={cfg['T']} beam={cfg['beam']}")
    eng, params = _engine(c, emu)
    n = cfg["n_hyp"]
    eng.begin(params, c["memory"], max_hyps=n, precision="fp32")
    cols = torch.from_numpy(z["cols"])
    for step in range(cfg["steps"]):
        ys = c["prefixes"][step]
        anc = None if step == 0 else torch.arange(n, dtype=torch.int32).repeat(step, 1)
        logp = eng.step(ys[:, -1].to(torch.int32), anc, step)
        mx, rms = err_stats(logp[:, cols], torch.from_numpy(z[f"dec_logp_f64_{step}"]))
        top = torch.equal(torch.topk(logp, 3, dim=-1)[1], torch.from_numpy(z[f"dec_top_f64_{step}"])[:, :3])
        print(f"  decoder step {step}: max|logp - reference fp64 batch_score| = {mx:.2e} (rms {rms:.2e}); top-3 tokens identical: {top}")
    logp = HO.ctc_log_softmax(c["memory"].float(), c["head_sd"])
    ce = CtcPrefixEngine(logp, 0, cfg["odim"] - 1, _lib=emu)
    r_prev, s_prev = ce.initial(n)
    for step in range(cfg["steps"]):
        cand = torch.from_numpy(z[f"ctc_cand_{step}"]).to(torch.int32)
        local, r, log_psi = ce.score(step, c["prefixes"][step][:, -1].to(torch.int32), r_prev, s_prev, cand)
        got = torch.gather(local, 1, cand.long())
        want = torch.from_numpy(z[f"ctc_local_f64_{step}"])
        live = (want > DO.LOGZERO / 2) & (want < -DO.LOGZERO / 2)
        mx, _ = err_stats(got[live], want[live])
        print(f"  CTC prefix step {step}: max|local - reference fp64 CTCPrefixScoreTH| = {mx:.2e} over {int(live.sum())} live (hyp, candidate) "
              f"pairs, |score| up to {float(want[live].abs().max()):.1f}")
        if f"ctc_keep_{step}" in z.files:
            keep = torch.from_numpy(z[f"ctc_keep_{step}"]).to(torch.int32)
            r_prev, s_prev = ce.select(r, log_psi, cand, torch.arange(n, dtype=torch.int32), keep)
    if name == "decoder_tiny":
        dec = _dropin_decoder(c, emu)
        nb = [h.asdict() for h in DeviceBeamSearch(dec, CpuCTC(c["head_sd"]), beam_size=cfg["beam"], vocab_size=cfg["odim"])(c["memory"])]
        k = len(z["nbest_len_f32"])
        same = all(nb[i]["yseq"] == z["nbest_yseq_f32"][i, :int(z["nbest_len_f32"][i])].tolist() for i in range(k))
        gap = max(abs(nb[i]["score"] - float(z["nbest_score_f32"][i])) for i in range(k))
        print(f"  DeviceBeamSearch: {len(nb)} ended hypotheses (reference {int(z['nbest_count_f32'])}); the {k} listed n-best sequences identical "
              f"and in the same order: {same}; max |score - reference fp32 score| = {gap:.2e}; {dec.engine().stats['step']} decoder steps")
print("\nthe reference's own BatchBeamSearch (oracle/_ref copy) over the drop-in scorers reproduces the same n-best: "
      "tests/test_decoder_dropin_cpu.py::test_reference_batch_beam_search_drives_the_dropin_scorers")
