#!/usr/bin/env python3
"""Generate tests/golden/decoder_batch_{tiny,full}.npz by running the UNMODIFIED reference on several utterances of
different lengths at once.  TEST INFRASTRUCTURE ONLY; build container only:

    PYTHONPATH=/root/reference python oracle/make_golden_decoder_batch.py

Per case it stores what the reference computed, in float64 and float32:
  * ``CTCPrefixScoreTH(x (U, T_max, O), xlens)`` (ctc_prefix_score.py:21-54) for a few steps over U utterances with
    n_hyp hypotheses each (the class needs equal counts): frames past xlens[u] carry only blank and ``<eos>`` reads
    frame xlens[u] - 1.  Local scores at the candidates and at ``<eos>``, states selected as
    ``CTCPrefixScorer.select_state`` does (scorers/ctc.py:40-63);
  * per utterance, the n-best list of ``BatchBeamSearch`` built like ``get_beam_search_decoder`` (lightning.py:126-157)
    on that utterance's own frames.
Weights and the (U, T_max, d) memory regenerate from seeds (``auto_avsr_b200.synthetic``); candidates and prefixes are
stored; only outputs are stored otherwise.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from espnet.nets.batch_beam_search import BatchBeamSearch  # noqa: E402
from espnet.nets.ctc_prefix_score import CTCPrefixScoreTH  # noqa: E402
from espnet.nets.pytorch_backend.ctc import CTC  # noqa: E402
from espnet.nets.pytorch_backend.decoder.transformer_decoder import TransformerDecoder  # noqa: E402
from espnet.nets.scorers.ctc import CTCPrefixScorer  # noqa: E402
from espnet.nets.scorers.length_bonus import LengthBonus  # noqa: E402

from auto_avsr_b200.synthetic import decoder_state_dict, encoder_input, head_state_dict  # noqa: E402

CASES = [
    dict(name="decoder_batch_tiny", odim=37, d_model=128, n_heads=2, linear_units=256, num_blocks=2, beam=5,
         wseed=51, xseed=71, steps=4, n_hyp=3, lengths=[1, 9, 23, 40]),
    dict(name="decoder_batch_full", odim=5049, d_model=768, n_heads=12, linear_units=3072, num_blocks=6, beam=40,
         wseed=52, xseed=72, steps=3, n_hyp=4, lengths=[5, 17, 30]),
]
NBEST_KEPT = 10


def build(case, dtype):
    dec = TransformerDecoder(odim=case["odim"], attention_dim=case["d_model"], attention_heads=case["n_heads"],
                             linear_units=case["linear_units"], num_blocks=case["num_blocks"])
    dec.load_state_dict(decoder_state_dict(case["wseed"], case["odim"], case["d_model"], case["n_heads"],
                                           case["linear_units"], case["num_blocks"]), strict=True)
    hsd = head_state_dict(case["wseed"], 64, case["d_model"], case["odim"])
    ctc = CTC(case["odim"], case["d_model"], 0.1, reduce=True)
    ctc.load_state_dict({"ctc_lo.weight": hsd["ctc.ctc_lo.weight"], "ctc_lo.bias": hsd["ctc.ctc_lo.bias"]}, strict=True)
    return dec.to(dtype).eval(), ctc.to(dtype).eval()


def script(case):
    """prefixes (steps + 1 of them, (U * n_hyp, step + 1), utterance-major rows) and per step the candidates
    (U * n_hyp, int(1.5 beam)): seeded distinct tokens off blank / <eos>, the row's next prefix token first"""
    U, n, odim = len(case["lengths"]), case["n_hyp"], case["odim"]
    g = torch.Generator().manual_seed(case["xseed"] * 7 + 1)
    body = torch.randint(1, odim - 1, (U * n, case["steps"]), generator=g)
    sos = torch.full((U * n, 1), odim - 1, dtype=torch.long)
    prefixes = [torch.cat([sos, body[:, :s]], dim=1) for s in range(case["steps"] + 1)]
    S = min(int(1.5 * case["beam"]), odim - 2)
    cands = []
    for step in range(case["steps"]):
        rows = []
        for i in range(U * n):
            nxt = int(body[i, step])
            rest = [t + 1 for t in torch.randperm(odim - 2, generator=g).tolist() if t + 1 != nxt]
            rows.append([nxt] + rest[:S - 1])
        cands.append(torch.tensor(rows))
    return prefixes, cands


def run_reference(case, dtype):
    dec, ctc = build(case, dtype)
    lengths, n, eos = case["lengths"], case["n_hyp"], case["odim"] - 1
    mem = encoder_input(lengths, case["d_model"], case["xseed"]).to(dtype)
    prefixes, cands = script(case)
    out = {}
    with torch.no_grad():
        ctc_logp = ctc.log_softmax(mem)                                         # (U, T_max, O)
        impl = CTCPrefixScoreTH(ctc_logp.clone(), torch.tensor(lengths), 0, eos)
        scorer = CTCPrefixScorer(ctc, eos)
        state = None
        for step in range(case["steps"]):
            if state is not None:                     # what batch_score_partial stacks (scorers/ctc.py:118-128)
                state = (torch.stack([s[0] for s in state], dim=2), torch.stack([s[1] for s in state]), state[0][2],
                         state[0][3])
            local, new_state = impl(prefixes[step], state, cands[step])
            out[f"ctc_local_{step}"] = local
            keep = cands[step][:, 0]                  # the next prefix token
            state = [scorer.select_state(new_state, i, int(keep[i])) for i in range(keep.numel())]
        token_list = [str(i) for i in range(case["odim"])]
        for u, T in enumerate(lengths):
            scorers = dict(decoder=dec, ctc=CTCPrefixScorer(ctc, eos), lm=None, length_bonus=LengthBonus(len(token_list)))
            weights = dict(decoder=0.9, ctc=0.1, lm=0.0, length_bonus=0)
            bs = BatchBeamSearch(beam_size=case["beam"], vocab_size=len(token_list), weights=weights, scorers=scorers,
                                 sos=eos, eos=eos, token_list=token_list, pre_beam_score_key="decoder")
            out[f"nbest_{u}"] = [h.asdict() for h in bs(mem[u, :T])]
    return out


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    only = sys.argv[1:]
    for case in CASES:
        if only and case["name"] not in only:
            continue
        r64 = run_reference(case, torch.float64)
        r32 = run_reference(case, torch.float32)
        prefixes, cands = script(case)
        eos = case["odim"] - 1
        store = {"lengths": np.asarray(case["lengths"])}
        for step in range(case["steps"]):
            cand = cands[step]
            store[f"ctc_prefix_{step}"] = prefixes[step].numpy()
            store[f"ctc_cand_{step}"] = cand.numpy()
            store[f"ctc_local_f64_{step}"] = torch.gather(r64[f"ctc_local_{step}"], 1, cand).numpy()
            store[f"ctc_local_f32_{step}"] = torch.gather(r32[f"ctc_local_{step}"], 1, cand).numpy()
            store[f"ctc_eos_f64_{step}"] = r64[f"ctc_local_{step}"][:, eos].numpy()
            store[f"ctc_eos_f32_{step}"] = r32[f"ctc_local_{step}"][:, eos].numpy()
        for tag, r in (("f64", r64), ("f32", r32)):
            for u in range(len(case["lengths"])):
                full = r[f"nbest_{u}"]
                nb = full[:NBEST_KEPT]
                width = max(len(h["yseq"]) for h in nb)
                store[f"nbest_len_{tag}_{u}"] = np.asarray([len(h["yseq"]) for h in nb])
                store[f"nbest_yseq_{tag}_{u}"] = np.asarray([h["yseq"] + [-1] * (width - len(h["yseq"])) for h in nb])
                store[f"nbest_score_{tag}_{u}"] = np.asarray([h["score"] for h in nb])
                store[f"nbest_dec_{tag}_{u}"] = np.asarray([h["scores"]["decoder"] for h in nb])
                store[f"nbest_ctc_{tag}_{u}"] = np.asarray([h["scores"]["ctc"] for h in nb])
                store[f"nbest_count_{tag}_{u}"] = np.asarray(len(full))
        meta = {k: v for k, v in case.items() if k not in ("name", "lengths")}
        np.savez_compressed(os.path.join(out_dir, case["name"] + ".npz"),
                            **store, **{"cfg_" + k: np.asarray(v) for k, v in meta.items()})
        for u in range(len(case["lengths"])):
            print(case["name"], "utterance", u, "nbest", len(r64[f"nbest_{u}"]), "best", r64[f"nbest_{u}"][0]["score"],
                  "f32", r32[f"nbest_{u}"][0]["score"],
                  "same best yseq f32/f64:", r64[f"nbest_{u}"][0]["yseq"] == r32[f"nbest_{u}"][0]["yseq"])


if __name__ == "__main__":
    main()
