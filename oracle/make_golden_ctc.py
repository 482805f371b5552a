#!/usr/bin/env python3
"""Generate tests/golden/ctc_loss_{tiny,full}.npz by running the UNMODIFIED reference CTC module
(espnet/nets/pytorch_backend/ctc.py:41-65, CTC.forward -> loss_fn) in float64, train mode, dropout p = 0.
TEST INFRASTRUCTURE ONLY.  Run where the reference tree or its oracle/_ref copy exists:

    python oracle/make_golden_ctc.py            (imports the reference from oracle/_ref, see oracle/build_ref.py)

Weights (``ctc.ctc_lo``) and encoder features regenerate from seeds via ``auto_avsr_b200.synthetic``; the label rows,
the loss (reduce=True and reduce=False) and the gradients of the reduce=True loss are stored: d hs_pad, d ctc_lo.bias,
and d ctc_lo.weight.  A large gradient is stored as a float32 subset (every FRAME_STEP-th frame of d hs_pad, every
ROW_STEP-th row of d ctc_lo.weight, the step stored beside it) plus [sum, sum |.|, sum of squares] of the whole array,
which keeps the full case's fixture small.

Cases
  tiny  d 128, odim 37, lengths [19, 12, 7, 1]: repeated tokens that need a blank between them, -1 in the middle of a
        row, a target too long for its frames (zero_infinity), an empty target
  full  d 768, odim 5049, B 4, ragged up to 400 frames, 60-100 labels per utterance
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from auto_avsr_b200.synthetic import encoder_input, head_state_dict  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
FRAME_STEP, ROW_STEP = 32, 128
CASES = {
    "ctc_loss_tiny": dict(d_model=128, odim=37, lengths=[19, 12, 7, 1], wseed=51, xseed=61),
    "ctc_loss_full": dict(d_model=768, odim=5049, lengths=[400, 370, 310, 260], wseed=52, xseed=62),
}


def labels(name):
    """(B, Lmax) int64 label rows, -1 = ignore_id."""
    if name == "ctc_loss_tiny":
        rows = [[5, 5, 9, -1, 9, 9, 3, 5, 5, 36],        # 19 frames; repeats need blanks; -1 inside the row
                [7, 2, -1, -1, 2, 30, -1, 1, -1, -1],     # 12 frames; several -1 between labels and at the end
                [4, 8, 8, 15, 16, 23, 42 % 37, 1, -1, -1],  # 7 frames, 8 labels: infeasible -> +inf -> 0
                [-1] * 10]                                # 1 frame, empty target
        return torch.tensor(rows, dtype=torch.long)
    g = torch.Generator().manual_seed(71)
    lens = [100, 87, 72, 60]
    ys = torch.full((4, max(lens)), -1, dtype=torch.long)
    for b, n in enumerate(lens):
        ys[b, :n] = torch.randint(1, CASES[name]["odim"], (n,), generator=g)
    ys[1, 10:13] = ys[1, 9]                               # a run of a repeated token
    return ys


def inputs(name):
    """-> (hs_pad (B, Tmax, d) float32, ctc_lo weight, bias float32, hlens int64, ys_pad int64)."""
    c = CASES[name]
    hs = encoder_input(c["lengths"], c["d_model"], c["xseed"])
    sd = head_state_dict(c["wseed"], 64, c["d_model"], c["odim"])
    return hs, sd["ctc.ctc_lo.weight"], sd["ctc.ctc_lo.bias"], torch.tensor(c["lengths"], dtype=torch.long), labels(name)


def import_reference_ctc():
    from oracle import build_ref
    build_ref.import_reference_encoder()             # puts the oracle/_ref copy first on sys.path
    from espnet.nets.pytorch_backend.ctc import CTC
    return CTC


def reference(name):
    """Run the reference CTC module in float64 -> dict of the stored arrays."""
    CTC = import_reference_ctc()
    c = CASES[name]
    hs, w, b, hlens, ys = inputs(name)
    out = {}
    for reduce in (True, False):
        ctc = CTC(c["odim"], c["d_model"], 0.0, reduce=reduce)
        ctc.load_state_dict({"ctc_lo.weight": w, "ctc_lo.bias": b}, strict=True)
        ctc = ctc.double().train()
        x = hs.double().clone().requires_grad_(reduce)
        loss, ys_hat = ctc(x, hlens, ys)
        if not reduce:
            out["loss_none"] = loss.detach().numpy()
            continue
        out["loss_sum"] = loss.detach().numpy()
        loss.backward()
        gh = x.grad.numpy()
        if gh.size > 500_000:
            out["d_hs__frames"] = gh[:, ::FRAME_STEP].astype(np.float32)
            out["d_hs__step"] = np.array(FRAME_STEP)
            out["d_hs__checksum"] = checksum(gh)
        else:
            out["d_hs"] = gh
        out["d_bias"] = ctc.ctc_lo.bias.grad.numpy()
        gw = ctc.ctc_lo.weight.grad.numpy()
        if gw.size > 500_000:
            out["d_weight__rows"] = gw[::ROW_STEP].astype(np.float32)
            out["d_weight__step"] = np.array(ROW_STEP)
            out["d_weight__checksum"] = checksum(gw)
        else:
            out["d_weight"] = gw
        out["ys_hat_shape"] = np.array(ys_hat.shape)
    return out


def checksum(g):
    """[sum, sum |.|, sum of squares] of a whole gradient (float64)"""
    return np.array([g.sum(), np.abs(g).sum(), (g ** 2).sum()])


def main():
    for name, c in CASES.items():
        res = reference(name)
        _, _, _, hlens, ys = inputs(name)
        np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), ys_pad=ys.numpy(), hlens=hlens.numpy(),
                            d_model=np.array(c["d_model"]), odim=np.array(c["odim"]), wseed=np.array(c["wseed"]),
                            xseed=np.array(c["xseed"]), **res)
        print(name, os.path.getsize(os.path.join(GOLDEN, name + ".npz")) // 1024, "KiB", "loss", float(res["loss_sum"]))


if __name__ == "__main__":
    main()
