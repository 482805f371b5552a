#!/usr/bin/env python3
"""Generate tests/golden/decoder_train_{tiny,full}.npz by running the UNMODIFIED reference TransformerDecoder.forward
(espnet/nets/pytorch_backend/decoder/transformer_decoder.py:229-258) and LabelSmoothingLoss (smoothing 0.1,
normalize_length=False; transformer/label_smoothing_loss.py:41-63) in float64, train mode, every dropout p = 0, on the
inputs E2E.forward builds (add_sos_eos, target_mask, the memory's prefix padding mask; e2e_asr_conformer.py:67-80).
TEST INFRASTRUCTURE ONLY.  Run where the reference tree or its oracle/_ref copy exists:

    python oracle/make_golden_decoder_train.py          (imports the reference from oracle/_ref, see oracle/build_ref.py)

Weights and encoder memory regenerate from seeds via ``auto_avsr_b200.synthetic``; the label rows are stored.  Stored:
the loss, pred_pad, d memory and the gradient of every parameter, in float32.  An array of more than the case's ``big``
elements is stored as a subset -- every r-th row and every c-th column of its leading-dimension-flattened 2-D form
((r, c) = the case's ``param_step``, or ``act_step`` for pred_pad / d memory; a vector is one row; both stored once) --
plus [sum, sum |.|, sum of squares] of the whole array in float64, which keeps the full case's fixture at about
200 KB.

Cases
  tiny  odim 37, d 128, H 2, ff 256, 2 layers, memory [23, 17, 9, 12], label rows of 7, 3, 0 (empty) and 5 tokens
  full  odim 5049, d 768, H 12, ff 3072, 6 layers, memory [300, 262, 190], 60 / 45 / 31 tokens
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from auto_avsr_b200.synthetic import decoder_state_dict, encoder_input  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
SMOOTHING, IGNORE_ID = 0.1, -1
CASES = {
    "decoder_train_tiny": dict(odim=37, d_model=128, n_heads=2, linear_units=256, num_blocks=2, mem=[23, 17, 9, 12],
                               labels=[7, 3, 0, 5], wseed=81, xseed=91, big=4096, param_step=(8, 1), act_step=(1, 1)),
    "decoder_train_full": dict(odim=5049, d_model=768, n_heads=12, linear_units=3072, num_blocks=6, mem=[300, 262, 190],
                               labels=[60, 45, 31], wseed=82, xseed=92, big=512, param_step=(128, 16),
                               act_step=(16, 16)),
}


def inputs(name):
    """-> (state dict float32, memory (B, T, d) float32, memory lengths int64, label rows (B, Lmax) int64 with -1)."""
    c = CASES[name]
    sd = decoder_state_dict(c["wseed"], c["odim"], c["d_model"], c["n_heads"], c["linear_units"], c["num_blocks"])
    mem = encoder_input(c["mem"], c["d_model"], c["xseed"])
    g = torch.Generator().manual_seed(c["xseed"] + 1)
    ys = torch.full((len(c["labels"]), max(max(c["labels"]), 1)), IGNORE_ID, dtype=torch.long)
    for b, n in enumerate(c["labels"]):
        ys[b, :n] = torch.randint(1, c["odim"] - 1, (n,), generator=g)
    return sd, mem, torch.tensor(c["mem"], dtype=torch.long), ys


def import_reference():
    from oracle import build_ref
    build_ref.import_reference_encoder()             # puts the oracle/_ref copy first on sys.path
    from espnet.nets.pytorch_backend.decoder.transformer_decoder import TransformerDecoder
    from espnet.nets.pytorch_backend.nets_utils import make_non_pad_mask
    from espnet.nets.pytorch_backend.transformer.add_sos_eos import add_sos_eos
    from espnet.nets.pytorch_backend.transformer.label_smoothing_loss import LabelSmoothingLoss
    from espnet.nets.pytorch_backend.transformer.mask import target_mask
    return TransformerDecoder, LabelSmoothingLoss, add_sos_eos, target_mask, make_non_pad_mask


def batch(name):
    """The decoder's inputs as E2E.forward builds them -> (ys_in_pad, ys_mask, memory_mask, ys_out_pad)."""
    _, _, add_sos_eos, target_mask, make_non_pad_mask = import_reference()
    c = CASES[name]
    _, _, mlen, ys = inputs(name)
    ys_in, ys_out = add_sos_eos(ys, c["odim"] - 1, c["odim"] - 1, IGNORE_ID)
    return ys_in, target_mask(ys_in, IGNORE_ID), make_non_pad_mask(mlen).unsqueeze(-2), ys_out


def _store(out, key, a, big, step):
    a = np.asarray(a)
    if a.size > big:
        out[key + "__rows"] = a.reshape(-1, a.shape[-1])[::step[0], ::step[1]].astype(np.float32)
        out[key + "__checksum"] = np.array([a.sum(), np.abs(a).sum(), (a ** 2).sum()])
    else:
        out[key] = a.astype(np.float32)


def reference(name):
    """Run the reference decoder + loss in float64 -> dict of the stored arrays."""
    TransformerDecoder, LabelSmoothingLoss, _, _, _ = import_reference()
    c = CASES[name]
    sd, mem, _, _ = inputs(name)
    ys_in, ys_mask, mem_mask, ys_out = batch(name)
    dec = TransformerDecoder(odim=c["odim"], attention_dim=c["d_model"], attention_heads=c["n_heads"],
                             linear_units=c["linear_units"], num_blocks=c["num_blocks"], dropout_rate=0.0,
                             positional_dropout_rate=0.0, self_attention_dropout_rate=0.0, src_attention_dropout_rate=0.0)
    dec.load_state_dict(sd, strict=True)
    dec = dec.double().train()
    crit = LabelSmoothingLoss(c["odim"], IGNORE_ID, SMOOTHING, False)
    x = mem.double().clone().requires_grad_(True)
    pred, _ = dec(ys_in, ys_mask, x, mem_mask)
    loss = crit(pred, ys_out)
    loss.backward()
    out = {"loss": loss.detach().numpy(), "ys_pad": inputs(name)[3].numpy(), "param_step": np.array(c["param_step"]),
           "act_step": np.array(c["act_step"])}
    _store(out, "pred_pad", pred.detach().numpy(), c["big"], c["act_step"])
    _store(out, "d_memory", x.grad.numpy(), c["big"], c["act_step"])
    for k, p in dec.named_parameters():
        _store(out, "d_" + k, p.grad.numpy(), c["big"], c["param_step"])
    return out


def main():
    for name in CASES:
        res = reference(name)
        np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), **res)
        print(name, os.path.getsize(os.path.join(GOLDEN, name + ".npz")) // 1024, "KiB", "loss", float(res["loss"]))


if __name__ == "__main__":
    main()
