"""Each residual stage of the fused f16 / tf32 / fp32 encoder layer (csrc/encoder.cu forward_body) against float64,
one stage at a time, at the bucket shapes and at the edges of the kernels' tiling.

A 2-layer full-size encoder (d 768, H 12, ff 3072, k 31) runs with layer-0 stage taps: g0..g4 are the residual stream
after the macaron FFN, the MHA, the conv module, the FFN and norm_final, and `out` is the output after layer 1 and
after_norm.  Each float64 reference starts from the GPU's own input to that stage (oracle/encoder_stages.py): r0 from
the embedded input xs * sqrt(d), r_s from g_{s-1}, and `out` from g4 through layer 1 (which runs the fused
norm_final + next norm_ff_macaron LayerNorm pair and layer 1's slice of the stacked linear_pos table).  A bound
therefore covers one stage's rounding, and a stage that goes wrong is named by the tap that fails.

Metrics (oracle/encoder_stages.errors): for the four residual blocks, max|g_s - r_s| over the block's own contribution
max|r_s - g_{s-1}| (the residual stream would hide an error in a block); for norm_final and the output, max-abs
relative to max|r|.  rms is recorded beside it, and the frame-outlier ratio (largest per-frame error over the median
per-frame error) catches a mistake confined to a tile or utterance edge.

Negative controls: for every case, references with one plausible kernel defect each (oracle/encoder_stages.DEFECTS)
must miss the GPU output by at least twice the stage's bound, so the bounds are shown to be tight enough to catch
them.  A defect that cannot change the result at a shape (ES.applies) is recorded as n/a; the few that clear the
bound but not twice it are listed in WEAK_CONTROLS.

Bounds are about 4x the largest value observed on an H100 over the nine shapes; every comparison is recorded with
helpers.record.
"""
import math

import pytest
import torch

from helpers import record
from oracle import conformer_oracle as O
from oracle import encoder_stages as ES

pytestmark = pytest.mark.gpu

PRECS = ["fp32", "tf32", "f16"]
D, H, FF, K = 768, 12, 3072, 31
WSEED = 11

# name -> (lengths, masked)
SHAPES = {
    "S1": ([100], False),                              # M < 128, no mask, 2 key tiles, Tp = 104
    "S2": ([400] * 4, True),                           # the benchmarked workload
    "S2r": ([400, 350, 300, 250, 300], True),          # padded query rows, ragged key tiles
    "S3": ([100] * 16, True),                          # utterance boundaries inside GEMM row tiles and QK row groups
    "S4": ([1600], False),                             # 25 key tiles, 3199-row pos table
    "E1": ([1], False),                                # T = 1
    "E2": ([65, 64, 63, 1], True),                     # query / key tile edges, a one-frame utterance
    "E3": ([33, 0, 33, 5, 33, 1, 33], True),           # odd T, utterances starting at rows != 0 mod 4, a length 0
    "E4": ([129, 128, 127], True),                     # 128-row GEMM tile edges
}

# (max, rms, frame-outlier ratio) per stage: max / rms relative to the block's contribution (stages 0-3) or to
# max|r| (norm_final, out).  About 4x the largest value over the nine shapes on an H100 80GB HBM3 (700 W).  tf32
# and f16 operands both carry a 10-bit mantissa and show the same errors.  The MHA's frame ratio is highest at E2
# and E3: a query with one valid key returns its V row unaveraged, with the full operand rounding of V.
TOL = {
    "fp32": {
        "ffn_macaron": (5e-05, 6.5e-06, 8.5),
        "mha": (7e-05, 7e-06, 8.5),           # the largest at S4, where the fp32 sinusoid table drifts most
        "conv": (5e-05, 7.5e-06, 8),
        "ffn": (4.5e-05, 6e-06, 8),
        "norm_final": (6.5e-07, 5e-08, 15),
        "out": (1.5e-06, 2.5e-07, 10),
    },
    "tf32": {
        "ffn_macaron": (2e-3, 5.5e-04, 6.5),
        "mha": (2e-3, 5.5e-04, 20),
        "conv": (1.5e-3, 2.5e-04, 7),
        "ffn": (2e-3, 4.5e-04, 7),
        "norm_final": (7e-07, 7.5e-08, 15),
        "out": (8e-4, 1.5e-04, 15),
    },
    "f16": {
        "ffn_macaron": (2e-3, 5.5e-04, 6.5),
        "mha": (2e-3, 5.5e-04, 20),
        "conv": (1.5e-3, 2.5e-04, 7),
        "ffn": (2e-3, 4.5e-04, 6.5),
        "norm_final": (6.5e-07, 7e-08, 15),
        "out": (8e-4, 1.5e-04, 15),
    },
}
CONTROL_MARGIN = 2.0
# Controls that miss the GPU output by more than the bound but by less than CONTROL_MARGIN times it: with 1600 keys,
# masking the last one moves the attention output by only ~1.85x the tf32 / f16 MHA bound on an H100.  They are
# recorded and must still exceed the bound itself.
WEAK_CONTROLS = {("S4", "tf32", "mha_drop_last_key"), ("S4", "f16", "mha_drop_last_key")}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "needs a GPU"
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def model(dev):
    from auto_avsr_b200 import ConformerEncoder
    from auto_avsr_b200.synthetic import encoder_state_dict
    sd = encoder_state_dict(WSEED, D, H, FF, num_blocks=2, cnn_kernel=K)
    enc = ConformerEncoder(attention_dim=D, attention_heads=H, linear_units=FF, num_blocks=2, cnn_module_kernel=K)
    enc.load_state_dict(sd, strict=True)
    enc = enc.to(dev).eval()
    sd64 = {k: (t.to(dev, torch.float64) if t.is_floating_point() else t.to(dev)) for k, t in sd.items()}
    return enc, sd64


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_encoder_stages_vs_fp64(dev, model, shape, prec):
    from auto_avsr_b200.synthetic import encoder_input
    enc, sd = model
    lengths, masked = SHAPES[shape]
    xs = encoder_input(lengths, D, 300 + list(SHAPES).index(shape)).to(dev)
    B, T, _ = xs.shape
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev) if masked else None
    enc.precision = prec
    enc.check_saturation = False

    # ---- bits: direct launches repeat, the CUDA-graph plan and the saturation-checked forward agree with them
    with torch.no_grad():
        taps = torch.empty(5, B * T, D, device=dev)
        out = enc(xs, mask, taps=taps)[0].clone()
        taps2 = torch.empty_like(taps)
        out2 = enc(xs, mask, taps=taps2)[0]
        assert torch.equal(taps, taps2) and torch.equal(out, out2), "repeated direct call differs"
        enc.use_graph, enc.graph_after = True, 1
        assert torch.equal(enc(xs, mask)[0], out), "CUDA-graph plan differs from direct launches"
        if prec == "f16":
            enc.check_saturation = True
            try:
                checked = enc(xs, mask)[0]               # raises SaturationError on a saturated fp16 operand
            finally:
                enc.check_saturation = False
            assert torch.equal(checked, out), "saturation-checked forward differs"
    assert torch.isfinite(taps).all() and torch.isfinite(out).all()

    # ---- stage-isolated float64 references
    pos = O.rel_sinusoid_table(T, D, torch.float64).to(dev)
    len_t = torch.tensor(lengths, dtype=torch.long, device=dev) if masked else None
    x0 = (xs * torch.tensor(math.sqrt(D), dtype=torch.float32, device=dev)).double()   # the kernel's embed scale
    g = [taps[s].view(B, T, D).double() for s in range(5)]
    ins = [x0] + g[:4]
    refs = [ES.stage(s, ins[s], pos, len_t, sd, "encoders.0.", H) for s in range(5)]
    ref_out = ES.layer_and_after_norm(g[4], pos, len_t, sd, 1, H)

    failures = []
    got = {}
    for key, gpu, ref, g_in in [*zip(ES.STAGES, g, refs, [*ins[:4], None]), ("out", out, ref_out, None)]:
        e = ES.errors(gpu, ref, g_in)
        got[key] = e
        tol = TOL[prec][key]
        record("encoder_stages", (shape, prec, key),
               {"max": e["max"], "rms": e["rms"], "frames": e["frames"], "worst_frame": divmod(e["worst"], T)},
               {"max": tol[0], "rms": tol[1], "frames": tol[2]})
        if not (e["max"] < tol[0] and e["rms"] < tol[1] and e["frames"] < tol[2]):
            failures.append(f"{key}: max {e['max']:.3e} rms {e['rms']:.3e} frames {e['frames']:.1f} vs {tol}")

    # ---- negative controls: a reference with one plausible defect must miss the GPU output clearly
    for defect, s in ES.DEFECTS.items():
        if not ES.applies(defect, B, T):
            record("encoder_stages_control", (shape, prec, defect), "n/a: no effect at this shape", CONTROL_MARGIN)
            continue
        bad = ES.stage(s, ins[s], pos, len_t, sd, "encoders.0.", H, defect=defect)
        miss = (g[s] - bad).abs().max().item() / got[ES.STAGES[s]]["scale"]
        margin = miss / TOL[prec][ES.STAGES[s]][0]
        need = 1.0 if (shape, prec, defect) in WEAK_CONTROLS else CONTROL_MARGIN
        record("encoder_stages_control", (shape, prec, defect), margin, need)
        if not margin >= need:
            failures.append(f"control {defect}: misses by {miss:.3e}, {margin:.2f}x the bound")
    assert not failures, f"{shape} {prec}: " + "; ".join(failures)
