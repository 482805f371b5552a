"""Each stage of the ResNet front-ends (csrc/frontend.cu) against float64 at the clip and waveform shapes the data
produces.

``avsr_frontend_forward_taps`` copies 10 stage outputs (stem, trunk input, the 8 BasicBlocks) as fp32.  Two checks per
case and precision, every error relative: max |gpu - ref| / max |ref| per tap, and for the (B, T, 512) output:
- isolated: each stage is fed the library's own previous tap promoted to float64 and compared with the oracle's stage
  (oracle/frontend_oracle.py), which measures that stage's own error.  The max-pool picks values, so its error is 0;
- chained: every tap against the oracle chained from the raw input, which shows how the error grows along the trunk.

Shapes: temporal edges of the video stem (1 to 9 frames per utterance), frame counts that leave the last 128-row tile of
each trunk layer with its fewest and most rows, the bucket shapes, odd frame sizes down to 1x1, waveforms around a
whole 640-sample frame, the audio bucket and 1600 frames, and audio shorter than one frame.  Then BatchNorm statistics as
training leaves them (running_var over six decades, means 5 standard deviations off, gammas near 0) with the f16
headroom to 65504 per tap; bit-identity under poisoned inputs past the cut and a NaN-filled workspace; and programmatic
dependent launch on and off for the front-end, the encoder, the fused head and the CTC loss.

Each case runs in a child process (its own CUDA context).  Bounds are about 4x the largest error observed on an H100
80GB HBM3 (tests/helpers.py record())."""
import math
import os
import subprocess
import sys
from collections import OrderedDict

import pytest
import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

pytestmark = pytest.mark.gpu

#: output pixels per frame of the 4 trunk layers of an 88x88 clip (22x22, 11x11, 6x6, 3x3)
TRUNK_PIXELS = {"layer1": 484, "layer2": 121, "layer3": 36, "layer4": 9}
CV_BM = 128            # output rows per CTA of the implicit-GEMM convolution


def tail_frame_counts():
    """{(layer, rows in the last tile): frames}: the fewest frames that leave the last 128-row M tile of a trunk layer
    with as few and as many rows as its pixels per frame allow (1 and 127 for odd counts; gcd(ppf, 128) and
    128 - gcd for even ones)."""
    out = {}
    for layer, ppf in TRUNK_PIXELS.items():
        g = math.gcd(ppf, CV_BM)
        for rows in (g, CV_BM - g):
            out[(layer, rows)] = next(n for n in range(1, CV_BM + 1) if n * ppf % CV_BM == rows)
    return out


def trained_like_state_dict(seed: int, modality: str) -> "OrderedDict[str, torch.Tensor]":
    """Synthetic front-end weights with BatchNorm statistics as training leaves them, fitted in float64 on a seeded
    calibration input (video 2 x 5 frames of 44x44, audio 2 x 6 frames).  Conv by conv in data-flow order, each output
    channel is rescaled so that its standard deviation over the calibration input is sqrt(running_var), with
    running_var log-uniform over [1e-4, 1e2]; running_mean is the channel's mean moved by up to +-5 of those standard
    deviations; gamma is uniform over [-2, 2] with every 8th channel within 1e-3 of 0; beta is N(0, 1).  fp32, under the
    reference's keys."""
    import torch.nn.functional as F
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    from oracle import frontend_oracle as O
    sd = OrderedDict((k, v.double() if v.is_floating_point() else v.clone())
                     for k, v in frontend_state_dict(seed, modality).items())
    g = torch.Generator().manual_seed(seed * 1009 + 7)

    def u(n, lo, hi):
        return torch.rand(n, generator=g, dtype=torch.float64) * (hi - lo) + lo

    def fit(conv, bn, h):
        C = h.shape[1]
        dims = [0] + list(range(2, h.dim()))
        var = 10.0 ** u(C, -4.0, 2.0)
        k = var.sqrt() / h.std(dim=dims)
        w = sd[conv + ".weight"]
        sd[conv + ".weight"] = w * k.view((-1,) + (1,) * (w.dim() - 1))
        sd[bn + ".running_var"] = var
        sd[bn + ".running_mean"] = h.mean(dim=dims) * k + u(C, -5.0, 5.0) * var.sqrt()
        gamma = u(C, -2.0, 2.0)
        gamma[::8] = u(gamma[::8].numel(), -1e-3, 1e-3)
        sd[bn + ".weight"] = gamma
        sd[bn + ".bias"] = torch.randn(C, generator=g, dtype=torch.float64)

    if modality == "video":
        x = frontend_input("video", 2, 5, 44, 44, seed, dtype=torch.float64)
        fit("frontend3D.0", "frontend3D.1",
            F.conv3d(x.transpose(1, 2), sd["frontend3D.0.weight"], stride=(1, 2, 2), padding=(2, 3, 3)))
        a = O.pool("video", O.stem(sd, "video", x))
    else:
        x = frontend_input("audio", 2, 640 * 6, seed=seed, dtype=torch.float64)
        fit("trunk.conv1", "trunk.bn1", F.conv1d(x.transpose(1, 2), sd["trunk.conv1.weight"], stride=4, padding=38))
        a = O.stem(sd, "audio", x)
    for i in range(8):
        p = O.block_name(i)
        stride = 2 if i in (2, 4, 6) else 1
        xin = O.from_channels_last(a, modality)
        fit(p + "conv1", p + "bn1", O.conv(xin, sd[p + "conv1.weight"], stride))
        h = O.silu(O.batch_norm(O.conv(xin, sd[p + "conv1.weight"], stride), sd, p + "bn1."))
        fit(p + "conv2", p + "bn2", O.conv(h, sd[p + "conv2.weight"], 1))
        if p + "downsample.0.weight" in sd:
            fit(p + "downsample.0", p + "downsample.1", O.conv(xin, sd[p + "downsample.0.weight"], stride))
        a = O.block(sd, modality, i, a)
    return OrderedDict((k, v.float() if v.is_floating_point() else v) for k, v in sd.items())


PRELUDE = f"""
import os, sys, math, torch
sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})
from helpers import record
from auto_avsr_b200 import _cabi
from auto_avsr_b200.frontend import PreparedFrontend, frontend_forward, frontend_tap_shape, frontend_workspace_bytes
from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
from oracle import frontend_oracle as O
from test_zz_gpu_frontend_stages import tail_frame_counts, trained_like_state_dict
dev = torch.device("cuda:0")
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
PRECS = ("fp32", "tf32", "f16")
# relative max error bounds per tap 0..9 and the output, about 4x the largest observed on an H100 80GB HBM3 over all
# shapes of this file with the synthetic weights (ISO: each stage fed the library's previous tap; CHAIN: from the raw
# input), and with trained-like BatchNorm statistics (ISO_BN, CHAIN_BN).  The max-pool's isolated error is 0.
ISO = {{"fp32": [3.2e-6, 0, 4.6e-6, 5.3e-6, 6.9e-6, 6.3e-6, 9e-6, 7.2e-6, 7.8e-6, 9.1e-6, 9.4e-7],
       "tf32": [2.9e-3, 0, 2.4e-3, 2.6e-3, 3.3e-3, 2.6e-3, 3.1e-3, 2.2e-3, 2.7e-3, 2.1e-3, 2.9e-7],
       "f16": [2.9e-3, 0, 2.4e-3, 2.5e-3, 3e-3, 2.5e-3, 3.3e-3, 2.3e-3, 2.6e-3, 2.3e-3, 3.5e-7]}}
CHAIN = {{"fp32": [3.2e-6, 3.2e-6, 4.7e-6, 5.8e-6, 6.6e-6, 7.8e-6, 1.1e-5, 9.7e-6, 1.04e-5, 9.9e-6, 4.5e-6],
         "tf32": [2.9e-3, 2.9e-3, 3.2e-3, 4e-3, 4.8e-3, 5.3e-3, 5.8e-3, 5.2e-3, 6.4e-3, 6.1e-3, 5.9e-3],
         "f16": [2.9e-3, 2.9e-3, 3.2e-3, 3.8e-3, 4.8e-3, 5.3e-3, 5.8e-3, 6.2e-3, 6.6e-3, 6.3e-3, 5.1e-3]}}
ISO_BN = {{"fp32": [1.7e-6, 0, 3.2e-6, 3.8e-6, 3.9e-6, 3.1e-6, 5e-6, 4.9e-6, 6.4e-6, 8.1e-6, 6.3e-7],
          "tf32": [1.5e-3, 0, 2.9e-3, 2.5e-3, 2.9e-3, 2.4e-3, 2.4e-3, 1.8e-3, 2.7e-3, 3e-3, 1.5e-7],
          "f16": [1.5e-3, 0, 2.9e-3, 2.5e-3, 2.8e-3, 2.3e-3, 2.5e-3, 1.6e-3, 3e-3, 2.6e-3, 1.5e-7]}}
CHAIN_BN = {{"fp32": [1.7e-6, 1.7e-6, 3.4e-6, 4.8e-6, 4.7e-6, 4.3e-6, 6.4e-6, 5.9e-6, 7.7e-6, 1.1e-5, 3.5e-6],
            "tf32": [1.5e-3, 1.5e-3, 3.5e-3, 4.2e-3, 4.9e-3, 5.4e-3, 5.7e-3, 4.5e-3, 7.9e-3, 6.8e-3, 2.9e-3],
            "f16": [1.5e-3, 1.5e-3, 3.5e-3, 4.2e-3, 5e-3, 5.4e-3, 5.8e-3, 5.7e-3, 6.2e-3, 7.4e-3, 2.8e-3]}}

def rel(a, b):
    b = b.double()
    return ((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()

class Lib:
    \"\"\"the library front-end on one state dict: out, taps = lib(x, prec)\"\"\"
    def __init__(self, modality, sd):
        from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
        m = Conv3dResNet() if modality == "video" else Conv1dResNet()
        m.load_state_dict(sd, strict=True)
        self.m, self.modality, self.prep = m.to(dev).eval(), modality, PreparedFrontend()
        self.sd64 = {{k: v.to(dev, torch.float64) for k, v in sd.items() if v.is_floating_point()}}

    def dims(self, x):
        return (x.shape[0], x.shape[1], x.shape[3], x.shape[4]) if self.modality == "video" else (x.shape[0], x.shape[1], 1, 1)

    def __call__(self, x, prec, taps=True, workspace=None):
        B, T, H, W = self.dims(x)
        t = [torch.empty(frontend_tap_shape(self.modality, B, T, H, W, i), device=dev) for i in range(O.N_TAPS)] if taps else None
        with torch.no_grad():
            out = frontend_forward(self.prep, self.modality, self.m.conv_bn_pairs(), x, prec, taps=t, workspace=workspace)
        torch.cuda.synchronize()
        return out, t

def check_stages(test, case, lib, x, precs, iso_bound=ISO, chain_bound=CHAIN, headroom=None):
    \"\"\"isolated and chained errors of every tap and the output, in each precision; returns the taps of the last one\"\"\"
    modality, sd64, B = lib.modality, lib.sd64, x.shape[0]
    x64 = x.double()
    with torch.no_grad():
        ref_taps, ref_out = O.taps(sd64, modality, x64)
    bad = []
    for prec in precs:
        out, t = lib(x, prec)
        assert out.shape == ref_out.shape, (out.shape, ref_out.shape)
        for k in range(O.N_TAPS):
            assert t[k].shape == ref_taps[k].shape, (k, t[k].shape, ref_taps[k].shape)
            assert torch.isfinite(t[k]).all(), (case, prec, "tap", k)
        assert torch.isfinite(out).all(), (case, prec)
        with torch.no_grad():
            iso = [rel(t[0], O.stem(sd64, modality, x64))]
            iso += [rel(t[k], O.next_tap(sd64, modality, k, t[k - 1].double())) for k in range(1, O.N_TAPS)]
            iso.append(rel(out, O.head_mean(modality, t[-1].double(), B)))
        chain = [rel(t[k], ref_taps[k]) for k in range(O.N_TAPS)] + [rel(out, ref_out)]
        record(test + "_isolated", (case, prec), iso, iso_bound[prec])
        record(test + "_chained", (case, prec), chain, chain_bound[prec])
        if modality == "video":
            assert iso[1] == 0.0, ("the max-pool picks values: its isolated error must be 0", case, prec, iso[1])
        else:
            assert torch.equal(t[0], t[1]), "audio taps 0 and 1 are the same activation"
        if headroom is not None and prec == "f16":
            peak = [t[k].abs().max().item() for k in range(O.N_TAPS)]
            record(headroom, case, peak, 65504.0)
            assert max(peak) < 65504.0, ("f16 activation saturated", case, peak)
        bad += [(prec, "isolated", k, e) for k, e in enumerate(iso) if not e <= iso_bound[prec][k]]
        bad += [(prec, "chained", k, e) for k, e in enumerate(chain) if not e <= chain_bound[prec][k]]
    assert not bad, (case, bad)
    return t
"""


def run_child(body, timeout=1200, env=None):
    r = subprocess.run([sys.executable, "-c", PRELUDE + body], capture_output=True, text=True, timeout=timeout,
                       cwd=ROOT, env=env)
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


# ---------------------------------------------------------------- video
def test_video_temporal_edges():
    """The 5-frame stem runs past both ends of utterances of 1 to 5 frames; its taps must stop at each utterance's
    edge and never read the neighbouring row (3 x 2, 2 x 9)."""
    run_child("""
lib = Lib("video", frontend_state_dict(51, "video"))
for B, T in ((1, 1), (1, 2), (1, 3), (1, 4), (1, 5), (3, 2), (2, 9)):
    x = frontend_input("video", B, T, 88, 88, 100 + 10 * B + T).to(dev)
    check_stages("frontend_stage_video", f"{B}x{T}", lib, x, PRECS)
print("CHILD-OK")
""")


def test_video_last_tile_rows():
    """Frame counts that leave the last 128-row M tile of each trunk layer with its fewest and most rows, derived from
    the pixels per frame of the four layers (484, 121, 36, 9)."""
    counts = tail_frame_counts()
    assert len(set(counts.values())) == len(counts)
    run_child(f"""
lib = Lib("video", frontend_state_dict(52, "video"))
for (layer, rows), n in sorted({counts!r}.items()):
    x = frontend_input("video", 1, n, 88, 88, 200 + n).to(dev)
    check_stages("frontend_stage_video", f"1x{{n}} ({{layer}} last tile {{rows}} rows)", lib, x, PRECS)
print("CHILD-OK")
""")


@pytest.mark.parametrize("B,T,precs", [(16, 100, ("fp32", "tf32", "f16")), (4, 400, ("fp32", "tf32", "f16")),
                                       (1, 1600, ("f16",))])
def test_video_bucket(B, T, precs):
    """The batch shapes of the video buckets; 4 x 400 is the max-frames bucket, here also in TF32 against float64."""
    run_child(f"""
lib = Lib("video", frontend_state_dict(53, "video"))
x = frontend_input("video", {B}, {T}, 88, 88, 300).to(dev)
check_stages("frontend_stage_video", "{B}x{T}", lib, x, {precs!r})
print("CHILD-OK")
""")


def test_video_odd_geometry():
    """Frame sizes whose trunk layers end at a single pixel (1x1, 2x3, 7x7, 9x9), odd sizes (45x61, 89x89) and 96x96."""
    run_child("""
lib = Lib("video", frontend_state_dict(54, "video"))
for H, W in ((1, 1), (2, 3), (7, 7), (9, 9), (45, 61), (89, 89), (96, 96)):
    x = frontend_input("video", 2, 3, H, W, 400 + H * W).to(dev)
    check_stages("frontend_stage_video", f"2x3 at {H}x{W}", lib, x, PRECS)
print("CHILD-OK")
""")


# ---------------------------------------------------------------- audio
def test_audio_frame_edges():
    """Waveforms of exactly one 640-sample frame, one sample more, and 3 frames + 639 samples: the tail past the last
    whole frame is cut before the stem."""
    run_child("""
lib = Lib("audio", frontend_state_dict(55, "audio"))
for B, S in ((1, 640), (2, 641), (2, 640 * 3 + 639)):
    x = frontend_input("audio", B, S, seed=500 + S).to(dev)
    check_stages("frontend_stage_audio", f"{B}x{S}", lib, x, PRECS)
print("CHILD-OK")
""")


@pytest.mark.parametrize("B,S", [(4, 256000), (1, 1024000)])
def test_audio_bucket(B, S):
    """The audio bucket (4 x 256,000 samples, also in TF32 against float64) and one 1600-frame utterance."""
    run_child(f"""
lib = Lib("audio", frontend_state_dict(56, "audio"))
x = frontend_input("audio", {B}, {S}, seed=600).to(dev)
check_stages("frontend_stage_audio", "{B}x{S}", lib, x, PRECS)
print("CHILD-OK")
""")


def test_audio_shorter_than_one_frame():
    """Fewer than 640 samples give (B, 0, 512) without a launch, and every tap is empty."""
    run_child("""
lib = Lib("audio", frontend_state_dict(57, "audio"))
for B, S in ((3, 639), (2, 1), (1, 0)):
    x = frontend_input("audio", B, S, seed=7).to(dev)
    for prec in PRECS:
        lib(x, prec)                                   # the first call per precision prepares the weights
        n0 = _cabi.launch_count()
        out, t = lib(x, prec)
        assert _cabi.launch_count() == n0, (B, S, prec)
        assert tuple(out.shape) == (B, 0, 512), out.shape
        assert all(a.numel() == 0 and a.shape[0] == B for a in t), [a.shape for a in t]
print("CHILD-OK")
""")


# ---------------------------------------------------------------- trained-like BatchNorm
@pytest.mark.parametrize("modality", ["video", "audio"])
def test_trained_like_batchnorm(modality):
    """BatchNorm statistics over six decades of running_var, means 5 standard deviations off and gammas near 0: the
    BN scale stays in fp32 outside the operand weights.  Records the largest |activation| per tap in f16."""
    run_child(f"""
lib = Lib({modality!r}, trained_like_state_dict(58, {modality!r}))
x = (frontend_input("video", 2, 5, 88, 88, 700) if {modality!r} == "video" else
     frontend_input("audio", 2, 640 * 5 + 100, seed=700)).to(dev)
check_stages("frontend_stage_trained_bn", {modality!r}, lib, x, PRECS, ISO_BN, CHAIN_BN,
             headroom="frontend_stage_f16_headroom")
print("CHILD-OK")
""")


# ---------------------------------------------------------------- bits that must not move
def test_poisoned_inputs_and_workspace_keep_bits():
    """Bit-identical outputs and taps: audio samples past the last whole frame set to NaN / +-1e30; the workspace filled
    with NaN (0xFF bytes) before the call, which catches a read of anything the call did not write; the taps entry
    against the plain entry."""
    run_child("""
for modality in ("video", "audio"):
    lib = Lib(modality, frontend_state_dict(59, modality))
    x = (frontend_input("video", 2, 5, 88, 88, 800) if modality == "video" else
         frontend_input("audio", 2, 640 * 4 + 333, seed=800)).to(dev)
    for prec in PRECS:
        out, t = lib(x, prec)
        plain, _ = lib(x, prec, taps=False)
        assert torch.equal(out, plain), (modality, prec, "taps entry vs plain entry")
        nbytes = frontend_workspace_bytes(modality, x, prec)
        for fill in (0x00, 0xFF):
            ws = torch.full((nbytes,), fill, dtype=torch.uint8, device=dev)
            o2, t2 = lib(x, prec, workspace=ws)
            assert torch.equal(out, o2), (modality, prec, fill)
            assert all(torch.equal(a, b) for a, b in zip(t, t2)), (modality, prec, fill)
        if modality == "audio":
            for v in (float("nan"), 1e30, -1e30):
                xp = x.clone()
                xp[:, 640 * 4:] = v
                o3, t3 = lib(xp, prec)
                assert torch.equal(out, o3), (prec, v)
                assert all(torch.equal(a, b) for a, b in zip(t, t3)), (prec, v)
print("CHILD-OK")
""")


# ---------------------------------------------------------------- programmatic dependent launch
PDL_BODIES = {
    "frontend": """
res = {}
for modality in ("video", "audio"):
    lib = Lib(modality, frontend_state_dict(60, modality))
    x = (frontend_input("video", 2, 7, 88, 88, 900) if modality == "video" else
         frontend_input("audio", 2, 640 * 7 + 3, seed=900)).to(dev)
    for prec in PRECS:
        out, t = lib(x, prec)
        res[f"{modality}_{prec}"] = out.cpu()
        res[f"{modality}_{prec}_taps"] = [a.cpu() for a in t]
""",
    "encoder": """
from helpers import load_case
from auto_avsr_b200 import ConformerEncoder
from oracle import conformer_oracle as CO
c = load_case("full2_ragged")
cfg = c["cfg"]
enc = ConformerEncoder(attention_dim=cfg["d_model"], attention_heads=cfg["n_heads"], linear_units=cfg["linear_units"],
                       num_blocks=cfg["num_blocks"], cnn_module_kernel=cfg["cnn_kernel"])
enc.load_state_dict(c["sd"], strict=True)
enc = enc.to(dev).eval()
enc.graph_after = 1
mask = CO.non_pad_mask(c["lengths"]).unsqueeze(1).to(dev)
res = {}
for prec in ("f16", "tf32"):
    enc.precision = prec
    for graph in (False, True):
        enc.use_graph = graph
        with torch.no_grad():
            res[f"{prec}_graph{int(graph)}"] = enc(c["xs"].to(dev), mask)[0].cpu()
""",
    "head": """
from helpers import load_head_case
from auto_avsr_b200 import ConformerEncoder, CTC, ProjEncoder
from auto_avsr_b200.head import features_to_log_probs
from oracle import conformer_oracle as CO
c = load_head_case("head_full")
cfg = c["cfg"]
enc = ConformerEncoder(attention_dim=cfg["d_model"], attention_heads=cfg["n_heads"], linear_units=cfg["linear_units"],
                       num_blocks=cfg["num_blocks"], cnn_module_kernel=cfg["cnn_kernel"])
enc.load_state_dict(c["enc_sd"], strict=True)
proj = ProjEncoder(cfg["idim"], cfg["d_model"])
proj.load_state_dict({"weight": c["head_sd"]["proj_encoder.weight"], "bias": c["head_sd"]["proj_encoder.bias"]})
ctc = CTC(cfg["odim"], cfg["d_model"], 0.1)
ctc.load_state_dict({"ctc_lo.weight": c["head_sd"]["ctc.ctc_lo.weight"], "ctc_lo.bias": c["head_sd"]["ctc.ctc_lo.bias"]})
proj, enc, ctc = (m.to(dev).eval() for m in (proj, enc, ctc))
mask = CO.non_pad_mask(c["lengths"]).unsqueeze(1).to(dev)
res = {}
for prec in ("f16", "fp32"):
    for m in (proj, enc, ctc):
        m.precision = prec
    with torch.no_grad():
        hs, logp, best = features_to_log_probs(proj, enc, ctc, c["feats"].to(dev), mask, want_argmax=True)
    res[prec] = [hs.cpu(), logp.cpu(), best.cpu()]
""",
    "ctc_loss": """
from auto_avsr_b200 import CTC
from oracle import make_golden_ctc as M
c = M.CASES["ctc_loss_full"]
hs, w, b, hlens, ys = M.inputs("ctc_loss_full")
res = {}
for prec in ("f16", "fp32"):
    ctc = CTC(c["odim"], c["d_model"], 0.0)
    ctc.load_state_dict({"ctc_lo.weight": w, "ctc_lo.bias": b}, strict=True)
    ctc = ctc.to(dev).train()
    ctc.precision = prec
    x = hs.to(dev).clone().requires_grad_(True)
    loss, _ = ctc(x, hlens.to(dev), ys.to(dev))
    loss.backward()
    res[prec] = [loss.detach().cpu(), x.grad.cpu(), ctc.ctc_lo.weight.grad.cpu(), ctc.ctc_lo.bias.grad.cpu()]
""",
}


@pytest.mark.parametrize("part", sorted(PDL_BODIES))
def test_pdl_off_gives_the_same_bits(part, tmp_path):
    """Every kernel AVSR_LAUNCH starts carries programmatic dependent launch; with AVSR_B200_PDL=0 none does.  The
    switch is read once per process, so each setting runs in its own child; the two must agree bit for bit."""
    got = {}
    for setting in ("default", "0"):
        env = {k: v for k, v in os.environ.items() if k != "AVSR_B200_PDL"}
        if setting == "0":
            env["AVSR_B200_PDL"] = "0"
        path = str(tmp_path / f"{part}_{setting}.pt")
        run_child(PDL_BODIES[part] + f"""
torch.save(res, {path!r})
print("CHILD-OK")
""", env=env)
        got[setting] = torch.load(path)

    def flat(v):
        return [t for x in v for t in flat(x)] if isinstance(v, (list, tuple)) else [v]

    assert got["default"].keys() == got["0"].keys()
    for k in got["default"]:
        a, b = flat(got["default"][k]), flat(got["0"][k])
        assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b)), (part, k)
