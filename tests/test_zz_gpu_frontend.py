"""GPU parity of the ResNet front-ends (csrc/frontend.cu): the per-op conv + BatchNorm [+ residual] + SiLU at every trunk
shape of both modalities, the whole front-end against the golden float64 outputs of the reference modules
(tests/golden/frontend_*.npz), the max-frames bucket against the reference module on the same GPU, the installed E2E
inference path, and determinism across calls and streams.

Each test runs in a child process (its own CUDA context).  Errors are relative: max |gpu - ref| / max |ref|.  The bounds
are about 4x the errors observed on the GPU (tests/helpers.py record())."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

pytestmark = pytest.mark.gpu

PRELUDE = f"""
import os, sys, math, torch
import numpy as np
sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})
from helpers import record
from auto_avsr_b200.frontend import conv_bn_act
from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
dev = torch.device("cuda:0")
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
# relative max error bounds, about 4x the largest observed on an H100 80GB HBM3: per-op conv (fp32 2.2e-6, tf32 / f16
# 6.1e-4: both round operands to a 10-bit mantissa),
# whole front-end vs the golden fp64 outputs (fp32 1.2e-6, tf32 8.3e-4, f16 6.5e-4), max-frames bucket vs the
# reference module in fp32 on the same GPU (fp32 1.6e-6, f16 7.3e-4)
TOL_OP = {{"fp32": 8e-6, "tf32": 2.5e-3, "f16": 2.5e-3}}
TOL_FE = {{"fp32": 5e-6, "tf32": 3.5e-3, "f16": 3.5e-3}}
TOL_BUCKET = {{"fp32": 7e-6, "f16": 3e-3}}

def rel(a, b):
    b = b.double().cpu()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()

def dropin(modality, sd):
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
    m = Conv3dResNet() if modality == "video" else Conv1dResNet()
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()
"""


def run_child(body, timeout=900):
    r = subprocess.run([sys.executable, "-c", PRELUDE + body], capture_output=True, text=True, timeout=timeout,
                       cwd=ROOT)
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, r.stdout[-2500:] + r.stderr[-2500:]


@pytest.mark.parametrize("prec", ["fp32", "tf32", "f16"])
def test_conv_bn_act_every_trunk_shape(prec):
    run_child(f"""
g = torch.Generator().manual_seed(1)
# (C_in, C_out, spatial size, KH, KW, stride): 3x3 s1 / s2 and 1x1 s2 at 22/11/6/3 px, 1-D at 160/80/40/20
video = [(c, c, s, 3, 3, 1) for c, s in ((64, 22), (128, 11), (256, 6), (512, 3))]
video += [(c, 2 * c, s, 3, 3, 2) for c, s in ((64, 22), (128, 11), (256, 6))]
video += [(c, 2 * c, s, 1, 1, 2) for c, s in ((64, 22), (128, 11), (256, 6))]
audio = [(c, c, s, 1, 3, 1) for c, s in ((64, 160), (128, 80), (256, 40), (512, 20))]
audio += [(c, 2 * c, s, 1, 3, 2) for c, s in ((64, 160), (128, 80), (256, 40))]
audio += [(c, 2 * c, s, 1, 1, 2) for c, s in ((64, 160), (128, 80), (256, 40))]
worst = (0.0, None)
for kind, shapes in (("video", video), ("audio", audio)):
    for cin, cout, s, kh, kw, stride in shapes:
        N = 5 if kind == "video" else 3
        H, W = (s, s) if kind == "video" else (1, s)
        x = torch.randn(N, H, W, cin, generator=g)
        w = torch.randn(cout, cin, kh, kw, generator=g) * math.sqrt(2.0 / (cin * kh * kw))
        scale = torch.rand(cout, generator=g) + 0.5
        shift = torch.randn(cout, generator=g) * 0.1
        ref = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), stride=stride,
                                         padding=((kh - 1) // 2, (kw - 1) // 2)).permute(0, 2, 3, 1)
        ref = ref * scale.double() + shift.double()
        for use_res, act in ((False, True), (True, True), (False, False)):
            res = torch.randn(ref.shape, generator=g) if use_res else None
            r = ref + res.double() if use_res else ref
            if act:
                r = r * torch.sigmoid(r)
            y = conv_bn_act(x.to(dev), w.to(dev), scale.to(dev), shift.to(dev), stride,
                            None if res is None else res.to(dev), act, {prec!r})
            assert y.shape == r.shape, (y.shape, r.shape)
            e = rel(y, r)
            if e > worst[0]:
                worst = (e, (kind, cin, cout, s, kh, kw, stride, use_res, act))
record("frontend_conv_op", ({prec!r},) + worst[1], worst[0], TOL_OP[{prec!r}])
assert worst[0] < TOL_OP[{prec!r}], worst
print("CHILD-OK")
""")


@pytest.mark.parametrize("prec", ["fp32", "tf32", "f16"])
@pytest.mark.parametrize("name", ["frontend_video_88", "frontend_video_t1", "frontend_video_45x61", "frontend_audio_ragged"])
def test_frontend_matches_golden(name, prec):
    run_child(f"""
z = np.load(os.path.join({HERE!r}, "golden", {name!r} + ".npz"))
modality = str(z["modality"])
B, T, H, W = (int(v) for v in z["shape"])
m = dropin(modality, frontend_state_dict(int(z["wseed"]), modality))
m.precision = {prec!r}
x = frontend_input(modality, B, T, H, W, int(z["xseed"])).to(dev)
with torch.no_grad():
    y = m(x)
ref = torch.from_numpy(z["out_f64"])
assert y.shape == ref.shape, (y.shape, ref.shape)
e = rel(y, ref)
record("frontend_golden", ({name!r}, {prec!r}), e, TOL_FE[{prec!r}])
assert torch.isfinite(y).all() and e < TOL_FE[{prec!r}], e
print("CHILD-OK")
""")


@pytest.mark.parametrize("modality", ["video", "audio"])
def test_max_frames_bucket_against_reference_on_gpu(modality):
    run_child(f"""
from oracle.make_golden_frontend import reference_module
sd = frontend_state_dict(31, {modality!r})
ref = reference_module({modality!r})
ref.load_state_dict(sd, strict=True)
ref = ref.to(dev).eval()
m = dropin({modality!r}, sd)
x = (frontend_input("video", 4, 400, 88, 88, 5) if {modality!r} == "video" else frontend_input("audio", 4, 256000, seed=5)).to(dev)
with torch.no_grad():
    r = ref(x)
    for prec in ("f16", "fp32"):
        m.precision = prec
        y = m(x)
        assert y.shape == r.shape and torch.isfinite(y).all(), prec
        e = rel(y, r)
        bound = TOL_BUCKET[prec]
        record("frontend_max_frames", ({modality!r}, prec), e, bound)
        assert e < bound, (prec, e)
print("CHILD-OK")
""")


def test_installed_e2e_inference_path_and_running_statistics():
    """E2E(odim, "video") with install() + install_head() + install_decoder() + install_frontend(), fp32: the
    frontend -> proj_encoder -> encoder path matches the un-installed reference model; a training step of the front-end
    updates the running statistics as in the reference; back in eval the output follows the new statistics."""
    run_child("""
os.environ["AVSR_B200_PRECISION"] = "fp32"
from oracle import build_ref
build_ref.import_reference_encoder()
from espnet.nets.pytorch_backend import e2e_asr_conformer as E
from espnet.nets.pytorch_backend.nets_utils import make_non_pad_mask
import auto_avsr_b200
torch.manual_seed(0)
ref = E.E2E(41, "video")
ref.frontend.load_state_dict(frontend_state_dict(41, "video"), strict=True)
auto_avsr_b200.install()
lib = E.E2E(41, "video")
lib.load_state_dict(ref.state_dict(), strict=True)
for f in (auto_avsr_b200.install_head, auto_avsr_b200.install_decoder, auto_avsr_b200.install_frontend):
    f(lib)
assert type(lib.frontend).__module__ == "auto_avsr_b200.espnet_dropin.resnet"
ref, lib = ref.to(dev).eval(), lib.to(dev).eval()
lengths = torch.tensor([7, 5])
x = frontend_input("video", 2, 7, 88, 88, 9).to(dev)
mask = make_non_pad_mask(lengths).to(dev).unsqueeze(-2)

def path(model):
    with torch.no_grad():
        f = model.frontend(x)
        h, _ = model.encoder(model.proj_encoder(f), mask)
    return f, h

fr, hr = path(ref)
fl, hl = path(lib)
ef, eh = rel(fl, fr), rel(hl[0, :7], hr[0, :7])
record("frontend_e2e_path", ("fp32",), [ef, eh], [5e-6, 5e-6])     # observed 1.2e-6, 1.1e-6
assert ef < 5e-6 and eh < 5e-6, (ef, eh)
torch.backends.cudnn.deterministic = True
for model in (ref, lib):
    model.frontend.train()
    model.frontend(x).square().mean().backward()
    model.frontend.eval()
for (k, a), (_, b) in zip(ref.frontend.named_buffers(), lib.frontend.named_buffers()):
    assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), k
with torch.no_grad():
    fr2, fl2 = ref.frontend(x), lib.frontend(x)
e2 = rel(fl2, fr2)
record("frontend_e2e_after_update", ("fp32",), e2, 5e-6)
assert e2 < 5e-6 and rel(fl2, fl) > 1e-3, (e2, rel(fl2, fl))
print("CHILD-OK")
""")


def test_repeatable_and_stream_independent():
    run_child("""
for modality, shape in (("video", (2, 5, 88, 88)), ("audio", (2, 640 * 7 + 3, 1, 1))):
    B, T, H, W = shape
    m = dropin(modality, frontend_state_dict(3, modality))
    x = frontend_input(modality, B, T, H, W, 4).to(dev)
    for prec in ("f16", "tf32", "fp32"):
        m.precision = prec
        with torch.no_grad():
            a = m(x).clone()
            b = m(x).clone()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                c = m(x)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
        assert torch.equal(a, b) and torch.equal(a, c), (modality, prec)
print("CHILD-OK")
""")
