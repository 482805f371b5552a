"""GPU parity of the front-ends' library training path (auto_avsr_b200/frontend_train.py, the training section of
csrc/frontend.cu): each conv unit at every trunk shape against torch autograd in float64, the whole front-end (both
modalities, ragged and zero-padded clips, odd frame sizes, a waveform that is not a multiple of 640) against the torch
modules in float64 on the CPU -- output, all 60 parameter gradients, the 40 running buffers and num_batches_tracked --,
determinism across steps and streams, and the refusals.

Each test runs in a child process (its own CUDA context).  Errors are relative: max |gpu - ref| / max |ref|, recorded
with tests/helpers.py record()."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

pytestmark = pytest.mark.gpu

PRELUDE = f"""
import copy, os, sys, math, torch
sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})
from helpers import record
from auto_avsr_b200.synthetic import frontend_state_dict
from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
from auto_avsr_b200 import frontend_train as FT
dev = torch.device("cuda:0")
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
# relative bounds, about 4x the largest errors observed on an H100 80GB HBM3
# (per unit: fp32 3.0e-6, tf32 / f16 6.7e-4; whole front-end: fp32 1.1e-5, tf32 / f16 7.5e-3, the video stem's
# gradients 5.1e-3 with the max-pool winners pinned)
TOL_UNIT = {{"fp32": 1.2e-5, "tf32": 2.7e-3, "f16": 2.7e-3}}
TOL_FE = {{"fp32": 5e-5, "tf32": 3e-2, "f16": 3e-2}}

def rel(a, b):
    b = b.double().cpu()
    return ((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()

def build(modality, seed=3):
    m = Conv3dResNet() if modality == "video" else Conv1dResNet()
    m.load_state_dict(frontend_state_dict(seed, modality), strict=True)
    return m.train()

def reference(modality, seed=3):
    from oracle.make_golden_frontend import reference_module
    m = reference_module(modality)
    m.load_state_dict(frontend_state_dict(seed, modality), strict=True)
    return m.train()

NBT0 = {{mod: frontend_state_dict(3, mod) for mod in ("video", "audio")}}     # the synthetic num_batches_tracked

def step(m, x, wts):
    out = m(x)
    loss = (out * wts).sum()
    loss.backward()
    grads = {{n: p.grad.detach().clone() for n, p in m.named_parameters()}}
    bufs = {{n: b.detach().clone() for n, b in m.named_buffers()}}
    m.zero_grad(set_to_none=True)
    return out.detach(), grads, bufs
"""


def run_child(body, timeout=1200):
    r = subprocess.run([sys.executable, "-c", PRELUDE + body], capture_output=True, text=True, timeout=timeout,
                       cwd=ROOT)
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize("prec", ["fp32", "tf32", "f16"])
def test_conv_unit_every_trunk_shape(prec):
    """conv -> BatchNorm(batch stats) -> [+ resid] -> [SiLU] against float64 autograd: output, batch mean / var through
    the running statistics, dW, d gamma, d beta, the input and residual gradients.  The 1-D cases of 129, 255 and 127
    output positions leave 1 and 127 rows in the last 128-row tile."""
    run_child(f"""
prec = {prec!r}
g = torch.Generator().manual_seed(5)
cases = []
for cin, cout, s, kh, kw, st in ((64, 64, 22, 3, 3, 1), (64, 128, 22, 3, 3, 2), (64, 128, 22, 1, 1, 2),
                                 (128, 128, 11, 3, 3, 1), (128, 256, 11, 3, 3, 2), (128, 256, 11, 1, 1, 2),
                                 (256, 256, 6, 3, 3, 1), (256, 512, 6, 3, 3, 2), (512, 512, 3, 3, 3, 1)):
    for N in (3, 7):
        cases.append(("video", N, s, s, cin, cout, kh, kw, st))
for cin, cout, L, st, k in ((64, 64, 160, 1, 3), (64, 128, 160, 2, 3), (64, 128, 160, 2, 1), (128, 128, 80, 1, 3),
                            (256, 512, 40, 2, 3), (512, 512, 20, 1, 3)):
    for N in (1, 5):
        cases.append(("audio", N, 1, L, cin, cout, 1, k, st))
for L, st in ((129, 1), (255, 1), (127, 1), (257, 2), (253, 2)):      # rows % 128 = 1, 127, 127, 1, 127
    cases.append(("audio", 1, 1, L, 64, 64, 1, 3, st))
worst = 0.0
for (mod, N, H, W, cin, cout, kh, kw, st) in cases:
    conv = (torch.nn.Conv2d(cin, cout, (kh, kw), st, ((kh - 1) // 2, (kw - 1) // 2), bias=False) if mod == "video"
            else torch.nn.Conv1d(cin, cout, kw, st, (kw - 1) // 2, bias=False))
    bn = torch.nn.BatchNorm2d(cout) if mod == "video" else torch.nn.BatchNorm1d(cout)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / math.sqrt(cin * kh * kw))
        bn.weight.copy_(1 + 0.2 * torch.randn(cout, generator=g)); bn.bias.copy_(0.2 * torch.randn(cout, generator=g))
        bn.running_mean.copy_(0.1 * torch.randn(cout, generator=g)); bn.running_var.copy_(1 + torch.rand(cout, generator=g))
    x = torch.randn(N, H, W, cin, generator=g) + 0.5
    spec = FT._Spec(0, N, 1, H, W, conv)
    res = torch.randn(N, spec.Ho, spec.Wo, cout, generator=g)
    dy = torch.randn(N, spec.Ho, spec.Wo, cout, generator=g)
    for act, use_res in ((True, False), (True, True), (False, False)):
        # float64 reference in torch's own layout
        c64, b64 = copy.deepcopy(conv).double(), copy.deepcopy(bn).double()
        xr = x.double().requires_grad_(True); rr = res.double().requires_grad_(True)
        xin = xr.permute(0, 3, 1, 2) if mod == "video" else xr[:, 0].permute(0, 2, 1)
        h = b64(c64(xin))
        h = h.permute(0, 2, 3, 1) if mod == "video" else h.permute(0, 2, 1)[:, None]
        if use_res: h = h + rr
        if act: h = torch.nn.functional.silu(h)
        h.backward(dy.double())
        # library
        cl, bl = copy.deepcopy(conv).to(dev), copy.deepcopy(bn).to(dev)
        xg = x.to(dev).requires_grad_(True); rg = res.to(dev).requires_grad_(True)
        y = FT.ConvBnActFn.apply(xg, rg if use_res else None, cl.weight, bl.weight, bl.bias, bl, spec, act, prec, None)
        y.backward(dy.to(dev))
        pairs = [("y", y, h), ("dx", xg.grad, xr.grad), ("dw", cl.weight.grad, c64.weight.grad),
                 ("dgamma", bl.weight.grad, b64.weight.grad), ("dbeta", bl.bias.grad, b64.bias.grad),
                 ("running_mean", bl.running_mean, b64.running_mean), ("running_var", bl.running_var, b64.running_var)]
        if use_res: pairs.append(("dres", rg.grad, rr.grad))
        assert int(bl.num_batches_tracked) == int(b64.num_batches_tracked) == 1
        for name, a, b in pairs:
            e = rel(a, b.detach())
            worst = max(worst, e)
            assert e < TOL_UNIT[prec], (mod, N, H, W, cin, cout, kh, kw, st, act, use_res, name, e)
record("conv_unit", prec, worst, TOL_UNIT[prec])
print("CHILD-OK")
""")


@pytest.mark.parametrize("prec", ["fp32", "tf32", "f16"])
def test_whole_frontend_vs_float64(prec):
    """One training step of each front-end against the reference modules in float64 on the CPU: video with 9 frames
    per utterance, 45x61 frames and all-zero padded frames (every max-pool window ties), video with 1 frame per
    utterance; audio with a waveform that is not a multiple of 640.  (Batches whose layer4 BatchNorm sees only a handful
    of positions per channel are left out: upstream error is amplified through the chain there; each unit on its own
    is checked at such batches in test_zz_gpu_frontend_train_stages.py.)  Output, the 60 parameter gradients, the 40
    running buffers and num_batches_tracked.  The float64 video chain's max-pool routes through the windows' winners
    the library recorded, whose float64 values must match float64 max_pool3d within the bound: with 11-bit operands
    a near-tie window can pick another winner than float64 does, and the stem's weight gradient (a sum with
    cancellation) would show the misrouted gradient, not the library's arithmetic."""
    run_child(f"""
from oracle.frontend_train_stages import pool_by_winner
prec = {prec!r}
g = torch.Generator().manual_seed(11)
cases = [("video", torch.randn(2, 9, 1, 45, 61, generator=g)), ("video", torch.randn(3, 1, 1, 88, 88, generator=g)),
         ("audio", torch.randn(2, 2 * 640 + 333, 1, generator=g))]
cases[0][1][1, 4:] = 0.0          # a zero-padded tail: constant stem output, every max-pool window ties
worst = worst_stem = worst_gap = 0.0
pool0 = FT.MaxPoolFn
class RecordWinners:
    @staticmethod
    def apply(x):
        y, idx = pool0.apply(x)
        winners.append(idx.cpu())
        return y, idx
for mod, x in cases:
    lib = build(mod).to(dev)
    lib.library_train, lib.precision = True, prec
    with torch.no_grad():
        out_shape = reference(mod).double()(x.double()).shape
    ref = reference(mod).double()
    wts = torch.randn(out_shape, generator=g)
    winners = []
    FT.MaxPoolFn = RecordWinners
    try:
        o, gl, bl = step(lib, x.to(dev), wts.to(dev))
    finally:
        FT.MaxPoolFn = pool0
    def pin(mod_, inp, out):
        pinned = pool_by_winner(inp[0], winners[0])
        # the library's winners hold a window maximum of the float64 stem output, up to the stem's own error
        gap.append(rel(pinned.detach(), out.detach()))
        return pinned
    gap = []
    for p in ref.modules():
        if isinstance(p, torch.nn.MaxPool3d):
            p.register_forward_hook(pin)
    o64, g64, b64 = step(ref, x.double(), wts.double())
    assert len(gl) == 60 and len([k for k in bl if not k.endswith("num_batches_tracked")]) == 40
    errs = {{"out": rel(o, o64)}}
    if gap:
        errs["pinned_pool_vs_max_pool3d"] = gap[0]
        worst_gap = max(worst_gap, gap[0])
    for k in g64: errs["grad." + k] = rel(gl[k], g64[k])
    for k in b64:
        if k.endswith("num_batches_tracked"):
            assert int(bl[k]) == int(b64[k]) == int(NBT0[mod][k]) + 1, k
        else:
            errs["buf." + k] = rel(bl[k], b64[k])
    print(mod, tuple(x.shape), sorted(errs.items(), key=lambda kv: -kv[1])[:5])
    name, e = max(errs.items(), key=lambda kv: kv[1])
    worst = max(worst, e)
    worst_stem = max([worst_stem] + [v for k, v in errs.items() if k.startswith("grad.frontend3D")])
    assert e < TOL_FE[prec], (mod, tuple(x.shape), name, e)
record("whole_frontend_train", prec, worst, TOL_FE[prec])
record("whole_frontend_train_video_stem_grads", prec, worst_stem, TOL_FE[prec])
record("whole_frontend_train_pinned_pool_vs_max_pool3d", prec, worst_gap, TOL_FE[prec])
print("CHILD-OK")
""")


def test_maxpool_ties_route_like_torch():
    """The recorded winner is torch's (first maximum in scan order): ties everywhere and a NaN, against
    torch.nn.functional.max_pool2d on the same GPU, forward and backward bit for bit."""
    run_child("""
g = torch.Generator().manual_seed(2)
x = torch.randn(3, 9, 13, 64, generator=g).round()        # many exact ties
x[1] = 0.25                                                # a constant frame: every window ties
x[2, 4, 5, 7] = float("nan")
x = x.to(dev)
dy = torch.randn(3, 5, 7, 64, generator=g).to(dev)
xr = x.clone().permute(0, 3, 1, 2).requires_grad_(True)
yr = torch.nn.functional.max_pool2d(xr, 3, 2, 1)
yr.backward(dy.permute(0, 3, 1, 2))
xl = x.clone().requires_grad_(True)
yl, _ = FT.MaxPoolFn.apply(xl)
yl.backward(dy)
assert torch.equal(yl.permute(0, 3, 1, 2).nan_to_num(7.0), yr.detach().nan_to_num(7.0))
assert torch.equal(xl.grad.permute(0, 3, 1, 2), xr.grad)
print("CHILD-OK")
""")


def test_deterministic_across_steps_and_streams():
    """Two identical steps, and one on a side stream, give bit-identical gradients and running statistics."""
    run_child("""
for mod, shape in (("video", (2, 5, 1, 40, 40)), ("audio", (2, 3 * 640, 1))):
    x = torch.randn(shape, generator=torch.Generator().manual_seed(4)).to(dev)
    res = []
    for side in (False, False, True):
        m = build(mod).to(dev)
        m.library_train, m.precision = True, "f16"
        wts = torch.ones(m(x).shape, device=dev)
        m = build(mod).to(dev)
        m.library_train, m.precision = True, "f16"
        if side:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                r = step(m, x, wts)
            torch.cuda.current_stream().wait_stream(s)
        else:
            r = step(m, x, wts)
        torch.cuda.synchronize()
        res.append(r)
    for r in res[1:]:
        assert torch.equal(r[0], res[0][0])
        for k in r[1]: assert torch.equal(r[1][k], res[0][1][k]), k
        for k in r[2]: assert torch.equal(r[2][k], res[0][2][k]), k
print("CHILD-OK")
""")


def test_no_grad_still_updates_running_statistics():
    """In train() under torch.no_grad() the batch statistics are used and the running statistics still move, as torch's."""
    run_child("""
x = torch.randn(2, 3, 1, 32, 32, generator=torch.Generator().manual_seed(8))
ref = build("video").double()
lib = build("video").to(dev)
lib.library_train, lib.precision = True, "fp32"
with torch.no_grad():
    o64 = ref(x.double()); o = lib(x.to(dev))
assert rel(o, o64) < 5e-5
for (k, a), (_, b) in zip(lib.named_buffers(), ref.named_buffers()):
    assert rel(a, b) < 5e-5 if a.is_floating_point() else int(a) == int(b) == int(NBT0["video"][k]) + 1, k
print("CHILD-OK")
""")


def test_momentum_none_is_cumulative_average():
    run_child("""
x1 = torch.randn(2, 2, 1, 24, 24, generator=torch.Generator().manual_seed(1))
x2 = torch.randn(2, 2, 1, 24, 24, generator=torch.Generator().manual_seed(2))
ref, lib = build("video").double(), build("video").to(dev)
for m in (ref, lib):
    for mod in m.modules():
        if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm): mod.momentum = None
lib.library_train, lib.precision = True, "fp32"
with torch.no_grad():
    for x in (x1, x2):
        ref(x.double()); lib(x.to(dev))
for (k, a), (_, b) in zip(lib.named_buffers(), ref.named_buffers()):
    assert rel(a, b) < 5e-5 if a.is_floating_point() else int(a) == int(b) == int(NBT0["video"][k]) + 2, k
print("CHILD-OK")
""")


def test_installed_e2e_train_step_then_eval_follows_new_statistics():
    """install_frontend(..., library_train=True) on a video front-end: the training step matches the torch path, and back
    in eval() the library forward follows the updated running statistics (the prepared-weights cache is refreshed)."""
    run_child("""
from auto_avsr_b200.install import install_frontend
class Holder(torch.nn.Module):
    def __init__(self):
        super().__init__(); self.frontend = build("video")
x = torch.randn(2, 4, 1, 32, 32, generator=torch.Generator().manual_seed(6)).to(dev)
h_ref, h_lib = Holder().to(dev), Holder().to(dev)
install_frontend(h_lib, library_train=True)
assert h_lib.frontend.library_train
h_lib.frontend.precision = h_ref.frontend.precision = "fp32"
wts = torch.randn(2, 4, 512, generator=torch.Generator().manual_seed(7)).to(dev)
torch.backends.cudnn.deterministic = True
o_ref, g_ref, b_ref = step(h_ref.frontend, x, wts)
o_lib, g_lib, b_lib = step(h_lib.frontend, x, wts)
assert rel(o_lib, o_ref) < 5e-5
for k in g_ref: assert rel(g_lib[k], g_ref[k]) < 5e-5, k
h_lib.eval(); h_ref.eval()
with torch.no_grad():
    e_lib = h_lib.frontend(x); e_ref = h_ref.frontend(x)       # both eval paths are the library's
assert rel(e_lib, e_ref) < 5e-5
print("CHILD-OK")
""")


def test_refusals_before_any_launch():
    run_child("""
from auto_avsr_b200._cabi import lib
m = build("video").to(dev)
m.library_train = True
x = torch.randn(1, 2, 1, 16, 16, device=dev)
def refused(fn):
    n0 = lib.avsr_launch_count()
    try:
        fn()
    except NotImplementedError:
        assert lib.avsr_launch_count() == n0
        return
    raise AssertionError("not refused")
refused(lambda: m(x.cpu()))
refused(lambda: m(x.clone().requires_grad_(True)))
m2 = build("video").to(dev); m2.library_train = True
m2.trunk.layer2[0].bn1.track_running_stats = False
m2.trunk.layer2[0].bn1.running_mean = None; m2.trunk.layer2[0].bn1.running_var = None
refused(lambda: m2(x))
m3 = build("audio").to(dev); m3.library_train = True
refused(lambda: m3(torch.randn(1, 2 * 640, 1)))
m4 = build("video").to(dev); m4.library_train = True
m4.trunk.relu_type = "prelu"
refused(lambda: m4(x))
# one value per channel in training: torch raises, so does the library (a 1x1 layer4 on one frame), before any launch
n0 = lib.avsr_launch_count()
try:
    m(torch.randn(1, 1, 1, 8, 8, device=dev))
    raise AssertionError("one value per channel was not refused")
except ValueError:
    pass
print("CHILD-OK")
""")


def test_eval_train_eval_refreshes_the_prepared_cache():
    """eval (prepares the library's weights), a library-train step (moves the running statistics), eval again: the
    second eval follows the new statistics, exactly as the torch-trained twin's does."""
    run_child("""
x = torch.randn(2, 4, 1, 40, 40, generator=torch.Generator().manual_seed(6)).to(dev)
a, b = build("video").to(dev), build("video").to(dev)
a.precision = b.precision = "fp32"
a.library_train = True
with torch.no_grad():
    e0 = a.eval()(x)
torch.backends.cudnn.deterministic = True
for m in (a, b):
    m.train()
    m(x).square().mean().backward()
    m.eval()
with torch.no_grad():
    ea, eb = a(x), b(x)
assert rel(ea, eb) < 5e-5 and rel(ea, e0) > 1e-3, (rel(ea, eb), rel(ea, e0))
print("CHILD-OK")
""")


def test_bucket_against_the_reference_module_on_the_gpu():
    """The max-frames buckets (video 4 x 400 frames of 88x88, audio 4 x 256,000 samples) in fp32 against the reference
    module on the same GPU in fp32 with cuDNN deterministic: every gradient and running buffer."""
    run_child("""
from auto_avsr_b200.synthetic import frontend_input
torch.backends.cudnn.deterministic = True
worst = 0.0
for mod, B, T in (("video", 4, 400), ("audio", 4, 256000)):
    x = frontend_input(mod, B, T).to(dev)
    ref, lib = reference(mod).to(dev), build(mod).to(dev)
    lib.library_train, lib.precision = True, "fp32"
    wts = torch.randn(B, T if mod == "video" else T // 640, 512, generator=torch.Generator().manual_seed(2)).to(dev)
    o_r, g_r, b_r = step(ref, x, wts)
    o_l, g_l, b_l = step(lib, x, wts)
    errs = {"out": rel(o_l, o_r)}
    errs.update({"grad." + k: rel(g_l[k], g_r[k]) for k in g_r})
    errs.update({"buf." + k: rel(b_l[k], b_r[k]) for k in b_r if b_r[k].is_floating_point()})
    assert all(int(b_l[k]) == int(b_r[k]) for k in b_r if not b_r[k].is_floating_point())
    name, e = max(errs.items(), key=lambda kv: kv[1])
    print(mod, name, e)
    worst = max(worst, e)
    assert e < 1e-3, (mod, name, e)     # two fp32 sums over up to 774 k pixels in different orders: observed 2.1e-4
    del ref, lib
    torch.cuda.empty_cache()
record("frontend_train_bucket", "fp32", worst, 1e-3)
print("CHILD-OK")
""")


def test_installed_e2e_loss_and_backward():
    """E2E(41, "video") with install(), install_head(), install_decoder() and install_frontend(library_train=True),
    dropout off, fp32: E2E.forward's loss and every gradient after backward() match the un-installed reference model."""
    run_child("""
os.environ["AVSR_B200_PRECISION"] = "fp32"
from oracle import build_ref
build_ref.import_reference_encoder()
from espnet.nets.pytorch_backend import e2e_asr_conformer as E
from auto_avsr_b200.synthetic import frontend_input
import auto_avsr_b200
torch.backends.cudnn.deterministic = True
torch.manual_seed(0)
ref = E.E2E(41, "video")
ref.frontend.load_state_dict(frontend_state_dict(41, "video"), strict=True)
auto_avsr_b200.install()
lib = E.E2E(41, "video")
lib.load_state_dict(ref.state_dict(), strict=True)
for model in (ref, lib):
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout): m.p = 0.0
    model.ctc.dropout_rate = 0.0
auto_avsr_b200.install_head(lib)
auto_avsr_b200.install_decoder(lib)
auto_avsr_b200.install_frontend(lib, library_train=True)
ref, lib = ref.to(dev).train(), lib.to(dev).train()
x = frontend_input("video", 2, 12, 88, 88, 9).to(dev)
lengths = torch.tensor([12, 9])
label = torch.tensor([[5, 7, 9, 11], [3, 4, -1, -1]]).to(dev)
lr = ref(x, lengths, label)[0]
lr.backward()
ll = lib(x, lengths, label)[0]
ll.backward()
el = abs(ll.item() - lr.item()) / abs(lr.item())
gr = dict(ref.named_parameters())
worst, wname = 0.0, None
gscale = max(q.grad.abs().max().item() for q in gr.values() if q.grad is not None)
for n, p in lib.named_parameters():
    # (the key biases' gradients are mathematically zero: the scale is floored at 1e-4 of the largest gradient)
    e = (p.grad.double().cpu() - gr[n].grad.double().cpu()).abs().max().item() / (gr[n].grad.abs().max().item() + 1e-4 * gscale)
    if e > worst: worst, wname = e, n
fe = max(rel(p.grad, gr["frontend." + n].grad) for n, p in lib.frontend.named_parameters())
print("loss", el, "worst grad", wname, worst, "worst frontend grad", fe)
# observed on an H100: loss 0, every gradient 3.7e-2 (the encoder's fp32 backward against torch's, scale floored), the
# front-end's gradients 2.2e-3
record("frontend_train_e2e", "fp32", [el, worst, fe], [1e-4, 1.5e-1, 9e-3])
assert el < 1e-4 and worst < 1.5e-1 and fe < 9e-3, (el, wname, worst, fe)
print("CHILD-OK")
""")


SYNC_WORKER = r"""
import os, sys, torch
sys.path.insert(0, ROOT)
import torch.distributed as dist
from auto_avsr_b200.synthetic import frontend_state_dict
from auto_avsr_b200.espnet_dropin.resnet import Conv3dResNet
rank, world = int(sys.argv[1]), 2
dist.init_process_group("gloo", init_method="file://" + sys.argv[2], rank=rank, world_size=world)
dev = torch.device("cuda:0")
torch.backends.cudnn.allow_tf32 = False
x = torch.randn(4, 5, 1, 40, 40, generator=torch.Generator().manual_seed(9)).to(dev)
wts = torch.randn(4, 5, 512, generator=torch.Generator().manual_seed(10)).to(dev)
m = Conv3dResNet(); m.load_state_dict(frontend_state_dict(3, "video"))
m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m).to(dev).train()
m.library_train, m.precision = True, "fp32"
half = slice(2 * rank, 2 * rank + 2)
(m(x[half]) * wts[half]).sum().backward()
grads = {n: p.grad.detach().cpu() for n, p in m.named_parameters()}
bufs = {n: b.detach().cpu() for n, b in m.named_buffers()}
torch.save((grads, bufs), sys.argv[3] + f".rank{rank}")
dist.barrier()
if rank == 0:
    whole = Conv3dResNet(); whole.load_state_dict(frontend_state_dict(3, "video"))
    whole = whole.to(dev).train()
    whole.library_train, whole.precision = True, "fp32"
    (whole(x) * wts).sum().backward()
    torch.save(({n: p.grad.detach().cpu() for n, p in whole.named_parameters()},
                {n: b.detach().cpu() for n, b in whole.named_buffers()}), sys.argv[3] + ".whole")
dist.destroy_process_group()
print("WORKER-OK", rank)
"""


def test_sync_batchnorm_two_processes():
    """SyncBatchNorm over two gloo processes on one GPU, half the batch each, loss a fixed weighted sum of the outputs:
    the running statistics equal those of one process with the whole batch, and the two ranks' parameter gradients
    sum to the whole-batch gradients.  Both processes are waited for (and killed on a timeout)."""
    import tempfile
    import torch
    with tempfile.TemporaryDirectory() as tmp:
        store, out = os.path.join(tmp, "store"), os.path.join(tmp, "res")
        code = f"ROOT = {ROOT!r}\n" + SYNC_WORKER
        procs = [subprocess.Popen([sys.executable, "-c", code, str(r), store, out], cwd=ROOT, stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True) for r in range(2)]
        logs = []
        try:
            for p in procs:
                logs.append(p.communicate(timeout=600)[0])
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                    p.wait()
        assert all(p.returncode == 0 for p in procs), "\n".join(l[-2000:] for l in logs)
        (g0, b0), (g1, b1) = torch.load(out + ".rank0"), torch.load(out + ".rank1")
        gw, bw = torch.load(out + ".whole")
    worst = 0.0
    for k in gw:
        s = g0[k].double() + g1[k].double()
        worst = max(worst, ((s - gw[k].double()).abs().max() / gw[k].double().abs().max()).item())
    for k in bw:
        if bw[k].is_floating_point():
            for b in (b0, b1):
                worst = max(worst, ((b[k].double() - bw[k].double()).abs().max() / bw[k].double().abs().max()).item())
        else:
            assert int(b0[k]) == int(b1[k]) == int(bw[k]), k
    print("sync batchnorm worst relative difference", worst)
    assert worst < 5e-5, worst
