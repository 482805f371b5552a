"""GPU parity of the CTC loss of the head (csrc/ctc_loss.cu; CTC.forward, ctc.py:41-65): against the fixtures generated
from the reference's own CTC module in float64 (tests/golden/ctc_loss_*.npz), against torch's ctc_loss in float64 on the
same GPU, bitwise repeatability, no host synchronisation, the no-grad (validation) path, and the reference E2E.forward
with install() + install_head().

Each test runs in a child process (its own CUDA context).  The bounds are about 4x the errors observed on the H100
(tests/helpers.py record())."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(ROOT, "oracle", "_ref")

pytestmark = pytest.mark.gpu

PRELUDE = f"""
import sys, math, numpy as np, torch
sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {HERE!r})
from helpers import err_stats, record
from auto_avsr_b200 import CTC
from auto_avsr_b200.train import CtcLossFn
from oracle import make_golden_ctc as M
dev = torch.device("cuda:0")

def head(name, prec, reduce=True, p=0.0):
    c = M.CASES[name]
    hs, w, b, hlens, ys = M.inputs(name)
    ctc = CTC(c["odim"], c["d_model"], p, reduce=reduce)
    ctc.load_state_dict({{"ctc_lo.weight": w, "ctc_lo.bias": b}}, strict=True)
    ctc = ctc.to(dev).train()
    ctc.precision = prec
    return ctc, hs.to(dev), hlens.to(dev), ys.to(dev)

def run(ctc, hs, hlens, ys):
    x = hs.clone().requires_grad_(True)
    ctc.ctc_lo.weight.grad = ctc.ctc_lo.bias.grad = None
    loss, ys_hat = ctc(x, hlens, ys)
    loss.backward()
    return loss.detach(), ys_hat, x.grad, ctc.ctc_lo.weight.grad, ctc.ctc_lo.bias.grad

def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()
"""


def run_child(body, timeout=900):
    r = subprocess.run([sys.executable, "-c", PRELUDE + body], capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2500:]


# relative max-abs error bounds (error / max |reference|) per precision: loss, d hs_pad, d weight / bias
TOL = {"fp32": (1e-6, 1e-4, 1e-4), "tf32": (2e-4, 1.4e-2, 5e-3), "f16": (4e-5, 6e-3, 4e-3)}


@pytest.mark.parametrize("prec", ["fp32", "tf32", "f16"])
@pytest.mark.parametrize("name", ["ctc_loss_tiny", "ctc_loss_full"])
def test_ctc_forward_backward_match_reference_golden(name, prec):
    tl, th, tw = TOL[prec]
    run_child(f"""
z = np.load(M.GOLDEN + "/" + {name!r} + ".npz")
ctc, hs, hlens, ys = head({name!r}, {prec!r})
loss, ys_hat, dh, dw, db = run(ctc, hs, hlens, ys)
assert tuple(ys_hat.shape) == tuple(z["ys_hat_shape"]) and loss.dim() == 0
e_loss = rel(loss, z["loss_sum"])
if "d_hs" in z.files:
    e_h = rel(dh, z["d_hs"])
else:
    e_h = rel(dh[:, ::int(z["d_hs__step"])], z["d_hs__frames"])
    cs = z["d_hs__checksum"]; g = dh.double().cpu()
    assert abs(g.sum().item() - cs[0]) <= 1e-2 * cs[1] and abs(g.abs().sum().item() - cs[1]) <= 1e-2 * cs[1]
if "d_weight" in z.files:
    e_w = rel(dw, z["d_weight"])
else:
    e_w = rel(dw[::int(z["d_weight__step"])], z["d_weight__rows"])
    cs = z["d_weight__checksum"]; g = dw.double().cpu()
    assert abs(g.abs().sum().item() - cs[1]) <= 1e-2 * cs[1] and abs((g * g).sum().item() - cs[2]) <= 2e-2 * cs[2]
e_b = rel(db, z["d_bias"])
ctc2, *_ = head({name!r}, {prec!r}, reduce=False)
ln, _ = ctc2(hs, hlens, ys)
e_none = rel(ln.detach(), z["loss_none"])
assert ln.shape == (hs.size(0),) and float(ln[2] if {name!r} == "ctc_loss_tiny" else 0) == 0.0
record("ctc_golden", ({name!r}, {prec!r}), [e_loss, e_none, e_h, e_w, e_b], [{tl}, {tl}, {th}, {tw}, {tw}])
assert e_loss < {tl} and e_none < {tl}, (e_loss, e_none)
assert e_h < {th} and e_w < {tw} and e_b < {tw}, (e_h, e_w, e_b)
print("CHILD-OK")
""")


def test_ctc_loss_fn_matches_torch_fp64_on_gpu():
    run_child("""
g = torch.Generator().manual_seed(3)
cases = [  # (hlens, label rows, odim, ld)
    ([12, 5, 7, 1, 0, 0], [[3, 3, -1, 5, 5, 5, 2, -1], [4, 4, 4, 4, -1, -1, -1, -1], [-1] * 8, [7] + [-1] * 7,
                           [1, 2, 3] + [-1] * 5, [-1] * 8], 9, 16),
    ([1], [[2]], 5, 8),
    ([40, 33, 20], None, 37, 40),
    ([400, 371, 300, 255], None, 5049, 5056),
]
worst_l, worst_g = 0.0, 0.0
for hl, rows, odim, ld in cases:
    B, T = len(hl), max(max(hl), 1)
    if rows is None:
        L = max(hl) // 4
        ys = torch.randint(1, odim, (B, L), generator=g)
        ys[torch.rand(B, L, generator=g) < 0.1] = -1
    else:
        ys = torch.tensor(rows)
    x = (torch.randn(B, T, ld, generator=g) * 2).to(dev)
    hlens = torch.tensor(hl, device=dev)
    dn = (torch.rand(B, generator=g) + 0.5).to(dev)
    xa = x.clone().requires_grad_(True)
    nll = CtcLossFn.apply(xa, hlens, ys.to(dev), odim, -1)
    (nll * dn).sum().backward()
    xr = x.double().clone().requires_grad_(True)
    lp = torch.log_softmax(xr[..., :odim], -1).transpose(0, 1)
    tg = [y[y != -1] for y in ys]
    flat = torch.cat(tg).to(dev)
    ref = torch.nn.functional.ctc_loss(lp, flat, hlens.long(), torch.tensor([len(t) for t in tg], device=dev),
                                       reduction="none", zero_infinity=True)
    (ref * dn.double()).sum().backward()
    el = ((nll.double() - ref).abs() / ref.abs().clamp_min(1.0)).max().item()
    eg = (xa.grad.double() - xr.grad).abs().max().item()
    assert (xa.grad[..., odim:] == 0).all()
    worst_l, worst_g = max(worst_l, el), max(worst_g, eg)
record("ctc_fn_vs_torch_fp64", "edge+random", [worst_l, worst_g], [2.5e-6, 1e-4])
assert worst_l < 2.5e-6 and worst_g < 1e-4, (worst_l, worst_g)
print("CHILD-OK")
""")


def test_ctc_loss_is_bitwise_repeatable_and_needs_no_host_sync():
    run_child("""
for prec in ("fp32", "f16"):
    ctc, hs, hlens, ys = head("ctc_loss_full", prec)
    a = run(ctc, hs, hlens, ys)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    b = run(ctc, hs, hlens, ys)
    torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    for u, v in zip(a, b):
        assert torch.equal(u, v), prec
print("CHILD-OK")
""")


def test_no_grad_and_eval_loss_equal_train_loss():
    run_child("""
for name in ("ctc_loss_tiny", "ctc_loss_full"):
    ctc, hs, hlens, ys = head(name, "f16")
    loss_train = run(ctc, hs, hlens, ys)[0]
    with torch.no_grad():
        loss_ng, ys_hat = ctc(hs, hlens, ys)
    ctc.eval()
    with torch.no_grad():
        loss_eval, _ = ctc(hs, hlens, ys)
    assert not loss_ng.requires_grad and ys_hat.shape == (hs.size(1), hs.size(0), ctc.ctc_lo.out_features)
    assert torch.equal(loss_ng, loss_train) and torch.equal(loss_eval, loss_train), (loss_ng, loss_eval, loss_train)
    assert ctc.loss is loss_eval
print("CHILD-OK")
""")


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "espnet")), reason="oracle/_ref not built")
def test_e2e_forward_backward_with_install_head_matches_reference():
    run_child(f"""
sys.path.insert(0, {REF!r})
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
from espnet.nets.pytorch_backend.e2e_asr_conformer import E2E
import auto_avsr_b200
odim = 41
torch.manual_seed(0)
ref = E2E(odim, "audio")                   # built before install(): the reference encoder
auto_avsr_b200.install()
ours = E2E(odim, "audio")
ours.load_state_dict(ref.state_dict(), strict=True)
auto_avsr_b200.install_head(ours)
assert type(ours.encoder).__module__.startswith("auto_avsr_b200") and type(ref.encoder).__module__.startswith("espnet")
for m in (ref, ours):
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
ref = ref.double().to(dev).train()
ours = ours.to(dev).train()
for mod in (ours.encoder, ours.proj_encoder, ours.ctc):
    mod.precision = "fp32"
g = torch.Generator().manual_seed(5)
lengths = torch.tensor([64, 47]) * 640
x = torch.randn(2, int(lengths.max()), 1, generator=g)
label = torch.randint(1, odim - 1, (2, 9), generator=g)
label[1, 6:] = -1
outs = {{}}
for tag, m, dt in (("ref", ref, torch.float64), ("ours", ours, torch.float32)):
    loss, loss_ctc, loss_att, acc = m(x.to(dev, dt), lengths.to(dev), label.to(dev))
    loss.backward()
    p = dict(m.named_parameters())
    outs[tag] = dict(loss=loss.detach(), loss_ctc=loss_ctc.detach(),
                     **{{k: p[k].grad for k in ("proj_encoder.weight", "proj_encoder.bias", "ctc.ctc_lo.weight",
                                              "ctc.ctc_lo.bias", "encoder.after_norm.weight", "encoder.after_norm.bias",
                                              "frontend.trunk.conv1.weight")}})
errs = {{k: rel(outs["ours"][k], outs["ref"][k]) for k in outs["ref"]}}
record("e2e_install_head_vs_ref_fp64", "fp32", errs, 2e-3)
for k, e in errs.items():
    assert e < 2e-3, (k, e, errs)
print("CHILD-OK")
""", timeout=1500)
