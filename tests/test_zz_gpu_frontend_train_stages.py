"""Each conv unit of the front-ends' library training path on its own inputs, against float64
(oracle/frontend_train_stages.py).

One library training step of a whole front-end runs with ``FT._unit``, ``FT.MaxPoolFn`` and ``FT.MeanRowsFn`` wrapped:
every unit's input, residual, geometry, output, pre-step running buffers and the gradient that reaches its output
(a tensor hook: for a BasicBlock output used twice, the sum autograd builds) are recorded.  Then, unit by unit:

- the capture is faithful: ``ConvBnActFn`` re-run alone on the recorded inputs and gradient, with a fresh copy of the
  BatchNorm, gives the chained step's output, dW, d gamma, d beta and running buffers bit for bit;
- the re-run's output, dx, d residual, dW, d gamma, d beta, running buffers and num_batches_tracked against the same
  inputs promoted to float64 (a bound covers one unit's rounding, and names the unit that fails).  The video stem gets
  the max-pool backward's result as its gradient, so the max-pool's winner choice is out of its comparison;
- negative controls: the float64 unit with one plausible kernel defect (``DEFECTS``) must miss the library by at
  least 2x the bound at every unit where the defect applies, except the BatchNorm-variance defects at BatchNorms over
  many positions (``WEAK_ABOVE``), which are recorded;
- torch's own fp32 unit with cuDNN TF32 on the same inputs (the reference implementation's training arithmetic),
  recorded next to the library's error, not asserted (cuDNN's choice of algorithm varies).

The max-pool and the final means are checked exactly: the pooled value is the recorded winner's, the backward equals a
float32 restatement of the fixed-order sum over the windows that named a pixel, and the means' backward is dout / P.

Each test runs in a child process.  Errors are relative, max |gpu - ref| / max |ref|, recorded with
tests/helpers.py record() under case / precision / modality / unit / quantity."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

pytestmark = pytest.mark.gpu

CHILD = r"""
import copy, sys, time, torch
sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
import torch.nn.functional as F
from helpers import record
from auto_avsr_b200._cabi import lib
from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
from auto_avsr_b200 import frontend_train as FT
from oracle import frontend_train_stages as S

dev = torch.device("cuda:0")
torch.backends.cuda.matmul.allow_tf32 = False
Q = ("y", "dx", "dres", "dw", "dgamma", "dbeta", "running_mean", "running_var")
# Relative bounds per quantity, about 4x the largest errors observed on an H100 80GB HBM3 (700 W), in two regimes.
# A BatchNorm that normalises few positions cancels strongly in its backward: "few" (<= 32 positions per channel, the
# 1x1 layer 4 of 5 to 32 frames) observed fp32 y 3.1e-6, dx 2.1e-6, dres 1.1e-6, dw 4.9e-6, d gamma 1.7e-6,
# d beta 1.3e-6, running mean / var 3.7e-7 / 2.3e-7; tf32 and f16 2.2e-3, 1.4e-3, 5.6e-4, 3.1e-3, 1.1e-3, 1.3e-3,
# 2.2e-4 / 1.2e-4.  Every other unit, buckets included: fp32 2.0e-6, 2.5e-6, 1.9e-6, 1.2e-6, 1.7e-6, 1.9e-6,
# 3.1e-7 / 2.0e-7; tf32 and f16 6.8e-4, 7.4e-4, 7.7e-4, 9.2e-4, 8.2e-4, 7.4e-4, 2.9e-4 / 8.2e-5.
FEW = 32
TOL = {
    ("fp32", "few"): dict(y=1.2e-5, dx=8.5e-6, dres=4.5e-6, dw=2e-5, dgamma=7e-6, dbeta=5.2e-6, running_mean=1.5e-6,
                          running_var=9.5e-7),
    ("fp32", "many"): dict(y=8e-6, dx=1e-5, dres=7.5e-6, dw=5e-6, dgamma=7e-6, dbeta=7.5e-6, running_mean=1.3e-6,
                           running_var=8e-7),
    ("tf32", "few"): dict(y=9e-3, dx=5.5e-3, dres=2.3e-3, dw=1.2e-2, dgamma=4.5e-3, dbeta=5e-3, running_mean=9e-4,
                          running_var=4.6e-4),
    ("tf32", "many"): dict(y=2.8e-3, dx=3e-3, dres=3.1e-3, dw=3.7e-3, dgamma=3.3e-3, dbeta=3e-3, running_mean=1.2e-3,
                           running_var=3.3e-4),
}
for k in ("few", "many"):
    TOL[("f16", k)] = TOL[("tf32", k)]      # the backward is the same TF32 code in both
# A negative control must miss the library by CONTROL_MARGIN x the bound at every unit it applies to, with one
# exception: the two BatchNorm-variance defects at a BatchNorm over more than WEAK_ABOVE[(defect, fp32 or tensor-core)]
# positions.  They move dz, d gamma and running_var by about 1 / positions (the factor n / (n - 1) between the biased
# and the unbiased variance), which a relative bound cannot resolve once 1 / positions falls below it.  Those are
# recorded with their margins, not asserted.  On an H100 every unit at or below these counts misses by >= 2.5x; the
# first weak ones: the unbiased backward at 80 positions (1.9x, tf32 / f16) and 81,312 (1.3x, fp32), running_var at
# 57 positions (0.56x, tf32 / f16) and 81,312 (2.0x, fp32).
CONTROL_MARGIN = 2.0
WEAK_ABOVE = {("bn_bwd_unbiased_var", "fp32"): 32768, ("running_var_biased", "fp32"): 32768,
              ("bn_bwd_unbiased_var", "tc"): 64, ("running_var_biased", "tc"): 40}
FAILS = []

def splits_of(g):
    Kw = -(-g.K // S.WG_T) * S.WG_T
    return (lib.avsr_frontend_train_wgrad_workspace_bytes(*g.args()) - 256) // (g.Cout * Kw * 4)

def capture_step(m, x, wts, prec):
    geoms = S.units(CASE)
    names = {id(conv): g.name for (conv, _), g in zip(m.conv_bn_pairs(), geoms)}
    rec, pool, mean = {}, {}, {}
    unit0, pool0, mean0 = FT._unit, FT.MaxPoolFn, FT.MeanRowsFn

    def unit(x, resid, pair, spec, act, precision):
        conv, bn = pair
        e = dict(x=x.detach(), resid=None if resid is None else resid.detach(), spec=spec, act=act, pair=pair,
                 rm=bn.running_mean.clone(), rv=bn.running_var.clone(), nbt=int(bn.num_batches_tracked))
        y = unit0(x, resid, pair, spec, act, precision)
        e["y"] = y.detach()
        y.register_hook(lambda gr, e=e: e.__setitem__("dy", gr.detach().clone()))
        rec[names[id(conv)]] = e
        return y

    class Pool:
        @staticmethod
        def apply(x):
            y, idx = pool0.apply(x)
            pool.update(x=x.detach(), y=y.detach(), idx=idx)
            y.register_hook(lambda gr: pool.__setitem__("dy", gr.detach().clone()))
            return y, idx

    class Mean:
        @staticmethod
        def apply(x, G, P):
            out = mean0.apply(x, G, P)
            mean.update(G=G, P=P)
            out.register_hook(lambda gr: mean.__setitem__("dout", gr.detach().clone()))
            return out

    FT._unit, FT.MaxPoolFn, FT.MeanRowsFn = unit, Pool, Mean
    try:
        (m(x) * wts).sum().backward()
    finally:
        FT._unit, FT.MaxPoolFn, FT.MeanRowsFn = unit0, pool0, mean0
    torch.cuda.synchronize()
    return geoms, rec, pool, mean

def check_pool_and_mean(geoms, rec, pool, mean):
    # forward: the recorded winner's value, and a maximum of its window
    sx = pool["x"]
    N, H, W, C = sx.shape
    win = S.pool_by_winner(sx.permute(3, 0, 1, 2)[None], pool["idx"])       # the N frames as one clip
    assert torch.equal(win[0].permute(1, 2, 3, 0), pool["y"])
    assert torch.equal(F.max_pool2d(sx.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1), pool["y"])
    # backward: in the kernel's order, windows (oy, ox) = (iy // 2 - 1 + a, ix // 2 - 1 + b), a then b
    Ho, Wo = pool["y"].shape[1:3]
    dy, idx = pool["dy"], pool["idx"].long()
    iy = torch.arange(H, device=dev)[:, None]
    ix = torch.arange(W, device=dev)[None, :]
    s = torch.zeros_like(sx)
    for a in range(3):
        for b in range(3):
            oy, ox = iy // 2 - 1 + a, ix // 2 - 1 + b
            ky, kx = iy - (2 * oy - 1), ix - (2 * ox - 1)
            ok = (oy >= 0) & (oy < Ho) & (ky >= 0) & (ky <= 2) & (ox >= 0) & (ox < Wo) & (kx >= 0) & (kx <= 2)
            oyc, oxc = oy.clamp(0, Ho - 1).expand(H, W), ox.clamp(0, Wo - 1).expand(H, W)
            sel = (idx[:, oyc, oxc] == (ky * 3 + kx).expand(H, W)[None, :, :, None]) & ok[None, :, :, None]
            s = s + torch.where(sel, dy[:, oyc, oxc], torch.zeros((), device=dev))
    assert torch.equal(s, rec["stem"]["dy"]), (s - rec["stem"]["dy"]).abs().max()
    # the means' backward: a broadcast of dout / P
    G, P = mean["G"], mean["P"]
    last = rec[geoms[-1].name]["dy"]
    dout = mean["dout"]      # divided by a tensor: torch multiplies by the reciprocal of a scalar divisor
    assert torch.equal(last.reshape(G, P, -1), (dout / torch.full_like(dout, P))[:, None].expand(G, P, dout.shape[-1]))

def run_case(prec):
    name, mod, B, T, H, W, tail, _ = CASE
    t0 = time.time()
    m = Conv3dResNet() if mod == "video" else Conv1dResNet()
    m.load_state_dict(frontend_state_dict(3, mod), strict=True)
    m = m.to(dev).train()
    m.library_train, m.precision = True, prec
    x = frontend_input(mod, B, T, H, W, seed=17)
    if tail is not None:
        x[1, tail:] = 0.0
    x = x.to(dev)
    G = B * T if mod == "video" else B * (T // 640)
    wts = torch.randn(G, 512, generator=torch.Generator().manual_seed(5)).to(dev).view(B, -1, 512)
    torch.cuda.reset_peak_memory_stats()
    geoms, rec, pool, mean = capture_step(m, x, wts, prec)
    if mod == "video":
        check_pool_and_mean(geoms, rec, pool, mean)
    else:
        G, P = mean["G"], mean["P"]
        last = rec[geoms[-1].name]["dy"]
        dout = mean["dout"]
        assert torch.equal(last.reshape(G, P, -1), (dout / torch.full_like(dout, P))[:, None].expand(G, P, 512))
    tag = f"{name}/{prec}/{mod}"
    weak = []
    for g in geoms:
        e = rec[g.name]
        conv, bn = e["pair"]
        assert e["spec"].args() == g.args(), (g.name, e["spec"].args(), g.args())
        # the capture is faithful: the unit alone reproduces the chained step bit for bit
        bn2 = copy.deepcopy(bn)
        bn2.running_mean.copy_(e["rm"]); bn2.running_var.copy_(e["rv"]); bn2.num_batches_tracked.fill_(e["nbt"])
        w, ga, be = (p.detach().clone().requires_grad_(True) for p in (conv.weight, bn.weight, bn.bias))
        xr = e["x"].clone().requires_grad_(g.stem == 0)
        rr = None if e["resid"] is None else e["resid"].clone().requires_grad_(True)
        y = FT.ConvBnActFn.apply(xr, rr, w, ga, be, bn2, e["spec"], e["act"], prec, None)
        y.backward(e["dy"])
        for a, b, what in ((y, e["y"], "y"), (w.grad, conv.weight.grad, "dw"), (ga.grad, bn.weight.grad, "dgamma"),
                           (be.grad, bn.bias.grad, "dbeta"), (bn2.running_mean, bn.running_mean, "running_mean"),
                           (bn2.running_var, bn.running_var, "running_var")):
            assert torch.equal(a, b), (tag, g.name, what, "re-run differs from the chained step")
        assert int(bn2.num_batches_tracked) == int(bn.num_batches_tracked) == e["nbt"] + 1
        got = dict(y=y.detach(), dx=xr.grad, dres=None if rr is None else rr.grad, dw=w.grad, dgamma=ga.grad,
                   dbeta=be.grad, running_mean=bn2.running_mean, running_var=bn2.running_var)
        del y, xr, rr
        # float64 on the same inputs
        factor = bn.momentum if bn.momentum is not None else 1.0 / (e["nbt"] + 1)
        d64 = lambda t: None if t is None else t.double()
        args = (d64(e["x"]), d64(e["resid"]), d64(conv.weight), d64(bn.weight), d64(bn.bias), d64(e["rm"]),
                d64(e["rv"]), factor, bn.eps, g, e["act"], d64(e["dy"]))
        ref = S.unit(*args, splits=splits_of(g))
        tol = TOL[(prec, "few" if g.rows <= FEW else "many")]
        errs = {q: S.rel(got[q], ref[q]) for q in Q if ref[q] is not None}
        # torch's fp32 unit with cuDNN TF32 (the reference implementation's training configuration): recorded only
        torch.backends.cudnn.allow_tf32 = True
        yard = S.torch_unit(*[a.float() if isinstance(a, torch.Tensor) else a for a in args])
        torch.backends.cudnn.allow_tf32 = False
        yerr = {q: S.rel(yard[q], ref[q]) for q in Q if ref[q] is not None}
        del yard
        for q, v in errs.items():
            record("frontend_train_units", f"{tag}/{g.name}/{q}", v, tol[q])
            record("frontend_train_units_cudnn_tf32", f"{tag}/{g.name}/{q}", yerr[q], None)
        FAILS.extend((tag, g.name, q, v, tol[q]) for q, v in errs.items() if not v < tol[q])
        # negative controls
        for d in S.DEFECTS:
            if not S.applies(d, g, e["act"], e["resid"] is not None):
                record("frontend_train_defects", f"{tag}/{g.name}/{d}", "n/a", CONTROL_MARGIN)
                continue
            bad = S.unit(*args, splits=splits_of(g), defect=d)
            margin = max(S.rel(got[q], bad[q]) / tol[q] for q in errs)
            del bad
            need = None if g.rows > WEAK_ABOVE.get((d, "fp32" if prec == "fp32" else "tc"), 1 << 62) else CONTROL_MARGIN
            record("frontend_train_defects", f"{tag}/{g.name}/{d}", {"margin": margin, "positions": g.rows}, need)
            if need is None:
                weak.append((g.name, d, round(margin, 3)))
            elif not margin >= need:
                FAILS.append((tag, g.name, d, "control not caught", margin))
        del ref, got
        torch.cuda.empty_cache()
    print(tag, "weak controls (recorded, not asserted)", weak)
    print(tag, "seconds", round(time.time() - t0, 1), "peak GiB", round(torch.cuda.max_memory_allocated() / 2**30, 2))
"""


def run_child(cases, precs, timeout=900):
    body = "ROOT, HERE = %r, %r\n" % (ROOT, HERE) + CHILD
    body += "for CASE in %r:\n    for prec in %r:\n        if prec in CASE[7]: run_case(prec)\n" % (cases, precs)
    body += "assert not FAILS, FAILS\nprint('CHILD-OK')\n"
    r = subprocess.run([sys.executable, "-c", body], capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    print(r.stdout[-6000:])
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def _cases(bucket):
    from oracle.frontend_train_stages import CASES
    return [c for c in CASES if (c[0] == "bucket") == bucket]


@pytest.mark.parametrize("prec", ["fp32", "tf32", "f16"])
def test_units_against_float64(prec):
    """Every unit of both modalities at every small case: one frame per utterance up to seven, zero-padded tails,
    45x61 and 89x89 frames, a 1x1 layer 4, layer-4 BatchNorms on 5 to 32 positions, empty trailing wgrad splits,
    statistics tiles ending in 1 and 255 rows; audio not a multiple of 640 and one frame per utterance."""
    run_child(_cases(False), [prec])


@pytest.mark.parametrize("modality", ["video", "audio"])
def test_bucket_units_against_float64(modality):
    """The max-frames buckets (video 4 x 400 frames of 88x88, audio 4 x 256,000 samples) in f16, the training default:
    the tensor-core wgrad at its full split counts."""
    run_child([c for c in _cases(True) if c[1] == modality], ["f16"])
