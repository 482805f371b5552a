"""CPU checks of the CTC loss (csrc/ctc_loss.cu) without a GPU: the label compaction, extended-label mapping, alpha / beta
recursion and gradient combination of csrc/ctc_loss_body.cuh, compiled into the host replay of tests/emu (same source,
the kernels' schedule as plain loops) and called through the package's ctypes signatures, against
torch.nn.functional.ctc_loss + autograd in float64.  Also: the reference-generated fixtures reproduce, and the C ABI
entries are bound as the header declares them.  The GPU parity is tests/test_zz_gpu_ctc_loss.py."""
import ctypes as C
import os
import re
import shutil

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "avsr_b200.h")
HAVE_NVCC = shutil.which("nvcc") is not None or os.path.exists("/usr/local/cuda/bin/nvcc")


@pytest.fixture(scope="module")
def emu():
    if not HAVE_NVCC:
        pytest.skip("nvcc is needed to build the host replay")
    from emu import build
    return build.load("ctc")


def emu_ctc(lib, logits, hlens, ys, odim, dnll, ignore_id=-1):
    """(B, T, ld) float32 logits -> (nll (B), dlogits (B, T, ld)) through the host replay."""
    logits = logits.float().contiguous()
    B, T, ld = logits.shape
    hl = hlens.to(torch.int32).contiguous()
    ys = ys.to(torch.int64).contiguous()
    L = ys.size(1)
    nll = torch.empty(B, dtype=torch.float32)
    state = torch.empty(int(lib.avsr_ctc_loss_state_bytes(B, T, L)), dtype=torch.uint8)
    rc = lib.avsr_ctc_loss_fwd(logits.data_ptr(), ld, hl.data_ptr(), ys.data_ptr(), B, T, L, odim, ignore_id, 1,
                               nll.data_ptr(), state.data_ptr(), state.numel(), None)
    assert rc == 0, lib.avsr_last_error()
    d = torch.empty_like(logits)
    dn = dnll.float().contiguous()
    rc = lib.avsr_ctc_loss_bwd(logits.data_ptr(), ld, hl.data_ptr(), ys.data_ptr(), B, T, L, odim, dn.data_ptr(),
                               state.data_ptr(), state.numel(), d.data_ptr(), ld, None)
    assert rc == 0, lib.avsr_last_error()
    return nll, d


def torch_ctc(logits, hlens, ys, odim, dnll, ignore_id=-1):
    """torch's own CTC loss (zero_infinity, blank 0) in float64 with autograd -> (nll, dlogits)."""
    x = logits.double().clone().requires_grad_(True)
    lp = torch.log_softmax(x[..., :odim], dim=-1).transpose(0, 1)
    tg = [y[y != ignore_id] for y in ys]
    olens = torch.tensor([len(t) for t in tg], dtype=torch.long)
    flat = torch.cat(tg) if sum(len(t) for t in tg) else torch.zeros(0, dtype=torch.long)
    nll = torch.nn.functional.ctc_loss(lp, flat, hlens.long(), olens, blank=0, reduction="none", zero_infinity=True)
    (nll * dnll.double()).sum().backward()
    return nll.detach(), x.grad


def check_case(lib, logits, hlens, ys, odim, seed=0, tol=2e-5):
    g = torch.Generator().manual_seed(seed)
    dnll = torch.rand(len(hlens), generator=g) + 0.5
    nll, d = emu_ctc(lib, logits, hlens, ys, odim, dnll)
    rn, rd = torch_ctc(logits, hlens, ys, odim, dnll)
    scale = max(1.0, rn.abs().max().item())
    assert (nll.double() - rn).abs().max().item() < tol * scale, (nll, rn)
    # the fp32 log-probs carry rounding of the size of |lp|; the state posteriors' error grows with the loss
    gtol = tol * max(1.0, scale / 30.0)
    assert (d.double() - rd).abs().max().item() < gtol, ((d.double() - rd).abs().max().item(), gtol)
    return nll, d


def rand_logits(B, T, ld, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T, ld, generator=g) * scale


def test_edge_cases_match_torch(emu):
    odim = 9
    ys = torch.tensor([[3, 3, -1, 5, 5, 5, 2, -1],      # repeats that need blanks, -1 inside the row
                       [4, 4, 4, 4, -1, -1, -1, -1],    # too long for 5 frames with the blanks it needs -> inf -> 0
                       [-1] * 8,                        # empty target
                       [7, -1, -1, -1, -1, -1, -1, -1],  # one label, one frame
                       [1, 2, 3, -1, -1, -1, -1, -1],   # no frame at all (hlen 0) -> 0
                       [-1] * 8])                       # empty target, no frame
    hlens = torch.tensor([12, 5, 7, 1, 0, 0])
    logits = rand_logits(6, 12, 16, 1)
    logits[..., odim:] = 1e4                            # padding columns of a padded GEMM output must be ignored
    nll, d = check_case(emu, logits, hlens, ys, odim)
    assert nll[1] == 0 and nll[4] == 0 and nll[5] == 0
    assert (d[1] == 0).all() and (d[4] == 0).all() and (d[:, :, odim:] == 0).all()
    for b, h in enumerate(hlens.tolist()):
        assert (d[b, h:] == 0).all()                    # frames past hlen


def test_single_frame_and_empty_targets(emu):
    for T, L in [(1, 0), (1, 1), (2, 1), (3, 2), (4, 0)]:
        ys = torch.randint(1, 6, (2, max(L, 1)), generator=torch.Generator().manual_seed(T * 10 + L))
        if L == 0:
            ys[:] = -1
        check_case(emu, rand_logits(2, T, 6, T + L), torch.tensor([T, T]), ys, 6, seed=T)


@pytest.mark.parametrize("seed", range(6))
def test_random_sweep_matches_torch(emu, seed):
    g = torch.Generator().manual_seed(100 + seed)
    B = int(torch.randint(1, 6, (1,), generator=g))
    T = int(torch.randint(1, 40, (1,), generator=g))
    odim = int(torch.randint(2, 50, (1,), generator=g))
    ld = odim + int(torch.randint(0, 9, (1,), generator=g))
    Lmax = int(torch.randint(0, 20, (1,), generator=g))
    hlens = torch.randint(0, T + 1, (B,), generator=g)
    hlens[0] = T
    ys = torch.randint(1, odim, (B, Lmax), generator=g)
    if Lmax:
        ys[torch.rand(B, Lmax, generator=g) < 0.25] = -1                 # ignore_id anywhere in a row
        if odim > 2:
            ys[:, 1::3] = ys[:, ::3][:, :ys[:, 1::3].size(1)]            # repeated neighbours
    check_case(emu, rand_logits(B, T, ld, seed, scale=float(1 + seed)), hlens, ys, odim, seed=seed)


def test_bad_labels_and_lengths_give_nan_without_touching_others(emu):
    odim = 7
    ys = torch.tensor([[1, 2, 3], [1, 9, 2], [0, 1, -1], [2, 2, 2]])     # 9 >= odim; 0 = blank in a target
    hlens = torch.tensor([6, 6, 6, 8])                                    # 8 > Tmax
    logits = rand_logits(4, 6, 7, 3)
    nll, d = emu_ctc(emu, logits, hlens, ys, odim, torch.ones(4))
    assert torch.isfinite(nll[0]) and torch.isnan(nll[1:]).all()
    rn, rd = torch_ctc(logits[:1], hlens[:1], ys[:1], odim, torch.ones(1))
    assert abs(nll[0].item() - rn.item()) < 1e-4
    assert (d[0].double() - rd[0]).abs().max() < 2e-5


def test_long_targets_use_several_state_chunks(emu):
    """300 labels -> 601 states; 250 frames (the device stages emissions a chunk of frames at a time)."""
    g = torch.Generator().manual_seed(9)
    ys = torch.randint(1, 40, (2, 300), generator=g)
    ys[1, 200:] = -1
    check_case(emu, rand_logits(2, 700, 40, 4), torch.tensor([700, 650]), ys, 40, tol=5e-5)


# ------------------------------------------------------------------ fixtures and ABI
def _have_ref():
    from oracle import build_ref
    return build_ref.available()


@pytest.mark.skipif(not _have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("name", ["ctc_loss_tiny", "ctc_loss_full"])
def test_fixtures_reproduce_from_reference_copy(name, golden_dir):
    import subprocess
    import sys
    code = f"""
import sys, numpy as np
sys.path.insert(0, {ROOT!r})
from oracle import make_golden_ctc as M
z = np.load({os.path.join(golden_dir, name + ".npz")!r})
got = M.reference({name!r})
assert set(got) <= set(z.files), (sorted(got), z.files)
for k, v in got.items():
    assert np.allclose(v, z[k], rtol=1e-6, atol=1e-9), k
print("OK")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr[-2000:]


def test_fixture_edge_cases_are_present(golden_dir):
    z = np.load(os.path.join(golden_dir, "ctc_loss_tiny.npz"))
    ys, hl = z["ys_pad"], z["hlens"]
    assert list(hl) == [19, 12, 7, 1] and int(z["odim"]) == 37 and int(z["d_model"]) == 128
    kept = [r[r != -1] for r in ys]
    assert any((r[:-1] == r[1:]).any() for r in kept)                                       # repeats need a blank
    assert any((r[:-1] == -1).any() and (r[np.argmax(r == -1):] != -1).any() for r in ys)  # -1 inside a row
    assert any(len(r) == 0 for r in kept)
    assert z["loss_none"][2] == 0 and len(kept[2]) > hl[2]                                   # zero_infinity
    zf = np.load(os.path.join(golden_dir, "ctc_loss_full.npz"))
    n = (zf["ys_pad"] != -1).sum(1)
    assert int(zf["odim"]) == 5049 and zf["hlens"].max() == 400 and n.min() >= 60 and n.max() <= 100


_CTYPE = {"int": C.c_int, "long": C.c_long, "size_t": C.c_size_t}


def test_ctc_loss_signatures_match_the_header():
    from auto_avsr_b200 import _cabi
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for name in ("avsr_ctc_loss_state_bytes", "avsr_ctc_loss_fwd", "avsr_ctc_loss_bwd"):
        m = re.search(r"(\w+)\s+" + name + r"\s*\(([^)]*)\)", src)
        assert m, name
        ret, params = m.group(1), [p.strip() for p in m.group(2).split(",")]
        want = [C.c_void_p if "*" in p else _CTYPE[p.split()[0]] for p in params]
        res, args = _cabi.SIGNATURES[name]
        assert res == _CTYPE[ret], name
        assert args == want, (name, args, want)
