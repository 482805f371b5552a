"""Stream-K (gemm_schedule.cuh) in the tensor-core GEMM, forced through AVSR_B200_TILE = "BN,sk".

Every CTA takes an equal share of the GEMM's (tile, k-block) steps; a tile shared by several CTAs is finished by the
last to arrive, which sums the pieces' fp32 partials in piece order.  Single residual GEMMs go through
avsr_linear_operands_split (the split workspace the encoder gives its residual GEMMs) at the encoder's w_2 / out
shapes and with M on tile edges: against float64, bit-identical on a second call, within tolerance of the
data-parallel "128,1", and bit-identical with programmatic dependent launch off.  The 12-layer encoder runs with every
residual GEMM on stream-K at the bench buckets: within the f16 / tf32 parity bounds of the data-parallel forward,
bit-identical run to run and between direct launches and the graph plan."""
import contextlib
import os
import subprocess
import sys

import pytest
import torch

from helpers import err_stats

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TOL_OP = {"tf32": 4e-3, "f16": 1.5e-3}                          # as tests/test_zz_gpu_gemm_cluster.py
TOL_ENC = {"tf32": (1.8e-2, 1.2e-3), "f16": (1.8e-2, 1.2e-3)}    # as tests/test_gpu_parity.py, 12 layers
# (M, N, K): FFN w_2 and out / pw2 at S2 (1600 rows), S1 (100), S2r (2000) and tile edges
SHAPES = [(1600, 768, 3072), (1600, 768, 768), (100, 768, 3072), (100, 768, 768), (2000, 768, 3072), (127, 136, 768),
          (128, 768, 3072), (129, 8, 64)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "needs a CUDA GPU"
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


@contextlib.contextmanager
def forced_tile(spec):
    old = os.environ.get("AVSR_B200_TILE")
    os.environ["AVSR_B200_TILE"] = spec
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("AVSR_B200_TILE", None)
        else:
            os.environ["AVSR_B200_TILE"] = old


def residual_gemm(M, N, K, prec, dev, seed=7):
    """-> (run(), float64 reference): y = resid + 0.5 * (x W^T + b) through the split entry"""
    from auto_avsr_b200 import _cabi
    from auto_avsr_b200.engine import PRECISIONS
    tdt = torch.float16 if prec == "f16" else torch.float32
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(tdt)
    w = ((torch.rand(N, K, generator=g) - 0.5) * 0.07).to(tdt)
    b = torch.randn(N, generator=g) * 0.1
    r = torch.randn(M, N, generator=g)
    ref = r.double() + 0.5 * (x.double() @ w.double().T + b.double())
    x, w, b, r = x.to(dev), w.to(dev), b.to(dev), r.to(dev)
    part = torch.full((_cabi.SPLIT_PLANES * M * N,), float("nan"), device=dev)
    cnt = torch.zeros(_cabi.SPLIT_COUNTERS, device=dev, dtype=torch.int32)

    def run():
        y = torch.empty(M, N, device=dev)
        _cabi.check(_cabi.lib.avsr_linear_operands_split(
            x.data_ptr(), w.data_ptr(), b.data_ptr(), r.data_ptr(), 0.5, y.data_ptr(), M, N, K, 0, 0, PRECISIONS[prec],
            part.data_ptr(), cnt.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
        torch.cuda.synchronize()
        assert not cnt.any(), "tile counters must be re-armed"
        return y
    return run, ref


@pytest.mark.parametrize("prec", ["f16", "tf32"])
@pytest.mark.parametrize("bn", [64, 128])
def test_single_gemm_streamk(dev, prec, bn):
    for M, N, K in SHAPES:
        run, ref = residual_gemm(M, N, K, prec, dev)
        with forced_tile(f"{bn},sk"):
            a, b = run(), run()
        with forced_tile("128,1"):
            dp = run()
        assert torch.equal(a, b), (M, N, K, "second call differs")
        scale = ref.abs().max().item()
        mx, _ = err_stats(a.cpu(), ref)
        assert mx < TOL_OP[prec] * scale, (M, N, K, mx, scale)
        mx_dp, _ = err_stats(a, dp)
        assert mx_dp < TOL_OP[prec] * scale, (M, N, K, mx_dp)


PDL_CHILD = r'''
import os, sys, torch
sys.path.insert(0, %(here)r); sys.path.insert(0, %(root)r)
from test_zz_gpu_gemm_streamk import residual_gemm, SHAPES
os.environ["AVSR_B200_TILE"] = "128,sk"
dev = torch.device("cuda:0")
out = [residual_gemm(M, N, K, prec, dev)[0]().cpu() for prec in ("f16", "tf32") for M, N, K in SHAPES]
torch.save(out, sys.argv[1])
'''


def test_single_gemm_streamk_same_bits_without_pdl(dev, tmp_path):
    outs = {}
    for pdl in ("1", "0"):
        path = str(tmp_path / f"pdl{pdl}.pt")
        r = subprocess.run([sys.executable, "-c", PDL_CHILD % dict(here=HERE, root=ROOT), path], capture_output=True,
                           text=True, env=dict(os.environ, AVSR_B200_PDL=pdl), timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr[-2000:]
        outs[pdl] = torch.load(path)
    for a, b in zip(outs["1"], outs["0"]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("prec", ["f16", "tf32"])
@pytest.mark.parametrize("shape", ["S1", "S2", "S2r", "S3", "S4"])
def test_encoder_streamk(dev, prec, shape):
    from auto_avsr_b200 import ConformerEncoder
    from auto_avsr_b200.synthetic import SHAPES as BUCKETS, encoder_input, encoder_state_dict
    from oracle import conformer_oracle as O
    lengths = BUCKETS[shape]
    enc = ConformerEncoder()
    enc.load_state_dict(encoder_state_dict(11), strict=True)
    enc = enc.to(dev).eval()
    enc.precision = prec
    xs = encoder_input(lengths, 768, 5).to(dev)
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)

    def fwd(graph):
        enc.use_graph = graph
        with torch.no_grad():
            return enc(xs, mask)[0].clone()
    dp = fwd(False)
    with forced_tile("128,sk"):
        direct = [fwd(False) for _ in range(2)]
        graphed = [fwd(True) for _ in range(3)]
    assert torch.equal(direct[0], direct[1])
    for g in graphed:
        assert torch.equal(g, direct[0]), "graph plan differs from direct launches"
    mx, rms = err_stats(direct[0], dp)
    assert mx < TOL_ENC[prec][0] and rms < TOL_ENC[prec][1], (shape, prec, mx, rms)
