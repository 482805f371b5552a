"""The tensor-core GEMM in 2-CTA and 4-CTA clusters (TMA multicast of the shared operand tiles) against the same GEMM
in 1 x 1 clusters at the same tile width, and against float64.

Multicast changes where an operand tile comes from, not the order in which each output element sums over K, so every
cluster shape must give exactly the bits of the 1 x 1 kernel, and the same bits on a second call.  The shapes put M and
N on tile edges (M = 1600 leaves the last 2 x 1 cluster with an empty partner; N smaller than one tile leaves a peer's
operand slice wholly outside the matrix) and K from one k-block to 48.  LINEAR (fp32 with residual, ReLU) and GLU go
through their C-ABI entries; QK, V^T and POS through a 2-layer encoder forward."""
import contextlib
import math
import os

import pytest
import torch

from helpers import err_stats

pytestmark = pytest.mark.gpu

TOL_OP = {"tf32": 4e-3, "f16": 1.5e-3}      # as tests/test_gpu_parity.py: single GEMMs, relative to output scale
CLUSTERS = ["1x1", "2x1", "1x2", "2x2"]


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


def run_all(fn, bn):
    """fn() under every cluster shape at tile width bn, twice each -> {cluster: output}; asserts repeat bits."""
    out = {}
    for cl in CLUSTERS:
        with forced_tile(f"{bn},1,{cl}"):
            a = fn()
            b = fn()
        torch.cuda.synchronize()
        assert torch.equal(a, b), ("second call differs", cl)
        out[cl] = a
    return out


LINEAR_SHAPES = [(1, 64, 64), (64, 200, 768), (127, 8, 768), (128, 384, 3072), (129, 72, 64), (1600, 3072, 768),
                 (1600, 768, 3072), (1601, 136, 768), (3200, 1536, 64)]


@pytest.mark.parametrize("prec", ["f16", "tf32"])
@pytest.mark.parametrize("bn", [64, 128])
def test_linear_clusters(dev, prec, bn):
    from auto_avsr_b200 import ops
    g = torch.Generator().manual_seed(11)
    for M, N, K in LINEAR_SHAPES:
        x = torch.randn(M, K, generator=g).to(dev)
        w = ((torch.rand(N, K, generator=g) * 2 - 1) / math.sqrt(K)).to(dev)
        b = (torch.randn(N, generator=g) * 0.1).to(dev)
        r = torch.randn(M, N, generator=g).to(dev)
        ref = x.double() @ w.double().T + b.double()
        scale = ref.abs().max().item()
        for relu, resid in ((False, None), (True, None), (False, r)):
            outs = run_all(lambda: ops.linear(x, w, b, relu=relu, residual=resid, alpha=0.5, precision=prec), bn)
            want = ref.clamp_min(0) if relu else ref
            if resid is not None:
                want = resid.double() + 0.5 * want
            assert err_stats(outs["1x1"].cpu(), want.cpu())[0] < TOL_OP[prec] * scale, (M, N, K, relu)
            for cl, y in outs.items():
                assert torch.equal(y, outs["1x1"]), (M, N, K, relu, resid is not None, cl)


@pytest.mark.parametrize("prec", ["f16", "tf32"])
def test_glu_clusters(dev, prec):
    from auto_avsr_b200 import ops
    g = torch.Generator().manual_seed(12)
    for rows, C in [(1, 128), (129, 768), (1600, 768), (1601, 256)]:
        x = torch.randn(rows, C, generator=g).to(dev)
        w = ((torch.rand(2 * C, C, 1, generator=g) * 2 - 1) / math.sqrt(C)).to(dev)
        b = (torch.randn(2 * C, generator=g) * 0.1).to(dev)
        full = x.double() @ w.squeeze(-1).double().T + b.double()
        ref = full[:, :C] * torch.sigmoid(full[:, C:])
        outs = run_all(lambda: ops.pointwise_glu(x, w, b, prec), 128)
        tol = TOL_OP[prec] * max(1.0, ref.abs().max().item())
        assert err_stats(outs["1x1"].cpu(), ref.cpu())[0] < tol, (rows, C)
        for cl, y in outs.items():
            assert torch.equal(y, outs["1x1"]), (rows, C, cl)


@pytest.mark.parametrize("prec", ["f16", "tf32"])
def test_encoder_clusters(dev, prec):
    """QK (head-major scatter + pos biases), V^T, POS and the rest at a ragged batch of 2 x ~400 frames."""
    from auto_avsr_b200 import ConformerEncoder
    from auto_avsr_b200.synthetic import encoder_input, encoder_state_dict
    from oracle import conformer_oracle as O
    lengths = [400, 263]
    enc = ConformerEncoder(num_blocks=2)
    enc.load_state_dict(encoder_state_dict(5, num_blocks=2), strict=True)
    enc = enc.to(dev).eval()
    enc.precision = prec
    enc.use_graph = False
    xs = encoder_input(lengths, 768, 9).to(dev)
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)

    def fwd():
        with torch.no_grad():
            return enc(xs, mask)[0].clone()
    outs = run_all(fwd, 128)
    for cl, y in outs.items():
        assert torch.equal(y, outs["1x1"]), cl
