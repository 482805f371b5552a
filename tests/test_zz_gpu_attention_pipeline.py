"""The pipelined rel-pos attention kernel (csrc/attention_tc.cu) against the float64 restatement at the edges of its
tiling: a CTA serves 64 queries, the K tile and position band of the next key tile load while the current one is
processed, and the V tile loads during the softmax.  Every case runs twice and the two outputs must be equal bit for
bit."""
import pytest
import torch

from helpers import err_stats
from oracle import conformer_oracle as O

pytestmark = pytest.mark.gpu

TOL_ATT = {"tf32": 4e-3, "f16": 4e-3}        # tests/test_gpu_parity.py: attention context, relative

CASES = [
    # (B, T, H, lengths): every tail of one and two 64-query tiles, and 1..25 key tiles
    *[(1, T, 2, None) for T in (1, 63, 64, 65, 127, 128, 129, 191, 400, 1600)],
    (2, 64, 2, [64, 40]),              # one full query tile, a ragged key tile
    (3, 65, 2, [65, 64, 1]),           # the second query tile holds a single row
    (4, 129, 2, [0, 1, 63, 64]),       # lengths 0, 1, 63 and 64
    (2, 300, 3, [300, 0]),
    (16, 200, 12, [200 - 11 * i for i in range(16)]),   # B * H = 192 (* query tiles) well above the SM count
]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "needs a GPU"
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


@pytest.mark.parametrize("prec", ["f16", "tf32"])
@pytest.mark.parametrize("B,T,H,lengths", CASES)
def test_pipelined_attention_vs_fp64(dev, prec, B, T, H, lengths):
    from auto_avsr_b200 import ops
    g = torch.Generator().manual_seed(1000 + T + B)
    D = H * 64
    q, k, v = (torch.randn(B, T, D, generator=g) for _ in range(3))
    p = torch.randn(2 * T - 1, D, generator=g)
    u, vb = torch.randn(H, 64, generator=g) * 0.3, torch.randn(H, 64, generator=g) * 0.3
    ln = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=dev)
    args = [t.to(dev) for t in (q, k, v, p, u, vb)]
    outs = [ops.relpos_attention(*args, ln, H, precision=prec).cpu() for _ in range(2)]
    assert torch.equal(outs[0], outs[1]), "repeated call differs"

    def heads(t):
        return t.double().view(B, T, H, 64).transpose(1, 2)
    scores = O.rel_attention_scores(heads(q), heads(k), p.double().view(2 * T - 1, H, 64).transpose(0, 1),
                                    u.double(), vb.double())
    if lengths is not None:
        pad = torch.arange(T)[None, :] >= torch.tensor(lengths)[:, None]
        scores = scores.masked_fill(pad[:, None, None, :], float("-inf"))
    attn = torch.softmax(scores, dim=-1)
    attn = torch.where(torch.isnan(attn), torch.zeros_like(attn), attn)       # fully masked rows -> 0
    ref = (attn @ heads(v)).transpose(1, 2).reshape(B, T, D)
    assert torch.isfinite(outs[0]).all()
    if lengths is not None:
        for b, L in enumerate(lengths):
            if L == 0:
                assert (outs[0][b] == 0).all()
    assert err_stats(outs[0], ref)[0] < TOL_ATT[prec] * max(1.0, ref.abs().max().item())
