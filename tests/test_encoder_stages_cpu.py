"""The stage-isolated references and negative controls of oracle/encoder_stages.py (used by
tests/test_zz_gpu_encoder_stages.py) checked on the CPU in float64: chained over their own outputs they reproduce the
whole-encoder oracle, and every defect moves its stage far above float64 noise."""
import math

import pytest
import torch

from auto_avsr_b200.synthetic import encoder_input, encoder_state_dict
from helpers import load_case
from oracle import conformer_oracle as O
from oracle import encoder_stages as ES


def _tiny():
    c = load_case("tiny_ragged")
    return c["sd"], c["xs"], c["lengths"], c["cfg"]["n_heads"]


def _full768():
    lengths = [30, 17]                       # B * T = 60; key tiles and the halo both see an utterance boundary
    return encoder_state_dict(21, num_blocks=2), encoder_input(lengths, 768, 77), lengths, 12


CASES = {"tiny_ragged": _tiny, "full768_b2": _full768}


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    sd, xs, lengths, H = CASES[request.param]()
    sd = {k: (t.double() if t.is_floating_point() else t) for k, t in sd.items()}
    xs = xs.double()
    B, T, D = xs.shape
    stages = []
    out = O.encoder_forward(sd, xs, lengths, H, stages=stages)
    return dict(name=request.param, sd=sd, x0=xs * math.sqrt(D), lengths=torch.tensor(lengths), H=H,
                pos=O.rel_sinusoid_table(T, D, torch.float64), stages=stages, out=out)


def test_stage_chain_reproduces_encoder_forward(case):
    ins = [case["x0"]] + case["stages"][:4]
    for s in range(5):
        r = ES.stage(s, ins[s], case["pos"], case["lengths"], case["sd"], "encoders.0.", case["H"])
        want = case["stages"][s]
        assert (r - want).abs().max().item() <= 1e-12 * want.abs().max().item(), (case["name"], s)
    out = ES.layer_and_after_norm(case["stages"][4], case["pos"], case["lengths"], case["sd"], 1, case["H"])
    assert (out - case["out"]).abs().max().item() <= 1e-12 * case["out"].abs().max().item()


def test_errors_metric():
    r = torch.zeros(4, 10, 8, dtype=torch.float64)
    g_in = r.clone()
    g_in[..., 0] = -2.0                       # the stage added 2 to channel 0
    g = r.clone()
    g[1, 3, 5] = 0.5                          # one frame off by 0.5, every other frame off by 0.01
    g[..., 7] += 0.01
    e = ES.errors(g, r, g_in)
    assert e["scale"] == 2.0 and e["max"] == pytest.approx(0.25)
    assert e["frames"] == pytest.approx(50.0) and e["worst"] == 1 * 10 + 3
    assert ES.errors(g_in, g_in)["frames"] == 1.0


@pytest.mark.parametrize("defect", list(ES.DEFECTS))
def test_defect_moves_its_stage(case, defect):
    s = ES.DEFECTS[defect]
    ins = [case["x0"]] + case["stages"][:4]
    B, T, _ = ins[s].shape
    assert ES.applies(defect, B, T)
    r = case["stages"][s]
    bad = ES.stage(s, ins[s], case["pos"], case["lengths"], case["sd"], "encoders.0.", case["H"], defect=defect)
    e = ES.errors(bad, r, ins[s] if s < 4 else None)
    # float64 rounding of a stage is ~1e-15 of its scale; the GPU bounds are 1e-6 (fp32) to 1e-2 (f16)
    assert e["max"] > 1e-4, (case["name"], defect, e)
    with pytest.raises(ValueError):
        ES.stage((s + 1) % 5, ins[s], case["pos"], case["lengths"], case["sd"], "encoders.0.", case["H"], defect=defect)


def test_defects_that_cannot_show_are_skipped():
    """The conv halo needs an utterance boundary; a bias or position-row slip needs more than one key.  Where
    applies() says no, the defect indeed changes nothing."""
    assert not ES.applies("conv_halo", 1, 50) and ES.applies("conv_halo", 2, 50)
    assert [d for d in ES.DEFECTS if not ES.applies(d, 1, 1)] == ["mha_uv_swap_last_head", "mha_relshift_tile",
                                                                  "conv_halo"]
    sd, xs, _, H = _tiny()
    sd = {k: (t.double() if t.is_floating_point() else t) for k, t in sd.items()}
    for B, T in [(1, 37), (3, 1)]:
        x = xs[:B, :T].double() * 4
        pos = O.rel_sinusoid_table(T, x.shape[-1], torch.float64)
        for d, s in ES.DEFECTS.items():
            if not ES.applies(d, B, T):
                good = ES.stage(s, x, pos, None, sd, "encoders.0.", H)
                assert torch.equal(ES.stage(s, x, pos, None, sd, "encoders.0.", H, defect=d), good), (d, B, T)
