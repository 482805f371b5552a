"""The float64 stage oracle of the ResNet front-ends (oracle/frontend_oracle.py) without a GPU: chaining its stages
reproduces the reference modules at every tap the library exposes (stem, trunk input, each BasicBlock) and at the
output, for both modalities, at small shapes including a ragged batch and a waveform with a cut tail, with the
synthetic weights and with trained-like BatchNorm statistics; and it reproduces the four golden front-end fixtures."""
import os

import numpy as np
import pytest
import torch

from oracle import build_ref
from oracle import frontend_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["frontend_video_88", "frontend_video_t1", "frontend_video_45x61", "frontend_audio_ragged"]

needs_ref = pytest.mark.skipif(not build_ref.available(), reason="oracle/_ref not built")


def _reference_taps(modality, sd, x):
    """the reference module in float64 with forward hooks: its 10 stage outputs in the taps' channels-last layout, and
    its output"""
    from oracle.make_golden_frontend import reference_module
    ref = reference_module(modality)
    ref.load_state_dict(sd, strict=True)
    ref = ref.double().eval()
    B, T = x.shape[:2]
    got = {}

    def keep(i):
        def hook(module, inputs, output):
            got[i] = output.detach().clone()
        return hook

    if modality == "video":
        stages = [ref.frontend3D[2], ref.frontend3D[3]]
    else:
        stages = [ref.trunk.relu, ref.trunk.relu]
    trunk = ref.trunk
    stages += [blk for layer in (trunk.layer1, trunk.layer2, trunk.layer3, trunk.layer4) for blk in layer]
    for i, m in enumerate(stages):
        if m not in stages[:i]:
            m.register_forward_hook(keep(i))
    with torch.no_grad():
        out = ref(x)
    got[1] = got.get(1, got[0])
    taps = []
    for i in range(O.N_TAPS):
        h = got[i]
        if h.dim() == 5:                                   # video stem (B, C, T, H, W) -> (B*T, H, W, C)
            taps.append(h.permute(0, 2, 3, 4, 1).reshape(B * T, h.shape[3], h.shape[4], h.shape[1]))
        else:
            taps.append(O.to_channels_last(h))
    return taps, out


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


CASES = [  # modality, B, T (frames or samples), H, W
    ("video", 2, 5, 24, 20),           # a ragged batch: lengths 5 and 2 padded to 5, the padding is data
    ("video", 1, 1, 17, 17),
    ("video", 3, 2, 9, 9),
    ("audio", 2, 640 * 3 + 317, 1, 1),  # a cut tail; lengths 3 frames + 317 samples and 1 frame padded
    ("audio", 1, 640, 1, 1),
]


@needs_ref
@pytest.mark.parametrize("weights", ["synthetic", "trained_like"])
@pytest.mark.parametrize("modality,B,T,H,W", CASES)
def test_oracle_stages_reproduce_reference_taps(modality, B, T, H, W, weights):
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    if weights == "synthetic":
        sd = frontend_state_dict(71, modality)
    else:
        from test_zz_gpu_frontend_stages import trained_like_state_dict
        sd = trained_like_state_dict(72, modality)
    x = frontend_input(modality, B, T, H, W, seed=73, dtype=torch.float64)
    ref_taps, ref_out = _reference_taps(modality, sd, x)
    sd64 = {k: v.double() for k, v in sd.items() if v.is_floating_point()}
    taps, out = O.taps(sd64, modality, x)
    for k in range(O.N_TAPS):
        assert taps[k].shape == ref_taps[k].shape, (k, taps[k].shape, ref_taps[k].shape)
        assert _rel(taps[k], ref_taps[k]) < 1e-12, (k, _rel(taps[k], ref_taps[k]))
        if k > 0:                                              # each stage on its own, from the reference's input
            assert _rel(O.next_tap(sd64, modality, k, ref_taps[k - 1]), ref_taps[k]) < 1e-12, k
    assert out.shape == ref_out.shape and _rel(out, ref_out) < 1e-12
    assert _rel(O.head_mean(modality, ref_taps[-1], B), ref_out) < 1e-12
    if weights == "trained_like":
        var = torch.cat([v for k, v in sd.items() if k.endswith("running_var")])
        gamma = torch.cat([v for k, v in sd.items() if k.endswith("bn1.weight") or k.endswith("bn2.weight")])
        assert var.min() < 2e-4 and var.max() > 50 and (gamma < 0).any() and gamma.abs().min() < 1e-3


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_golden(name):
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    modality = str(z["modality"])
    B, T, H, W = (int(v) for v in z["shape"])
    sd = {k: v.double() for k, v in frontend_state_dict(int(z["wseed"]), modality).items() if v.is_floating_point()}
    x = frontend_input(modality, B, T, H, W, int(z["xseed"]), dtype=torch.float64)
    out = O.forward(sd, modality, x).numpy()
    ref = z["out_f64"]
    assert out.shape == ref.shape
    assert np.abs(out - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


def test_library_tap_shapes_match_oracle():
    """avsr_frontend_tap_shape (host-only) states the geometry the oracle's stages produce, down to 1x1 frames and
    waveforms shorter than one frame."""
    from auto_avsr_b200.frontend import frontend_tap_shape
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    for modality, B, T, H, W in (("video", 2, 3, 1, 1), ("video", 1, 2, 2, 3), ("video", 2, 1, 7, 7),
                                 ("video", 1, 1, 9, 9), ("video", 1, 2, 45, 61), ("video", 1, 1, 89, 89),
                                 ("video", 1, 1, 96, 96), ("audio", 2, 641, 1, 1), ("audio", 1, 640 * 3 + 639, 1, 1)):
        sd = {k: v.double() for k, v in frontend_state_dict(1, modality).items() if v.is_floating_point()}
        taps, out = O.taps(sd, modality, frontend_input(modality, B, T, H, W, dtype=torch.float64))
        assert [frontend_tap_shape(modality, B, T, H, W, k) for k in range(O.N_TAPS)] == [tuple(t.shape) for t in taps]
    assert frontend_tap_shape("audio", 3, 639, 1, 1, 9) == (3, 1, 0, 512)
