"""The ResNet front-end drop-ins without a GPU: state-dict contract against the reference modules, install_frontend's
re-homing, train-mode equality with the reference, refusals, and the golden fixtures reproduced by the reference copy."""
import os

import numpy as np
import pytest
import torch

from oracle import build_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

pytestmark = pytest.mark.skipif(not build_ref.available(), reason="oracle/_ref not built")

PARAMS = {"video": 11182784, "audio": 3848576}


def _ref(modality):
    from oracle.make_golden_frontend import reference_module
    return reference_module(modality)


def _dropin(modality):
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
    return Conv3dResNet() if modality == "video" else Conv1dResNet()


@pytest.mark.parametrize("modality", ["video", "audio"])
def test_state_dicts_load_strictly_both_ways(modality):
    from auto_avsr_b200.synthetic import frontend_state_dict
    ref, new = _ref(modality), _dropin(modality)
    assert sum(p.numel() for p in ref.parameters()) == PARAMS[modality]
    assert sum(p.numel() for p in new.parameters()) == PARAMS[modality]
    sd = frontend_state_dict(5, modality)
    assert list(sd) == list(ref.state_dict()) == list(new.state_dict())
    for k, v in ref.state_dict().items():
        assert new.state_dict()[k].shape == v.shape, k
    new.load_state_dict(sd, strict=True)
    ref.load_state_dict(new.state_dict(), strict=True)
    for k, v in ref.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert len(new.conv_bn_pairs()) == 20
    assert all(isinstance(bn, torch.nn.modules.batchnorm._BatchNorm) for _, bn in new.conv_bn_pairs())


@pytest.mark.parametrize("modality", ["video", "audio"])
def test_train_forward_backward_equal_reference_bit_for_bit(modality):
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    torch.manual_seed(0)
    sd = frontend_state_dict(6, modality)
    ref, new = _ref(modality), _dropin(modality)
    ref.load_state_dict(sd)
    new.load_state_dict(sd)
    ref.train(); new.train()
    x = frontend_input(modality, 2, 3 if modality == "video" else 640 * 3 + 11, 44, 40, seed=3)
    xr, xn = x.clone().requires_grad_(), x.clone().requires_grad_()
    yr, yn = ref(xr), new(xn)
    assert torch.equal(yr, yn)
    g = torch.randn_like(yr)
    yr.backward(g); yn.backward(g)
    assert torch.equal(xr.grad, xn.grad)
    for (k, pr), (_, pn) in zip(ref.named_parameters(), new.named_parameters()):
        assert torch.equal(pr.grad, pn.grad), k
    for (k, br), (_, bn) in zip(ref.named_buffers(), new.named_buffers()):
        assert torch.equal(br, bn), k                      # running statistics updated identically


def test_eval_refuses_cpu_tensors_and_non_swish():
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
    from auto_avsr_b200.synthetic import frontend_input
    for m, x in ((Conv3dResNet(), frontend_input("video", 1, 2, 20, 20)), (Conv1dResNet(), frontend_input("audio", 1, 1280))):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            m.eval()(x)
    for relu_type in ("relu", "prelu"):
        with pytest.raises(NotImplementedError):
            Conv3dResNet(relu_type=relu_type)
        with pytest.raises(NotImplementedError):
            Conv1dResNet(relu_type=relu_type)


@pytest.mark.parametrize("modality", ["video", "audio"])
def test_install_frontend_keeps_parameters_buffers_and_state_dict(modality):
    import auto_avsr_b200
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet

    class Shell(torch.nn.Module):                 # the member of E2E that install_frontend re-homes
        def __init__(self):
            super().__init__()
            self.frontend = _ref(modality)
            self.proj_encoder = torch.nn.Linear(512, 768)

    m = Shell()
    m.frontend.train()
    m.frontend.trunk.layer2[0].bn1.eval()         # per-module modes survive
    m.frontend.trunk.layer3[1].bn2.eps = 1e-3
    before = {k: v for k, v in m.state_dict().items()}
    params = {k: p for k, p in m.named_parameters()}
    buffers = {k: b for k, b in m.named_buffers()}
    out = auto_avsr_b200.install_frontend(m)
    assert out is m and isinstance(m.frontend, Conv3dResNet if modality == "video" else Conv1dResNet)
    assert list(m.state_dict()) == list(before)
    for k, v in m.state_dict().items():
        assert v.data_ptr() == before[k].data_ptr(), k
    for k, p in m.named_parameters():
        assert p is params[k], k
    for k, b in m.named_buffers():
        assert b is buffers[k], k
    assert m.frontend.training and not m.frontend.trunk.layer2[0].bn1.training
    assert m.frontend.trunk.layer3[1].bn2.eps == 1e-3


@pytest.mark.parametrize("name", ["frontend_video_88", "frontend_video_t1", "frontend_video_45x61", "frontend_audio_ragged"])
def test_reference_copy_reproduces_golden(name):
    from oracle.make_golden_frontend import CASES, reference_output
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    modality, wseed, xseed, B, T, H, W, lengths = CASES[name]
    assert str(z["modality"]) == modality and int(z["wseed"]) == wseed and int(z["xseed"]) == xseed
    assert list(z["shape"]) == [B, T, H, W] and list(z["lengths"]) == lengths
    out = reference_output(name)
    assert out.shape == z["out_f64"].shape
    assert np.abs(out - z["out_f64"]).max() <= 1e-12 * max(1.0, np.abs(z["out_f64"]).max())
