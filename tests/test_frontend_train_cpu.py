"""The front-ends' library-train switch without a GPU: install_frontend(library_train=True) keeps the same Parameter and
buffer objects and state dict, the default stays the torch path, and the new C entries' workspace sizes and argument
refusals (probed in a child process with no visible device)."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Holder(torch.nn.Module):
    def __init__(self, frontend):
        super().__init__()
        self.frontend = frontend


def _video():
    from auto_avsr_b200.espnet_dropin.resnet import Conv3dResNet
    from auto_avsr_b200.synthetic import frontend_state_dict
    m = Conv3dResNet()
    m.load_state_dict(frontend_state_dict(2, "video"), strict=True)
    return m


def test_install_library_train_keeps_parameters_buffers_and_state_dict():
    from auto_avsr_b200.install import install_frontend
    old = _video()
    h = _Holder(old)
    params = {n: p for n, p in old.named_parameters()}
    bufs = {n: b for n, b in old.named_buffers()}
    sd = {k: v.clone() for k, v in h.state_dict().items()}
    install_frontend(h, library_train=True)
    assert h.frontend is not old and h.frontend.library_train
    for n, p in h.frontend.named_parameters():
        assert p is params[n], n
    for n, b in h.frontend.named_buffers():
        assert b is bufs[n], n
    assert list(h.state_dict()) == list(sd)
    for k, v in h.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_default_is_the_torch_path():
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet
    from auto_avsr_b200.install import install_frontend
    h = _Holder(_video())
    install_frontend(h)
    assert h.frontend.library_train is False and Conv1dResNet.library_train is False
    x = torch.randn(1, 2, 1, 16, 16)
    ref = _video().train()
    h.frontend.train()
    assert torch.equal(h.frontend(x), ref(x))          # CPU train(): torch sub-modules, as before


def test_library_train_refuses_cpu_tensors():
    import pytest
    m = _video().train()
    m.library_train = True
    with pytest.raises(NotImplementedError):
        m(torch.randn(1, 2, 1, 16, 16))


PROBE = r"""
import json, sys
sys.path.insert(0, %r)
from auto_avsr_b200._cabi import lib
out = {}
out["conv_ws_trunk"] = lib.avsr_frontend_train_conv_workspace_bytes(0, 4, 1, 22, 22, 64, 64, 3, 3, 1, 2)
out["conv_ws_vstem"] = lib.avsr_frontend_train_conv_workspace_bytes(1, 8, 4, 88, 88, 1, 64, 0, 0, 0, 1)
out["conv_ws_astem"] = lib.avsr_frontend_train_conv_workspace_bytes(2, 2, 1, 1, 1280, 1, 64, 0, 0, 0, 0)
out["conv_ws_bad_cin"] = lib.avsr_frontend_train_conv_workspace_bytes(0, 4, 1, 22, 22, 3, 64, 3, 3, 1, 2)
out["conv_ws_bad_stride"] = lib.avsr_frontend_train_conv_workspace_bytes(0, 4, 1, 22, 22, 64, 64, 3, 3, 3, 2)
out["conv_ws_bad_prec"] = lib.avsr_frontend_train_conv_workspace_bytes(0, 4, 1, 22, 22, 64, 64, 3, 3, 1, 9)
out["conv_ws_bad_audio"] = lib.avsr_frontend_train_conv_workspace_bytes(2, 2, 1, 1, 1000, 1, 64, 0, 0, 0, 0)
out["conv_ws_bad_video_T"] = lib.avsr_frontend_train_conv_workspace_bytes(1, 7, 4, 88, 88, 1, 64, 0, 0, 0, 1)
out["dgrad_ws"] = lib.avsr_frontend_train_dgrad_workspace_bytes(4, 22, 22, 64, 128, 3, 3, 2, 1)
out["dgrad_ws_bad"] = lib.avsr_frontend_train_dgrad_workspace_bytes(4, 22, 22, 64, 100, 3, 3, 2, 1)
out["wgrad_ws"] = lib.avsr_frontend_train_wgrad_workspace_bytes(0, 4, 1, 22, 22, 64, 128, 1, 1, 2)
out["wgrad_ws_bad"] = lib.avsr_frontend_train_wgrad_workspace_bytes(0, -1, 1, 22, 22, 64, 128, 1, 1, 2)
out["bn_ws"] = lib.avsr_bn_train_workspace_bytes(1000, 64)
out["bn_ws_bad"] = lib.avsr_bn_train_workspace_bytes(1000, 0)
P = 1 << 20          # a non-NULL pointer value: every call below is refused before it could be dereferenced
need = out["conv_ws_trunk"]
out["rc_conv_null"] = lib.avsr_frontend_train_conv_fwd(None, P, P, P, 0, 4, 1, 22, 22, 64, 64, 3, 3, 1, P, need, 2, None)
out["rc_conv_small"] = lib.avsr_frontend_train_conv_fwd(P, P, P, P, 0, 4, 1, 22, 22, 64, 64, 3, 3, 1, P, need - 1, 2, None)
out["rc_conv_shape"] = lib.avsr_frontend_train_conv_fwd(P, P, P, P, 0, 4, 1, 22, 22, 65, 64, 3, 3, 1, P, need, 2, None)
out["rc_dgrad_small"] = lib.avsr_frontend_train_conv_dgrad(P, P, P, 4, 22, 22, 64, 128, 3, 3, 2, P, out["dgrad_ws"] - 1, 1, None)
out["rc_wgrad_null"] = lib.avsr_frontend_train_conv_wgrad(P, None, P, 0, 4, 1, 22, 22, 64, 128, 1, 1, 2, P, out["wgrad_ws"], 1, None)
out["rc_wgrad_prec"] = lib.avsr_frontend_train_conv_wgrad(P, P, P, 0, 4, 1, 22, 22, 64, 128, 1, 1, 2, P, out["wgrad_ws"], 7, None)
out["rc_bn_sums_small"] = lib.avsr_bn_train_bwd_sums(P, P, P, P, P, P, None, 1, P, 1000, 64, P, out["bn_ws"] - 1, None)
out["rc_finalize_bad"] = lib.avsr_bn_train_finalize(P, 0, 64, 1e-5, 0.1, None, None, P, P, None)
out["rc_finalize_half"] = lib.avsr_bn_train_finalize(P, 1, 64, 1e-5, 0.1, P, None, P, P, None)
out["rc_bn_fwd_null"] = lib.avsr_bn_train_act_fwd(P, P, P, P, None, None, 1, P, 10, 64, None)
out["rc_bn_dx_null"] = lib.avsr_bn_train_bwd_dx(P, P, P, P, P, P, None, 1, None, 0.1, P, None, 10, 64, None)
out["rc_pool_null"] = lib.avsr_frontend_train_maxpool_fwd(P, P, None, 1, 4, 4, 64, None)
out["rc_pool_bwd_shape"] = lib.avsr_frontend_train_maxpool_bwd(P, P, P, 1, 0, 4, 64, None)
out["rc_mean_null"] = lib.avsr_frontend_train_mean_rows(None, P, 2, 20, 512, None)
out["rc_mean_bwd_shape"] = lib.avsr_frontend_train_mean_rows_bwd(P, P, 2, 0, 512, None)
out["launches"] = lib.avsr_launch_count()
print(json.dumps(out))
""" % ROOT


def test_workspace_sizes_and_refusals_without_a_device():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", PROBE], capture_output=True, text=True, env=env, cwd=ROOT, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    for k in ("conv_ws_trunk", "conv_ws_vstem", "conv_ws_astem", "dgrad_ws", "wgrad_ws", "bn_ws"):
        assert out[k] > 0, k
    for k in ("conv_ws_bad_cin", "conv_ws_bad_stride", "conv_ws_bad_prec", "conv_ws_bad_audio", "conv_ws_bad_video_T",
              "dgrad_ws_bad", "wgrad_ws_bad", "bn_ws_bad"):
        assert out[k] == 0, k
    # the trunk conv's workspace holds the f16 input copy, the f16 weight rows, the unit scale / shift and the partials
    assert out["conv_ws_trunk"] >= 4 * 22 * 22 * 64 * 2 + 64 * 576 * 2
    assert out["rc_conv_small"] == 3 and out["rc_dgrad_small"] == 3 and out["rc_bn_sums_small"] == 3
    for k in ("rc_conv_null", "rc_conv_shape", "rc_wgrad_null", "rc_wgrad_prec", "rc_finalize_bad", "rc_finalize_half", "rc_bn_fwd_null",
              "rc_bn_dx_null", "rc_pool_null", "rc_pool_bwd_shape", "rc_mean_null", "rc_mean_bwd_shape"):
        assert out[k] == 1, k
    assert out["launches"] == 0
