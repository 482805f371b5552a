"""The bf16 precision mode without a GPU: the host-side contract of AVSR_PREC_BF16 (= 16) against AVSR_PREC_F16 (= 2),
the host replay's bf16 operand store against torch's rounding, and the Python surface that resolves "bf16".

Every probe runs in a subprocess with CUDA_VISIBLE_DEVICES="", so no call can reach a device."""
import ctypes as C
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(ROOT, "auto_avsr_b200", "csrc", "libavsr_b200.so")
PF16, PBF16 = 2, 16

needs_nvcc = pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"),
                                reason="nvcc is needed to build the host replay")

# Runs the host-contract probe table of test_host_contract_cpu.py against a library with one precision constant of
# that module replaced ("P32" for the decoder probes, which all run in fp32, "PF16" for the rest): the refused calls
# must answer exactly as with the original constant.
_PROBE = r"""
import json, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {here!r})
import ctypes as C
import test_host_contract_cpu as H
if {const!r}:
    setattr(H, {const!r}, {value!r})
lib = C.CDLL({lib!r})
print(json.dumps(H._probe(lib, {decoder_only!r}), sort_keys=True))
"""


def _probe(lib, const=None, value=None, decoder_only=False):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    code = _PROBE.format(root=ROOT, here=HERE, const=const, value=value, lib=lib, decoder_only=decoder_only)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _sizes(lib):
    """every *_bytes entry that takes a precision, over the host-contract grid, at f16 and at bf16"""
    from auto_avsr_b200 import _cabi as A
    for name, (res, args) in A.SIGNATURES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    pairs = []
    for rows, n, k in ((0, 8, 64), (37, 768, 3072), (5, 0, 64), (1600, 3072, 768)):
        pairs.append(("avsr_linear_workspace_bytes", (rows, n, k)))
    for mod in (0, 1, 2):
        pairs.append(("avsr_frontend_prepared_bytes", (mod,)))
        for B, T, H, W in ((2, 29, 88, 88), (1, 1, 45, 61), (2, 16000, 1, 1), (0, 5, 88, 88), (1, 5, 0, 88),
                           (-1, 5, 88, 88)):
            pairs.append(("avsr_frontend_workspace_bytes", (mod, B, T, H, W)))
    for g in ((2, 22, 22, 64, 64, 3, 3, 1), (2, 22, 22, 64, 128, 1, 1, 2), (0, 22, 22, 64, 64, 3, 3, 1),
              (2, 0, 22, 64, 64, 3, 3, 1), (2, 22, 22, 64, 64, 3, 3, 0)):
        pairs.append(("avsr_conv_bn_act_workspace_bytes", g))
    for g in ((1, 2, 29, 88, 88, 1, 64, 7, 7, 2), (0, 2, 1, 22, 22, 64, 64, 3, 3, 1), (0, 2, 1, 22, 22, 64, 128, 1, 1, 2),
              (1, 2, 1, 1, 16000, 1, 64, 1, 80, 4), (0, 0, 1, 22, 22, 64, 64, 3, 3, 1)):
        pairs.append(("avsr_frontend_train_conv_workspace_bytes", g))
    for g in ((2, 22, 22, 64, 64, 3, 3, 1), (2, 22, 22, 64, 128, 3, 3, 2), (2, 22, 22, 64, 128, 1, 1, 2)):
        pairs.append(("avsr_frontend_train_dgrad_workspace_bytes", g))
    out = {}
    for name, a in pairs:
        if not hasattr(lib, name):
            continue
        out[f"{name}{a!r}"] = [int(getattr(lib, name)(*a, p)) for p in (PF16, PBF16)]
    return out


_SIZES = r"""
import json, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {here!r})
import ctypes as C
import test_bf16_cpu as T
print(json.dumps(T._sizes(C.CDLL({lib!r}))))
"""


def test_every_bytes_entry_gives_the_f16_value():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", _SIZES.format(root=ROOT, here=HERE, lib=LIB)], capture_output=True,
                       text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    table = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(table) >= 38
    assert any(v[0] > 0 for v in table.values())
    diff = {k: v for k, v in table.items() if v[0] != v[1]}
    assert not diff, diff


def _norm(text):
    return text.replace("AVSR_PREC_BF16", "AVSR_PREC_F16")


def test_refused_calls_answer_as_with_f16():
    """Every call of the host-contract table that runs at AVSR_PREC_F16 (refused before launch: too small, NULL, bad
    shape) answers with the same code and, up to the precision's name, the same text at AVSR_PREC_BF16."""
    base = _probe(LIB)
    bf = _probe(LIB, "PF16", PBF16)
    assert set(base) == set(bf)
    diff = {k: (base[k], bf[k]) for k in base
            if (base[k] != bf[k] if not isinstance(base[k], list) else
                (base[k][0], _norm(base[k][1])) != (bf[k][0], _norm(bf[k][1])))}
    assert not diff, diff


@needs_nvcc
def test_emu_decoder_probes_with_bf16_match_product():
    """The decoder probes rerun at AVSR_PREC_BF16: the host replay answers each as the product library does, and both
    answer as they do in fp32."""
    from emu import build
    emu = build.build("decoder_batch")
    prod_bf = _probe(LIB, "P32", PBF16, decoder_only=True)
    emu_bf = _probe(emu, "P32", PBF16, decoder_only=True)
    prod_32 = _probe(LIB, decoder_only=True)
    assert set(prod_bf) == set(emu_bf) == set(prod_32)
    diff = {k: (prod_bf[k], emu_bf[k]) for k in prod_bf if prod_bf[k] != emu_bf[k]}
    assert not diff, diff
    diff = {k: (prod_bf[k], prod_32[k]) for k in prod_bf if prod_bf[k] != prod_32[k]}
    assert not diff, diff


def _edge_values():
    bmax = float(torch.finfo(torch.bfloat16).max)
    vals = [1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 1.0 + 2.0 ** -9, 2.0 ** 100 * (1 + 2.0 ** -8),
            1.0 + 2.0 ** -8 + 2.0 ** -20,                                            # ties and just past a tie
            0.0, -0.0, 1e-40, -1e-40, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -126 * 0.75, 2.0 ** -133 * 1.5,   # subnormals
            float("inf"), -float("inf"), float("nan"), -float("nan"),
            65504.0 * 4, -65504.0 * 4, 65520.0, 65536.0,
            bmax, -bmax, float(np.nextafter(np.float32(bmax), np.float32(np.inf))), 3.3961e38,
            float(np.finfo(np.float32).max), -float(np.finfo(np.float32).max)]
    g = torch.Generator().manual_seed(4)
    rand = (torch.randn(4096 - len(vals), generator=g) * torch.exp2(torch.randint(-30, 30, (4096 - len(vals),),
                                                                                  generator=g).float()))
    return torch.cat([torch.tensor(vals, dtype=torch.float32), rand.float()])


@needs_nvcc
def test_emu_store_operand_bf16_matches_torch_bits():
    """The host replay's store_operand (what avsr_prepare_decoder converts weights with) against torch's CPU
    .to(torch.bfloat16): bit for bit except NaN's payload (both NaN)."""
    from emu import build
    from auto_avsr_b200 import _cabi as A
    lib = build.load("decoder")
    cfg = A.DecoderConfig(64, 2, 128, 2, 11)
    D = 64
    v = _edge_values()
    assert v.numel() == D * D
    keep = []

    def buf(n, src=None):
        t = torch.zeros(n, dtype=torch.float32) if src is None else src.contiguous()
        keep.append(t)
        return t.data_ptr()

    fields = [buf(D * D, v) if f == "self_q_w" else buf(4096) for f, _ in A.DECODER_LAYER_FIELDS]
    layers = (A.DecoderLayerParams * 2)(*[A.DecoderLayerParams(*fields)] * 2)
    nbytes = int(lib.avsr_decoder_prepared_bytes(C.byref(cfg)))
    prep = torch.zeros(nbytes, dtype=torch.uint8)
    rc = lib.avsr_prepare_decoder(C.byref(cfg), layers, buf(11 * D), buf(D), buf(D), buf(11 * D), buf(11),
                                  prep.data_ptr(), nbytes, PBF16, None)
    assert rc == 0, lib.avsr_last_error()
    got = prep[:2 * D * D].view(torch.bfloat16)           # layer 0's q rows lead its q|k|v block
    want = v.to(torch.bfloat16)
    nan = torch.isnan(want.float())
    assert torch.equal(torch.isnan(got.float()), nan)
    assert torch.equal(got[~nan].view(torch.int16), want[~nan].view(torch.int16))


def test_python_resolves_bf16_everywhere(monkeypatch):
    from auto_avsr_b200 import _cabi, engine, train
    assert engine.PRECISIONS["bf16"] == _cabi.PREC_BF16 == 16
    assert len(set(engine.PRECISIONS.values())) == len(engine.PRECISIONS)      # cache keys never alias
    assert train.bwd_precision("bf16") == "tf32"
    monkeypatch.setenv("AVSR_B200_PRECISION", "bf16")
    assert engine.default_precision() == "bf16"
    from auto_avsr_b200 import ConformerEncoder, CTC, TransformerDecoder
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet
    for m in (ConformerEncoder(num_blocks=1), CTC(11, 768, 0.0), TransformerDecoder(11, 64, 2, 128, 1), Conv1dResNet()):
        assert engine.PRECISIONS[getattr(m, "precision", None) or engine.default_precision()] == 16
