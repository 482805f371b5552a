"""Build the host replays of tests/emu into tests/emu/_build/ and bind them with the SAME ctypes signatures the package
uses for libavsr_b200.so.  TEST INFRASTRUCTURE ONLY.

Targets:
  decoder        decoder_emu.cu        the one-utterance decoder / CTC-prefix entries (csrc/decoder_body.cuh)
  decoder_batch  decoder_batch_emu.cu  the same plus the batched entries
  ctc            ctc_loss_emu.cu       the CTC loss schedule (csrc/ctc_loss_body.cuh)
  decoder_train  decoder_train_emu.cu  the decoder-training kernels' schedule (csrc/decoder_train_body.cuh)

A replay library is rebuilt when any csrc/*.cuh, include/avsr_b200.h or tests/emu/*.cu is newer than it."""
import ctypes as C
import glob
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
TARGETS = {"decoder": "decoder_emu.cu", "decoder_batch": "decoder_batch_emu.cu", "ctc": "ctc_loss_emu.cu",
           "decoder_train": "decoder_train_emu.cu"}


def _deps():
    return (glob.glob(os.path.join(ROOT, "auto_avsr_b200", "csrc", "*.cuh")) +
            [os.path.join(ROOT, "include", "avsr_b200.h")] + glob.glob(os.path.join(HERE, "*.cu")))


def build(target: str) -> str:
    src = os.path.join(HERE, TARGETS[target])
    out = os.path.join(HERE, "_build", "libavsr_" + TARGETS[target].replace(".cu", ".so"))
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in _deps()):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC",
               "--expt-relaxed-constexpr", "-shared", "-o", out, src]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"{target} emu build failed:\n{r.stdout}\n{r.stderr}")
    return out


def load(target: str = "decoder"):
    """the replay library of `target`, every symbol of _cabi.SIGNATURES it defines bound like the package binds it"""
    from auto_avsr_b200 import _cabi
    lib = C.CDLL(build(target))
    for name, (res, args) in _cabi.SIGNATURES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return lib
