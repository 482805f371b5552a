"""Build tests/emu/_build/libavsr_decoder_train_emu.so (the host replay of csrc/decoder_train_body.cuh) and bind it with
the SAME ctypes signatures the package uses for libavsr_b200.so.  A third target beside the decoder and CTC replays
(tests/emu/build.py, tests/emu/build_ctc.py), built the same way.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC = os.path.join(HERE, "decoder_train_emu.cu")
OUT = os.path.join(HERE, "_build", "libavsr_decoder_train_emu.so")
CSRC = os.path.join(ROOT, "auto_avsr_b200", "csrc")
DEPS = [SRC, os.path.join(CSRC, "decoder_train_body.cuh"), os.path.join(CSRC, "decoder_body.cuh"),
        os.path.join(CSRC, "common.cuh"), os.path.join(ROOT, "include", "avsr_b200.h")]
EMU_SYMBOLS = ["avsr_last_error", "avsr_mha_core_fwd", "avsr_mha_core_bwd_workspace_bytes", "avsr_mha_core_bwd",
               "avsr_label_smoothing_fwd", "avsr_label_smoothing_bwd", "avsr_embed_fwd", "avsr_embed_bwd_workspace_bytes",
               "avsr_embed_bwd"]


def build() -> str:
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in DEPS):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC",
               "--expt-relaxed-constexpr", "-shared", "-o", OUT, SRC]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"decoder-train emu build failed:\n{r.stdout}\n{r.stderr}")
    return OUT


def load():
    from auto_avsr_b200 import _cabi
    lib = C.CDLL(build())
    for name in EMU_SYMBOLS:
        res, args = _cabi.SIGNATURES[name]
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib
