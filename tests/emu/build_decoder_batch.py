"""Build tests/emu/_build/libavsr_decoder_batch_emu.so (the host replay of csrc/decoder_body.cuh's one-utterance AND
batched entries) and bind it with the SAME ctypes signatures the package uses for libavsr_b200.so.  Built like
tests/emu/build.py.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC = os.path.join(HERE, "decoder_batch_emu.cu")
OUT = os.path.join(HERE, "_build", "libavsr_decoder_batch_emu.so")
DEPS = [SRC, os.path.join(HERE, "decoder_emu.cu"), os.path.join(ROOT, "auto_avsr_b200", "csrc", "decoder_body.cuh"),
        os.path.join(ROOT, "auto_avsr_b200", "csrc", "common.cuh"), os.path.join(ROOT, "include", "avsr_b200.h")]
EMU_SYMBOLS = ["avsr_last_error", "avsr_launch_count", "avsr_decoder_prepared_bytes", "avsr_prepare_decoder",
               "avsr_decoder_session_bytes", "avsr_decoder_begin", "avsr_decoder_step_workspace_bytes",
               "avsr_decoder_step", "avsr_ctc_prefix_init", "avsr_ctc_prefix_score", "avsr_ctc_prefix_select",
               "avsr_decoder_batch_session_bytes", "avsr_decoder_batch_step_workspace_bytes", "avsr_decoder_batch_begin",
               "avsr_decoder_batch_step", "avsr_ctc_prefix_batch_init", "avsr_ctc_prefix_batch_score"]


def build() -> str:
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in DEPS):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC",
               "--expt-relaxed-constexpr", "-shared", "-o", OUT, SRC]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"decoder-batch emu build failed:\n{r.stdout}\n{r.stderr}")
    return OUT


def load():
    from auto_avsr_b200 import _cabi
    lib = C.CDLL(build())
    for name in EMU_SYMBOLS:
        res, args = _cabi.SIGNATURES[name]
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib
