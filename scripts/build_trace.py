#!/usr/bin/env python3
"""Diagnostic build: the same sources compiled with -DAVSR_TRACE into auto_avsr_b200/csrc/libavsr_b200_trace.so.
The GEMM and the elementwise kernels then record %globaltimer when a CTA opens, when its dependency resolved and when
it is done, one record per CTA (common.cuh, "phase trace"); avsr_trace_set binds the buffer.  Use with
AVSR_B200_LIB=<that file>."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

OUT = os.path.join(g.CSRC, "libavsr_b200_trace.so")


def main() -> None:
    objdir = os.path.join(g.CSRC, "build_trace")
    os.makedirs(objdir, exist_ok=True)
    nvcc = g._nvcc()

    def one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc] + g.NVCC_FLAGS + ["-DAVSR_TRACE"] + (["-DAVSR_TRACE_EPI"] if os.environ.get("AVSR_TRACE_EPI") else []) + ["-c", os.path.join(g.CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise SystemExit(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(one, g.SOURCES))
    r = subprocess.run([nvcc, "-shared", "-o", OUT] + objs, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(f"link failed:\n{r.stdout}\n{r.stderr}")
    print(OUT)


if __name__ == "__main__":
    main()
