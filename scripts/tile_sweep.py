#!/usr/bin/env python3
"""Time the encoder's GEMM shapes for every CTA tile shape (AVSR_B200_TILE override), warm L2, CUDA events."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BODY = r'''
import sys, torch
sys.path.insert(0, %(root)r)
from auto_avsr_b200 import _cabi
from auto_avsr_b200.engine import PRECISIONS
dev = torch.device("cuda:0"); prec = %(prec)r
tdt = torch.float16 if prec == "f16" else torch.float32
st = torch.cuda.current_stream(dev).cuda_stream
def run(name, M, N, K, relu, opdest, resid):
    x = torch.randn(M, K, device=dev).to(tdt)
    ws = [(torch.randn(N, K, device=dev) * 0.03).to(tdt) for _ in range(8)]
    b = torch.zeros(N, device=dev)
    y = torch.zeros(M, N, device=dev, dtype=tdt if opdest else torch.float32)
    r = y if resid else None
    def go(w):
        _cabi.check(_cabi.lib.avsr_linear_operands(x.data_ptr(), w.data_ptr(), b.data_ptr(), None if r is None else r.data_ptr(),
                                                   0.5, y.data_ptr(), M, N, K, relu, opdest, PRECISIONS[prec], st))
    global st
    for w in ws[:2]: go(w)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()          # replay from a graph: the python/ctypes launch path is slower than the kernel
    with torch.cuda.graph(g):
        st = torch.cuda.current_stream(dev).cuda_stream
        for w in ws: go(w)
    st = torch.cuda.current_stream(dev).cuda_stream
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / 40
    print(f"{name:8s} {us:7.2f} us  {2.0*M*N*K/us/1e6:7.1f} TFLOP/s")
run("ffn1", 1600, 3072, 768, 1, 1, 0)
run("ffn2", 1600, 768, 3072, 0, 0, 1)
run("out", 1600, 768, 768, 0, 0, 1)
run("n1536", 1600, 1536, 768, 0, 1, 0)
'''
prec = sys.argv[1] if len(sys.argv) > 1 else "f16"
for tile in (sys.argv[2:] or ["auto", "64", "128"]):          # AVSR_B200_TILE = "BN[,SPLITS]"
    env = dict(os.environ)
    if tile != "auto":
        env["AVSR_B200_TILE"] = tile
    r = subprocess.run([sys.executable, "-c", BODY % dict(root=ROOT, prec=prec)], capture_output=True, text=True, env=env,
                       timeout=300)
    print(f"== tile {tile}\n{r.stdout}{r.stderr[-600:] if r.returncode else ''}", flush=True)
