#!/usr/bin/env python3
"""On-GPU bring-up diagnostics for the tensor-core (wgmma) kernels: each case runs in its own subprocess (a trapped kernel
poisons the CUDA context) and prints the error structure against the fp32 CUDA-core path of the same library."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {
    "linear_small": "linear(128, 64, 32)",
    "linear_k": "linear(128, 64, 256)",
    "linear_mtail": "linear(200, 128, 128)",
    "linear_ffn1": "linear(1600, 3072, 768)",
    "linear_ffn2": "linear(1600, 768, 3072)",
    "linear_qk": "linear(1600, 1536, 768)",
    "linear_out": "linear(1600, 768, 768)",
    "attn_small": "attn(1, 64, 1, None)",
    "attn_130": "attn(1, 130, 2, None)",
    "attn_masked": "attn(2, 200, 2, [200, 77])",
    "attn_400": "attn(2, 400, 12, [400, 301])",
}

BODY = r'''
import sys, math, torch
sys.path.insert(0, %(root)r)
from auto_avsr_b200 import ops
dev = torch.device("cuda:0")
torch.manual_seed(0)
import os
PREC = os.environ.get("TC_PREC", "f16")

def report(name, y, ref):
    d = (y.double() - ref.double()).abs()
    scale = ref.abs().max().item()
    print(f"{name}: max-abs {d.max().item():.3e} rms {d.pow(2).mean().sqrt().item():.3e} (ref scale {scale:.3e})"
          f" finite={bool(torch.isfinite(y).all())}")
    if d.max().item() > 5e-3 * scale:
        bad = d > 5e-3 * scale
        print("  bad fraction", bad.float().mean().item())
        if y.dim() == 2:
            rows = bad.any(1).nonzero().flatten()[:16].tolist(); cols = bad.any(0).nonzero().flatten()[:16].tolist()
            print("  first bad rows", rows, "first bad cols", cols)
            print("  bad per 32-col chunk", bad.float().view(bad.size(0), -1, 32).mean((0, 2))[:12].tolist() if bad.size(1) %% 32 == 0 else "")
            print("  bad per 8-row group", bad.float()[: (bad.size(0)//8)*8].view(-1, 8, bad.size(1)).mean((1, 2))[:16].tolist())
            print("  y[0,:8]", y[0,:8].tolist()); print("  r[0,:8]", ref[0,:8].tolist())
            print("  ratio y/ref[0,:8]", (y[0,:8]/ref[0,:8]).tolist())

def linear(M, N, K):
    x = torch.randn(M, K, device=dev); w = torch.randn(N, K, device=dev) / math.sqrt(K); b = torch.randn(N, device=dev)
    ref = ops.linear(x, w, b, precision="fp32")
    y = ops.linear(x, w, b, precision=PREC)
    torch.cuda.synchronize()
    report(f"linear {M}x{N}x{K}", y, ref)

def attn(B, T, H, lengths):
    D = H * 64
    q, k, v = (torch.randn(B, T, D, device=dev) * 0.5 for _ in range(3))
    p = torch.randn(2 * T - 1, D, device=dev) * 0.5
    u, vb = torch.randn(H, 64, device=dev) * 0.3, torch.randn(H, 64, device=dev) * 0.3
    ln = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=dev)
    ref = ops.relpos_attention(q, k, v, p, u, vb, ln, H, precision="fp32")
    y = ops.relpos_attention(q, k, v, p, u, vb, ln, H, precision=PREC)
    torch.cuda.synchronize()
    report(f"attn B{B} T{T} H{H} {lengths}", y.view(B * T, D), ref.view(B * T, D))

%(call)s
'''

def main():
    names = sys.argv[1:] or list(CASES)
    for n in names:
        code = BODY % dict(root=ROOT, call=CASES[n])
        try:
            r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
            out = (r.stdout + ("\n" + r.stderr[-1500:] if r.returncode else "")).strip()
        except subprocess.TimeoutExpired:
            out = "TIMEOUT (hang)"
        print(f"== {n}\n{out}", flush=True)

if __name__ == "__main__":
    main()
