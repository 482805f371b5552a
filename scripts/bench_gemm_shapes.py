#!/usr/bin/env python3
"""Time the S2 encoder's GEMMs at their real shapes, per tile / cluster shape, for one or more builds of the library.

    python scripts/bench_gemm_shapes.py [--lib NAME=PATH ...] [--tiles auto 128,1,2x1 ...] [--precision f16]

Each (build, tile) runs in its own process (AVSR_B200_LIB selects the build, AVSR_B200_TILE = "BN[,SPLITS[,CMxCN]]"
or "BN,sk" (stream-K) the tile; "auto" is the cost model's pick).  The residual shapes (w_2, out / pw2) go through
avsr_linear_operands_split with the encoder's split workspace, so they take the schedule they take in the forward.  Every shape replays a CUDA graph of 24 launches over 24 distinct weight
matrices, as bench.py's roofline does, and reports us per launch, TFLOP/s, the modelled L2 -> SM operand bytes of the
tile and cluster shape (each CTA pulls 1/CN of its A tile and 1/CM of its weight tile) and the implied GB/s.  QKV and
pw1 run here as plain LINEAR GEMMs with operand-typed output at the QKV / pw1 shapes; their scatter and GLU epilogues
write the same bytes."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# name, M, N, K, relu, operand-typed output, residual
SHAPES = [("ffn_w1", 1600, 3072, 768, 1, 1, 0), ("ffn_w2", 1600, 768, 3072, 0, 0, 1), ("qkv", 1600, 2304, 768, 0, 1, 0),
          ("pw1", 1600, 1536, 768, 0, 1, 0), ("out_pw2", 1600, 768, 768, 0, 0, 1)]

BODY = r'''
import json, sys, torch
sys.path.insert(0, %(root)r)
from auto_avsr_b200 import _cabi
from auto_avsr_b200.engine import PRECISIONS
dev = torch.device("cuda:0"); prec = %(prec)r
tdt = {"f16": torch.float16, "bf16": torch.bfloat16}.get(prec, torch.float32)
res = {}
for name, M, N, K, relu, opdest, resid in %(shapes)r:
    g = torch.Generator().manual_seed(7)
    x = torch.randn(M, K, generator=g).to(dev).to(tdt)
    ws = [((torch.rand(N, K, generator=g) - 0.5) * 0.07).to(dev).to(tdt) for _ in range(24)]
    b = torch.zeros(N, device=dev)
    y = torch.zeros(M, N, device=dev, dtype=tdt if opdest else torch.float32)
    r = y if resid else None
    # the residual GEMMs get the encoder's split workspace, so they take the schedule they take in the forward
    part = torch.empty(_cabi.SPLIT_PLANES * M * N, device=dev)
    cnt = torch.zeros(_cabi.SPLIT_COUNTERS, device=dev, dtype=torch.int32)
    st = torch.cuda.current_stream(dev).cuda_stream
    def go(w):
        if resid:
            _cabi.check(_cabi.lib.avsr_linear_operands_split(x.data_ptr(), w.data_ptr(), b.data_ptr(), r.data_ptr(),
                                                             0.5, y.data_ptr(), M, N, K, relu, opdest,
                                                             PRECISIONS[prec], part.data_ptr(), cnt.data_ptr(), st))
        else:
            _cabi.check(_cabi.lib.avsr_linear_operands(x.data_ptr(), w.data_ptr(), b.data_ptr(), None, 0.5,
                                                       y.data_ptr(), M, N, K, relu, opdest, PRECISIONS[prec], st))
    for w in ws[:3]: go(w)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st = torch.cuda.current_stream(dev).cuda_stream
        for w in ws: go(w)
    graph.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    e0.record()
    for _ in range(reps): graph.replay()
    e1.record(); torch.cuda.synchronize()
    res[name] = e0.elapsed_time(e1) * 1e3 / (reps * len(ws))
print("RESULT " + json.dumps(res))
'''


def tile_bytes(M, N, K, esz, tile):
    bn, cm, cn = 128, 1, 1
    if tile != "auto":
        parts = tile.split(",")
        bn = int(parts[0])
        if len(parts) > 2:
            cm, cn = (int(v) for v in parts[2].split("x"))
    tiles_m, tiles_n = -(-M // 128), -(-N // bn)
    # every CTA tile (edge tiles of a cluster included) pulls its share of A and W for the whole K
    ctiles = (-(-tiles_m // cm) * cm) * (-(-tiles_n // cn) * cn)
    return ctiles * (128 / cn + bn / cm) * K * esz


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="NAME=PATH of a libavsr_b200.so build")
    ap.add_argument("--tiles", nargs="*", default=["auto"])
    ap.add_argument("--precision", default="f16", choices=["f16", "bf16", "tf32"])
    args = ap.parse_args()
    libs = [tuple(s.split("=", 1)) for s in args.lib] or [("this", os.path.join(ROOT, "auto_avsr_b200", "csrc",
                                                                                   "libavsr_b200.so"))]
    esz = 2 if args.precision in ("f16", "bf16") else 4
    rows = []
    for name, path in libs:
        for tile in args.tiles:
            env = dict(os.environ, AVSR_B200_LIB=os.path.abspath(path))
            env.pop("AVSR_B200_TILE", None)
            if tile != "auto":
                env["AVSR_B200_TILE"] = tile
            r = subprocess.run([sys.executable, "-c", BODY % dict(root=ROOT, prec=args.precision, shapes=SHAPES)],
                               capture_output=True, text=True, env=env, timeout=600)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
            if r.returncode or not line:
                print(f"== {name} tile {tile}: FAILED\n{r.stdout[-800:]}{r.stderr[-1500:]}", flush=True)
                continue
            us = json.loads(line[0][7:])
            for sname, M, N, K, *_ in SHAPES:
                t = us[sname]
                by = tile_bytes(M, N, K, esz, tile)
                rows.append(dict(lib=name, tile=tile, shape=sname, us=round(t, 2),
                                 tflops=round(2.0 * M * N * K / t / 1e6, 1), mbytes=round(by / 1e6, 1),
                                 gbs=round(by / t / 1e3, 0)))
                print(f"{name:6s} {tile:10s} {sname:8s} {t:8.2f} us {rows[-1]['tflops']:7.1f} TFLOP/s "
                      f"{rows[-1]['mbytes']:8.1f} MB {rows[-1]['gbs']:8.0f} GB/s", flush=True)
    print("JSON " + json.dumps(rows))


if __name__ == "__main__":
    main()
