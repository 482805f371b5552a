#!/usr/bin/env python3
"""Per-kernel attribution of the encoder forward on the GPU, for one or more builds of the library.

    python scripts/profile_forward.py [--lib NAME=PATH ...] [--shapes S2 S2r S3 S4] [--precision f16 bf16 tf32]
                                      [--steps N] [--dump DIR]

Each build runs in its own process (AVSR_B200_LIB selects it, as in scripts/bench_gemm_shapes.py).  For every shape and
precision the 12-layer encoder (bench.py's synthetic weights and inputs, eval) runs WITHOUT its CUDA graph, so every
launch is a kernel of its own in the trace:
  1. ms per forward from CUDA events, profiler off;
  2. a separate window under torch.profiler (CUDA activity only): each kernel's device time per forward and its share
     of the summed kernel time (the forked linear_pos branch overlaps the main stream, so the shares are of kernel
     time, not of wall time);
  3. the attention kernel's us per launch and its rate on executed FLOPs (every 64-query x 64-key tile that holds a
     row < T and a key < L_b: S 64x64x64, G 64x128x64 over the rel-pos band, P.V 64x64x64) and on the FLOPs
     bench.algorithmic_flops credits (4 * 64 * L_b^2 per head), against the data-sheet dense peak of the operand type.
Kernels launch with programmatic dependent launch (PDL) in the product: a kernel starts while its predecessor drains
and waits inside, so its trace duration includes that wait.  The attribution therefore runs with AVSR_B200_PDL=0
(each kernel's own duration; the events time is then the PDL-off forward too) unless --pdl is given.
The card name, power limit and max SM clock are read in the same process.  --dump DIR writes every shape's encoder
output to DIR/<build>/<shape>_<precision>.npy so that two builds can be compared byte for byte."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ATTN = "attention_wg_kernel"   # the rel-pos attention kernel (csrc/attention_tc.cu)
PEAK_TFLOPS = {"f16": 989.0, "bf16": 989.0, "tf32": 495.0}   # NVIDIA H100 SXM data sheet, dense, at a 700 W power limit


def attention_flops(lengths, heads=12):
    """(executed, credited) attention FLOPs of ONE layer."""
    T = max(lengths)
    tile = 2 * 64 * 64 * 64 + 2 * 64 * 128 * 64 + 2 * 64 * 64 * 64
    executed = sum(heads * -(-T // 64) * -(-L // 64) * tile for L in lengths)
    credited = 4 * 64 * heads * sum(L * L for L in lengths)
    return executed, credited


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = (c.strip() for c in r.stdout.splitlines()[0].split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:      # noqa: BLE001
        return {"error": f"{type(e).__name__}: {e}"}


def child(args):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from auto_avsr_b200 import ConformerEncoder
    from auto_avsr_b200.synthetic import SHAPES, encoder_input, encoder_state_dict

    assert torch.cuda.is_available(), "profile_forward.py needs a GPU"
    dev = torch.device("cuda:0")
    cfg = dict(d_model=768, n_heads=12, linear_units=3072, num_blocks=12, cnn_kernel=31)
    enc = ConformerEncoder(attention_dim=768, attention_heads=12, linear_units=3072, num_blocks=12, cnn_module_kernel=31)
    enc.load_state_dict(encoder_state_dict(0, **cfg), strict=True)
    enc = enc.to(dev).eval()
    enc.use_graph = False
    enc.assume_frozen = True
    out = {"card": card(), "rows": []}
    for prec in args.precision:
        enc.precision = prec
        for name in args.shapes:
            lengths = list(SHAPES[name])
            xs = encoder_input(lengths, 768, 1234).to(dev)
            mask = (torch.arange(max(lengths), device=dev)[None, :] <
                    torch.tensor(lengths, device=dev)[:, None]).unsqueeze(1)
            with torch.no_grad():
                for _ in range(5):
                    y, _ = enc(xs, mask)
                torch.cuda.synchronize()
                if args.dump:
                    os.makedirs(args.dump, exist_ok=True)
                    np.save(os.path.join(args.dump, f"{name}_{prec}.npy"), y.float().cpu().numpy())
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    enc(xs, mask)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.steps
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.steps):
                        enc(xs, mask)
                    torch.cuda.synchronize()
            kernels = {}
            for ev in prof.key_averages():
                t = ev.self_device_time_total
                if t > 0:
                    k = kernels.setdefault(ev.key, [0.0, 0])
                    k[0] += t / args.steps
                    k[1] += ev.count / args.steps
            total = sum(v[0] for v in kernels.values())
            table = sorted(({"kernel": k, "us_per_forward": v[0], "launches_per_forward": v[1], "share": v[0] / total}
                            for k, v in kernels.items()), key=lambda r: -r["us_per_forward"])
            row = {"shape": name, "precision": prec, "lengths": lengths, "ms_per_forward": ms,
                   "kernel_us_per_forward": total, "kernels": table}
            att = [r for r in table if ATTN in r["kernel"]]
            if att:
                a = att[0]
                us = a["us_per_forward"] / a["launches_per_forward"]
                ex, cr = attention_flops(lengths)
                row["attention"] = {"kernel": a["kernel"], "us_per_launch": us, "share": a["share"],
                                    "tflops_executed": ex / us / 1e6, "tflops_credited": cr / us / 1e6,
                                    "frac_of_datasheet_peak_executed": ex / us / 1e6 / PEAK_TFLOPS[prec]}
            out["rows"].append(row)
    print("RESULT " + json.dumps(out))


def short(k, n=60):
    return k if len(k) <= n else k[:n - 3] + "..."


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="NAME=PATH of a libavsr_b200.so build")
    ap.add_argument("--shapes", nargs="*", default=["S2", "S2r", "S3", "S4"])
    ap.add_argument("--precision", nargs="*", default=["f16"], choices=["f16", "bf16", "tf32"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--top", type=int, default=12, help="kernels listed per shape")
    ap.add_argument("--dump", metavar="DIR", default=None)
    ap.add_argument("--pdl", action="store_true", help="keep programmatic dependent launch on (durations overlap)")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    libs = [tuple(s.split("=", 1)) for s in args.lib] or [("this", os.path.join(ROOT, "auto_avsr_b200", "csrc",
                                                                               "libavsr_b200.so"))]
    results = {}
    for name, path in libs:
        env = dict(os.environ, AVSR_B200_LIB=os.path.abspath(path))
        if not args.pdl:
            env["AVSR_B200_PDL"] = "0"
        cmd = [sys.executable, os.path.abspath(__file__), "--child", "--steps", str(args.steps),
               "--shapes", *args.shapes, "--precision", *args.precision]
        if args.dump:
            cmd += ["--dump", os.path.join(args.dump, name)]
        r = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=1800)
        line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
        if r.returncode or not line:
            print(f"== {name}: FAILED\n{r.stdout[-800:]}{r.stderr[-2000:]}", flush=True)
            continue
        res = results[name] = json.loads(line[0][7:])
        print(f"== {name} ({path}) on {res['card']}, PDL {'on' if args.pdl else 'off'}", flush=True)
        for row in res["rows"]:
            print(f"-- {row['shape']} {row['precision']}: {row['ms_per_forward']:.3f} ms/forward (events, no profiler), "
                  f"kernel time {row['kernel_us_per_forward']:.1f} us/forward")
            for k in row["kernels"][:args.top]:
                print(f"   {k['us_per_forward']:9.1f} us {100 * k['share']:5.1f} % {k['launches_per_forward']:6.1f}x  "
                      f"{short(k['kernel'])}")
            a = row.get("attention")
            if a:
                print(f"   attention: {a['us_per_launch']:.2f} us/launch, {100 * a['share']:.1f} % of kernel time, "
                      f"{a['tflops_executed']:.1f} TFLOP/s executed ({100 * a['frac_of_datasheet_peak_executed']:.1f} % "
                      f"of the {PEAK_TFLOPS[row['precision']]:.0f} TFLOP/s data sheet), "
                      f"{a['tflops_credited']:.1f} TFLOP/s credited", flush=True)
    print("JSON " + json.dumps(results))


if __name__ == "__main__":
    main()
