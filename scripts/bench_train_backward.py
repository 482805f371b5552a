"""Where the encoder's backward spends its time, default backward against ``backward_precision="bf16"``.

  attention   the rel-pos attention backward per call at the bucket shapes of synthetic.SHAPES (12 heads): the fp32
              CUDA-core kernels (avsr_relpos_attention_bwd) against the tensor-core bf16 kernels
              (avsr_relpos_attention_bwd_tc), CUDA events around many launches after a warm-up
  step        the 12-layer encoder training step (forward + backward) at S2 with the reference's dropout rates and
              batch-statistics BatchNorm, the two backwards alternated in one process for --rounds rounds; medians
  --profile   instead: a torch.profiler kernel table of one step of each (run it on its own: tracing slows the host)

Prints the card name and power limit with the numbers, and one JSON line at the end.

    python scripts/bench_train_backward.py [--rounds 7] [--steps 3] [--calls 20] [--profile] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:              # noqa: BLE001
        q = torch.cuda.get_device_name(0) + ", power limit not readable"
    return q


def attention_per_call(calls):
    import torch
    from auto_avsr_b200.synthetic import SHAPES
    from auto_avsr_b200.train import relpos_attention_bwd
    dev = torch.device("cuda:0")
    H = 12
    out = {}
    for name, lengths in SHAPES.items():
        B, T = len(lengths), max(lengths)
        g = torch.Generator(device=dev).manual_seed(1)
        q, k, v, o, r = (torch.randn(B, T, H * 64, device=dev, generator=g) for _ in range(5))
        p = torch.randn(2 * T - 1, H * 64, device=dev, generator=g)
        u, vb = (torch.randn(H, 64, device=dev, generator=g) for _ in range(2))
        ln = torch.tensor(lengths, dtype=torch.int32, device=dev)
        row = {}
        for prec in ("fp32", "bf16"):
            run = lambda: relpos_attention_bwd(q, k, v, p, u, vb, ln, o, r, H, precision=prec)   # noqa: E731
            for _ in range(3):
                run()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(calls):
                run()
            e1.record()
            torch.cuda.synchronize()
            row[prec + "_ms"] = e0.elapsed_time(e1) / calls
        row["speedup"] = row["fp32_ms"] / row["bf16_ms"]
        out[f"{name} (B {B}, T {T}, H {H})"] = row
        print(f"attention backward {name:4s} B {B:2d} T {T:4d}: fp32 {row['fp32_ms']:8.3f} ms  bf16 {row['bf16_ms']:7.3f} ms"
              f"  x{row['speedup']:.1f}", flush=True)
    return out


def make_encoder():
    import torch
    from auto_avsr_b200 import ConformerEncoder
    from auto_avsr_b200.synthetic import SHAPES, encoder_input, encoder_state_dict
    from oracle import conformer_oracle as O
    dev = torch.device("cuda:0")
    lengths = SHAPES["S2"]
    enc = ConformerEncoder(num_blocks=12)              # reference dropout rates (0.1, 0.1, 0.0)
    enc.load_state_dict(encoder_state_dict(3, num_blocks=12), strict=True)
    enc = enc.to(dev).train()
    xs = encoder_input(lengths, 768, 7).to(dev)
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)
    return enc, xs, mask


def step(enc, xs, mask):
    enc.zero_grad(set_to_none=True)
    enc(xs, mask)[0].pow(2).mean().backward()


def train_step(rounds, steps):
    import statistics
    import torch
    enc, xs, mask = make_encoder()
    times = {"default": [], "bf16": []}
    for label in times:                                # warm-up of both
        enc.backward_precision = None if label == "default" else "bf16"
        for _ in range(2):
            step(enc, xs, mask)
    torch.cuda.synchronize()
    for rnd in range(rounds):
        for label in (("default", "bf16") if rnd % 2 == 0 else ("bf16", "default")):
            enc.backward_precision = None if label == "default" else "bf16"
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                step(enc, xs, mask)
            torch.cuda.synchronize()
            times[label].append((time.perf_counter() - t0) / steps * 1e3)
    out = {k: {"median_ms": statistics.median(v), "runs_ms": v} for k, v in times.items()}
    out["speedup"] = out["default"]["median_ms"] / out["bf16"]["median_ms"]
    print(f"S2 training step: default {out['default']['median_ms']:.1f} ms  bf16 backward {out['bf16']['median_ms']:.1f} ms"
          f"  x{out['speedup']:.2f}  (medians of {rounds} alternated rounds of {steps} steps)", flush=True)
    return out


def profile(outdir):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    enc, xs, mask = make_encoder()
    result = {}
    for label, bp in (("default", None), ("bf16", "bf16")):
        enc.backward_precision = bp
        for _ in range(2):
            step(enc, xs, mask)
        torch.cuda.synchronize()
        with tprof(activities=[ProfilerActivity.CUDA]) as prof:
            step(enc, xs, mask)
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)
        print(f"---- kernel table, one S2 training step, backward {label}\n{table}", flush=True)
        total = sum(e.device_time_total for e in prof.key_averages())
        result[label] = {"kernels_us_total": total,
                         "top": [{"name": e.key[:90], "us": e.device_time_total, "calls": e.count}
                                 for e in sorted(prof.key_averages(), key=lambda e: -e.device_time_total)[:25]]}
        if outdir:
            with open(os.path.join(outdir, f"train_step_kernels_{label}.txt"), "w") as f:
                f.write(table)
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the kernel tables and the JSON result")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_train_backward.py needs a CUDA GPU")
    import __graft_entry__ as g
    g.build()
    info = card()
    print(f"card: {info}", flush=True)
    res = {"card": info}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    if a.profile:
        res["profile"] = profile(a.out)
    else:
        res["attention_backward"] = attention_per_call(a.calls)
        res["train_step_s2"] = train_step(a.rounds, a.steps)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(os.path.join(a.out, "bench_train_backward" + ("_profile" if a.profile else "") + ".json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
