#!/usr/bin/env python3
"""Time the CTC head of the training step (CTC.forward + backward: hs_pad -> ctc_lo -> CTC loss -> gradients of hs_pad,
ctc_lo.weight, ctc_lo.bias) with CUDA events, for the drop-in and for the reference module on the same GPU.

    python scripts/bench_ctc_loss.py [--steps 50] [--warmup 10] [--shapes S2,S3]

Shapes are SURVEY.md's S2 (4 x 400 frames) and S3 (16 x 100), d 768, odim 5049, label length a quarter of the frames.
Arms: the drop-in (auto_avsr_b200.CTC) at f16 / tf32 / fp32 GEMM precision; the reference CTC (ctc.py: eager ctc_lo,
log_softmax, torch.nn.CTCLoss) in fp32 and with allow_tf32, imported from oracle/_ref when it was built (skipped
otherwise).  Also the time of each library kernel of the loss (torch.profiler, a separate run) next to the bound from
shapes: the forward reads the valid logits once, the backward reads them again and writes dlogits, at the H100 SXM's
3.35 TB/s.  The kernels are profiled in a child process without programmatic dependent launch.  Prints one JSON
object with the device name and its power limit; writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from auto_avsr_b200 import CTC  # noqa: E402
from auto_avsr_b200.synthetic import SHAPES, encoder_input, head_state_dict  # noqa: E402
from auto_avsr_b200.train import ctc_loss_backward, ctc_loss_forward  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
D, ODIM = 768, 5049


def device_info():
    p = torch.cuda.get_device_properties(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"device": p.name, "power_limit": pl or "unknown", "sm_count": p.multi_processor_count}


def inputs(shape, dev):
    lengths = list(SHAPES[shape])
    B, T = len(lengths), max(lengths)
    g = torch.Generator().manual_seed(7)
    L = T // 4
    ys = torch.randint(1, ODIM, (B, L), generator=g)
    hs = encoder_input(lengths, D, 11).to(dev)
    return hs, torch.tensor(lengths, device=dev), ys.to(dev)


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def step_fn(module, hs, hlens, ys):
    x = hs.clone().requires_grad_(True)

    def fn():
        module.ctc_lo.weight.grad = module.ctc_lo.bias.grad = x.grad = None
        loss, _ = module(x, hlens, ys)
        loss.backward()
    return fn


def reference_ctc():
    from oracle import build_ref
    if not build_ref.available():
        return None
    build_ref.import_reference_encoder()
    from espnet.nets.pytorch_backend.ctc import CTC as RefCTC
    return RefCTC


def kernel_times(hs, hlens, ys, module, steps):
    """per-kernel mean device time (us) of the loss's library kernels from one profiled run"""
    with torch.no_grad():
        logits = torch.nn.functional.linear(hs, module.ctc_lo.weight, module.ctc_lo.bias).contiguous()
    dnll = torch.full((hs.size(0),), 1.0 / hs.size(0), device=hs.device)
    for _ in range(3):
        nll, saved = ctc_loss_forward(logits, hlens, ys, ODIM, -1, want_grad=True)
        ctc_loss_backward(logits, saved, ODIM, dnll)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            nll, saved = ctc_loss_forward(logits, hlens, ys, ODIM, -1, want_grad=True)
            ctc_loss_backward(logits, saved, ODIM, dnll)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "ctc_" in ev.key and "kernel" in ev.key:
            name = ev.key.split("(")[0].split("::")[-1]
            out[name] = round(ev.device_time_total / max(ev.count, 1), 2)
    return out


def kernel_times_child(shape):
    """kernel_times in a child process with programmatic dependent launch off (AVSR_B200_PDL=0): under PDL a kernel
    starts early and waits for its predecessor, which the profiler would count as the kernel's own time"""
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernels-only", shape], capture_output=True, text=True,
                       env=dict(os.environ, AVSR_B200_PDL="0"), timeout=600)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-2000:])
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--shapes", default="S2,S3")
    ap.add_argument("--kernels-only", metavar="SHAPE", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ctc_loss.py needs a CUDA GPU")
    dev = torch.device("cuda:0")
    sd = head_state_dict(0, 512, D, ODIM)
    if args.kernels_only:
        hs, hlens, ys = inputs(args.kernels_only, dev)
        ours = CTC(ODIM, D, 0.0).to(dev)
        ours.load_state_dict({"ctc_lo.weight": sd["ctc.ctc_lo.weight"], "ctc_lo.bias": sd["ctc.ctc_lo.bias"]})
        print(json.dumps(kernel_times(hs, hlens, ys, ours, 20)))
        return
    RefCTC = reference_ctc()
    result = dict(device_info(), steps=args.steps, warmup=args.warmup, shapes={})
    for shape in args.shapes.split(","):
        hs, hlens, ys = inputs(shape, dev)
        B, T = hs.shape[:2]
        row = {"B": B, "T": T, "labels": ys.size(1), "ms": {}}
        ours = CTC(ODIM, D, 0.0).to(dev).train()
        ours.load_state_dict({"ctc_lo.weight": sd["ctc.ctc_lo.weight"], "ctc_lo.bias": sd["ctc.ctc_lo.bias"]})
        for prec in ("f16", "tf32", "fp32"):
            ours.precision = prec
            row["ms"][f"dropin_{prec}"] = round(time_ms(step_fn(ours, hs, hlens, ys), args.steps, args.warmup), 4)
        if RefCTC is not None:
            ref = RefCTC(ODIM, D, 0.0).to(dev).train()
            ref.load_state_dict({"ctc_lo.weight": sd["ctc.ctc_lo.weight"], "ctc_lo.bias": sd["ctc.ctc_lo.bias"]})
            for tag, tf32 in (("reference_fp32", False), ("reference_tf32", True)):
                old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
                torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
                row["ms"][tag] = round(time_ms(step_fn(ref, hs, hlens, ys), args.steps, args.warmup), 4)
                torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
        else:
            row["reference"] = "oracle/_ref not built: reference arm skipped"
        logit_bytes = B * T * ODIM * 4
        row["kernel_us"] = kernel_times_child(shape)
        row["bound_us"] = {"forward_reads_logits": round(logit_bytes / HBM_BYTES_PER_S * 1e6, 2),
                           "backward_reads_logits_writes_dlogits": round(2 * logit_bytes / HBM_BYTES_PER_S * 1e6, 2),
                           "logits_MB": round(logit_bytes / 1e6, 1)}
        result["shapes"][shape] = row
    print(json.dumps(result))


if __name__ == "__main__":
    main()
