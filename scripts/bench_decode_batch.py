#!/usr/bin/env python3
"""Decoding a corpus one utterance at a time vs in lock-step batches (DeviceBeamSearch.forward vs forward_batch).

A seeded corpus of 64 encoder outputs of 25..155 frames (d 768) is decoded with synthetic weights (decoder_state_dict(4),
head_state_dict(4): 6-layer d=768 attention decoder + CTC prefix scorer, odim 5049, beam 40, ctc_weight 0.1) by
  sequential       forward() per utterance
  batch_U          forward_batch() over the corpus sorted by length and cut into batches of U = 1, 4, 8, 16, 32
Reports utterances/s, search steps, ms per step and the largest batch session per arm, checks in the same run that every
arm returns the sequential arm's n-best (token sequences and scores), and reads the GPU name and power limit.

  python scripts/bench_decode_batch.py [--sizes 1,4,8,16,32] [--utts 64]
  python scripts/bench_decode_batch.py --profile [--out DIR]   torch.profiler traces (to a temporary directory) of one
                                                              batch at U = 1 and U = 16, separate from the timing: top
                                                              kernels, device busy / idle time per step
AVSR_BENCH_DECODE_DRYRUN=1: CPU dry run of this script's plumbing on the tests' host replay (tiny sizes, no timing
value)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                   # noqa: BLE001
        return f"unavailable ({type(e).__name__})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,4,8,16,32")
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--beam", type=int, default=40)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "decode_batch_profile"))
    args = ap.parse_args()
    import torch
    from auto_avsr_b200 import CTC, TransformerDecoder
    from auto_avsr_b200.beam_search import DeviceBeamSearch
    from auto_avsr_b200.synthetic import decoder_state_dict, head_state_dict

    dry = os.environ.get("AVSR_BENCH_DECODE_DRYRUN") == "1"
    dev = torch.device("cpu" if dry else "cuda:0")
    sync = (lambda: None) if dry else torch.cuda.synchronize
    if dry:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from emu import build
        lib = build.load("decoder_batch")
        odim, d, H, ff, L, lo, hi = 37, 64, 1, 64, 1, 2, 9
        dsd = decoder_state_dict(4, odim, d, H, ff, L)
        hsd = head_state_dict(4, 64, d, odim)
    else:
        odim, d, H, ff, L, lo, hi = 5049, 768, 12, 3072, 6, 25, 155
        dsd, hsd = decoder_state_dict(4), head_state_dict(4)
    g = torch.Generator().manual_seed(2024)
    lengths = torch.randint(lo, hi + 1, (args.utts,), generator=g).tolist()
    corpus = [torch.randn(T, d, generator=g).to(dev) for T in lengths]
    dec = TransformerDecoder(odim=odim, attention_dim=d, attention_heads=H, linear_units=ff, num_blocks=L)
    dec.load_state_dict(dsd, strict=True)
    ctc = CTC(odim, d, 0.1)
    ctc.load_state_dict({"ctc_lo.weight": hsd["ctc.ctc_lo.weight"], "ctc_lo.bias": hsd["ctc.ctc_lo.bias"]})
    dec, ctc = dec.to(dev).eval(), ctc.to(dev).eval()
    if dry:
        class _CpuCTC(torch.nn.Module):                       # the drop-in CTC refuses CPU tensors
            def __init__(self, lo_):
                super().__init__()
                self.ctc_lo = lo_

            @torch.no_grad()
            def log_softmax(self, hs):
                return torch.log_softmax(self.ctc_lo(hs), dim=-1)
        ctc = _CpuCTC(ctc.ctc_lo)
        dec._lib, dec.precision = lib, "fp32"
    bs = DeviceBeamSearch(dec, ctc, beam_size=args.beam, vocab_size=odim)
    order = sorted(range(len(corpus)), key=lambda i: (lengths[i], i))

    def batches(U):
        for b in range(0, len(order), U):
            ids = order[b:b + U]
            lens = [lengths[i] for i in ids]
            xs = torch.zeros(len(ids), max(lens), d, device=dev)
            for row, i in enumerate(ids):
                xs[row, :lens[row]] = corpus[i]
            yield ids, xs, lens

    def run_sequential():
        return {i: bs.forward(corpus[i]) for i in range(len(corpus))}

    def run_batched(U):
        res = {}
        for ids, xs, lens in batches(U):
            for i, nb in zip(ids, bs.forward_batch(xs, lens)):
                res[i] = nb
        return res

    def key(res):
        return {i: [(h.yseq.tolist(), h.score, h.scores["decoder"], h.scores["ctc"]) for h in nb] for i, nb in res.items()}

    sizes = [int(s) for s in args.sizes.split(",")]
    out = {"what": f"decode {len(corpus)} utterances of {lo}..{hi} frames, beam {args.beam}, odim {odim}, d {d}, "
                   f"{L} layers, ctc_weight 0.1, synthetic weights", "gpu": "cpu dry run" if dry else gpu_info(),
           "precision": dec.precision or "f16 (default)", "frames": sum(lengths)}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.out, exist_ok=True)
        run_batched(16)                                       # warm-up
        for U in (1, 16):
            ids, xs, lens = next(batches(U)) if U == 1 else list(batches(U))[len(corpus) // U // 2]
            s0 = bs.stats["steps"]
            sync()
            acts = [ProfilerActivity.CPU] + ([] if dry else [ProfilerActivity.CUDA])
            with profile(activities=acts) as prof:
                bs.forward_batch(xs, lens)
                sync()
            steps = bs.stats["steps"] - s0
            path = os.path.join(args.out, f"decode_batch_U{U}.pt.trace.json")
            prof.export_chrome_trace(path)
            ev = [e for e in prof.key_averages() if (e.device_time_total if hasattr(e, "device_time_total") else 0) > 0]
            ev.sort(key=lambda e: -e.device_time_total)
            kern = [e for e in prof.events() if e.device_type.name == "CUDA"] if not dry else []
            busy = sum(k.time_range.elapsed_us() for k in kern)
            span = (max(k.time_range.end for k in kern) - min(k.time_range.start for k in kern)) if kern else 0
            out[f"profile_U{U}"] = {
                "utterances": len(ids), "steps": steps, "trace": path,
                "kernels_per_step": len(kern) / max(steps, 1),
                "kernel_us_per_step": busy / max(steps, 1),            # summed kernel / copy durations
                "device_span_us_per_step": span / max(steps, 1),       # first start to last end, over the steps
                "top_kernels_us_per_step": [(e.key[:90], e.device_time_total / max(steps, 1)) for e in ev[:12]]}
        print("DECODE-BATCH-JSON " + json.dumps(out))
        return
    ref = None
    arms = [("sequential", run_sequential)] + [(f"batch_{U}", (lambda U=U: run_batched(U))) for U in sizes]
    for name, fn in arms:
        if name == "sequential":                              # warm-up: the first utterance / batch of the arm
            bs.forward(corpus[order[0]])
        else:
            _, xs, lens = next(batches(int(name.split("_")[1])))
            bs.forward_batch(xs, lens)
        sync()
        s0 = bs.stats["steps"]
        t0 = time.perf_counter()
        res = fn()
        sync()
        dt = time.perf_counter() - t0
        steps = bs.stats["steps"] - s0
        arm = {"s": dt, "utterances_per_s": len(corpus) / dt, "steps": steps, "ms_per_step": dt * 1e3 / max(steps, 1)}
        if name != "sequential":
            U = int(name.split("_")[1])
            arm["max_session_bytes"] = max(dec.engine().batch_session_bytes(lens, U * args.beam, max(lens) + 1)
                                           for _, _, lens in batches(U))
            arm["same_nbest_as_sequential"] = key(res) == ref
        else:
            ref = key(res)
        out[name] = arm
    seq = out["sequential"]["s"]
    out["speedup_vs_sequential"] = {n: seq / out[n]["s"] for n, _ in arms[1:]}
    print("DECODE-BATCH-JSON " + json.dumps(out))


if __name__ == "__main__":
    main()
