#!/usr/bin/env python3
"""Time the attention decoder's share of the training step -- TransformerDecoder.forward + LabelSmoothingLoss + backward
(e2e_asr_conformer.py:77-80): token ids and encoder memory -> loss -> gradients of the memory and of every decoder
parameter -- with CUDA events, for the drop-in and for the reference modules in eager PyTorch on the same GPU.

    python scripts/bench_decoder_train.py [--steps 30] [--warmup 5] [--profile]

Synthetic bucket: memory lengths [400, 350, 300, 250, 300] (S2-like), label lengths [80, 70, 60, 50, 60], d 768, 12 heads,
ff 3072, 6 layers, odim 5049, dropout as E2E builds the decoder (0.1 everywhere, attention probabilities included).
Arms: the drop-in at f16 / tf32 / fp32 GEMM precision, and at f16 with backward_precision="bf16"; the reference decoder + LabelSmoothingLoss (oracle/_ref, skipped
when it was not built) in fp32 and with allow_tf32.  Also the arithmetic of one step counted from shapes (GEMMs and
attention, forward + backward), and the per-call device time of the attention core's backward, fp32 kernels
(avsr_mha_core_bwd) against the tensor-core kernels (avsr_mha_core_bwd_tc), at the bucket's self and source attention
and at a long bucket.  ``--profile`` adds one step each of the default and the bf16 backward under torch.profiler: the
device time per kernel, and its split into attention-core kernels, GEMMs and the rest.  Prints one JSON object with the
device name and its power limit; writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from auto_avsr_b200 import LabelSmoothingLoss, TransformerDecoder  # noqa: E402
from auto_avsr_b200.synthetic import decoder_state_dict, encoder_input  # noqa: E402

MEM, LAB = [400, 350, 300, 250, 300], [80, 70, 60, 50, 60]
D, H, FF, NL, ODIM = 768, 12, 3072, 6, 5049


def device_info():
    p = torch.cuda.get_device_properties(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"device": p.name, "power_limit": pl or "unknown", "sm_count": p.multi_processor_count}


def batch(dev):
    """ys_in / ys_out (add_sos_eos), tgt_mask (target_mask), memory mask, memory -- as E2E.forward builds them."""
    g = torch.Generator().manual_seed(3)
    eos = ODIM - 1
    L = max(LAB) + 1
    ys_in = torch.full((len(LAB), L), eos, dtype=torch.long)
    ys_out = torch.full((len(LAB), L), -1, dtype=torch.long)
    for b, n in enumerate(LAB):
        r = torch.randint(1, ODIM - 1, (n,), generator=g)
        ys_in[b, 1:n + 1] = r
        ys_out[b, :n] = r
        ys_out[b, n] = eos
    tgt_mask = torch.tril(torch.ones(L, L, dtype=torch.bool))[None].expand(len(LAB), L, L).contiguous()
    mem_mask = (torch.arange(max(MEM))[None, :] < torch.tensor(MEM)[:, None])[:, None, :]
    mem = encoder_input(MEM, D, 5)
    return [t.to(dev) for t in (ys_in, tgt_mask, mem, mem_mask, ys_out)]


def flops_per_step():
    """Forward + backward arithmetic from shapes (2 flops per multiply-add; backward = 2x forward for GEMMs)."""
    rows_l, rows_t = len(LAB) * (max(LAB) + 1), len(MEM) * max(MEM)
    gemm = NL * (rows_l * D * 3 * D + rows_l * D * D * 2 + rows_t * D * 2 * D + rows_l * 2 * D * FF) + rows_l * D * ODIM
    Lq = max(LAB) + 1
    attn = NL * len(LAB) * H * 64 * (Lq * Lq + Lq * max(MEM)) * 2        # QK^T and PV per attention, self + source
    return {"gemm_gflop": 3 * 2 * gemm / 1e9, "attention_gflop": 3 * 2 * attn / 1e9}


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


def step_fn(dec, crit, data):
    ys_in, tgt_mask, mem, mem_mask, ys_out = data
    x = mem.clone().requires_grad_(True)

    def fn():
        dec.zero_grad(set_to_none=True)
        x.grad = None
        pred, _ = dec(ys_in, tgt_mask, x, mem_mask)
        crit(pred, ys_out).backward()
    return fn


def attention_core_calls(dev, steps):
    """ms per call (CUDA events over `steps` calls after a warm-up) of the two attention-core backwards on the same
    stored probabilities, dropout 0.1 as in training."""
    from auto_avsr_b200 import decoder_train as DT
    shapes = {"self_5x81x81": (LAB, max(LAB) + 1, max(LAB) + 1, True),
              "source_5x81x400": (MEM, max(LAB) + 1, max(MEM), False),
              "source_long_5x151x600": ([600, 550, 500, 450, 500], 151, 600, False)}
    g = torch.Generator(device=dev).manual_seed(1)
    out = {}
    for tag, (klen, Lq, Lk, causal) in shapes.items():
        B = len(klen)
        if causal:
            src = torch.randn(B, Lq, 3 * D, device=dev, generator=g)
            q, k, v = src[..., :D], src[..., D:2 * D], src[..., 2 * D:]
            ln = torch.tensor([n + 1 for n in LAB], dtype=torch.int32, device=dev)
        else:
            q = torch.randn(B, Lq, D, device=dev, generator=g)
            kv = torch.randn(B, Lk, 2 * D, device=dev, generator=g)
            k, v = kv[..., :D], kv[..., D:]
            ln = torch.tensor(klen, dtype=torch.int32, device=dev)
        dctx = torch.randn(B, Lq, D, device=dev, generator=g)
        keep, scale = DT.draw_keep_mask(0.1, (B, H, Lq, Lk), dev), 1.0 / 0.9
        ctx, probs = DT.mha_core_forward(q, k, v, H, causal, ln, keep, scale, want_probs=True)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        fp32 = lambda: DT.mha_core_backward(q, k, v, H, causal, ln, keep, scale, probs, dctx, dq, dk, dv)   # noqa: E731
        tc = lambda: DT.mha_core_backward_tc(q, k, v, H, causal, ln, keep, scale, probs, ctx, dctx, dq, dk, dv)  # noqa
        t32, ttc = time_ms(fp32, steps, 5), time_ms(tc, steps, 5)
        out[tag] = {"fp32_ms": round(t32, 4), "bf16_tc_ms": round(ttc, 4), "speedup": round(t32 / ttc, 2)}
    return out


def profile_steps(dec, crit, data):
    """One step each of the default and the bf16 backward under torch.profiler -> device ms per kernel and the split."""
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for tag, backward in (("default", None), ("bf16", "bf16")):
        dec.backward_precision = backward
        fn = step_fn(dec, crit, data)
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            if t > 0:
                kernels[e.key] = round(t / 1e3, 4)
        split = {"attention_core": 0.0, "gemm": 0.0, "other": 0.0}
        for name, ms in kernels.items():
            kind = ("attention_core" if "mha_" in name else
                    "gemm" if ("gemm" in name or "pack" in name or "linear" in name) else "other")
            split[kind] += ms
        res[tag] = {"split_ms": {k: round(v, 3) for k, v in split.items()},
                    "kernels_ms": dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:25])}
    dec.backward_precision = None
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decoder_train: needs a CUDA device")
    dev = torch.device("cuda:0")
    data = batch(dev)
    sd = decoder_state_dict(1, ODIM, D, H, FF, NL)
    out = {"bench": "decoder_train", "memory_lengths": MEM, "label_lengths": LAB, **device_info(), **flops_per_step(),
           "ms_per_step": {}}
    dec = TransformerDecoder(ODIM, D, H, FF, NL)
    dec.load_state_dict(sd, strict=True)
    dec = dec.to(dev).train()
    crit = LabelSmoothingLoss(ODIM, -1, 0.1, False)
    for prec in ("f16", "tf32", "fp32"):
        dec.precision = prec
        out["ms_per_step"]["dropin_" + prec] = round(time_ms(step_fn(dec, crit, data), args.steps, args.warmup), 3)
    dec.precision, dec.backward_precision = "f16", "bf16"
    out["ms_per_step"]["dropin_f16_bwd_bf16"] = round(time_ms(step_fn(dec, crit, data), args.steps, args.warmup), 3)
    dec.backward_precision = None
    out["attention_core_bwd_ms_per_call"] = attention_core_calls(dev, max(args.steps, 20))
    if args.profile:
        out["profile_one_step"] = profile_steps(dec, crit, data)
    del dec
    try:
        from oracle import build_ref
        build_ref.import_reference_encoder()
        from espnet.nets.pytorch_backend.decoder.transformer_decoder import TransformerDecoder as RefDecoder
        from espnet.nets.pytorch_backend.transformer.label_smoothing_loss import LabelSmoothingLoss as RefLS
    except ImportError as e:
        out["reference"] = f"not measured ({e})"
    else:
        ref = RefDecoder(ODIM, D, H, FF, NL)
        ref.load_state_dict(sd, strict=True)
        ref = ref.to(dev).train()
        rcrit = RefLS(ODIM, -1, 0.1, False)
        for tag, tf32 in (("reference_fp32", False), ("reference_allow_tf32", True)):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            out["ms_per_step"][tag] = round(time_ms(step_fn(ref, rcrit, data), args.steps, args.warmup), 3)
        torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps(out))


if __name__ == "__main__":
    main()
