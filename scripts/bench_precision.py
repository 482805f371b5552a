"""f16 / bf16 / tf32 side by side on one GPU, in one process, the three precisions alternated round by round and timed
with CUDA events:

  encoder_s2   the 12-layer encoder forward at S2 (4 x 400 frames), CUDA-graph replay
  ffn_w1       one FFN w_1 GEMM (1600 x 3072 x 768, ReLU, operand-typed output) per launch: avsr_linear_operands on
               operands already in the precision's storage, as the encoder runs it
  attention    one layer's rel-pos attention at S2 (B 4, T 400, 12 heads) per call of avsr_relpos_attention: the fp32
               inputs split into heads and converted, the attention kernel, the context converted back
  video_fe     the video front-end inference at the bucket (2 clips x 29 frames of 88 x 88)
  train_step   one 2-layer encoder training step (forward + backward, dropouts 0) at 4 x 400 frames

The precision that runs first in a round rotates from round to round (the first timing after a change of workload runs
slower).  Prints the card's name and power limit, then one JSON line per (workload, precision) with the median and the spread
over rounds, and the bf16 / f16 ratio of the medians.

    python scripts/bench_precision.py [--rounds 15] [--iters 20] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PRECS = ("f16", "bf16", "tf32")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def workloads(dev):
    import torch
    from auto_avsr_b200 import ConformerEncoder, ops
    from auto_avsr_b200._cabi import check, lib
    from auto_avsr_b200.engine import PRECISIONS
    from auto_avsr_b200.espnet_dropin.resnet import Conv3dResNet
    from auto_avsr_b200.synthetic import SHAPES, encoder_input, encoder_state_dict, frontend_input, frontend_state_dict
    from oracle import conformer_oracle as O
    lengths = list(SHAPES["S2"])
    xs = encoder_input(lengths, 768, 1234).to(dev)
    mask = O.non_pad_mask(lengths).unsqueeze(1).to(dev)
    encs = {}
    sd = encoder_state_dict(0)
    for p in PRECS:
        e = ConformerEncoder().to(dev).eval()
        e.load_state_dict(sd)
        e.precision, e.graph_after = p, 1
        encs[p] = e
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1600, 768, generator=g)
    w1 = torch.randn(3072, 768, generator=g) * 0.03
    storage = {"f16": torch.float16, "bf16": torch.bfloat16, "tf32": torch.float32}
    gemm_in = {p: (x.to(dev, storage[p]), w1.to(dev, storage[p]), torch.empty(1600, 3072, device=dev, dtype=storage[p]))
               for p in PRECS}
    bias = torch.zeros(3072, device=dev)
    B, T, H = 4, 400, 12
    q, k, v = (torch.randn(B, T, H * 64, generator=g).to(dev) for _ in range(3))
    pp = torch.randn(2 * T - 1, H * 64, generator=g).to(dev)
    u, vb = (torch.randn(H, 64, generator=g).to(dev) * 0.3 for _ in range(2))
    fe = Conv3dResNet().to(dev).eval()
    fe.load_state_dict(frontend_state_dict(0, "video"))
    clip = frontend_input("video", 2, 29, 88, 88, 0).to(dev)
    tr = {}
    for p in PRECS:
        e = ConformerEncoder(num_blocks=2, dropout_rate=0.0, positional_dropout_rate=0.0, attention_dropout_rate=0.0)
        e.load_state_dict(encoder_state_dict(0, num_blocks=2))
        e = e.to(dev).train()
        e.precision = p
        tr[p] = e

    def enc_fwd(p):
        with torch.no_grad():
            encs[p](xs, mask)

    def ffn(p):
        a, w, y = gemm_in[p]
        check(lib.avsr_linear_operands(a.data_ptr(), w.data_ptr(), bias.data_ptr(), None, 1.0, y.data_ptr(), 1600, 3072,
                                       768, 1, 1, PRECISIONS[p], torch.cuda.current_stream(dev).cuda_stream))

    def attn(p):
        ops.relpos_attention(q, k, v, pp, u, vb, None, H, precision=p)

    def video(p):
        fe.precision = p
        with torch.no_grad():
            fe(clip)

    def train_step(p):
        xg = xs.detach().requires_grad_(True)
        y, _ = tr[p](xg, mask)
        y.sum().backward()

    return {"encoder_s2": enc_fwd, "ffn_w1": ffn, "attention": attn, "video_fe": video, "train_step": train_step}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_precision.py measures on a GPU; there is no CPU fallback"
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda:0")
    print("card:", card())
    wl = workloads(dev)
    times = {(n, p): [] for n in wl for p in PRECS}
    for n, fn in wl.items():               # warm-up: modules, prepared weights, graphs of every shape
        for p in PRECS:
            for _ in range(3):
                fn(p)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.rounds):
        order = PRECS[r % 3:] + PRECS[:r % 3]     # rotate who goes first: the first timing after a switch of workload
        for n, fn in wl.items():
            for p in order:
                e0.record()
                for _ in range(args.iters):
                    fn(p)
                e1.record()
                e1.synchronize()
                times[(n, p)].append(e0.elapsed_time(e1) / args.iters)
    rows = []
    for n in wl:
        med = {p: statistics.median(times[(n, p)]) for p in PRECS}
        for p in PRECS:
            t = sorted(times[(n, p)])
            rows.append({"workload": n, "precision": p, "ms_median": med[p], "ms_min": t[0], "ms_max": t[-1],
                         "bf16_over_f16": med["bf16"] / med["f16"]})
            print(json.dumps(rows[-1]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
