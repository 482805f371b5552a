#!/usr/bin/env python3
"""ResNet front-ends: libavsr_b200 (avsr_frontend_forward) against the reference module on the same GPU.

Workloads: the max-frames bucket (4 x 400 frames: video 88x88 clips, audio 4 x 256,000 samples) and the config-1 clip
(B = 1, 100 frames of 88x88 video).  Arms:
  lib_f16, lib_tf32       the drop-in Conv3dResNet / Conv1dResNet in eval on prepared weights
  ref_fp32                the reference module, eager fp32, cuDNN TF32 off
  ref_tf32                the same with torch.backends.cudnn.allow_tf32
  ref_cl_autocast_f16     channels_last + autocast f16 + cudnn.benchmark: cuDNN's best stock configuration
Times are device events around `--steps` calls after `--warmup` calls; ms/step, frames/s and algorithmic TFLOP/s (MACs
counted from the layer shapes below, 2 FLOP per MAC).  Also times raw clip -> CTC log-probs for the config-1 clip through
an E2E(5049, "video") with install() + install_head(), with and without install_frontend().  The card's name and power
limit are read (nvidia-smi, read-only) in the same run.  Writes bench_frontend.json under --out.

  python scripts/bench_frontend.py --out DIR [--steps 20] [--warmup 5]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                   # noqa: BLE001
        return f"unavailable ({type(e).__name__})"


def frontend_macs(modality, B, T, H=88, W=88):
    """Multiply-accumulates of one forward, from the layer shapes (stem, 16 trunk convs, 3 downsample convs)."""
    if modality == "video":
        frames, h, w = B * T, (H - 1) // 2 + 1, (W - 1) // 2 + 1
        macs = frames * h * w * 64 * 245
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        k = 9
    else:
        frames, h, w = B, 1, (T // 640 * 640) // 4
        macs = frames * w * 64 * 80
        k = 3
    cin = 64
    for i, planes in enumerate((64, 128, 256, 512)):
        for b in range(2):
            s = 2 if (i > 0 and b == 0) else 1
            ho = (h - 1) // s + 1 if modality == "video" else 1
            wo = (w - 1) // s + 1
            macs += frames * ho * wo * planes * (k * cin + k * planes + (cin if s == 2 else 0))
            h, w, cin = ho, wo, planes
    return macs


def time_it(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    from oracle.make_golden_frontend import reference_module

    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "workloads": {}}
    workloads = [("video_max_frames", "video", 4, 400), ("audio_max_frames", "audio", 4, 256000),
                 ("video_config1", "video", 1, 100)]
    for name, modality, B, T in workloads:
        sd = frontend_state_dict(0, modality)
        ref = reference_module(modality)
        ref.load_state_dict(sd)
        ref = ref.to(dev).eval()
        lib = (Conv3dResNet() if modality == "video" else Conv1dResNet())
        lib.load_state_dict(sd)
        lib = lib.to(dev).eval()
        x = frontend_input(modality, B, T, 88, 88, 1).to(dev)
        frames = B * T if modality == "video" else B * (T // 640)
        flop = 2.0 * frontend_macs(modality, B, T)
        arms = {}

        def lib_arm(prec):
            lib.precision = prec
            return lambda: lib(x)

        def ref_arm(tf32):
            def run():
                torch.backends.cudnn.allow_tf32 = tf32
                return ref(x)
            return run

        ref_cl = reference_module(modality)
        ref_cl.load_state_dict(sd)
        ref_cl = ref_cl.to(dev).eval()
        if modality == "video":                          # 1-D convs have no channels-last layout
            ref_cl.trunk.to(memory_format=torch.channels_last)
            ref_cl.frontend3D.to(memory_format=torch.channels_last_3d)

        def ref_autocast():
            torch.backends.cudnn.benchmark = True
            with torch.autocast("cuda", dtype=torch.float16):
                return ref_cl(x)

        with torch.no_grad():
            for arm, fn in (("lib_f16", lib_arm("f16")), ("lib_tf32", lib_arm("tf32")), ("ref_fp32", ref_arm(False)),
                            ("ref_tf32", ref_arm(True)), ("ref_cl_autocast_f16", ref_autocast)):
                ms = time_it(fn, args.steps, args.warmup)
                torch.backends.cudnn.benchmark = False
                torch.backends.cudnn.allow_tf32 = False
                arms[arm] = {"ms_per_step": round(ms, 4), "frames_per_s": round(frames / ms * 1e3, 1),
                             "tflops": round(flop / ms / 1e9, 2)}
                print(name, arm, arms[arm], flush=True)
            lib.precision = "f16"
            y = lib(x).double()
            r = ref(x).double()
            err = ((y - r).abs().max() / r.abs().max()).item()
        res["workloads"][name] = {"modality": modality, "B": B, "T": T, "frames": frames,
                                  "gflop": round(flop / 1e9, 1), "arms": arms, "lib_f16_rel_err_vs_ref_fp32": err}
        del ref, ref_cl, lib, x
        torch.cuda.empty_cache()

    # raw clip -> CTC log-probs, config-1 clip, with and without install_frontend
    from oracle import build_ref
    build_ref.import_reference_encoder()
    import auto_avsr_b200
    from auto_avsr_b200.head import features_to_log_probs
    auto_avsr_b200.install()
    from espnet.nets.pytorch_backend import e2e_asr_conformer as E
    torch.manual_seed(0)
    model = E.E2E(5049, "video")
    model.frontend.load_state_dict(frontend_state_dict(0, "video"))
    auto_avsr_b200.install_head(model)
    model = model.to(dev).eval()
    x = frontend_input("video", 1, 100, 88, 88, 2).to(dev)
    e2e = {}

    def clip_to_logp():
        feats = model.frontend(x)
        return features_to_log_probs(model.proj_encoder, model.encoder, model.ctc, feats, None, want_features=False)[1]

    with torch.no_grad():
        e2e["reference_frontend_fp32"] = round(time_it(clip_to_logp, args.steps, args.warmup), 4)
        auto_avsr_b200.install_frontend(model)
        model.frontend.to(dev)
        e2e["install_frontend_f16"] = round(time_it(clip_to_logp, args.steps, args.warmup), 4)
    res["clip_to_ctc_logprobs_ms"] = e2e
    print("clip -> CTC log-probs (ms):", e2e)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_frontend.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
