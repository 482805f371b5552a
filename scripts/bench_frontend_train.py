#!/usr/bin/env python3
"""One training step of the ResNet front-ends (forward, backward, running-statistics update): the library training
path (``library_train``) against the reference module on the same GPU.

Workloads: the max-frames bucket (video 4 x 400 frames of 88x88, audio 4 x 256,000 samples) and the config-1 clip
(1 x 100 frames).  Arms:
  lib_f16, lib_tf32        the drop-in with library_train = True (forward convs in f16 / TF32, dgrad TF32)
  ref_tf32                 the reference module as training runs it: fp32, cudnn.allow_tf32 at its default (True)
  ref_fp32                 the same with cuDNN TF32 off
  ref_cl_autocast_f16      channels_last + autocast f16 + cudnn.benchmark
Times are device events around `--steps` steps after `--warmup` steps: ms/step, algorithmic TFLOP/s (forward + dgrad
+ wgrad MACs from the layer shapes; the stem has no dgrad) and peak memory (max_memory_allocated) per arm.  The card's
name and power limit are read in the same run.  Writes bench_frontend_train.json under --out.

--profile: instead, a torch.profiler run of `--steps` library steps (f16) on the video bucket, CUDA time per kernel.
--e2e: instead, one E2E(5049, "video") forward + backward at the S2 bucket (4 x 400 frames of 88x88, 100 labels per
utterance) with install(), install_head(), install_decoder() and install_frontend(library_train = False / True), f16.

  python scripts/bench_frontend_train.py --out DIR [--steps 10] [--warmup 3] [--only video_max_frames] [--profile | --e2e]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_frontend import frontend_macs, gpu_info, time_it  # noqa: E402


def stem_macs(modality, B, T, H=88, W=88):
    if modality == "video":
        return B * T * ((H - 1) // 2 + 1) * ((W - 1) // 2 + 1) * 64 * 245
    return B * ((T // 640 * 640) // 4) * 64 * 80


def train_macs(modality, B, T):
    """forward + wgrad of every conv + dgrad of every conv but the stem"""
    f = frontend_macs(modality, B, T)
    return 3 * f - stem_macs(modality, B, T)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--e2e", action="store_true")
    args = ap.parse_args()
    if args.profile:
        return profile(args)
    if args.e2e:
        return e2e(args)
    import torch
    from auto_avsr_b200.espnet_dropin.resnet import Conv1dResNet, Conv3dResNet
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    from oracle.make_golden_frontend import reference_module

    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "workloads": {}}
    workloads = [("video_max_frames", "video", 4, 400), ("audio_max_frames", "audio", 4, 256000),
                 ("video_config1", "video", 1, 100)]
    for name, modality, B, T in workloads:
        if args.only and name != args.only:
            continue
        sd = frontend_state_dict(0, modality)
        x = frontend_input(modality, B, T).to(dev)
        macs = train_macs(modality, B, T)
        arms = {}

        def run_arm(label, module, fn_ctx=None, cl=False, tf32=True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cudnn.benchmark = label == "ref_cl_autocast_f16"
            module = module.to(dev).train()
            if cl and modality == "video":
                module.frontend3D.to(memory_format=torch.channels_last_3d)
                module.trunk.to(memory_format=torch.channels_last)
            with torch.no_grad():
                wts = torch.randn(module(x).shape, device=dev)

            def step():
                module.zero_grad(set_to_none=True)
                if fn_ctx is not None:
                    with fn_ctx():
                        out = module(x)
                else:
                    out = module(x)
                (out.float() * wts).sum().backward()

            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            ms = time_it(step, args.steps, args.warmup)
            peak = torch.cuda.max_memory_allocated(dev)
            arms[label] = {"ms": ms, "tflops": 2 * macs / ms / 1e9, "peak_gib": peak / 2 ** 30}
            print(name, label, json.dumps(arms[label]), flush=True)
            del module
            torch.cuda.empty_cache()

        for prec in ("f16", "tf32"):
            m = Conv3dResNet() if modality == "video" else Conv1dResNet()
            m.load_state_dict(sd)
            m.library_train, m.precision = True, prec
            run_arm(f"lib_{prec}", m)
        for label, tf32 in (("ref_tf32", True), ("ref_fp32", False)):
            r = reference_module(modality)
            r.load_state_dict(sd)
            run_arm(label, r, tf32=tf32)
        r = reference_module(modality)
        r.load_state_dict(sd)
        run_arm("ref_cl_autocast_f16", r, fn_ctx=lambda: torch.autocast("cuda", dtype=torch.float16), cl=True)
        torch.backends.cudnn.allow_tf32 = True
        torch.backends.cudnn.benchmark = False
        res["workloads"][name] = {"B": B, "T": T, "train_gmac": macs / 1e9, "arms": arms}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_frontend_train.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


def _dump(args, name, res):
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, name), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


def profile(args):
    import torch
    from torch.profiler import ProfilerActivity
    from auto_avsr_b200.espnet_dropin.resnet import Conv3dResNet
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    dev = torch.device("cuda:0")
    m = Conv3dResNet()
    m.load_state_dict(frontend_state_dict(0, "video"))
    m = m.to(dev).train()
    m.library_train, m.precision = True, "f16"
    x = frontend_input("video", 4, 400).to(dev)
    wts = torch.randn(4, 400, 512, device=dev)

    def step():
        m.zero_grad(set_to_none=True)
        (m(x) * wts).sum().backward()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", 0) or getattr(ev, "cuda_time_total", 0)
        if t > 0 and ev.device_type == torch.autograd.DeviceType.CUDA:
            rows[ev.key[:90]] = rows.get(ev.key[:90], 0.0) + t / 1e3 / args.steps
    total = sum(rows.values())
    top = sorted(rows.items(), key=lambda kv: -kv[1])[:20]
    _dump(args, "bench_frontend_train_profile.json", {"gpu": gpu_info(), "steps": args.steps, "ms_per_step_total": total,
                                                       "kernels_ms_per_step": dict(top)})


def e2e(args):
    import torch
    from oracle import build_ref
    build_ref.import_reference_encoder()
    import auto_avsr_b200
    auto_avsr_b200.install()
    from espnet.nets.pytorch_backend import e2e_asr_conformer as E
    from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "arms": {}}
    x = frontend_input("video", 4, 400).to(dev)
    lengths = torch.tensor([400, 380, 350, 300])
    label = torch.randint(1, 5048, (4, 100), generator=torch.Generator().manual_seed(1)).to(dev)
    for library_train in (False, True):
        torch.manual_seed(0)
        model = E.E2E(5049, "video")
        model.frontend.load_state_dict(frontend_state_dict(0, "video"))
        auto_avsr_b200.install_head(model)
        auto_avsr_b200.install_decoder(model)
        auto_avsr_b200.install_frontend(model, library_train=library_train)
        model = model.to(dev).train()

        def step():
            model.zero_grad(set_to_none=True)
            model(x, lengths, label)[0].backward()

        torch.cuda.reset_peak_memory_stats(dev)
        ms = time_it(step, args.steps, args.warmup)
        res["arms"]["library_train" if library_train else "torch_frontend"] = {
            "ms": ms, "peak_gib": torch.cuda.max_memory_allocated(dev) / 2 ** 30}
        print(library_train, ms, flush=True)
        del model
        torch.cuda.empty_cache()
    _dump(args, "bench_frontend_train_e2e.json", res)


if __name__ == "__main__":
    main()
