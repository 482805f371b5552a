#!/usr/bin/env python3
"""Golden fixtures of the ResNet front-ends: the UNMODIFIED reference modules (oracle/_ref, copied by build_ref.py) in
float64 on the CPU, eval mode, on seeded weights (synthetic.frontend_state_dict) and inputs (synthetic.frontend_input).
Each tests/golden/frontend_<modality>_<case>.npz holds the seeds, the input shape, the utterance lengths the batch
stands for (the front-end itself takes none: padded frames are data) and the fp64 output.
Run:  python oracle/make_golden_frontend.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import build_ref  # noqa: E402
from auto_avsr_b200.synthetic import frontend_input, frontend_state_dict  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")

#: name -> (modality, wseed, xseed, B, T (frames or samples), H, W, lengths)
CASES = {
    "frontend_video_88": ("video", 11, 21, 2, 9, 88, 88, [9, 4]),
    "frontend_video_t1": ("video", 12, 22, 1, 1, 88, 88, [1]),
    "frontend_video_45x61": ("video", 13, 23, 2, 3, 45, 61, [3, 2]),
    "frontend_audio_ragged": ("audio", 14, 24, 2, 640 * 6 + 317, 1, 1, [640 * 6 + 317, 640 * 3 + 5]),
}


def reference_module(modality):
    build_ref.import_reference_encoder()
    if modality == "video":
        from espnet.nets.pytorch_backend.frontend.resnet import video_resnet
        return video_resnet()
    from espnet.nets.pytorch_backend.frontend.resnet1d import audio_resnet
    return audio_resnet()


def reference_output(name):
    modality, wseed, xseed, B, T, H, W, _ = CASES[name]
    ref = reference_module(modality)
    ref.load_state_dict(frontend_state_dict(wseed, modality), strict=True)
    ref = ref.double().eval()
    with torch.no_grad():
        return ref(frontend_input(modality, B, T, H, W, xseed, dtype=torch.float64)).numpy()


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    for name, (modality, wseed, xseed, B, T, H, W, lengths) in CASES.items():
        out = reference_output(name)
        np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), modality=np.array(modality), wseed=np.int64(wseed),
                            xseed=np.int64(xseed), shape=np.array([B, T, H, W], dtype=np.int64),
                            lengths=np.array(lengths, dtype=np.int64), out_f64=out)
        print(name, out.shape, float(np.abs(out).max()))


if __name__ == "__main__":
    main()
