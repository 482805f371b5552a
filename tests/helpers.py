"""Shared test helpers: load a golden case and regenerate its weights/inputs from seeds."""
import os

import numpy as np
import torch

from auto_avsr_b200.synthetic import encoder_input, encoder_state_dict, frontend_features, head_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_case(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    d_model, n_heads, linear_units, num_blocks, cnn_kernel = (int(v) for v in z["config"])
    lengths = [int(v) for v in z["lengths"]]
    masked = bool(int(z["masked"]))
    sd = encoder_state_dict(int(z["wseed"]), d_model, n_heads, linear_units, num_blocks, cnn_kernel)
    xs = encoder_input(lengths, d_model, int(z["xseed"]))
    return dict(z=z, cfg=dict(d_model=d_model, n_heads=n_heads, linear_units=linear_units,
                              num_blocks=num_blocks, cnn_kernel=cnn_kernel),
                lengths=lengths, masked=masked, sd=sd, xs=xs)


def load_head_case(name):
    """Golden case of the steps either side of the encoder (oracle/make_golden_head.py)."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = {k[4:]: int(z[k]) for k in z.files if k.startswith("cfg_")}
    lengths = [int(v) for v in z["lengths"]]
    enc_sd = encoder_state_dict(cfg["wseed"], cfg["d_model"], cfg["n_heads"], cfg["linear_units"], cfg["num_blocks"],
                                cfg["cnn_kernel"])
    head_sd = head_state_dict(cfg["wseed"], cfg["idim"], cfg["d_model"], cfg["odim"])
    feats = frontend_features(lengths, cfg["idim"], cfg["xseed"])
    return dict(z=z, cfg=cfg, lengths=lengths, masked=bool(cfg["masked"]), enc_sd=enc_sd, head_sd=head_sd, feats=feats)


def err_stats(a, b):
    d = (a.double() - b.double()).abs()
    return d.max().item(), d.pow(2).mean().sqrt().item()


_OBS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")


def record(test, case, observed, bound):
    """Print the observed error next to its bound and append it to gpurun_out/parity_observed.jsonl (the GPU runs'
    scratch directory) so that the bounds in the tests can be kept at about 4x what the GPU actually produces."""
    import json
    line = {"test": test, "case": str(case), "observed": observed, "bound": bound}
    print("PARITY", json.dumps(line))
    try:
        os.makedirs(_OBS, exist_ok=True)
        with open(os.path.join(_OBS, "parity_observed.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")
    except OSError:
        pass


def load_decoder_case(name):
    """Golden case of the attention-decoder scoring path (oracle/make_golden_decoder.py): config, the regenerated
    decoder / CTC weights, the (T, d) memory and the fixed prefixes of every stored step."""
    from auto_avsr_b200.synthetic import decoder_state_dict
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = {k[4:]: int(z[k]) for k in z.files if k.startswith("cfg_")}
    dec_sd = decoder_state_dict(cfg["wseed"], cfg["odim"], cfg["d_model"], cfg["n_heads"], cfg["linear_units"],
                                cfg["num_blocks"])
    head_sd = head_state_dict(cfg["wseed"], 64, cfg["d_model"], cfg["odim"])
    memory = encoder_input([cfg["T"]], cfg["d_model"], cfg["xseed"])[0]
    g = torch.Generator().manual_seed(cfg["xseed"] * 7 + 1)
    body = torch.randint(1, cfg["odim"] - 1, (cfg["n_hyp"], cfg["steps"]), generator=g)
    sos = torch.full((cfg["n_hyp"], 1), cfg["odim"] - 1, dtype=torch.long)
    prefixes = [torch.cat([sos, body[:, :s]], dim=1) for s in range(cfg["steps"] + 1)]
    return dict(z=z, cfg=cfg, dec_sd=dec_sd, head_sd=head_sd, memory=memory, prefixes=prefixes)
