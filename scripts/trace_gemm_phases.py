#!/usr/bin/env python3
"""Per-CTA phases of every tensor-core GEMM launch in one S2 encoder forward, reduced per GEMM kind.

    python scripts/build_trace.py
    AVSR_B200_LIB=auto_avsr_b200/csrc/libavsr_b200_trace.so python scripts/trace_gemm_phases.py [--precision f16]
        [--out FILE.json]

Runs the 12-layer encoder at S2 (4 x 400 frames) through its graph plan with programmatic dependent launch on, with
the diagnostic build's trace buffer bound (common.cuh, "phase trace"), and reads the %globaltimer stamps each GEMM CTA
leaves: open, dependency resolved (slot 10), first ring stage landed (1), last main loop retired (3), done (11).
Per launch, averaged over its CTAs:
  ramp       dependency resolved -> first stage landed
  main loop  first stage landed -> last main loop retired (earlier epilogues run under it)
  epilogue   last main loop retired -> CTA done (the exposed epilogue)
  idle tail  CTA done -> the launch's last CTA done
and the launch span, first dependency resolved -> last CTA done.  Each is the mean over the launches of that kind.
The GEMM kind is (epilogue mode, N, K)."""
import argparse
import ctypes as C
import json
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = {400: "LINEAR", 401: "QK", 402: "VT", 403: "GLU", 404: "POS"}
KINDS = {("LINEAR", 3072, 768): "FFN w_1", ("LINEAR", 768, 3072): "FFN w_2", ("QK", 2304, 768): "QKV",
         ("GLU", 1536, 768): "pw1 + GLU", ("LINEAR", 768, 768): "out / pw2"}
WORDS = 16


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="f16")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if "trace" not in os.environ.get("AVSR_B200_LIB", ""):
        raise SystemExit("set AVSR_B200_LIB to the diagnostic build (scripts/build_trace.py)")
    import torch
    from auto_avsr_b200._cabi import lib
    from auto_avsr_b200.engine import EncoderEngine
    from auto_avsr_b200.synthetic import SHAPES, encoder_input, encoder_state_dict
    dev = torch.device("cuda:0")
    lengths = SHAPES["S2"]
    xs = encoder_input(lengths, 768, 5).to(dev)
    lens = torch.tensor(lengths, dtype=torch.int32, device=dev)
    eng = EncoderEngine(768, 12, 3072, 12, 31)
    eng.graph_after = 1
    buf = eng.prepare({k: v.to(dev) for k, v in encoder_state_dict(11).items()}, dev, args.precision)
    for _ in range(3):
        eng.forward(buf, xs, lens, args.precision)          # builds and warms the plan
    torch.cuda.synchronize()
    cap = 200000
    tb = torch.zeros(2 + cap * WORDS, dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    lib.avsr_trace_set.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    lib.avsr_trace_set.restype = C.c_int
    assert lib.avsr_trace_set(tb.data_ptr(), tb.numel(), st) == 0
    eng.forward(buf, xs, lens, args.precision)
    torch.cuda.synchronize()
    lib.avsr_trace_set(None, 0, st)
    t = tb.cpu().numpy().astype("uint64")
    n = min(int(t[0]), cap)
    recs = t[2:2 + n * WORDS].reshape(n, WORDS)

    # (kind, blockIdx) -> its records in time order; the i-th record of each block belongs to launch i of the kind
    per_block = defaultdict(list)
    for r in recs:
        kid = int(r[0])
        if kid not in MODES:
            continue
        aux = int(r[1]) >> 32
        kind = KINDS.get((MODES[kid], aux & 0xFFFF, aux >> 16), f"{MODES[kid]} N={aux & 0xFFFF} K={aux >> 16}")
        per_block[(kind, int(r[1]) & 0xFFFFFFFF)].append(r)
    launches = defaultdict(lambda: defaultdict(list))
    for (kind, _), rs in per_block.items():
        rs.sort(key=lambda r: int(r[3]))
        for i, r in enumerate(rs):
            launches[kind][i].append(r)

    table = {}
    for kind, ls in sorted(launches.items()):
        acc = defaultdict(list)
        for rs in ls.values():
            dep = [int(r[14]) for r in rs]
            first = [int(r[4 + 1]) for r in rs]
            ret = [int(r[4 + 3]) for r in rs]
            done = [int(r[15]) for r in rs]
            end = max(done)
            ok = [i for i in range(len(rs)) if first[i] and ret[i]]
            if not ok:
                continue
            mean = lambda v: sum(v) / len(v) / 1000.0            # ns -> us
            acc["ramp"].append(mean([first[i] - dep[i] for i in ok]))
            acc["main"].append(mean([ret[i] - first[i] for i in ok]))
            acc["epilogue"].append(mean([done[i] - ret[i] for i in ok]))
            acc["tail"].append(mean([end - done[i] for i in ok]))
            acc["span"].append((end - min(dep)) / 1000.0)
            acc["ctas"].append(len(rs))
        table[kind] = {k: sum(v) / len(v) for k, v in acc.items()}
        table[kind]["launches"] = len(acc["span"])
    print(f"{'GEMM':<22}{'launches':>9}{'CTAs':>6}{'ramp':>8}{'main':>8}{'epi':>8}{'tail':>8}{'span':>8}   (us)")
    for kind, v in table.items():
        print(f"{kind:<22}{v['launches']:>9}{v['ctas']:>6.0f}{v['ramp']:>8.2f}{v['main']:>8.2f}{v['epilogue']:>8.2f}"
              f"{v['tail']:>8.2f}{v['span']:>8.2f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"precision": args.precision, "prologue": os.environ.get("AVSR_B200_PROLOGUE", "1"),
                       "gpu": torch.cuda.get_device_name(0), "kinds": table}, f, indent=1)


if __name__ == "__main__":
    main()
