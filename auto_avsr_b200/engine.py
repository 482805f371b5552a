"""Host-side driver of the C-ABI encoder: owns the prepared-weight buffer, per-(B,T) workspaces and CUDA-graph
plans.  torch is used for device memory and streams only; all arithmetic happens in libavsr_b200.so."""
from __future__ import annotations

import ctypes as C
import os
from collections import OrderedDict
from typing import Dict, Optional, Tuple

import torch

from . import _cabi
from ._cabi import EncoderConfig, LayerParams, LAYER_FIELDS, PREC_BF16, PREC_F16, PREC_FP32, PREC_TF32, check, lib

#: precision name -> AVSR_PREC_* code.  "bf16" has f16's bytes and tensor-core rate with fp32's exponent range (unit
#: roundoff 2^-8 against f16's 2^-11): the mode for activations that outgrow f16's +-65504.
PRECISIONS = {"fp32": PREC_FP32, "tf32": PREC_TF32, "f16": PREC_F16, "bf16": PREC_BF16}


def default_precision() -> str:
    return os.environ.get("AVSR_B200_PRECISION", "f16")


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream_handle(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(
            f"{what}: tensor is on {t.device}; the CUDA encoder path has no CPU fallback "
            "(move the module and its inputs to a CUDA device)")
    if t.dtype != torch.float32:
        raise TypeError(f"{what}: expected float32, got {t.dtype}")


class PlanCache:
    """Which shapes get a CUDA-graph plan.  A shape key runs on direct launches (``get`` returns None) until it has been
    seen ``graph_after`` times (the caller's threshold); then ``build()`` makes its entry, a tuple whose first item is the plan handle.  At most
    ``max_plans`` entries are kept, the least recently used evicted first; ``_seen`` remembers at most 64 * max_plans
    keys, so a stream of one-off shapes (the B = 1 eval loop) does not grow it.  Evicted and cleared plans are destroyed
    with avsr_plan_destroy."""

    def __init__(self, max_plans: int):
        self.max_plans = max_plans
        self._plans: "OrderedDict[tuple, tuple]" = OrderedDict()
        self._seen: "OrderedDict[tuple, int]" = OrderedDict()
        self._capture_stream: Dict[int, torch.cuda.Stream] = {}

    def __del__(self):
        try:
            self.clear()
        except Exception:
            pass

    def get(self, key: tuple, graph_after: int, build) -> Optional[tuple]:
        hit = self._plans.get(key)
        if hit is not None:
            self._plans.move_to_end(key)
            return hit
        seen = self._seen.get(key, 0) + 1
        self._seen[key] = seen
        self._seen.move_to_end(key)
        while len(self._seen) > 64 * self.max_plans:
            self._seen.popitem(last=False)
        if seen < graph_after:
            return None
        entry = self._plans[key] = build()
        while len(self._plans) > self.max_plans:
            _, old = self._plans.popitem(last=False)
            lib.avsr_plan_destroy(old[0])
        return entry

    def clear(self) -> None:
        for entry in self._plans.values():
            lib.avsr_plan_destroy(entry[0])
        self._plans.clear()

    def capture_stream(self, device: torch.device) -> torch.cuda.Stream:
        """the stream plans of `device` are captured on (the legacy default stream cannot capture), ordered after the
        current stream's work"""
        idx = device.index or 0
        if idx not in self._capture_stream:
            self._capture_stream[idx] = torch.cuda.Stream(device=device)
        cs = self._capture_stream[idx]
        cs.wait_stream(torch.cuda.current_stream(device))
        return cs


class SaturationError(OverflowError):
    """The fp16 operand path left its range (+-65504) for these weights / inputs: use precision "bf16" (fp32's range
    at f16's speed), "tf32" or "fp32"."""


class EncoderEngine:
    """Runs ConformerEncoder.forward (eval) for one parameter set on one device.

    Shape policy (the reference's eval path feeds B=1 with a different T per utterance, lightning.py:72): a (B, T)
    shape runs on direct launches -- one growable workspace per device, no capture cost -- until it has been seen
    ``graph_after`` times; only then a CUDA-graph plan (own ~85 KB/frame workspace, ~190-node capture) is built for it.
    Plans live in an LRU of ``MAX_PLANS`` (env AVSR_B200_MAX_PLANS).  Fixed-shape loops (training buckets, bench)
    reach the graph after ``graph_after - 1`` calls; ``graph_after=1`` captures at first sight."""

    MAX_PLANS = int(os.environ.get("AVSR_B200_MAX_PLANS", "16"))
    GRAPH_AFTER = int(os.environ.get("AVSR_B200_GRAPH_AFTER", "3"))

    def __init__(self, d_model: int, n_heads: int, linear_units: int, num_blocks: int, cnn_kernel: int):
        self.cfg = EncoderConfig(d_model, n_heads, linear_units, num_blocks, cnn_kernel)
        need = lib.avsr_prepared_bytes(C.byref(self.cfg))
        if need == 0:
            check(_cabi.E_INVALID)
        self.prepared_bytes = need
        self._prepared: Dict[Tuple[int, int], torch.Tensor] = {}      # (device index, precision) -> buffer
        self._workspaces: "OrderedDict[tuple, torch.Tensor]" = OrderedDict()
        self._plans = PlanCache(self.MAX_PLANS)
        self._sat: Dict[int, torch.Tensor] = {}
        self.graph_after = self.GRAPH_AFTER
        self.stats = {"direct": 0, "graph": 0, "plans_built": 0}

    # ---- weights -------------------------------------------------------------------------------
    def invalidate(self) -> None:
        """Forget prepared weights (and the plans that bake their addresses)."""
        self._plans.clear()
        self._prepared.clear()

    def prepare(self, state, device: torch.device, precision: str) -> torch.Tensor:
        """state: reference-keyed tensors ('encoders.{l}.<suffix>', 'after_norm.*') living on `device`, or a
        callable returning them (only called when the prepared copy for (device, precision) is missing)."""
        key = (device.index or 0, PRECISIONS[precision])
        buf = self._prepared.get(key)
        if buf is not None:
            return buf
        if callable(state):
            state = state()
        L = self.cfg.num_blocks
        arr = (LayerParams * L)()
        keep = []
        for l in range(L):
            for field, suffix in LAYER_FIELDS:
                t = state[f"encoders.{l}.{suffix}"]
                require_cuda(t, suffix)
                if t.device != device:
                    raise RuntimeError(f"encoder parameter {suffix} (layer {l}) lives on {t.device} but the input is on "
                                       f"{device}: move the module with .to(device) first")
                t = t.detach().contiguous()
                keep.append(t)
                setattr(arr[l], field, t.data_ptr())
        aw = state["after_norm.weight"].detach().contiguous()
        ab = state["after_norm.bias"].detach().contiguous()
        buf = torch.empty(self.prepared_bytes, dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            check(lib.avsr_prepare_weights(C.byref(self.cfg), arr, aw.data_ptr(), ab.data_ptr(), buf.data_ptr(),
                                           self.prepared_bytes, PRECISIONS[precision], _stream_handle(device)))
        self._prepared[key] = buf
        return buf

    # ---- buffers -------------------------------------------------------------------------------
    def _workspace(self, B: int, T: int, device: torch.device, stream: int) -> torch.Tensor:
        """The direct-launch workspace: ONE buffer per (device, stream), grown to the largest shape seen (its layout
        is carved per call by the library, so any buffer that is large enough serves every shape)."""
        key = (device.index or 0, stream)
        nbytes = max(int(lib.avsr_workspace_bytes(C.byref(self.cfg), B, T)), 256)
        ws = self._workspaces.get(key)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(nbytes + nbytes // 4, dtype=torch.uint8, device=device)   # 25 % slack: fewer regrowths
            self._workspaces[key] = ws
        return ws

    # ---- forward -------------------------------------------------------------------------------
    def forward(self, prepared: torch.Tensor, xs: torch.Tensor, lengths: Optional[torch.Tensor], precision: str,
                use_graph: bool = True, taps: Optional[torch.Tensor] = None, check_saturation: bool = False) -> torch.Tensor:
        require_cuda(xs, "xs")
        if xs.dim() != 3 or xs.size(2) != self.cfg.d_model:
            raise ValueError(f"xs must be (B, T, {self.cfg.d_model}), got {tuple(xs.shape)}")
        B, T, D = xs.shape
        device = xs.device
        xs = xs.contiguous()
        out = torch.empty_like(xs)
        if B == 0 or T == 0:
            return out
        if lengths is not None:
            if lengths.device != device or lengths.dtype != torch.int32 or lengths.numel() != B:
                raise ValueError("lengths must be an int32 tensor of B elements on the input's device")
            lengths = lengths.contiguous()
        prec = PRECISIONS[precision]
        with torch.cuda.device(device):
            st = _stream_handle(device)
            plan = None
            if use_graph and taps is None and not check_saturation:
                plan = self._plan(prepared, B, T, device, prec, st)
            if plan is not None:
                self.stats["graph"] += 1
                check(lib.avsr_plan_forward(plan, xs.data_ptr(), _ptr(lengths), out.data_ptr(), st))
            else:
                self.stats["direct"] += 1
                ws = self._workspace(B, T, device, st)
                if check_saturation:
                    cnt = self._sat.get(device.index or 0)
                    if cnt is None:
                        cnt = self._sat[device.index or 0] = torch.zeros(1, dtype=torch.int64, device=device)
                    check(lib.avsr_encoder_forward_checked(C.byref(self.cfg), prepared.data_ptr(), xs.data_ptr(),
                                                           _ptr(lengths), B, T, out.data_ptr(), ws.data_ptr(),
                                                           ws.numel(), prec, cnt.data_ptr(), st))
                    n = int(cnt.item())                      # host sync: this is the diagnostic path
                    if n:
                        raise SaturationError(
                            f"{n} fp16 operand value(s) saturated at +-65504 (or NaN) in this forward: the f16 path "
                            "is outside its range for these weights / inputs -- use precision='bf16' (fp32's range), 'tf32' or "
                            "'fp32'")
                elif taps is None:
                    check(lib.avsr_encoder_forward(C.byref(self.cfg), prepared.data_ptr(), xs.data_ptr(), _ptr(lengths),
                                                   B, T, out.data_ptr(), ws.data_ptr(), ws.numel(), prec, st))
                else:
                    check(lib.avsr_encoder_forward_taps(C.byref(self.cfg), prepared.data_ptr(), xs.data_ptr(),
                                                        _ptr(lengths), B, T, out.data_ptr(), taps.data_ptr(),
                                                        ws.data_ptr(), ws.numel(), prec, st))
        return out

    def _plan(self, prepared: torch.Tensor, B: int, T: int, device: torch.device, prec: int, stream: int):
        """The plan for this shape, or None while the shape has been seen fewer than ``graph_after`` times.  A plan's
        workspace is private to it and to the stream it was built for (two streams never share one)."""
        key = (device.index or 0, B, T, prec, prepared.data_ptr(), stream)

        def build():
            self.stats["plans_built"] += 1
            ws = torch.empty(int(lib.avsr_workspace_bytes(C.byref(self.cfg), B, T)), dtype=torch.uint8, device=device)
            cs = self._plans.capture_stream(device)
            plan = C.c_void_p()
            check(lib.avsr_plan_create(C.byref(self.cfg), prepared.data_ptr(), B, T, ws.data_ptr(), ws.numel(), prec,
                                       cs.cuda_stream, C.byref(plan)))
            cs.synchronize()
            return plan, ws

        hit = self._plans.get(key, self.graph_after, build)
        return None if hit is None else hit[0]
