"""Unit-isolated float64 references of the front-ends' training path, the plausible kernel defects to check them
against, and the geometry of every conv unit a front-end runs.

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

The library trains a front-end as a chain of conv units (``auto_avsr_b200/frontend_train.py``: conv -> BatchNorm with
batch statistics -> [+ residual] -> [SiLU]).  ``unit(...)`` evaluates one unit from given inputs and a given gradient at
its output, so a unit the library ran inside a whole training step can be compared with a reference that starts from
the library's own inputs: the comparison carries one unit's rounding and names the unit that is wrong.

The BatchNorm backward is written out (not autograd) so that ``unit(..., defect=name)`` can make one mistake of the
kind a kernel change could make (see ``DEFECTS``); the convolutions' gradients are torch autograd.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor

WG_T = 64            # wgrad tile: 64 C_out x 64 k columns
WGT_PB = 32          # pixels per wgrad K-block: a split is a multiple of it
FT_ROWS = 256        # rows per BatchNorm statistics tile, at most (stats_tile_rows)


def stats_tile_rows(rows: int, C: int) -> int:
    """Rows per BatchNorm statistics tile (csrc/train.cu bn_tile_rows): FT_ROWS, halved down to 32 while the grid of
    tiles x ceil(C / 128) CTAs would hold fewer than two per SM of 132."""
    h = FT_ROWS
    while h > 32 and -(-rows // h) * -(-C // 128) < 2 * 132:
        h //= 2
    return h


DEFECTS: Dict[str, str] = {
    "wgrad_drop_split": "dW without the partial of one full-size pixel split (a slipped split offset)",
    "stem_no_utterance_mask": "the video stem's temporal taps read across utterances: the B*T frames act as one clip",
    "stem_drop_last_ktile": "the stem's dW without its last, partly masked 64-wide k tile",
    "dgrad_zero_parity_class": "one stride-2 parity class of dx left zero (the last class that receives gradient)",
    "bn_bwd_unbiased_var": "the BatchNorm backward normalises with the unbiased variance",
    "silu_grad_before_residual": "the SiLU gradient taken at the pre-residual value",
    "running_var_biased": "running_var moves toward the biased variance",
}


class Geom:
    """One conv unit: stem 0 (trunk; x (N, H, W, C_in), a 1-D conv when H = 1 and the module is 1-D), 1 (video stem,
    x (N = B * T, H, W)) or 2 (audio stem, x (N, W)); the same arguments as ``frontend_train._Spec.args()``."""

    def __init__(self, name: str, stem: int, N: int, T: int, H: int, W: int, Cin: int, Cout: int, KH: int, KW: int,
                 stride: int, dims: int):
        self.name, self.stem, self.N, self.T, self.H, self.W = name, stem, N, T, H, W
        self.Cin, self.Cout, self.KH, self.KW, self.stride, self.dims = Cin, Cout, KH, KW, stride, dims
        if stem == 1:
            self.Ho, self.Wo, self.K = (H - 1) // 2 + 1, (W - 1) // 2 + 1, 245
        elif stem == 2:
            self.Ho, self.Wo, self.K = 1, W // 4, 80
        else:
            self.Ho = (H + 2 * ((KH - 1) // 2) - KH) // stride + 1
            self.Wo = (W + 2 * ((KW - 1) // 2) - KW) // stride + 1
            self.K = KH * KW * Cin

    def args(self):
        return (self.stem, self.N, self.T, self.H, self.W, self.Cin, self.Cout, self.KH, self.KW, self.stride)

    @property
    def rows(self) -> int:
        return self.N * self.Ho * self.Wo

    def split_rows(self, splits: int) -> int:
        """Pixels per wgrad split (the library's rule): an even share rounded up to whole K-blocks."""
        return (-(-self.rows // splits) + WGT_PB - 1) // WGT_PB * WGT_PB

    def split_ranges(self, splits: int) -> List[Tuple[int, int]]:
        per = self.split_rows(splits)
        return [(min(s * per, self.rows), min((s + 1) * per, self.rows)) for s in range(splits)]


def _trunk_units(N: int, H: int, W: int, dims: int) -> List[Geom]:
    out, cin = [], 64
    for layer, planes in enumerate((64, 128, 256, 512)):
        for b in range(2):
            st = 2 if layer > 0 and b == 0 else 1
            pfx = f"layer{layer + 1}.{b}"
            kh = 3 if dims == 2 else 1
            c1 = Geom(pfx + ".conv1", 0, N, 1, H, W, cin, planes, kh, 3, st, dims)
            out.append(c1)
            out.append(Geom(pfx + ".conv2", 0, N, 1, c1.Ho, c1.Wo, planes, planes, kh, 3, 1, dims))
            if st == 2:
                out.append(Geom(pfx + ".downsample", 0, N, 1, H, W, cin, planes, 1, 1, 2, dims))
            H, W, cin = c1.Ho, c1.Wo, planes
    return out


def video_units(B: int, T: int, H: int, W: int) -> List[Geom]:
    """Every conv unit of a video front-end step on (B, T, 1, H, W), in the order of ``conv_bn_pairs()``."""
    stem = Geom("stem", 1, B * T, T, H, W, 1, 64, 0, 0, 0, 2)
    Hp, Wp = (stem.Ho - 1) // 2 + 1, (stem.Wo - 1) // 2 + 1
    return [stem] + _trunk_units(B * T, Hp, Wp, 2)


def audio_units(B: int, L: int) -> List[Geom]:
    """Every conv unit of an audio front-end step on (B, L, 1), in the order of ``conv_bn_pairs()``."""
    Lt = L // 640 * 640
    stem = Geom("stem", 2, B, 1, 1, Lt, 1, 64, 0, 0, 0, 1)
    return [stem] + _trunk_units(B, 1, stem.Wo, 1)


def units(case) -> List[Geom]:
    return video_units(*case[2:6]) if case[1] == "video" else audio_units(case[2], case[3])


#: (name, modality, B, T frames (video) or samples (audio), H, W, zero-padded tail from frame, precisions).  Each
#: case is here for an edge of the training kernels; tests/test_frontend_train_stages_cpu.py shows every edge is reached.
CASES = [
    # the video bucket: 132 stem splits of 23,488 pixels across frames and utterances; the layer-3 downsample's last
    # split empty; 17 layer-4 downsample splits
    ("bucket", "video", 4, 400, 88, 88, None, ("f16",)),
    # one frame per utterance (the stem's temporal taps all masked); layer 4 is 1x1 on 5 positions
    ("t1_24", "video", 5, 1, 24, 24, None, ("fp32", "tf32", "f16")),
    ("t2_32", "video", 4, 2, 32, 32, None, ("fp32", "tf32", "f16")),
    # 57 frames: layer 2's 513 rows leave 1 row in the last statistics tile
    ("t3_24", "video", 19, 3, 24, 24, None, ("fp32", "tf32", "f16")),
    # 89x89: stride-2 dgrad on odd H and W (layer 2's 23x23 input); 15 frames leave layer 1's last statistics tile one
    # row short; the second utterance's last two frames are zero padding
    ("t5_89", "video", 3, 5, 89, 89, 3, ("fp32", "tf32", "f16")),
    # non-square; layer 4's BatchNorm sees 32 positions per channel
    ("t4_45x61", "video", 2, 4, 45, 61, None, ("fp32", "tf32", "f16")),
    # 42 frames of 88x88: layer 1 runs 59 splits, the last one empty; the stem 132, four of them empty
    ("t7_42", "video", 6, 7, 88, 88, None, ("fp32", "tf32", "f16")),
    ("bucket", "audio", 4, 256000, 1, 1, None, ("f16",)),
    ("ragged", "audio", 2, 2 * 640 + 333, 1, 1, None, ("fp32", "tf32", "f16")),
    ("one_frame", "audio", 2, 640, 1, 1, None, ("fp32", "tf32", "f16")),
]


# ------------------------------------------------------------------ the unit in float64
def _stem_channels(x: Tensor, T: int, masked: bool = True) -> Tensor:
    """(B * T, H, W) frames -> (B * T, 5, H, W): frame t's five temporal taps t - 2 .. t + 2 as channels, zero outside
    its utterance (``masked=False``: outside the whole B * T sequence).  The video stem's Conv3d is then a Conv2d."""
    N = x.shape[0]
    n = torch.arange(N, device=x.device)
    taps = []
    for dt in range(5):
        src = n + dt - 2
        ok = (src >= 0) & (src < N)
        if masked:
            t = n % T
            ok &= (t + dt - 2 >= 0) & (t + dt - 2 < T)
        taps.append(torch.where(ok[:, None, None], x[src.clamp(0, N - 1)], torch.zeros((), dtype=x.dtype,
                                                                                        device=x.device)))
    return torch.stack(taps, 1)


def conv(x: Tensor, w: Tensor, g: Geom, defect: Optional[str] = None) -> Tensor:
    """The unit's convolution on channels-last x, in torch's weight layout: (N, Ho, Wo, C_out)."""
    if g.stem == 1:
        xs = _stem_channels(x, g.T, masked=defect != "stem_no_utterance_mask")
        return F.conv2d(xs, w.reshape(64, 5, 7, 7), stride=2, padding=3).permute(0, 2, 3, 1)
    if g.stem == 2:
        return F.conv1d(x[:, None], w, stride=4, padding=38).permute(0, 2, 1)[:, None]
    if g.dims == 2:
        return F.conv2d(x.permute(0, 3, 1, 2), w, stride=g.stride, padding=(g.KH - 1) // 2).permute(0, 2, 3, 1)
    return F.conv1d(x[:, 0].permute(0, 2, 1), w, stride=g.stride, padding=(g.KW - 1) // 2).permute(0, 2, 1)[:, None]


def parity_class(g: Geom) -> Optional[Tuple[int, int]]:
    """The stride-2 parity class (ry, rx) of dx that ``dgrad_zero_parity_class`` zeroes: the last one that receives
    gradient (None: no stride-2 dgrad at this unit)."""
    if g.stem != 0 or g.stride != 2:
        return None
    r = 1 if g.KW == 3 else 0
    return (r if g.H > 1 else 0, r)


def applies(defect: str, g: Geom, act: bool, has_resid: bool) -> bool:
    """Whether ``defect`` can change anything at this unit."""
    if defect == "stem_no_utterance_mask":
        return g.stem == 1 and g.N > g.T
    if defect == "stem_drop_last_ktile":
        # the video stem's last k tile (k >= 192) holds the temporal taps t + 1 and t + 2 only: all masked when T = 1
        return g.stem == 2 or (g.stem == 1 and g.T > 1)
    if defect == "dgrad_zero_parity_class":
        return parity_class(g) is not None
    if defect == "silu_grad_before_residual":
        return act and has_resid
    return True


def unit(x: Tensor, resid: Optional[Tensor], w: Tensor, gamma: Tensor, beta: Tensor, running_mean: Tensor,
         running_var: Tensor, momentum: float, eps: float, g: Geom, act: bool, dy: Tensor, splits: int = 1,
         defect: Optional[str] = None) -> Dict[str, Optional[Tensor]]:
    """conv -> BatchNorm (batch statistics) -> [+ resid] -> [SiLU] and its backward for the gradient ``dy`` at the
    output, in the dtype of the inputs.  Returns y, dx (trunk units), dres (with a residual), dw, dgamma, dbeta and the
    running statistics after the step (``momentum`` is the averaging factor of this step).  ``splits`` is the library's
    wgrad pixel-split count (only ``wgrad_drop_split`` reads it)."""
    if defect is not None and defect not in DEFECTS:
        raise ValueError(f"unknown defect {defect}")
    xg = x.detach().requires_grad_(g.stem == 0)
    wg = w.detach().requires_grad_(True)
    z = conv(xg, wg, g, defect)
    C = z.shape[-1]
    zf = z.detach().reshape(-1, C)
    n = zf.shape[0]
    mean = zf.mean(0)
    d = zf - mean
    var_b = d.square().mean(0)
    var_u = d.square().sum(0) / (n - 1)
    invstd = (var_b + eps).rsqrt()
    xh = d * invstd
    h = xh * gamma + beta
    pre = h
    if resid is not None:
        h = h + resid.reshape(-1, C)
    y = h * torch.sigmoid(h) if act else h
    ds = dy.reshape(-1, C)
    if act:
        at = pre if defect == "silu_grad_before_residual" else h
        s = torch.sigmoid(at)
        ds = ds * s * (1 + at * (1 - s))
    if defect == "bn_bwd_unbiased_var":
        invstd = (var_u + eps).rsqrt()
        xh = d * invstd
    dbeta, dgamma = ds.sum(0), (ds * xh).sum(0)
    dz = (gamma * invstd * (ds - (dbeta + xh * dgamma) / n)).reshape(z.shape)
    rv_to = var_b if defect == "running_var_biased" else var_u
    out = {"y": y.reshape(z.shape), "dres": ds.reshape(z.shape) if resid is not None else None,
           "dgamma": dgamma, "dbeta": dbeta,
           "running_mean": (1 - momentum) * running_mean + momentum * mean,
           "running_var": (1 - momentum) * running_var + momentum * rv_to}
    if g.stem == 0:
        dx, dw = torch.autograd.grad(z, (xg, wg), dz, retain_graph=defect == "wgrad_drop_split")
        pc = parity_class(g) if defect == "dgrad_zero_parity_class" else None
        if pc is not None:
            dx = dx.clone()
            dx[:, pc[0]::2, pc[1]::2] = 0
        out["dx"] = dx
    else:
        (dw,) = torch.autograd.grad(z, (wg,), dz, retain_graph=defect == "wgrad_drop_split")
        out["dx"] = None
    if defect == "wgrad_drop_split":
        # the middle of the non-empty splits, rounded down: a full-size split whenever there are two or more
        full = [r for r in g.split_ranges(splits) if r[1] > r[0]]
        lo, hi = full[(len(full) - 1) // 2]
        mask = torch.zeros(n, 1, dtype=dz.dtype, device=dz.device)
        mask[lo:hi] = 1
        (part,) = torch.autograd.grad(z, (wg,), (dz.reshape(-1, C) * mask).reshape(z.shape))
        dw = dw - part
    if defect == "stem_drop_last_ktile":
        dw = dw.reshape(64, -1).clone()
        dw[:, (g.K - 1) // WG_T * WG_T:] = 0
        dw = dw.reshape(w.shape)
    out["dw"] = dw
    return out


def torch_unit(x: Tensor, resid: Optional[Tensor], w: Tensor, gamma: Tensor, beta: Tensor, running_mean: Tensor,
               running_var: Tensor, momentum: float, eps: float, g: Geom, act: bool,
               dy: Tensor) -> Dict[str, Optional[Tensor]]:
    """The same unit as torch's own modules compute it (Conv3d / Conv2d / Conv1d, ``F.batch_norm`` in training mode,
    ``F.silu``, autograd), in the dtype of the inputs and torch's layout: the reference for ``unit`` and, in fp32 with
    cuDNN TF32, the reference implementation's training arithmetic."""
    xg = x.detach().requires_grad_(g.stem == 0)
    rg = resid.detach().requires_grad_(True) if resid is not None else None
    wg, gg, bg = (t.detach().requires_grad_(True) for t in (w, gamma, beta))
    rm, rv = running_mean.clone(), running_var.clone()
    if g.stem == 1:
        B = g.N // g.T
        z = F.conv3d(xg.reshape(B, 1, g.T, g.H, g.W), wg, stride=(1, 2, 2), padding=(2, 3, 3))
        h = F.batch_norm(z, rm, rv, gg, bg, True, momentum, eps)
        h = h.permute(0, 2, 3, 4, 1).reshape(g.N, g.Ho, g.Wo, 64)
    elif g.stem == 2:
        h = F.batch_norm(F.conv1d(xg[:, None], wg, stride=4, padding=38), rm, rv, gg, bg, True, momentum, eps)
        h = h.permute(0, 2, 1)[:, None]
    elif g.dims == 2:
        z = F.conv2d(xg.permute(0, 3, 1, 2), wg, stride=g.stride, padding=(g.KH - 1) // 2)
        h = F.batch_norm(z, rm, rv, gg, bg, True, momentum, eps).permute(0, 2, 3, 1)
    else:
        z = F.conv1d(xg[:, 0].permute(0, 2, 1), wg, stride=g.stride, padding=(g.KW - 1) // 2)
        h = F.batch_norm(z, rm, rv, gg, bg, True, momentum, eps).permute(0, 2, 1)[:, None]
    if rg is not None:
        h = h + rg
    y = F.silu(h) if act else h
    inputs = [t for t in (xg, rg, wg, gg, bg) if t is not None and t.requires_grad]
    grads = dict(zip([id(t) for t in inputs], torch.autograd.grad(y, inputs, dy)))
    return {"y": y.detach(), "dx": grads.get(id(xg)), "dres": grads.get(id(rg)) if rg is not None else None,
            "dw": grads[id(wg)], "dgamma": grads[id(gg)], "dbeta": grads[id(bg)], "running_mean": rm,
            "running_var": rv}


def pool_by_winner(x: Tensor, idx: Tensor) -> Tensor:
    """MaxPool((1, 3, 3), (1, 2, 2), (0, 1, 1)) of torch-layout x (B, C, T, H, W) whose window winners are given:
    idx (B * T, Ho, Wo, C) holds the window index dy * 3 + dx the library recorded.  Differentiable in x, so a float64
    chain through it routes every gradient to the library's winner."""
    B, C, T, H, W = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = F.pad(x, (1, 1, 1, 1), value=float("-inf"))
    cand = torch.stack([xp[..., dy:dy + 2 * Ho - 1:2, dx:dx + 2 * Wo - 1:2] for dy in range(3) for dx in range(3)])
    sel = idx.long().reshape(B, T, Ho, Wo, C).permute(0, 4, 1, 2, 3)[None]
    return cand.gather(0, sel)[0]


def rel(a: Optional[Tensor], b: Optional[Tensor]) -> float:
    """max |a - b| / max |b|, in float64."""
    b = b.double()
    return ((a.double().to(b.device) - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()
