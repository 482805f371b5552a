"""Stage-isolated references of one Conformer encoder layer, and plausible kernel defects to check them against.

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

The encoder layer is five residual stages (``conformer_oracle.encoder_layer``): the macaron FFN, the rel-pos MHA, the
conv module, the FFN and norm_final.  ``stage(s, x_in, ...)`` evaluates stage ``s`` alone from a given input, so a
GPU tap can be compared with a reference that starts from the GPU's own input to that stage: the comparison then
carries one stage's rounding instead of everything upstream of it.

``stage(..., defect=name)`` evaluates the same stage with one deliberate mistake of the kind a kernel change could
make (see ``DEFECTS``).  A test shows that its bound would catch such a mistake by checking that the defective
reference misses the GPU output by a clear margin.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import conformer_oracle as O

Tensor = torch.Tensor

STAGES = ("ffn_macaron", "mha", "conv", "ffn", "norm_final")
TILE = 64   # query rows of one attention CTA

# defect name -> the stage it applies to
DEFECTS: Dict[str, int] = {
    "ffn_macaron_b2_block": 0,   # w_2 bias missing on the last 64 output columns (a stale bias tile in the epilogue)
    "mha_uv_swap_last_head": 1,  # pos_bias_u and pos_bias_v swapped for the last head (a QK-epilogue scatter slip)
    "mha_relshift_tile": 1,      # rel-shift one row off for the queries of the last 64-query tile
    "mha_drop_last_key": 1,      # the last valid key of every utterance masked out
    "conv_halo": 2,              # depthwise halo reads the neighbouring utterance instead of zeros (B > 1 only)
    "ffn_b2_block": 3,           # as ffn_macaron_b2_block, in the second FFN
    "ln_unbiased_var": 4,        # norm_final divides the variance by d - 1
}


def applies(defect: str, B: int, T: int) -> bool:
    """Whether ``defect`` changes anything at B utterances of T frames: the conv halo needs an utterance boundary,
    and with a single key the softmax is 1 whatever the score, so a wrong bias or position row does nothing."""
    if defect == "conv_halo":
        return B > 1
    if defect in ("mha_uv_swap_last_head", "mha_relshift_tile"):
        return T > 1
    return True


def _ln(x: Tensor, sd, pfx: str, name: str) -> Tensor:
    return O.layer_norm(x, sd[pfx + name + ".weight"], sd[pfx + name + ".bias"])


def _ln_unbiased(x: Tensor, w: Tensor, b: Tensor) -> Tensor:
    mean = x.mean(dim=-1, keepdim=True)
    var = (x - mean).pow(2).sum(dim=-1, keepdim=True) / (x.shape[-1] - 1)
    return (x - mean) / torch.sqrt(var + O.LN_EPS) * w + b


def _without_bias_block(sd, key: str):
    sd = dict(sd)
    b = sd[key].clone()
    b[-TILE:] = 0
    sd[key] = b
    return sd


def _swap_uv_last_head(sd, pfx: str):
    sd = dict(sd)
    u, v = sd[pfx + "pos_bias_u"].clone(), sd[pfx + "pos_bias_v"].clone()
    u[-1], v[-1] = sd[pfx + "pos_bias_v"][-1], sd[pfx + "pos_bias_u"][-1]
    sd[pfx + "pos_bias_u"], sd[pfx + "pos_bias_v"] = u, v
    return sd


def _mha(x: Tensor, pos_emb: Tensor, lengths: Optional[Tensor], sd, pfx: str, n_heads: int,
         defect: Optional[str]) -> Tensor:
    B, T, _ = x.shape
    if defect == "mha_uv_swap_last_head":
        return O.rel_mha(x, pos_emb, lengths, _swap_uv_last_head(sd, pfx), pfx, n_heads)
    if defect == "mha_drop_last_key":
        full = torch.full((B,), T, dtype=torch.long, device=x.device) if lengths is None else lengths
        return O.rel_mha(x, pos_emb, (full - 1).clamp_min(0), sd, pfx, n_heads)
    out = O.rel_mha(x, pos_emb, lengths, sd, pfx, n_heads)
    if defect == "mha_relshift_tile":
        # linear_pos has no bias and a query row's output depends on its own scores only, so reading row m + 1 of the
        # projected table for some queries is the same as running those queries against the table moved up one row
        # (the last row repeated: a kernel would read past the band there)
        idx = torch.arange(1, 2 * T, device=x.device).clamp_max(2 * T - 2)
        slipped = O.rel_mha(x, pos_emb[idx], lengths, sd, pfx, n_heads)
        t0 = (T - 1) // TILE * TILE
        out = out.clone()
        out[:, t0:] = slipped[:, t0:]
    return out


def stage(s: int, x: Tensor, pos_emb: Tensor, lengths: Optional[Tensor], sd, pfx: str, n_heads: int,
          defect: Optional[str] = None) -> Tensor:
    """Residual stage ``s`` of the encoder layer at ``pfx`` applied to its input ``x`` (B, T, d), optionally with one
    of ``DEFECTS`` (which must belong to stage ``s``)."""
    if defect is not None and DEFECTS[defect] != s:
        raise ValueError(f"defect {defect} belongs to stage {DEFECTS[defect]}, not {s}")
    if s == 0:
        if defect:
            sd = _without_bias_block(sd, pfx + "feed_forward_macaron.w_2.bias")
        return x + 0.5 * O.feed_forward(_ln(x, sd, pfx, "norm_ff_macaron"), sd, pfx + "feed_forward_macaron.")
    if s == 1:
        return x + _mha(_ln(x, sd, pfx, "norm_mha"), pos_emb, lengths, sd, pfx + "self_attn.", n_heads, defect)
    if s == 2:
        h = _ln(x, sd, pfx, "norm_conv")
        if defect:
            # one long sequence of B*T frames: the depthwise conv reads across every utterance boundary
            B, T, D = h.shape
            return x + O.conv_module(h.reshape(1, B * T, D), sd, pfx + "conv_module.").reshape(B, T, D)
        return x + O.conv_module(h, sd, pfx + "conv_module.")
    if s == 3:
        if defect:
            sd = _without_bias_block(sd, pfx + "feed_forward.w_2.bias")
        return x + 0.5 * O.feed_forward(_ln(x, sd, pfx, "norm_ff"), sd, pfx + "feed_forward.")
    if s == 4:
        if defect:
            return _ln_unbiased(x, sd[pfx + "norm_final.weight"], sd[pfx + "norm_final.bias"])
        return _ln(x, sd, pfx, "norm_final")
    raise ValueError(f"stage {s}")


def layer_and_after_norm(x: Tensor, pos_emb: Tensor, lengths: Optional[Tensor], sd, layer: int,
                         n_heads: int) -> Tensor:
    """Encoder layer ``layer`` applied to ``x``, then after_norm: the output of a ``layer + 1``-layer encoder whose
    previous layers produced ``x``."""
    y = O.encoder_layer(x, pos_emb, lengths, sd, f"encoders.{layer}.", n_heads)
    return O.layer_norm(y, sd["after_norm.weight"], sd["after_norm.bias"])


def errors(g: Tensor, r: Tensor, g_in: Optional[Tensor] = None) -> Dict[str, float]:
    """How far ``g`` is from the reference ``r`` (both (..., d)).

    ``max`` / ``rms``: max-abs and rms of g - r over a scale.  With ``g_in`` (the stage's input) the scale is the
    stage's own contribution max|r - g_in|, because the residual stream it is added to would hide an error in it;
    without, the scale is max|r|.
    ``frames``: per frame, the max over channels of |g - r|; the largest frame value over the median frame value.  A
    mistake at a tile or utterance edge shows up as a few outlier frames, rounding noise does not.  ``worst`` is
    the flat (b * T + t) index of the largest frame.
    """
    d = (g.double() - r).abs().reshape(-1, r.shape[-1])
    scale = ((r - g_in.double()) if g_in is not None else r).abs().max().item()
    frame = d.amax(dim=1)
    top, med = frame.max().item(), frame.median().item()
    return {"max": top / scale, "rms": d.pow(2).mean().sqrt().item() / scale,
            "frames": 1.0 if top == 0 else (top / med if med > 0 else float("inf")), "scale": scale,
            "worst": int(frame.argmax())}
