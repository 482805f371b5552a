"""Teacher-forced training pass of the attention decoder and its LabelSmoothingLoss (e2e_asr_conformer.py:77-80):
``torch.autograd.Function``s whose forward AND backward run in libavsr_b200 (csrc/decoder_train.cu), composed with the
encoder path's ``LinearFn`` / ``LayerNormFn`` / ``feed_forward_train`` into ``TransformerDecoder.forward``
(transformer_decoder.py:229-258).

- ``MhaCoreFn``: masked multi-head attention core (attention.py:59-88) on the projected q / k / v, read in place from the
  fused self q|k|v and source k|v GEMM outputs; dropout on the probabilities is live (E2E builds the decoder with
  self / source attention dropout 0.1), with keep-masks drawn by torch (``draw_keep_mask``).
- ``EmbedFn``: Embedding * sqrt(d) + PositionalEncoding (embedding.py:60-90); the backward groups positions by token on
  the device and sums them in a fixed order.
- ``LabelSmoothingFn``: LabelSmoothingLoss(normalize_length=False) (label_smoothing_loss.py:41-63) = sum of the
  per-row KL divergences / B, with no host synchronisation (the reference's ``.item()`` is not needed for the
  batch-size denominator).

torch supplies device memory, the autograd tape, dropout masks and the residual adds.  Gradients land on the original
``Parameter``s; the memory gradient flows back into the encoder.  Under ``torch.no_grad()`` or in ``eval()`` the same
kernels run without storing probabilities and without dropout.

``TransformerDecoder.backward_precision = "bf16"`` gives every backward GEMM of the decoder bf16 operands and runs the
attention core's backward on the tensor cores (avsr_mha_core_bwd_tc); None (the default) keeps the TF32 / fp32 backward.
Embedding, LayerNorm and the label-smoothing loss keep their fp32 kernels."""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from ._cabi import check, lib
from .engine import _ptr, _stream_handle
from .engine import PRECISIONS
from .train import LayerNormFn, LinearFn, _c, _workspace, feed_forward_train


def draw_keep_mask(p: float, shape, device) -> torch.Tensor:
    """uint8 keep-mask of dropout rate ``p`` (1 = kept), drawn from torch's generator like ``torch.nn.Dropout``."""
    return (torch.rand(shape, device=device) < 1.0 - p).view(torch.uint8)


def _rows(t: torch.Tensor, vector_rows: bool = True):
    """(B, L, cols) fp32 view -> (tensor, row stride) the kernels can read in place: unit column stride, rows evenly
    spaced across the batch and, for the attention kernels' float4 loads (``vector_rows``), 16-byte aligned rows;
    anything else is copied."""
    B, L, _ = t.shape
    ld = t.stride(1)
    ok = t.stride(2) == 1 and (B <= 1 or t.stride(0) == L * ld) and ld >= t.size(2)
    if vector_rows:
        ok = ok and ld % 4 == 0 and t.data_ptr() % 16 == 0
    if not ok:
        t = t.contiguous()
        ld = t.size(2)
    return t, ld


# ------------------------------------------------------------------------------------------------ raw ops
def mha_core_forward(q, k, v, n_heads: int, causal: bool, lengths: Optional[torch.Tensor], keep: Optional[torch.Tensor],
                     keep_scale: float, want_probs: bool):
    """avsr_mha_core_fwd: q (B, Lq, H*64), k / v (B, Lk, H*64) (views with a row stride are read in place), int32 key
    lengths (B) or None -> (ctx (B, Lq, H*64), probs (B, H, Lq, Lk) or None)."""
    (q, ldq), (k, ldk), (v, ldv) = _rows(q.detach()), _rows(k.detach()), _rows(v.detach())
    B, Lq, D = q.shape
    Lk = k.size(1)
    ctx = torch.empty(B, Lq, D, dtype=torch.float32, device=q.device)
    probs = torch.empty(B, n_heads, Lq, Lk, dtype=torch.float32, device=q.device) if want_probs else None
    with torch.cuda.device(q.device):
        check(lib.avsr_mha_core_fwd(q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv, B, n_heads, Lq, Lk,
                                    int(causal), _ptr(lengths), _ptr(keep), float(keep_scale), ctx.data_ptr(), _ptr(probs),
                                    _stream_handle(q.device)))
    return ctx, probs


def mha_core_backward(q, k, v, n_heads: int, causal: bool, lengths, keep, keep_scale: float, probs, dctx, dq, dk, dv):
    """avsr_mha_core_bwd into the (possibly strided) views dq (B, Lq, H*64) and dk / dv (B, Lk, H*64), which must share
    one row stride."""
    (q, ldq), (k, ldk), (v, ldv) = _rows(q.detach()), _rows(k.detach()), _rows(v.detach())
    B, Lq, _ = q.shape
    Lk = k.size(1)
    dctx = _c(dctx)
    assert dk.stride(1) == dv.stride(1)
    ws = _workspace(q.device, int(lib.avsr_mha_core_bwd_workspace_bytes(B, n_heads, Lq)))
    with torch.cuda.device(q.device):
        check(lib.avsr_mha_core_bwd(q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv, B, n_heads, Lq, Lk,
                                    int(causal), _ptr(lengths), _ptr(keep), float(keep_scale), probs.data_ptr(),
                                    dctx.data_ptr(), dq.data_ptr(), dq.stride(1), dk.data_ptr(), dv.data_ptr(), dk.stride(1),
                                    ws.data_ptr(), ws.numel(), _stream_handle(q.device)))


def mha_core_backward_tc(q, k, v, n_heads: int, causal: bool, lengths, keep, keep_scale: float, probs, out, dctx, dq, dk,
                         dv):
    """avsr_mha_core_bwd_tc (bf16 operands on the tensor cores, fp32 accumulation): ``mha_core_backward`` plus the
    forward's output ``out`` (B, Lq, H*64), from which Delta = rowsum(dctx o out) is taken."""
    (q, ldq), (k, ldk), (v, ldv) = _rows(q.detach()), _rows(k.detach()), _rows(v.detach())
    B, Lq, _ = q.shape
    Lk = k.size(1)
    dctx, out = _c(dctx), _c(out)
    assert dk.stride(1) == dv.stride(1)
    prec = PRECISIONS["bf16"]
    ws = _workspace(q.device, int(lib.avsr_mha_core_bwd_tc_workspace_bytes(B, n_heads, Lq, Lk, prec)))
    with torch.cuda.device(q.device):
        check(lib.avsr_mha_core_bwd_tc(q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv, B, n_heads, Lq, Lk,
                                       int(causal), _ptr(lengths), _ptr(keep), float(keep_scale), probs.data_ptr(),
                                       out.data_ptr(), dctx.data_ptr(), dq.data_ptr(), dq.stride(1), dk.data_ptr(),
                                       dv.data_ptr(), dk.stride(1), prec, ws.data_ptr(), ws.numel(),
                                       _stream_handle(q.device)))


def _split(qsrc, kvsrc, self_attn: bool, D: int):
    if self_attn:
        return qsrc[..., :D], qsrc[..., D:2 * D], qsrc[..., 2 * D:3 * D]
    return qsrc, kvsrc[..., :D], kvsrc[..., D:2 * D]


class MhaCoreFn(torch.autograd.Function):
    """ctx = dropout(softmax(q k^T / 8, mask)) v  (attention.py:59-88).  Self attention: ``qsrc`` is the (B, L, 3d)
    q|k|v GEMM output and ``kvsrc`` the same tensor; source attention: ``qsrc`` (B, L, d) and ``kvsrc`` the (B, T, 2d)
    k|v GEMM output.  The gradient comes back in the same fused layouts (no slicing copies).  Backward: the fp32 kernels
    (``mha_core_backward``), or with ``backward="bf16"`` the tensor-core kernels (``mha_core_backward_tc``), which also
    need the output, so only then is it saved."""

    @staticmethod
    def forward(ctx_, qsrc, kvsrc, self_attn: bool, n_heads: int, causal: bool, lengths, keep, keep_scale: float,
                backward: Optional[str] = None):
        D = n_heads * 64
        q, k, v = _split(qsrc, kvsrc, self_attn, D)
        out, probs = mha_core_forward(q, k, v, n_heads, causal, lengths, keep, keep_scale, want_probs=True)
        ctx_.save_for_backward(qsrc, kvsrc, lengths, keep, probs, out if backward == "bf16" else None)
        ctx_.cfg = (self_attn, n_heads, causal, keep_scale)
        ctx_.backward = backward
        return out

    @staticmethod
    def backward(ctx_, dout):
        qsrc, kvsrc, lengths, keep, probs, out = ctx_.saved_tensors
        self_attn, n_heads, causal, keep_scale = ctx_.cfg
        D = n_heads * 64
        q, k, v = _split(qsrc, kvsrc, self_attn, D)

        def core_bwd(dq, dk, dv):
            if ctx_.backward == "bf16":
                mha_core_backward_tc(q, k, v, n_heads, causal, lengths, keep, keep_scale, probs, out, dout, dq, dk, dv)
            else:
                mha_core_backward(q, k, v, n_heads, causal, lengths, keep, keep_scale, probs, dout, dq, dk, dv)

        if self_attn:
            dsrc = torch.empty(qsrc.shape, dtype=torch.float32, device=qsrc.device)
            core_bwd(*_split(dsrc, None, True, D))
            return dsrc, None, None, None, None, None, None, None, None
        dq = torch.empty(qsrc.shape, dtype=torch.float32, device=qsrc.device)
        dkv = torch.empty(kvsrc.shape, dtype=torch.float32, device=kvsrc.device)
        core_bwd(dq, dkv[..., :D], dkv[..., D:])
        return dq, dkv, None, None, None, None, None, None, None


def mha_core(qsrc, kvsrc, self_attn: bool, n_heads: int, causal: bool, lengths, keep, keep_scale: float,
             backward: Optional[str] = None):
    """``MhaCoreFn`` when a gradient is wanted; otherwise the forward kernel alone (no probabilities stored)."""
    if torch.is_grad_enabled() and (qsrc.requires_grad or kvsrc.requires_grad):
        return MhaCoreFn.apply(qsrc, kvsrc, self_attn, n_heads, causal, lengths, keep, keep_scale, backward)
    q, k, v = _split(qsrc, kvsrc, self_attn, n_heads * 64)
    return mha_core_forward(q, k, v, n_heads, causal, lengths, keep, keep_scale, want_probs=False)[0]


class EmbedFn(torch.autograd.Function):
    """x = embed.weight[tokens] * sqrt(d) + pe[:L]  (transformer_decoder.py:250, embedding.py:60-90) on (B, L) int64
    tokens.  A token outside [0, odim) gives a NaN row (and no gradient)."""

    @staticmethod
    def forward(ctx, tokens, weight):
        tokens = tokens.to(torch.int64).contiguous()
        w = _c(weight)
        odim, D = w.shape
        B, L = tokens.shape
        x = torch.empty(B, L, D, dtype=torch.float32, device=w.device)
        with torch.cuda.device(w.device):
            check(lib.avsr_embed_fwd(tokens.data_ptr(), w.data_ptr(), B * L, max(L, 1), D, odim, x.data_ptr(),
                                     _stream_handle(w.device)))
        ctx.save_for_backward(tokens)
        ctx.wshape = (odim, D)
        return x

    @staticmethod
    def backward(ctx, dx):
        (tokens,) = ctx.saved_tensors
        odim, D = ctx.wshape
        dx = _c(dx)
        dw = torch.empty(odim, D, dtype=torch.float32, device=dx.device)
        rows = tokens.numel()
        ws = _workspace(dx.device, int(lib.avsr_embed_bwd_workspace_bytes(rows, odim)))
        with torch.cuda.device(dx.device):
            check(lib.avsr_embed_bwd(tokens.data_ptr(), dx.data_ptr(), rows, D, odim, dw.data_ptr(), ws.data_ptr(),
                                     ws.numel(), _stream_handle(dx.device)))
        return None, dw


class LabelSmoothingFn(torch.autograd.Function):
    """LabelSmoothingLoss(size=odim, padding_idx=ignore_id, smoothing, normalize_length=False)(x, target)
    (label_smoothing_loss.py:41-63): sum over the non-ignored rows of KL(smoothed target || softmax(x)), divided by
    ``batch``.  ``x`` (B, L, odim) may be a column slice of a wider (B, L, ld) tensor (the padded output-layer GEMM):
    it is read in place, and its gradient is returned in the same layout."""

    @staticmethod
    def forward(ctx, x, target, ignore_id: int, smoothing: float, batch: int):
        xs, ld = _rows(x.detach(), vector_rows=False)
        B, L, odim = xs.shape
        rows = B * L
        tgt = target.reshape(-1).to(device=xs.device, dtype=torch.int64).contiguous()
        if tgt.numel() != rows:
            raise ValueError(f"LabelSmoothingLoss: target has {tgt.numel()} entries for {rows} rows")
        row_loss = torch.empty(rows, dtype=torch.float32, device=xs.device)
        lse = torch.empty(rows, dtype=torch.float32, device=xs.device)
        with torch.cuda.device(xs.device):
            check(lib.avsr_label_smoothing_fwd(xs.data_ptr(), ld, tgt.data_ptr(), rows, odim, int(ignore_id),
                                               float(smoothing), row_loss.data_ptr(), lse.data_ptr(),
                                               _stream_handle(xs.device)))
        ctx.save_for_backward(xs, tgt, lse)
        ctx.cfg = (ld, ignore_id, smoothing, batch)
        return row_loss.sum() / batch

    @staticmethod
    def backward(ctx, dloss):
        xs, tgt, lse = ctx.saved_tensors
        ld, ignore_id, smoothing, batch = ctx.cfg
        B, L, odim = xs.shape
        dscale = (dloss.to(torch.float32) / batch).reshape(1).contiguous()       # stays on the device
        dx = torch.empty(B, L, ld, dtype=torch.float32, device=xs.device)
        with torch.cuda.device(xs.device):
            check(lib.avsr_label_smoothing_bwd(xs.data_ptr(), ld, tgt.data_ptr(), B * L, odim, int(ignore_id),
                                               float(smoothing), lse.data_ptr(), dscale.data_ptr(), dx.data_ptr(), ld,
                                               _stream_handle(xs.device)))
        return dx[..., :odim], None, None, None, None


# ------------------------------------------------------------------------------------------------ masks
def target_lengths(tgt_mask: torch.Tensor, B: int, L: int, check_mask: bool = False) -> torch.Tensor:
    """(B, L, L) ``target_mask`` (mask.py:27-37: key-prefix AND lower-triangular) -> int32 key lengths (B), read from its
    last row, without a host sync.  ``check_mask`` verifies the form (one host sync) and raises otherwise."""
    if tgt_mask is None:
        raise NotImplementedError("TransformerDecoder.forward: tgt_mask=None (no causal mask) is not supported; pass "
                                  "target_mask(ys_in_pad, ignore_id)")
    if tgt_mask.dim() != 3 or tuple(tgt_mask.shape) != (B, L, L):
        raise NotImplementedError(f"TransformerDecoder.forward: tgt_mask must be (B, L, L) = {(B, L, L)} from target_mask, "
                                  f"got {tuple(tgt_mask.shape)}")
    m = tgt_mask.to(torch.bool)
    lengths = m[:, -1, :].sum(dim=-1, dtype=torch.int32)
    if check_mask:
        ar = torch.arange(L, device=m.device)
        want = (ar[None, None, :] < lengths[:, None, None]) & (ar[None, None, :] <= ar[None, :, None])
        if not bool(torch.equal(want, m)):
            raise NotImplementedError("tgt_mask is not a key-prefix AND causal mask (target_mask); the CUDA path takes "
                                      "a causal flag and key lengths")
    return lengths


# ------------------------------------------------------------------------------------------------ module forwards
def _keep(m, B: int, Lq: int, Lk: int, device):
    p = m.dropout.p
    if not m.training or p == 0.0:
        return None, 1.0
    return draw_keep_mask(p, (B, m.h, Lq, Lk), device), (1.0 / (1.0 - p) if p < 1.0 else 0.0)


def _check_heads(m):
    if m.d_k != 64:
        raise NotImplementedError(f"decoder attention: d_k = 64 only (got {m.d_k})")


def self_attention_train(m, x, lengths, precision: str, backward: Optional[str] = None):
    """MultiHeadedAttention(x, x, x, tgt_mask) (attention.py:90-110) with the causal target mask: one q|k|v GEMM."""
    _check_heads(m)
    B, L, _ = x.shape
    w = torch.cat([m.linear_q.weight, m.linear_k.weight, m.linear_v.weight])
    b = torch.cat([m.linear_q.bias, m.linear_k.bias, m.linear_v.bias])
    qkv = LinearFn.apply(x, w, b, False, precision, backward)
    keep, scale = _keep(m, B, L, L, x.device)
    ctx = mha_core(qkv, qkv, True, m.h, True, lengths, keep, scale, backward)
    return LinearFn.apply(ctx, m.linear_out.weight, m.linear_out.bias, False, precision, backward)


def source_attention_train(m, x, memory, mem_lengths, precision: str, backward: Optional[str] = None):
    """MultiHeadedAttention(x, memory, memory, memory_mask): q GEMM on x, one k|v GEMM on the memory."""
    _check_heads(m)
    B, L, _ = x.shape
    q = LinearFn.apply(x, m.linear_q.weight, m.linear_q.bias, False, precision, backward)
    kv = LinearFn.apply(memory, torch.cat([m.linear_k.weight, m.linear_v.weight]),
                        torch.cat([m.linear_k.bias, m.linear_v.bias]), False, precision, backward)
    keep, scale = _keep(m, B, L, memory.size(1), x.device)
    ctx = mha_core(q, kv, False, m.h, False, mem_lengths, keep, scale, backward)
    return LinearFn.apply(ctx, m.linear_out.weight, m.linear_out.bias, False, precision, backward)


def decoder_layer_train(layer, x, tgt_lengths, memory, mem_lengths, precision: str, backward: Optional[str] = None):
    """DecoderLayer.forward (transformer_decoder.py:65-128): pre-norm, concat_after=False, no cache."""
    if getattr(layer.feed_forward, "backward_precision", None) is not None:
        raise ValueError("feed_forward.backward_precision is set on a decoder layer: the per-module knob is an encoder "
                         "option; set TransformerDecoder.backward_precision for the whole decoder")
    h = LayerNormFn.apply(x, layer.norm1.weight, layer.norm1.bias)
    x = x + layer.dropout(self_attention_train(layer.self_attn, h, tgt_lengths, precision, backward))
    h = LayerNormFn.apply(x, layer.norm2.weight, layer.norm2.bias)
    x = x + layer.dropout(source_attention_train(layer.src_attn, h, memory, mem_lengths, precision, backward))
    h = LayerNormFn.apply(x, layer.norm3.weight, layer.norm3.bias)
    return x + layer.dropout(feed_forward_train(layer.feed_forward, h, precision, backward))


def decoder_forward(dec, tgt, tgt_lengths, memory, mem_lengths, precision: str, backward: Optional[str] = None):
    """TransformerDecoder.forward (transformer_decoder.py:229-258) -> (B, L, odim) logits: a column view of the
    (B, L, odim padded to a multiple of 8) output-layer GEMM.  ``backward`` (None | "bf16") goes to every GEMM and
    attention core of the pass."""
    emb = dec.embed[0].weight
    x = dec.embed[1].dropout(EmbedFn.apply(tgt, emb))
    for layer in dec.decoders:
        x = decoder_layer_train(layer, x, tgt_lengths, memory, mem_lengths, precision, backward)
    x = LayerNormFn.apply(x, dec.after_norm.weight, dec.after_norm.bias)
    w, b = dec.output_layer.weight, dec.output_layer.bias
    odim = w.size(0)
    npad = (odim + 7) // 8 * 8
    if npad != odim:
        w, b = F.pad(w, (0, 0, 0, npad - odim)), F.pad(b, (0, npad - odim))
    return LinearFn.apply(x, w, b, False, precision, backward)[..., :odim]


def label_smoothing_loss(x, target, ignore_id: int, smoothing: float):
    """LabelSmoothingLoss(normalize_length=False) of (B, L, odim) logits -> scalar loss (divided by B)."""
    return LabelSmoothingFn.apply(x, target, ignore_id, smoothing, x.size(0))
