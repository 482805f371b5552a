"""Drop-in for RelPositionMultiHeadedAttention of espnet.nets.pytorch_backend.transformer.attention
(reference attention.py:107-193; base-class projections :31-34)."""
from typing import Optional

import torch
from torch import nn

from .. import ops
from ..engine import default_precision


def mask_to_lengths(mask: torch.Tensor, B: int, T: int, check: bool = False) -> torch.Tensor:
    """(B,1,T) bool key mask from make_non_pad_mask (nets_utils.py:183; True = valid, prefix-contiguous)
    -> int32 lengths (B) on the same device, without a host sync.

    Restriction (INTEGRATION.md): the mask must be a PREFIX mask (valid frames first), which is what every caller in
    the reference passes (e2e_asr_conformer.py:67).  A mask with holes or left padding cannot be expressed as lengths;
    ``check=True`` (ConformerEncoder.check_mask / AVSR_B200_CHECK_MASK=1) verifies the property at the cost of one
    host sync and raises instead of computing attention over the wrong keys."""
    if mask.dim() != 3 or mask.size(0) != B or mask.size(1) != 1 or mask.size(2) != T:
        raise NotImplementedError(f"only (B,1,T) key-padding masks are supported, got {tuple(mask.shape)}")
    m = mask[:, 0, :].to(torch.bool)
    lengths = m.to(torch.int32).sum(dim=-1, dtype=torch.int32)
    if check:
        prefix = torch.arange(T, device=mask.device)[None, :] < lengths[:, None]
        if not bool(torch.equal(prefix, m)):
            raise NotImplementedError("key mask is not prefix-contiguous (holes / left padding): the CUDA path takes "
                                      "lengths, i.e. make_non_pad_mask-style masks only")
    return lengths


class RelPositionMultiHeadedAttention(nn.Module):
    """Transformer-XL style rel-pos self-attention with learnable biases u, v.

    Parameter names match the reference: linear_{q,k,v,out} (with bias), linear_pos (no bias),
    pos_bias_u / pos_bias_v (h, d_k).  ``forward`` computes
    softmax_j(((q_i+u).k_j + (q_i+v).p[i-j]) / sqrt(d_k)) @ v in one fused kernel (no (T x 2T) tensor, no
    rel_shift copy) with the key-length mask applied inside."""

    def __init__(self, n_head, n_feat, dropout_rate, zero_triu=False):
        super().__init__()
        assert n_feat % n_head == 0
        self.d_k = n_feat // n_head
        self.h = n_head
        self.linear_q = nn.Linear(n_feat, n_feat)
        self.linear_k = nn.Linear(n_feat, n_feat)
        self.linear_v = nn.Linear(n_feat, n_feat)
        self.linear_out = nn.Linear(n_feat, n_feat)
        self.attn = None            # the reference stores the (B,H,T,T) probabilities here; nothing reads them
        self.dropout = nn.Dropout(p=dropout_rate)
        self.zero_triu = zero_triu
        self.linear_pos = nn.Linear(n_feat, n_feat, bias=False)
        self.pos_bias_u = nn.Parameter(torch.empty(self.h, self.d_k))
        self.pos_bias_v = nn.Parameter(torch.empty(self.h, self.d_k))
        torch.nn.init.xavier_uniform_(self.pos_bias_u)
        torch.nn.init.xavier_uniform_(self.pos_bias_v)
        self.precision: Optional[str] = None
        self.backward_precision: Optional[str] = None     # None (default backward) | "bf16"; see train.py

    def forward(self, query, key, value, pos_emb, mask, residual: Optional[torch.Tensor] = None):
        """query (B,T,d); key/value must be the same tensor (self-attention) or None; pos_emb (1,2T-1,d);
        mask (B,1,T) bool or None.  ``residual`` (extension) is added in the output projection's epilogue."""
        if self.zero_triu or self.d_k != 64:
            raise NotImplementedError("RelPositionMultiHeadedAttention: zero_triu=False and d_k=64 only")
        for other in (key, value):
            if other is not None and other is not query:
                raise NotImplementedError("RelPositionMultiHeadedAttention: self-attention only (query is key is value)")
        prec = self.precision or default_precision()
        B, T, _ = query.shape
        if self.training:                       # forward + backward in libavsr_b200 (auto_avsr_b200/train.py)
            from ..train import attention_train, module_backward_precision
            y = attention_train(self, query, pos_emb, mask, prec, module_backward_precision(self))
            return y if residual is None else residual + y
        q = ops.linear(query, self.linear_q.weight, self.linear_q.bias, precision=prec)
        k = ops.linear(query, self.linear_k.weight, self.linear_k.bias, precision=prec)
        v = ops.linear(query, self.linear_v.weight, self.linear_v.bias, precision=prec)
        p = ops.linear(pos_emb.reshape(2 * T - 1, -1), self.linear_pos.weight, None, precision=prec)
        lengths = None if mask is None else mask_to_lengths(mask, B, T)
        ctx = ops.relpos_attention(q, k, v, p, self.pos_bias_u, self.pos_bias_v, lengths, self.h, precision=prec)
        return ops.linear(ctx, self.linear_out.weight, self.linear_out.bias, residual=residual, precision=prec)
