"""Native drop-in for the attention operator of the reference's ``Attention(attn_op=...)`` seam
(module/attention.py:136-139,225-242): TE ``DotProductAttention``'s constructor, ``forward`` and
``set_context_parallel_group``, running ``g3c_attn_fwd_sbhd``.

    attn_op = gen3c_b200.attention_op.DotProductAttention(heads, 128)

Supported: bf16 CUDA ``sbhd`` tensors, head_dim 128, any batch and any query / key count, no mask, no dropout, no bias,
as many key heads as query heads, and context parallelism (K and V all-gathered over the group).  Anything else raises
``NotImplementedError`` (unsupported configuration) or ``ValueError`` (malformed tensor); there is no fallback.

Differentiable like TE's operator: gradients reach q, k and v through the native backward kernels
(``ops.attention_sbhd``), and under context parallelism the K/V gather's backward reduce-scatters the gathered
gradients over the group, so each rank receives the gradient of its own K/V slice."""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import ops


class _GatherSequence(torch.autograd.Function):
    """all_gather_into_tensor over `group` along dim 0 (rank order); backward: reduce_scatter_tensor (sum) of the
    gradient, so each rank gets the sum over ranks of the gradient of its own slice."""

    @staticmethod
    def forward(ctx, t, group):
        ctx.group = group
        world = torch.distributed.get_world_size(group)
        out = torch.empty((world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        torch.distributed.all_gather_into_tensor(out, t.contiguous(), group=group)
        return out

    @staticmethod
    def backward(ctx, grad):
        world = torch.distributed.get_world_size(ctx.group)
        out = torch.empty((grad.shape[0] // world,) + tuple(grad.shape[1:]), dtype=grad.dtype, device=grad.device)
        torch.distributed.reduce_scatter_tensor(out, grad.contiguous(), op=torch.distributed.ReduceOp.SUM,
                                                group=ctx.group)
        return out, None


class DotProductAttention(torch.nn.Module):
    """softmax(q k^T * softmax_scale) v on [s, b, h, d] inputs, returning [s, b, h*d] (TE DotProductAttention with
    qkv_format="sbhd", attn_mask_type="no_mask", attention_dropout=0)."""

    def __init__(self, num_attention_heads: int, kv_channels: int, num_gqa_groups: Optional[int] = None,
                 attention_dropout: float = 0.0, qkv_format: str = "sbhd", attn_mask_type: str = "no_mask",
                 tp_size: int = 1, tp_group=None, sequence_parallel: bool = False,
                 softmax_scale: Optional[float] = None, **kwargs):
        super().__init__()
        if attention_dropout > 0:
            raise NotImplementedError(f"attention_dropout={attention_dropout}: dropout is not implemented")
        if attn_mask_type != "no_mask":
            raise NotImplementedError(f"attn_mask_type={attn_mask_type!r}: only 'no_mask' is implemented")
        if num_gqa_groups is not None and num_gqa_groups != num_attention_heads:
            raise NotImplementedError(f"num_gqa_groups={num_gqa_groups} for {num_attention_heads} heads: "
                                      "GQA is not implemented")
        if qkv_format != "sbhd":
            raise NotImplementedError(f"qkv_format={qkv_format!r}: only 'sbhd' is implemented")
        if kv_channels != 128:
            raise NotImplementedError(f"kv_channels={kv_channels}: only head_dim 128 is implemented")
        self.num_attention_heads = num_attention_heads
        self.kv_channels = kv_channels
        self.tp_size, self.tp_group, self.sequence_parallel = tp_size, tp_group, sequence_parallel
        self.softmax_scale = 1.0 / math.sqrt(kv_channels) if softmax_scale is None else float(softmax_scale)
        self.cp_group = self.cp_ranks = self.cp_stream = None

    def set_context_parallel_group(self, cp_group, cp_ranks, cp_stream) -> None:
        """Each rank holds a contiguous slice of the sequence (its queries, keys and values).  forward then
        all-gathers K and V over `cp_group` in rank order, so every rank attends to all keys and returns the output
        of its own queries.  cp_group=None switches context parallelism off.  The gather runs on the current stream;
        cp_stream is kept for the interface only."""
        self.cp_group, self.cp_ranks, self.cp_stream = cp_group, cp_ranks, cp_stream

    def _gather(self, t: torch.Tensor) -> torch.Tensor:
        return _GatherSequence.apply(t, self.cp_group)

    def forward(self, query_layer: torch.Tensor, key_layer: torch.Tensor, value_layer: torch.Tensor,
                core_attention_bias_type: str = "no_bias",
                core_attention_bias: Optional[torch.Tensor] = None) -> torch.Tensor:
        if core_attention_bias_type != "no_bias" or core_attention_bias is not None:
            raise NotImplementedError(f"core_attention_bias_type={core_attention_bias_type!r}: "
                                      "attention bias is not implemented")
        k, v = key_layer, value_layer
        if self.cp_group is not None:
            k, v = self._gather(k), self._gather(v)
        return ops.attention_sbhd(query_layer, k, v, self.softmax_scale)
