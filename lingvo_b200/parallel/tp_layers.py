"""Tensor-parallel building blocks for model layers (SURVEY K5/K6; ref
`lingvo/core/gshard_builder.py:2281-2320`: `mhd_w_split / mh_wi_split / hm_wo_split` put
the attention heads and the FFN hidden dim on the model axis of the device mesh).

GSPMD derives the collectives from sharding annotations; here they are explicit. A
column-parallel GEMM (weights split on the output dim) followed by a row-parallel GEMM
(weights split on the input dim) needs exactly two collectives per block:

    x (replicated) ──f──▶ x ─▶ [x·W1_shard] ─▶ act ─▶ [h_shard·W2_shard] ──g──▶ y (replicated)

  * `CopyToTensorParallel`  (f): identity forward, **all-reduce(sum) backward** — the input
    gradient is the sum of the partial gradients of the shards;
  * `ReduceFromTensorParallel` (g): **all-reduce(sum) forward** of the partial outputs,
    identity backward.

Both run on `ctx.tp_group` (NCCL over NVLink on the device, gloo in CPU tests). The local
GEMMs are the framework's wgmma kernels. The fully fused variant — collectives inside the
GEMM kernel over peer memory — lives in `parallel/tp.py` (`TpEngine`); it is selected with
`LINGVO_B200_TP_FUSED=1` for geometries it supports and is otherwise an experimental path:
the NCCL + wgmma-GEMM composition is the default.
"""

from __future__ import annotations

import torch
import torch.distributed as dist


class _CopyToTp(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, group):
    ctx.group = group
    return x.view_as(x)

  @staticmethod
  def backward(ctx, dy):
    dy = dy.contiguous()
    dist.all_reduce(dy, group=ctx.group)
    return dy, None


class _ReduceFromTp(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, group):
    x = x.contiguous()
    # out-of-place: the partial product may be needed by autograd of the producer
    y = x.clone()
    dist.all_reduce(y, group=group)
    return y

  @staticmethod
  def backward(ctx, dy):
    return dy, None


def CopyToTensorParallel(x, tp_ctx):
  """f: replicated activation entering a tensor-parallel region."""
  if tp_ctx is None:
    return x
  return _CopyToTp.apply(x, tp_ctx.tp_group)


def ReduceFromTensorParallel(x, tp_ctx):
  """g: partial results leaving a tensor-parallel region → replicated sum."""
  if tp_ctx is None:
    return x
  return _ReduceFromTp.apply(x, tp_ctx.tp_group)


def MarkSharded(var, tp_ctx, dim, logical_size):
  """Tags `var` as this rank's slice along `dim` of a logical tensor: consumed by the
  data-parallel sync (reduce over replicas only), the global gradient norm (sum over the TP
  group) and the checkpointer (gather / slice)."""
  var.tp_shard = (tp_ctx.tp_rank, tp_ctx.tp_size, dim, logical_size)
  return var


def GatherShards(t, tp_ctx, dim):
  """All-gathers the shards of `t` along `dim` (checkpoint export, tests)."""
  parts = [torch.empty_like(t) for _ in range(tp_ctx.tp_size)]
  dist.all_gather(parts, t.contiguous(), group=tp_ctx.tp_group)
  return torch.cat(parts, dim=dim)


def AllReduceScalar(t, tp_ctx):
  """Sums a small tensor over the TP group (gradient-norm contributions of sharded vars)."""
  if tp_ctx is None:
    return t
  t = t.clone()
  dist.all_reduce(t, group=tp_ctx.tp_group)
  return t
