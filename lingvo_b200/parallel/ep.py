"""Expert parallelism: tokens ⇄ experts across ranks.

Reference: GShard's `GSEC,GSM->EGCM` einsum + G-sharded→E-sharded reshard =
XLA all-to-all (`gshard_layers.py:3072-3161`), TPU-only. Here it is explicit:

* `mode='nccl'`  — stock baseline: local index-dispatch into `[E, G_l·C, M]`,
  `all_to_all_single`, grouped expert GEMMs, `all_to_all_single`, local
  index-combine (`gshard_layers.MoEApplyIndexed`, with `ToExperts` /
  `FromExperts` below as the two exchanges).
* `mode='fused'` — the H100 path (`ops/moe.py` + `parallel/symm.py`): the
  dispatch kernel writes every routed token row **directly into the owning
  rank's expert buffer over NVLink** (peer stores into symmetric memory), the
  second expert GEMM's epilogue stores each output row straight back into the
  *source* rank's combine buffer (row-pointer table), and flags replace the
  collective's implicit barrier. Falls back to `nccl` when peer memory is
  unavailable (e.g. gloo/CPU tests).

Slot convention (shared with `gshard_layers`): expert buffer on the owner is
`[E_local, G_total·C, M]` with row `(e_l·G_total + g_global)·C + c`.
"""

from __future__ import annotations

import torch
import torch.distributed as dist


class _AllToAll(torch.autograd.Function):
  """Equal-split all_to_all over dim 0; backward is the reverse exchange."""

  @staticmethod
  def forward(ctx, x, group):
    ctx.group = group
    out = torch.empty_like(x)
    dist.all_to_all_single(out, x.contiguous(), group=group)
    return out

  @staticmethod
  def backward(ctx, dy):
    out = torch.empty_like(dy)
    dist.all_to_all_single(out, dy.contiguous(), group=ctx.group)
    return out, None


class _ScaleGrad(torch.autograd.Function):
  """Identity forward; multiplies the gradient by a constant (expert weights under EP get
  the sum over all ranks' tokens — 1/ep makes it the mean, like the replicated variables)."""

  @staticmethod
  def forward(ctx, w, scale):
    ctx.scale = scale
    return w.view_as(w)

  @staticmethod
  def backward(ctx, dw):
    return dw * ctx.scale, None


class ExpertParallel:
  """EP engine shared by all MoE layers with the same (E, ep) geometry."""

  def __init__(self, ctx, num_experts: int, ep_size: int):
    assert num_experts % ep_size == 0, (num_experts, ep_size)
    assert ctx.world % ep_size == 0
    self.ctx = ctx
    self.num_experts = num_experts
    self.ep_size = ep_size
    self.num_local_experts = num_experts // ep_size
    if ep_size == ctx.world:
      self.group = None            # default (world) group
      self.ep_rank = ctx.rank
    else:
      # Consecutive ranks form an EP group; groups are data-parallel replicas.
      self.group = None
      for start in range(0, ctx.world, ep_size):
        g = dist.new_group(list(range(start, start + ep_size)))
        if start <= ctx.rank < start + ep_size:
          self.group = g
      self.ep_rank = ctx.rank % ep_size
    self._fused = None

  def GetExchange(self, device):
    """The fused peer-memory exchange, or None (NCCL baseline / CPU)."""
    if self._fused is None:
      self._fused = False
      if self.ctx.mode == 'fused' and device.type == 'cuda':
        from lingvo_b200.parallel import symm
        self._fused = symm.MoeExchange(self, device=device)
    return self._fused or None

  def ScaleExpertGrad(self, w):
    """Local expert weights whose gradient is scaled by 1/ep while training."""
    if self.ep_size > 1 and torch.is_grad_enabled():
      return _ScaleGrad.apply(w, 1.0 / self.ep_size)
    return w

  def ToExperts(self, xin):
    """This rank's expert inputs `[E, G_l·C, M]` → the local experts' inputs
    from every rank `[E_local, ep·G_l·C, M]`."""
    _, rows, m = xin.shape
    ep, el = self.ep_size, self.num_local_experts
    recv = _AllToAll.apply(xin.reshape(ep, el * rows, m), self.group)
    return recv.reshape(ep, el, rows, m).transpose(0, 1).reshape(el, ep * rows, m)

  def FromExperts(self, ye):
    """Inverse of `ToExperts`: `[E_local, ep·G_l·C, M]` → `[E, G_l·C, M]`."""
    el, ep = self.num_local_experts, self.ep_size
    rows, m = ye.shape[1] // ep, ye.shape[2]
    back = ye.reshape(el, ep, rows, m).transpose(0, 1).reshape(ep, el * rows, m)
    return _AllToAll.apply(back, self.group).reshape(self.num_experts, rows, m)
