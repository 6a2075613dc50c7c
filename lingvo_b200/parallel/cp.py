"""Context (sequence) parallel attention — a capability the reference does not have
(SURVEY §5.7: no ring / context-parallel attention; only single-device sub-quadratic
variants and GSPMD annotations nobody uses on the length dim).

Every rank holds a contiguous `L/W` slice of each sequence. Attention needs all keys and
values, so K and V are all-gathered along the length dim (NVSwitch gives every rank full
bandwidth to every peer, so one flat all-gather beats a W-step ring on this fabric) while
queries stay local: rank r computes rows `[r·L/W, (r+1)·L/W)` of softmax(QKᵀ)V. In
backward the gathered dK/dV are reduce-scattered back to their owners. Packed-segment and
causal masks are built from *global* positions, so results match the single-device layer
bit-for-bit up to reduction order.

`AllGatherSeq` / `ReduceScatterSeq` are autograd functions (each is the other's backward),
so any attention implementation can sit between them; `Attention()` wires the common case
through `torch.nn.functional.scaled_dot_product_attention` (cuDNN flash on H100).
"""

from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist
import torch.nn.functional as F


def _World(group):
  if not (dist.is_available() and dist.is_initialized()):
    return 1, 0
  return dist.get_world_size(group), dist.get_rank(group)


def _AllGather(x, dim, group):
  w, _ = _World(group)
  if w == 1:
    return x
  x = x.contiguous()
  parts = [torch.empty_like(x) for _ in range(w)]
  dist.all_gather(parts, x, group=group)
  return torch.cat(parts, dim=dim)


def _ReduceScatter(x, dim, group):
  w, r = _World(group)
  if w == 1:
    return x
  chunks = [c.contiguous() for c in x.chunk(w, dim=dim)]
  out = torch.empty_like(chunks[r])
  if dist.get_backend(group) == 'gloo':        # gloo has no reduce_scatter
    full = torch.cat(chunks, dim=dim).contiguous()
    dist.all_reduce(full, group=group)
    return full.chunk(w, dim=dim)[r].contiguous()
  dist.reduce_scatter(out, chunks, group=group)
  return out


class AllGatherSeq(torch.autograd.Function):
  """[..., L/W, ...] → [..., L, ...] along `dim`; backward reduce-scatters."""

  @staticmethod
  def forward(ctx, x, dim, group):
    ctx.dim, ctx.group = dim, group
    return _AllGather(x, dim, group)

  @staticmethod
  def backward(ctx, dy):
    return _ReduceScatter(dy, ctx.dim, ctx.group), None, None


class ReduceScatterSeq(torch.autograd.Function):
  """Sum over ranks, keep this rank's slice of `dim`; backward all-gathers."""

  @staticmethod
  def forward(ctx, x, dim, group):
    ctx.dim, ctx.group = dim, group
    return _ReduceScatter(x, dim, group)

  @staticmethod
  def backward(ctx, dy):
    return _AllGather(dy, ctx.dim, ctx.group), None, None


def ShardSequence(x, dim=1, group=None):
  """This rank's contiguous slice of a replicated `[B, L, ...]` tensor."""
  w, r = _World(group)
  assert x.shape[dim] % w == 0, (x.shape, w)
  return x.chunk(w, dim=dim)[r].contiguous()


def Attention(q, k, v, *, causal: bool = True, segment_ids: Optional[torch.Tensor] = None,
              bias: Optional[torch.Tensor] = None, scale: Optional[float] = None, group=None):
  """Context-parallel attention.

  q, k, v: local shards `[B, L/W, H, D]`. segment_ids: local `[B, L/W]` (0 = padding) for
  packed inputs. bias: optional additive `[H or 1, L/W, L]` rows for the local queries
  (e.g. a relative-position table sliced by global row). Returns the local `[B, L/W, H, D]`.
  """
  w, r = _World(group)
  b, lq, h, d = q.shape
  k_full = AllGatherSeq.apply(k, 1, group)
  v_full = AllGatherSeq.apply(v, 1, group)
  lk = k_full.shape[1]
  q_pos = torch.arange(lq, device=q.device) + r * lq
  k_pos = torch.arange(lk, device=q.device)
  allowed = torch.ones(lq, lk, dtype=torch.bool, device=q.device)
  if causal:
    allowed = k_pos.unsqueeze(0) <= q_pos.unsqueeze(1)
  allowed = allowed.unsqueeze(0).unsqueeze(0)                     # [1, 1, Lq, Lk]
  if segment_ids is not None:
    seg_full = _AllGather(segment_ids, 1, group)                  # [B, L]
    same = segment_ids.unsqueeze(-1) == seg_full.unsqueeze(1)      # [B, Lq, Lk]
    same = same & (segment_ids.unsqueeze(-1) != 0)
    allowed = allowed & same.unsqueeze(1)
  mask = torch.zeros(allowed.shape, dtype=q.dtype, device=q.device).masked_fill(~allowed, -1e9)
  if bias is not None:
    mask = mask + bias.to(q.dtype).reshape(1, -1, lq, lk)
  out = F.scaled_dot_product_attention(
      q.transpose(1, 2), k_full.transpose(1, 2), v_full.transpose(1, 2), attn_mask=mask,
      scale=scale)
  return out.transpose(1, 2).contiguous()


def AttentionRef(q, k, v, *, causal=True, segment_ids=None, bias=None, scale=None):
  """Single-device oracle on the full (unsharded) tensors."""
  b, l, h, d = q.shape
  pos = torch.arange(l, device=q.device)
  allowed = torch.ones(l, l, dtype=torch.bool, device=q.device)
  if causal:
    allowed = pos.unsqueeze(0) <= pos.unsqueeze(1)
  allowed = allowed.unsqueeze(0).unsqueeze(0)
  if segment_ids is not None:
    same = (segment_ids.unsqueeze(-1) == segment_ids.unsqueeze(1)) & (segment_ids.unsqueeze(-1) != 0)
    allowed = allowed & same.unsqueeze(1)
  logits = torch.einsum('blhd,bmhd->bhlm', q.float(), k.float()) * (scale or d ** -0.5)
  if bias is not None:
    logits = logits + bias.float().reshape(1, -1, l, l)
  logits = logits.masked_fill(~allowed, -1e9)
  return torch.einsum('bhlm,bmhd->blhd', torch.softmax(logits, -1), v.float()).to(q.dtype)
