"""Tensor-parallel FFN with the collectives fused into the wgmma GEMM (SURVEY K5/K6).

GShard shards the FFN weights `wi[M, H]` / `wo[H, M]` on H and keeps the
activations between layers sharded on the model dim M (`blm_split`,
ref `lingvo/core/gshard_builder.py:2040-2090`). XLA SPMD lowers that to
all-gather → einsum and einsum → reduce-scatter. Here both collectives live
inside the GEMM kernel:

* all-gather → GEMM: the A operand's K range is covered by one TMA tensor map
  per rank; the producer warp pulls each K-block straight out of the owning
  peer's HBM over NVLink (`a_peer_ptrs`). The gathered activation is never
  materialised.
* GEMM → reduce-scatter: every 128×256 output tile belongs to exactly one
  owner rank; the epilogue stores it into that rank's partial slab
  (`nblk_ptrs`), and the owner sums the W slabs (`tp_reduce_slabs`), or sums
  and re-broadcasts (`tp_reduce_bcast`) when the consumer wants the result
  replicated (all-reduce).

Forward and backward are mirror images (dgrad of AG→GEMM is GEMM→RS and vice
versa), so the whole fwd+bwd FFN is 6 GEMM launches + 4 slab reductions + 8
flag syncs, with no NCCL call.
"""

from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from lingvo_b200 import ops
from lingvo_b200.ops import gemm as gemm_lib
from lingvo_b200.parallel import symm as symm_lib
from lingvo_b200.parallel import zero as zero_lib

_TILE_N = 256


class TpEngine:
  """Symmetric buffers and tile→owner tables for one [tokens, M] / H geometry."""

  def __init__(self, tokens: int, model_dim: int, hidden_dim: int,
               device: torch.device, group=None):
    self.world = dist.get_world_size(group)
    self.rank = dist.get_rank(group)
    w = self.world
    assert model_dim % (w * _TILE_N) == 0, (
        'model_dim must be a multiple of world*256 for tile ownership')
    assert hidden_dim % w == 0
    self.t, self.m, self.h = tokens, model_dim, hidden_dim
    self.ms, self.hs = model_dim // w, hidden_dim // w
    bf = torch.bfloat16
    shard_b = tokens * self.ms * 2
    self.arena = symm_lib.SymmArena(2 * shard_b * (1 + w) + tokens * model_dim * 2
                                    + (1 << 16), device, group)
    a = self.arena
    # Two sets (forward / backward) so a backward never races the next forward.
    self.sets = []
    for _ in range(2):
      xoff, soff = a.Alloc(shard_b), a.Alloc(shard_b * w)
      self.sets.append(dict(
          x=a.Local(xoff, (tokens, self.ms), bf),
          x_peers=torch.tensor([b + xoff for b in a.peer_base], dtype=torch.int64),
          slab=a.Local(soff, (w, tokens, self.ms), bf),
          nblk=self._TileTable(soff)))
    yoff = a.Alloc(tokens * model_dim * 2)
    self.full = a.Local(yoff, (tokens, model_dim), bf)
    self.full_peers = torch.tensor([b + yoff for b in a.peer_base], dtype=torch.int64)
    self.chan = zero_lib._Channels(a, w, self.rank, n=8)   # pylint: disable=protected-access
    dist.barrier(group)

  def _TileTable(self, slab_off):
    """Destination base of every 256-column output tile: owner's slab[my rank]."""
    ptrs = []
    for nb in range(self.m // _TILE_N):
      n0 = nb * _TILE_N
      owner = n0 // self.ms
      ptrs.append(self.arena.peer_base[owner] + slab_off +
                  (self.rank * self.t * self.ms + (n0 - owner * self.ms)) * 2)
    return torch.tensor(ptrs, dtype=torch.int64, device=self.arena.device)

  # -- primitives -------------------------------------------------------------
  def AgGemm(self, s, w, w_kmajor, act=0, aux=None, aux_mode=0):
    """(all-gather_M of set-s shard) · W. Caller has filled `sets[s].x`."""
    st = self.sets[s]
    self.chan.Sync(2 * s)                    # every rank's shard is in place
    return gemm_lib.gemm(st['x'], w, True, w_kmajor, act=act, aux=aux,
                         aux_mode=aux_mode, a_peer_ptrs=st['x_peers'])

  def GemmRs(self, s, a, w, w_kmajor, bcast=False):
    """reduce-scatter_M(a · W) → my [T, M/W] shard (or the all-reduced [T, M])."""
    st = self.sets[s]
    gemm_lib.gemm(a, w, True, w_kmajor, nblk_ptrs=st['nblk'], nblk_ld=self.ms)
    self.chan.Sync(2 * s + 1)                # all partial tiles have landed
    nat = ops.native()
    if not bcast:
      return nat.tp_reduce_slabs(st['slab'], self.world)
    nat.tp_reduce_bcast(st['slab'], self.world, self.full_peers, self.m,
                        self.rank * self.ms)
    self.chan.Sync(4 + s)                    # every column block has arrived
    return self.full

  def PeerShard(self, s, r):
    """Rank r's set-s activation shard, readable by TMA over NVLink."""
    if r == self.rank:
      return self.sets[s]['x']
    raw = ops.native().symm_view(int(self.sets[s]['x_peers'][r]),
                                 self.t * self.ms * 2, self.arena.device.index)
    return raw.view(torch.bfloat16).view(self.t, self.ms)


class _TpFfnFn(torch.autograd.Function):
  """y_shard = RS_M( relu( AG_M(x_shard) · wi_shard ) · wo_shard )."""

  @staticmethod
  def forward(ctx, eng, x_shard, wi, wo, replicated_out):
    eng.sets[0]['x'].copy_(x_shard)
    h = eng.AgGemm(0, wi, False, act=1)                       # [T, H/W]
    y = eng.GemmRs(0, h, wo, False, bcast=replicated_out)
    ctx.eng, ctx.rep = eng, replicated_out
    ctx.save_for_backward(x_shard, wi, wo, h)
    return y.clone() if replicated_out else y

  @staticmethod
  def backward(ctx, dy):
    eng = ctx.eng
    x_shard, wi, wo, h = ctx.saved_tensors
    w, r, ms = eng.world, eng.rank, eng.ms
    if ctx.rep:      # replicated consumer: my shard of dy is a column slice
      dy = dy[:, r * ms:(r + 1) * ms]
    eng.sets[1]['x'].copy_(dy)
    # dh = AG(dy)·woᵀ ⊙ relu'(h)
    dh = eng.AgGemm(1, wo, True, aux=h, aux_mode=gemm_lib.AUX_RELU_MASK)
    # dwo[:, cols of rank q] = hᵀ · dy_q  (B tiles read from peer q by TMA)
    dwo = torch.empty_like(wo)
    for q in range(w):
      gemm_lib.gemm(h, eng.PeerShard(1, q), False, False,
                    out=dwo[:, q * ms:(q + 1) * ms])
    # dx_shard = RS(dh · wiᵀ)
    dx = eng.GemmRs(1, dh, wi, True)
    # dwi[rows of rank q] = x_qᵀ · dh. Set-0 shards still hold this layer's x
    # only if no other forward ran in between; use the saved copy for mine and
    # re-stage (cheap) so peers can read it.
    eng.sets[0]['x'].copy_(x_shard)
    eng.chan.Sync(6)
    dwi = torch.empty_like(wi)
    for q in range(w):
      gemm_lib.gemm(eng.PeerShard(0, q), dh, False, False,
                    out=dwi[q * ms:(q + 1) * ms])
    eng.chan.Sync(7)                         # peers are done reading my shards
    return None, dx, dwi, dwo, None


def TpFfn(eng: TpEngine, x_shard, wi_shard, wo_shard, replicated_out=False):
  """Tensor-parallel relu-FFN on an M-sharded activation `[T, M/W]`."""
  return _TpFfnFn.apply(eng, x_shard, wi_shard, wo_shard, replicated_out)


def TpFfnNccl(x_shard, wi_shard, wo_shard, group=None):
  """NCCL + cuBLAS baseline of the same computation (for parity / speed tests)."""
  w = dist.get_world_size(group)
  parts = [torch.empty_like(x_shard) for _ in range(w)]
  dist.all_gather(parts, x_shard.contiguous(), group=group)
  x = torch.cat(parts, dim=1)
  h = torch.relu(x @ wi_shard)
  y = h @ wo_shard
  ms = y.shape[1] // w
  out = torch.empty(y.shape[0], ms, dtype=y.dtype, device=y.device)
  dist.reduce_scatter(out, [c.contiguous() for c in y.split(ms, dim=1)], group=group)
  return out
