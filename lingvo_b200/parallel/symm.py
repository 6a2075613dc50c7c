"""Symmetric (peer-mapped) memory + the fused MoE exchange.

`SymmArena` — one `cudaMalloc` slab per rank whose CUDA-IPC handle is
exchanged once; every rank maps every peer's slab, so kernels can `st`/`ld`
straight into peers over NVLink 4 / NVSwitch (uniform any-to-any bandwidth ⇒
flat one-hop algorithms). Buffers are bump-allocated at identical offsets on
all ranks.

`MoeExchange` — the fused expert-parallel MoE FFN (SURVEY K1–K4):

  forward   gate+dispatch kernel  : top-2 gate, slot scan, **peer stores** of
                                    every (expert, group, slot) row
            signal / wait flags   : replaces the all-to-all's barrier
            grouped wgmma GEMM  : h = relu(xe · wi)
            grouped wgmma GEMM  : (h · wo) with a **row-pointer epilogue**
                                    that stores each output row into the
                                    *source* rank's combine buffer
            signal / wait, combine: gated 2-row gather (local)
  backward  mirrors it: gate-scaled slot scatter of dy to the experts, dgrad
            GEMM with fused ReLU-mask epilogue, two wgrad GEMMs, dgrad GEMM
            with the row-pointer epilogue back to the sources, token gather.

With a single rank the very same kernels run on local pointers.
"""

from __future__ import annotations

import logging
from typing import Dict, Optional

import torch
import torch.distributed as dist
import torch.nn.functional as F

from lingvo_b200 import ops
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.ops import gemm

_ALIGN = 1024


class SymmArena:
  """Per-rank slab mapped by all ranks of `group`."""

  def __init__(self, nbytes: int, device: torch.device, group=None):
    self.device = device
    self.group = group
    self.world = dist.get_world_size(group) if (
        dist.is_available() and dist.is_initialized()) else 1
    self.rank = dist.get_rank(group) if self.world > 1 else 0
    self.nbytes = int(nbytes)
    nat = ops.native()
    if self.world > 1:
      self._slab = nat.symm_alloc(self.nbytes, device.index)
      handle = nat.symm_export(self._slab)
      handles = [None] * self.world
      dist.all_gather_object(handles, handle, group=group)
      self.peer_base = []
      for r, h in enumerate(handles):
        if r == self.rank:
          self.peer_base.append(self._slab.data_ptr())
        else:
          self.peer_base.append(nat.symm_import(h, device.index))
    else:
      self._slab = torch.zeros(self.nbytes, dtype=torch.uint8, device=device)
      self.peer_base = [self._slab.data_ptr()]
    self._off = 0

  def Alloc(self, nbytes: int) -> int:
    off = (self._off + _ALIGN - 1) // _ALIGN * _ALIGN
    if off + nbytes > self.nbytes:
      raise MemoryError('SymmArena exhausted: need %d more bytes' %
                        (off + nbytes - self.nbytes))
    self._off = off + nbytes
    return off

  def Local(self, off: int, shape, dtype) -> torch.Tensor:
    n = 1
    for s in shape:
      n *= s
    nb = n * torch.empty((), dtype=dtype).element_size()
    return self._slab[off:off + nb].view(dtype).view(*shape)

  def PeerPtrs(self, off: int, loopback: bool = False) -> torch.Tensor:
    """Device table of every peer's address of offset `off`; `loopback` points all
    entries at this rank's own slab (timing-only mode: same stores, no NVLink)."""
    bases = [self.peer_base[self.rank]] * self.world if loopback else self.peer_base
    return torch.tensor([b + off for b in bases], dtype=torch.int64,
                        device=self.device)


class _LayerBufs:
  """Symmetric buffers + static tables of one MoE layer."""

  def __init__(self, ex: 'MoeExchange', g_l, s, c, m):
    a = ex.arena
    el, ep, e = ex.e_local, ex.ep, ex.num_experts
    g_t = ep * g_l
    bf = torch.bfloat16
    self.xe_off = a.Alloc(el * g_t * c * m * 2)
    self.yc_off = a.Alloc(e * g_l * c * m * 2)
    self.xe = a.Local(self.xe_off, (el, g_t * c, m), bf)
    self.yc = a.Local(self.yc_off, (e, g_l * c, m), bf)
    self._peer_xe = {False: a.PeerPtrs(self.xe_off)}
    self._row_ptrs_yc = {False: ex.RowPtrTable(self.yc_off, g_l, c, m)}
    self._ex, self._geom = ex, (g_l, c, m)
    self.chan = ex.NewChannels(4)
    self.seq = [0, 0, 0, 0]

  @property
  def peer_xe(self):
    lb = self._ex.loopback
    if lb not in self._peer_xe:
      self._peer_xe[lb] = self._ex.arena.PeerPtrs(self.xe_off, loopback=True)
    return self._peer_xe[lb]

  @property
  def row_ptrs_yc(self):
    lb = self._ex.loopback
    if lb not in self._row_ptrs_yc:
      self._row_ptrs_yc[lb] = self._ex.RowPtrTable(self.yc_off, *self._geom, loopback=True)
    return self._row_ptrs_yc[lb]


class MoeExchange:
  """Fused EP MoE FFN for one (E, ep) geometry; shared by all MoE layers."""

  def __init__(self, ep_engine=None, num_experts: Optional[int] = None,
               device: Optional[torch.device] = None):
    if ep_engine is not None:
      self.ep = ep_engine.ep_size
      self.rank = ep_engine.ep_rank
      self.num_experts = ep_engine.num_experts
      self.group = ep_engine.group
    else:
      self.ep, self.rank, self.num_experts, self.group = 1, 0, num_experts, None
    self.e_local = self.num_experts // self.ep
    self.device = device or torch.device('cuda', torch.cuda.current_device())
    self.arena = None
    self._layers: Dict[int, _LayerBufs] = {}
    self._next_chan = 0
    self._geom = None
    self._counters = None
    # Timing-only mode used to measure the *exposed* cost of the exchange: every peer
    # pointer is redirected to this rank's own buffers and the flag waits are skipped, so
    # a step does exactly the same work with zero NVLink traffic and zero peer waiting.
    # (Numerically meaningless; `bench.py` reports step(normal) − step(loopback).)
    self.loopback = False

  # -------------------------------------------------------------- plumbing --
  def _EnsureArena(self, g_l, s, c, m, n_layers_hint=8):
    if self.arena is not None:
      return
    el, ep, e = self.e_local, self.ep, self.num_experts
    per_layer = (el * ep * g_l * c * m + e * g_l * c * m) * 2 + 2 * _ALIGN
    scratch = 2 * (el * ep * g_l * c * m) * 2 + 2 * _ALIGN
    flags = 256 * max(ep, 1) * 4 + _ALIGN
    self.arena = SymmArena(per_layer * n_layers_hint + scratch + flags,
                           self.device, self.group)
    a = self.arena
    self.flags_off = a.Alloc(256 * ep * 4)
    self.flags = a.Local(self.flags_off, (256 * ep,), torch.int32)
    self.peer_flags = a.PeerPtrs(self.flags_off)
    g_t = ep * g_l
    self.dye_off = a.Alloc(el * g_t * c * m * 2)
    self.dxc_off = a.Alloc(e * g_l * c * m * 2)
    self.dye = a.Local(self.dye_off, (el, g_t * c, m), torch.bfloat16)
    self.dxc = a.Local(self.dxc_off, (e, g_l * c, m), torch.bfloat16)
    self._peer_dye = {False: a.PeerPtrs(self.dye_off), True: a.PeerPtrs(self.dye_off, True)}
    self._row_ptrs_dxc = {False: self.RowPtrTable(self.dxc_off, g_l, c, m),
                          True: self.RowPtrTable(self.dxc_off, g_l, c, m, loopback=True)}
    self._geom = (g_l, s, c, m)
    if self.ep > 1:
      dist.barrier(group=self.group)

  @property
  def peer_dye(self):
    return self._peer_dye[self.loopback]

  @property
  def row_ptrs_dxc(self):
    return self._row_ptrs_dxc[self.loopback]

  def WgradScale(self, groups, rows):
    """fp32 `[groups, rows]` filled with 1/ep (None when ep == 1)."""
    if self.ep <= 1:
      return None
    key = (groups, rows)
    cache = self.__dict__.setdefault('_wscale', {})
    if key not in cache:
      cache[key] = torch.full((groups, rows), 1.0 / self.ep, dtype=torch.float32,
                              device=self.device)
    return cache[key]

  def NewChannels(self, n):
    base = self._next_chan
    self._next_chan += n
    assert self._next_chan <= 256, 'out of flag channels'
    return list(range(base, base + n))

  def RowPtrTable(self, dst_off, g_l, c, m, loopback=False):
    """Pointer of the destination row for every local expert-buffer row.

    Expert-buffer row (e_l, g_glob, c) → rank g_glob // G_l, combine-layout
    row (e·G_l + g_loc)·C + c of the buffer at `dst_off`.
    """
    el, ep = self.e_local, self.ep
    dev = self.device
    bases = self.arena.peer_base
    if loopback:
      bases = [bases[self.arena.rank]] * len(bases)
    base = torch.tensor([b + dst_off for b in bases], dtype=torch.int64, device=dev)
    e_l = torch.arange(el, device=dev).view(el, 1, 1)
    g_glob = torch.arange(ep * g_l, device=dev).view(1, ep * g_l, 1)
    cc = torch.arange(c, device=dev).view(1, 1, c)
    dest = g_glob // g_l
    g_loc = g_glob % g_l
    e = self.rank * el + e_l
    row = (e * g_l + g_loc) * c + cc
    ptr = base[dest] + row * (m * 2)
    return ptr.reshape(el, ep * g_l * c).contiguous()

  def _Bufs(self, key, g_l, s, c, m) -> _LayerBufs:
    self._EnsureArena(g_l, s, c, m)
    assert self._geom == (g_l, s, c, m), (
        'MoeExchange geometry changed: %s vs %s' % (self._geom, (g_l, s, c, m)))
    if key not in self._layers:
      self._layers[key] = _LayerBufs(self, g_l, s, c, m)
    return self._layers[key]

  def _Sync(self, bufs: _LayerBufs, phase: int):
    """Release-signal all peers on this channel, then acquire-wait on all."""
    ch = bufs.chan[phase]
    if self.ep > 1 and not self.loopback:
      if self._counters is None:
        self._counters = torch.zeros(4096, dtype=torch.int32, device=self.flags.device)
      ops.native().moe_sync(self.peer_flags, self.flags, self._counters, self.ep, self.rank, ch)

  # ------------------------------------------------------------------ apply --
  def GateAndDispatch(self, key, x2d, logits, paddings, capacity, legacy):
    """Runs the fused gate + peer-store dispatch kernel (non-differentiable)."""
    g_l, s, e = logits.shape
    m = x2d.shape[-1]
    bufs = self._Bufs(key, g_l, s, capacity, m)
    idx, pos, gate, slot_token = ops.native().moe_gate_dispatch(
        logits.detach().float().contiguous(), paddings, x2d.detach(),
        bufs.peer_xe, capacity, self.e_local, self.rank, self.ep, legacy)
    return bufs, NestedMap(index=idx, pos=pos, keep=gate != 0,
                           slot_token=slot_token, capacity=capacity)

  def Apply(self, key, x2d, logits, paddings, capacity, legacy, wi, wo):
    """x2d `[G_l·S, M]`, logits `[G_l, S, E]` → (y `[G_l·S, M]`, aux_loss)."""
    g_l, s, e = logits.shape
    bufs, g = self.GateAndDispatch(key, x2d, logits, paddings, capacity, legacy)
    # Differentiable gate values (tiny [G,S,E] tensors) for the chosen experts.
    raw = torch.softmax(logits.float(), dim=-1)
    nonpad = None if paddings is None else (1.0 - paddings.float())
    i1, i2 = g.index[0].long(), g.index[1].long()
    g1 = raw.gather(-1, i1.unsqueeze(-1)).squeeze(-1)
    g2 = raw.gather(-1, i2.unsqueeze(-1)).squeeze(-1)
    oh1 = F.one_hot(i1, e).float()
    proxy = raw
    if nonpad is not None:
      g1, g2 = g1 * nonpad, g2 * nonpad
      oh1 = oh1 * nonpad.unsqueeze(-1)
      proxy = raw * nonpad.unsqueeze(-1)
    if legacy:
      den = g1 + g2 + 1e-9
      g1, g2 = g1 / den, g2 / den
    g1 = g1 * g.keep[0].float()
    g2 = g2 * g.keep[1].float()
    if not legacy:
      den = g1 + g2
      den = torch.where(den > 0, den, torch.ones_like(den))
      g1, g2 = g1 / den, g2 / den
    if legacy:
      dden = 1.0
    else:
      imp = nonpad if nonpad is not None else torch.ones_like(g1)
      dden = imp.mean(1)[:, None] + 1e-6
    aux_loss = ((proxy.mean(1) / dden) * (oh1.mean(1) / dden)).mean() * (e * e)
    gate = torch.stack([g1, g2]).reshape(2, g_l * s)
    y = _MoeFn.apply(x2d, gate, wi, wo, self, bufs, g, g_l, s)
    return y, aux_loss


class _MoeFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x2d, gate, wi, wo, ex: MoeExchange, bufs: _LayerBufs,
              g: NestedMap, g_l, s):
    nat = ops.native()
    c = g.capacity
    ex._Sync(bufs, 0)                                   # dispatch rows landed
    h = gemm.gemm(bufs.xe, wi, True, False, act='RELU')  # [El, A, H]
    gemm.gemm(h, wo, True, False, row_ptrs=bufs.row_ptrs_yc)   # → peers' yc
    ex._Sync(bufs, 1)                                   # combine rows landed
    gate_v = gate.detach().float().contiguous()
    idx = g.index.reshape(2, -1).contiguous()
    pos = g.pos.reshape(2, -1).contiguous()
    y = nat.moe_combine(bufs.yc, g.index, g.pos, gate_v.view(2, g_l, s), s, g_l,
                        c)
    ctx.save_for_backward(gate_v, wi, wo, h)
    ctx.ex, ctx.bufs, ctx.g, ctx.dims = ex, bufs, g, (g_l, s, c)
    # xe / yc stay in the layer's symmetric buffers until backward.
    return y

  @staticmethod
  def backward(ctx, dy):
    nat = ops.native()
    gate_v, wi, wo, h = ctx.saved_tensors
    ex, bufs, g = ctx.ex, ctx.bufs, ctx.g
    g_l, s, c = ctx.dims
    dy = dy.contiguous()
    gate3 = gate_v.view(2, g_l, s)
    dgate = nat.moe_combine_bwd_gate(bufs.yc, dy, g.index, g.pos, gate3, s, g_l,
                                     c)
    nat.moe_scatter_rows(dy, g.slot_token, g.index.reshape(2, -1).contiguous(),
                         gate_v, ex.peer_dye, ex.e_local, ex.rank, ex.ep)
    ex._Sync(bufs, 2)
    dye = ex.dye
    dh = gemm.gemm(dye, wo, True, True, aux=h, aux_mode=gemm.AUX_RELU_MASK)
    # Every rank's tokens reach these experts while the replicated variables get the
    # *mean* gradient over ranks: the same 1/ep goes on the expert weight gradients, for
    # free in the wgrad epilogue (`row_scale`), so the global norm is consistent.
    dwo = gemm.gemm(h, dye, False, False, row_scale=ex.WgradScale(h.shape[0], h.shape[-1]))
    dwi = gemm.gemm(bufs.xe, dh, False, False,
                    row_scale=ex.WgradScale(dh.shape[0], bufs.xe.shape[-1]))
    # Peer-store GEMM last: once peers see the flag, every read of this
    # layer's xe/h/dye on this rank has been issued before it in stream order.
    gemm.gemm(dh, wi, True, True, row_ptrs=ex.row_ptrs_dxc)
    ex._Sync(bufs, 3)
    dx = nat.moe_gather_rows(ex.dxc, g.index, g.pos, gate3, s, g_l, c)
    return dx, dgate.view_as(gate_v), dwi, dwo, None, None, None, None, None


_LOCAL: Dict[int, MoeExchange] = {}


def LocalExchange(num_experts: int, device) -> MoeExchange:
  """Single-rank exchange (all experts local) for `num_experts`."""
  key = (num_experts, device.index)
  if key not in _LOCAL:
    _LOCAL[key] = MoeExchange(None, num_experts, device)
  return _LOCAL[key]
