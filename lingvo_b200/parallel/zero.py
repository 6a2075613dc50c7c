"""Data-parallel gradient sync over NVLink peer memory (SURVEY K11).

Two engines, both built on `comm_kernels.cu` + the flag protocol:

* `FusedAllReduce` — flat bf16 gradient buffer in symmetric memory; one
  two-shot all-reduce kernel (peer loads, fp32 accumulate, scale, peer
  stores); the (fused) optimizer then runs replicated. Used with Adafactor,
  whose factored statistics need whole rows/columns.
* `ZeroAdam` — reduce-scatter (+ global-norm partial) → device-side clip
  scale → **one kernel** doing partitioned Adam on the fp32 master shard and
  storing the new bf16 weights into every peer's parameter replica
  (all-gather fused). Optimizer state and master weights are sharded 1/W.
"""

from __future__ import annotations

import math
from typing import List

import torch
import torch.distributed as dist

from lingvo_b200 import ops
from lingvo_b200.core import py_utils
from lingvo_b200.parallel import symm as symm_lib


def _ReplicatedVars(task) -> List[torch.nn.Parameter]:
  vs = [v for v in task.vars.Flatten()
        if v.requires_grad and not getattr(v, 'expert_parallel', False)]
  return sorted(vs, key=lambda v: v.var_name)


class _Flat:
  """Layout of variables inside a flat buffer (each slot 8-element aligned)."""

  def __init__(self, variables, world):
    self.vars = variables
    self.offsets = []
    off = 0
    for v in variables:
      self.offsets.append(off)
      off += (v.numel() + 7) // 8 * 8
    unit = world * 8
    self.total = (off + unit - 1) // unit * unit
    self.shard = self.total // world

  def Views(self, buf):
    return [buf[o:o + v.numel()].view(v.shape)
            for v, o in zip(self.vars, self.offsets)]


class _Channels:
  """Flag channels (signal all peers / wait for all peers)."""

  def __init__(self, arena, world, rank, n=8):
    self.world, self.rank = world, rank
    self.off = arena.Alloc(n * world * 4)
    self.flags = arena.Local(self.off, (n * world,), torch.int32)
    self.peer_flags = arena.PeerPtrs(self.off)
    # Sequence numbers live on the device (bumped by the sync kernel itself), so a Sync
    # has no step-dependent launch argument and replays correctly from a CUDA graph.
    self.counters = torch.zeros(n, dtype=torch.int32, device=self.flags.device)

  def Sync(self, ch):
    ops.native().moe_sync(self.peer_flags, self.flags, self.counters, self.world,
                          self.rank, ch)


class FusedAllReduce:
  """`learner.grad_sync` implementation: mean all-reduce of replicated grads, bucketed
  and **overlapped with backward**.

  Gradients are produced by autograd in a fixed order. Tensor hooks on the differentiated
  leaves (the bf16 compute copies) store each gradient straight into its slot of the
  symmetric bf16 buffer the moment it exists; slots are laid out in arrival order, so a
  bucket is a contiguous range and is complete as soon as its last gradient arrived. The
  hook that completes a bucket launches, on the communication stream (a parallel branch
  of the step's CUDA graph), `flag sync → two-shot all-reduce kernel over NVLink peer
  memory → flag sync` for just that range, capped at `_COMM_BLOCKS` CTAs so the GEMMs of
  the remaining backward keep the SMs. After backward only the last bucket is exposed.

  The arrival order is learned during the first step (which runs the monolithic path).
  """

  _COMM_BLOCKS = 48
  _MAX_BUCKETS = 60

  def __init__(self, task, ctx, bucket_bytes: int = 48 << 20):
    self.ctx = ctx
    self.world, self.rank = ctx.world, ctx.rank
    dev = task.Device()
    self.flat = _Flat(_ReplicatedVars(task), self.world)
    self.arena = symm_lib.SymmArena(
        self.flat.total * 2 + (2 * self._MAX_BUCKETS + 16) * self.world * 4 + 65536, dev)
    self.goff = self.arena.Alloc(self.flat.total * 2)
    self.gbuf = self.arena.Local(self.goff, (self.flat.total,), torch.bfloat16)
    self.gviews = self.flat.Views(self.gbuf)
    self.peers = torch.tensor([b + self.goff for b in self.arena.peer_base],
                              dtype=torch.int64)
    self.chan = _Channels(self.arena, self.world, self.rank, n=2 * self._MAX_BUCKETS + 8)
    self._index = {id(v): i for i, v in enumerate(self.flat.vars)}
    self._overlap = dev.type == 'cuda'
    self._bucket_bytes = int(bucket_bytes)
    self._arrival: List[int] = []
    self._phase = 0                      # 0: learning the order, 1: overlapped
    self._buckets = []                   # (start_elem, n_elems, [var indices])
    self._bucket_of = {}
    self._pending = []
    self._launched = []
    self._seen = set()
    self.comm = torch.cuda.Stream(dev) if self._overlap else None
    self._hooks = []
    if self._overlap:
      for i, v in enumerate(self.flat.vars):
        leaf = getattr(v, 'compute', None)
        leaf = leaf if leaf is not None else v
        self._hooks.append(leaf.register_hook(self._MakeHook(i)))
    dist.barrier()

  # ---------------------------------------------------------------- hooks --
  def _MakeHook(self, i):
    def hook(g):
      if self._phase == 0:
        self._arrival.append(i)
        return None
      if i in self._seen:                # a second backward through the same leaf
        return None
      self._seen.add(i)
      with torch.no_grad():
        self.gviews[i].copy_(g)          # cast → bf16 slot, on the backward's stream
      b = self._bucket_of[i]
      self._pending[b] -= 1
      if self._pending[b] == 0:
        self._LaunchBucket(b)
      return None
    return hook

  def _LaunchBucket(self, b):
    start, n, _ = self._buckets[b]
    cur = torch.cuda.current_stream(self.gbuf.device)
    ev = torch.cuda.Event()
    ev.record(cur)
    self.comm.wait_event(ev)
    with torch.cuda.stream(self.comm), torch.no_grad():
      self.chan.Sync(2 * b)                                   # every rank staged bucket b
      ops.native().allreduce_mean_bf16(
          self._bucket_peers[b], n // self.world, self.rank, self.world, 1.0 / self.world,
          self.gbuf.device.index, True, None, self._COMM_BLOCKS)
      self.chan.Sync(2 * b + 1)                               # every shard written everywhere
    self._launched[b] = True

  def _PlanBuckets(self):
    """Re-lays the flat buffer out in gradient-arrival order and cuts it into buckets."""
    order, seen = [], set()
    for i in self._arrival:
      if i not in seen:
        seen.add(i)
        order.append(i)
    order += [i for i in range(len(self.flat.vars)) if i not in seen]   # never arrived: last
    variables = [self.flat.vars[i] for i in order]
    unit = self.world * 8
    offsets, buckets = [], []
    off = start = 0
    members = []
    target = max(self._bucket_bytes // 2, (self.flat.total * 2) // self._MAX_BUCKETS + 1)
    for k, v in enumerate(variables):
      offsets.append(off)
      members.append(k)
      off += (v.numel() + 7) // 8 * 8
      if (off - start) * 2 >= target or k == len(variables) - 1:
        off = (off + unit - 1) // unit * unit                 # bucket = multiple of W·8
        buckets.append((start, off - start, members))
        start, members = off, []
    if off > self.flat.total:
      return False                                            # padding does not fit: keep monolithic
    self.flat.vars = variables
    self.flat.offsets = offsets
    self.gviews = self.flat.Views(self.gbuf)
    self._index = {id(v): i for i, v in enumerate(self.flat.vars)}
    self._buckets = buckets
    self._bucket_of = {k: b for b, (_, _, ms) in enumerate(buckets) for k in ms}
    self._bucket_peers = [
        torch.tensor([base + self.goff + s * 2 for base in self.arena.peer_base],
                     dtype=torch.int64) for s, _, _ in buckets]
    # hooks were registered with the old indices: re-register in the new order
    for h in self._hooks:
      h.remove()
    self._hooks = []
    for i, v in enumerate(self.flat.vars):
      leaf = getattr(v, 'compute', None)
      leaf = leaf if leaf is not None else v
      self._hooks.append(leaf.register_hook(self._MakeHook(i)))
    self._ResetStep()
    return True

  def _ResetStep(self):
    self._pending = [len(ms) for _, _, ms in self._buckets]
    self._launched = [False] * len(self._buckets)
    self._seen = set()

  # ------------------------------------------------------------------ call --
  def _Monolithic(self, leaves):
    dst = [self.gviews[self._index[id(vg.var)]] for vg in leaves]
    with torch.no_grad():
      torch._foreach_copy_(dst, [vg.grad for vg in leaves])   # cast → bf16 slots
      self.chan.Sync(2 * self._MAX_BUCKETS)                   # all copies staged
      ops.native().allreduce_mean_bf16(
          self.peers, self.flat.shard, self.rank, self.world, 1.0 / self.world,
          self.gbuf.device.index, True, None)
      self.chan.Sync(2 * self._MAX_BUCKETS + 1)               # all shards written
    return dst

  def __call__(self, var_grads):
    leaves = [vg for vg in var_grads.Flatten()
              if isinstance(vg, py_utils.VarGrad) and vg.grad is not None and
              id(vg.var) in self._index]
    if self._phase == 0 or not self._overlap:
      dst = self._Monolithic(leaves)
      if self._overlap and self._arrival:
        # Every rank saw the same autograd order; switch to the overlapped schedule.
        torch.cuda.synchronize()
        dist.barrier()
        if self._PlanBuckets():
          self._phase = 1
          dst = [self.gviews[self._index[id(vg.var)]] for vg in leaves]
          # this step's reduced values live at the old offsets: re-reduce in the new layout
          dst = self._Monolithic(leaves)
        else:
          self._overlap = False
    else:
      with torch.no_grad():
        for b, (start, n, ms) in enumerate(self._buckets):
          if self._launched[b]:
            continue
          for k in ms:                                       # gradients that never arrived
            if k not in self._seen:
              self.gviews[k].zero_()
          self._LaunchBucket(b)
      torch.cuda.current_stream(self.gbuf.device).wait_stream(self.comm)
      dst = [self.gviews[self._index[id(vg.var)]] for vg in leaves]
      self._ResetStep()
    for vg, view in zip(leaves, dst):
      vg.grad = view
    from lingvo_b200.parallel import dp as dp_lib  # pylint: disable=g-import-not-at-top
    dp_lib._ReduceExpertReplicas(   # pylint: disable=protected-access
        [vg for vg in var_grads.Flatten() if isinstance(vg, py_utils.VarGrad) and
         vg.grad is not None], self.ctx)
    return var_grads


class ZeroAdam:
  """Takes over a learner whose optimizer is Adam (sharded states, fused RS+Adam+AG)."""

  def __init__(self, task, learner, ctx):
    self.ctx = ctx
    self.world, self.rank = ctx.world, ctx.rank
    self.learner = learner
    self.opt_p = learner.optimizer.params
    dev = task.Device()
    self.flat = _Flat(_ReplicatedVars(task), self.world)
    n, shard = self.flat.total, self.flat.shard
    self.arena = symm_lib.SymmArena(n * 4 + 65536, dev)
    self.goff = self.arena.Alloc(n * 2)
    self.poff = self.arena.Alloc(n * 2)
    self.gbuf = self.arena.Local(self.goff, (n,), torch.bfloat16)
    self.pbuf = self.arena.Local(self.poff, (n,), torch.bfloat16)
    self.gviews = self.flat.Views(self.gbuf)
    self.pviews = self.flat.Views(self.pbuf)
    self.gpeers = torch.tensor([b + self.goff for b in self.arena.peer_base],
                               dtype=torch.int64)
    self.gself = torch.tensor([self.arena.peer_base[self.rank] + self.goff],
                              dtype=torch.int64)
    self.ppeers = torch.tensor([b + self.poff for b in self.arena.peer_base],
                               dtype=torch.int64)
    self.chan = _Channels(self.arena, self.world, self.rank)
    # fp32 master shard + Adam moments for my 1/W slice of the flat space.
    full = torch.zeros(n, dtype=torch.float32, device=dev)
    for v, o in zip(self.flat.vars, self.flat.offsets):
      full[o:o + v.numel()] = v.data.reshape(-1).float()
    self.master = full[self.rank * shard:(self.rank + 1) * shard].clone()
    self.m = torch.zeros_like(self.master)
    self.v = torch.zeros_like(self.master)
    self.pbuf.copy_(full)
    del full
    # The model computes with the replica views; gradients flow to them.
    for var, view in zip(self.flat.vars, self.pviews):
      var.compute = view.requires_grad_(True)
    for _, layer in task.Walk():
      for name, var in layer._private_vars.items():  # pylint: disable=protected-access
        if getattr(var, 'compute', None) is not None:
          layer.SetThetaOverride(name, var.compute)
    self.sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
    self.step = 0
    self._index = {id(v): i for i, v in enumerate(self.flat.vars)}
    dist.barrier()

  def Apply(self, lr, var_grads, clip_norm: float = 0.0):
    """Fused step. Returns the global gradient norm (device scalar)."""
    p = self.opt_p
    nat = ops.native()
    leaves = [vg for vg in var_grads.Flatten()
              if isinstance(vg, py_utils.VarGrad) and vg.grad is not None and
              id(vg.var) in self._index]
    dst = [self.gviews[self._index[id(vg.var)]] for vg in leaves]
    with torch.no_grad():
      torch._foreach_copy_(dst, [vg.grad for vg in leaves])
      self.chan.Sync(0)
      self.sumsq.zero_()
      nat.allreduce_mean_bf16(self.gpeers, self.flat.shard, self.rank,
                              self.world, 1.0 / self.world,
                              self.gbuf.device.index, False, self.sumsq)
      dist.all_reduce(self.sumsq)                       # 4-byte scalar
      gnorm = self.sumsq.sqrt()
      if clip_norm:
        scale = torch.clamp(clip_norm / gnorm, max=1.0)
      else:
        scale = torch.ones_like(gnorm)
      scale = torch.where(torch.isfinite(gnorm), scale, torch.zeros_like(scale))
      self.step += 1
      t = self.step
      lr_t = float(lr) * math.sqrt(1 - p.beta2**t) / (1 - p.beta1**t)
      nat.zero_adam(self.gself, self.ppeers, self.master, self.m, self.v,
                    self.rank, self.world, 1, 1.0, scale, lr_t, p.beta1,
                    p.beta2, p.epsilon)
      self.chan.Sync(1)
    return gnorm

  # -- checkpoint hooks (called through core/train_engine.py) -------------------------------
  def _Full(self, shard):
    full = torch.empty(self.flat.total, dtype=torch.float32, device=shard.device)
    dist.all_gather_into_tensor(full, shard)
    return full

  def PreSave(self):
    """Makes `var.data` (fp32 masters) and the optimizer's `<var>/Adam`, `<var>/Adam_1`
    slots authoritative on every rank, so the checkpoint has the reference layout."""
    from lingvo_b200.core import optimizer as optimizer_lib  # pylint: disable=g-import-not-at-top
    self.GatherMasters()
    opt = self.learner.optimizer
    fm, fv = self._Full(self.m), self._Full(self.v)
    with torch.no_grad():
      for var, o in zip(self.flat.vars, self.flat.offsets):
        n = var.numel()
        slots = opt._slots.setdefault(optimizer_lib._VarKey(var), {})  # pylint: disable=protected-access
        slots['m'] = fm[o:o + n].view(var.shape).clone()
        slots['v'] = fv[o:o + n].view(var.shape).clone()
    opt._step_count = self.step   # pylint: disable=protected-access

  def PostSave(self):
    """Drops the gathered full-size moments again (they only exist for the snapshot)."""
    from lingvo_b200.core import optimizer as optimizer_lib  # pylint: disable=g-import-not-at-top
    opt = self.learner.optimizer
    for var in self.flat.vars:
      slots = opt._slots.get(optimizer_lib._VarKey(var), {})  # pylint: disable=protected-access
      slots.pop('m', None)
      slots.pop('v', None)

  def PostRestore(self):
    """Re-shards masters / moments / step from the restored variables and slots."""
    from lingvo_b200.core import optimizer as optimizer_lib  # pylint: disable=g-import-not-at-top
    opt = self.learner.optimizer
    n, shard = self.flat.total, self.flat.shard
    dev = self.master.device
    lo, hi = self.rank * shard, (self.rank + 1) * shard
    full = torch.zeros(n, dtype=torch.float32, device=dev)
    fm, fv = torch.zeros_like(full), torch.zeros_like(full)
    with torch.no_grad():
      for var, o in zip(self.flat.vars, self.flat.offsets):
        k = var.numel()
        full[o:o + k] = var.data.reshape(-1).float()
        slots = opt._slots.get(optimizer_lib._VarKey(var), {})  # pylint: disable=protected-access
        if 'm' in slots:
          fm[o:o + k] = slots['m'].reshape(-1).float().to(dev)
        if 'v' in slots:
          fv[o:o + k] = slots['v'].reshape(-1).float().to(dev)
      self.master.copy_(full[lo:hi])
      self.m.copy_(fm[lo:hi])
      self.v.copy_(fv[lo:hi])
      self.pbuf.copy_(full)
    self.step = int(opt._step_count)   # pylint: disable=protected-access

  def GatherMasters(self):
    """fp32 masters of all shards → `var.data` (for checkpointing)."""
    full = torch.empty(self.flat.total, dtype=torch.float32,
                       device=self.master.device)
    dist.all_gather_into_tensor(full, self.master)
    with torch.no_grad():
      for v, o in zip(self.flat.vars, self.flat.offsets):
        v.data.copy_(full[o:o + v.numel()].view(v.shape))
