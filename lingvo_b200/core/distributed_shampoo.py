"""Distributed Shampoo: approximate full-matrix AdaGrad per layer
(ref `lingvo/core/distributed_shampoo.py`; "Second-order optimization made practical", Anil
et al. 2019) and the lingvo wrapper (ref `optimizer.py:689`).

For a rank-k (block of a) parameter with gradient G, one statistics matrix per preconditioned
axis i accumulates `S_i += G ·_{≠i} G` (contraction over all other axes); the preconditioned
gradient is G multiplied along each such axis by `S_i^{-1/(2k)}`. Everything else follows the
reference:

  * `TensorPartitioner` (:61): axes larger than `block_partition_threshold_size` are cut into
    `block_size` pieces; each block has its own statistics / preconditioners.
  * fall-backs (:233-264): rank ≤ 1, any dim > `max_any_dim`, or all-ones shapes use the
    diagonal AdaGrad update only; inside a preconditioned tensor an axis larger than
    `fallback_to_diagonal_dim` (or of size 1) simply gets no preconditioner.
  * grafting (:586): the preconditioned step is rescaled to the l2 norm of the diagonal
    AdaGrad step of the same tensor; two momentum buffers (diagonal / preconditioned).
  * warm-up (:213): before `start_preconditioning_steps` the diagonal update is used, then the
    two are blended linearly over another `start_preconditioning_steps` steps.
  * `second_moment_averaging` < 1 turns the statistics sums into moving averages,
    `statistics_computation_frequency` thins the statistics updates, `exponent_multiplier`
    scales the inverse-root exponent.

H100 design. The statistics updates are `tensordot`s — GEMMs on the tensor cores, fp32
accumulate. The inverse p-th roots are the only super-linear part; they run every
`preconditioning_compute_steps`:
  * synchronously with the coupled Newton iteration of `matrix_functions` (all matmuls), or
  * `async_preconditioning=True`: queued on `preconditioner_captain`'s low-priority CUDA
    stream (the reference ships them to CPU workers through `x_ops.compute_preconditioners`);
    the step keeps using the last finished preconditioners and swaps new ones in with the
    same `success` masking as the reference (:427-444). No host synchronisation either way.
"""

from __future__ import annotations

import re
from typing import Dict, List

import torch

from lingvo_b200.core import matrix_functions
from lingvo_b200.core import optimizer
from lingvo_b200.core import py_utils


class PartitionConfig:
  """Config for `TensorPartitioner` (ref :32)."""

  def __init__(self, max_dim_size, partition_size):
    if partition_size < 1 or partition_size > max_dim_size:
      raise ValueError('Partition size must be no less than 1 and no greater than max_dim.')
    self.max_dim_size = max_dim_size
    self.partition_size = partition_size


class PartitionMetadata:
  """Split sizes per axis of a partitioned tensor (ref :46)."""

  def __init__(self, split_sizes_per_dim, num_splits_per_dim):
    self.split_sizes_per_dim = split_sizes_per_dim
    self.num_splits_per_dim = num_splits_per_dim


class TensorPartitioner:
  """Cuts a tensor into blocks along every axis longer than `max_dim_size` and puts them back
  together (ref :61). Blocks are views, so partitioning moves no data."""

  @classmethod
  def partition_metadata(cls, tensor, partition_info) -> PartitionMetadata:
    split_sizes_per_dim = []
    for dim in tensor.shape:
      dim = int(dim)
      sizes = [dim]
      if dim > partition_info.max_dim_size:
        n = dim // partition_info.partition_size
        if n > 0:
          sizes = [partition_info.partition_size] * n
          if dim % partition_info.partition_size:
            sizes.append(dim % partition_info.partition_size)
      split_sizes_per_dim.append(sizes)
    return PartitionMetadata(split_sizes_per_dim, [len(v) for v in split_sizes_per_dim])

  @classmethod
  def partition_tensor(cls, tensor, partition_info) -> List[torch.Tensor]:
    meta = cls.partition_metadata(tensor, partition_info)
    parts = [tensor]
    rank = len(meta.num_splits_per_dim)
    for axis in range(rank - 1, -1, -1):                  # last axis first, as the reference
      if meta.num_splits_per_dim[axis] > 1:
        nxt = []
        for item in parts:
          nxt += list(torch.split(item, meta.split_sizes_per_dim[axis], dim=axis))
        parts = nxt
    return parts

  @classmethod
  def reform_tensor(cls, partitioned_tensors, num_splits_per_dim) -> torch.Tensor:
    parts = list(partitioned_tensors)
    for axis, n in enumerate(num_splits_per_dim):
      if n > 1:
        parts = [torch.cat(parts[i * n:(i + 1) * n], dim=axis)
                 for i in range(len(parts) // n)]
    assert len(parts) == 1
    return parts[0]


class DistributedShampoo(optimizer.Base):
  """Approximates full-matrix AdaGrad per layer (ref optimizer.py:689)."""

  SLOT_SUFFIX = {'accumulator': 'accumulator', 'momentum': 'momentum',
                 'precond_grad_momentum': 'precond_grad_momentum'}
  EXTRA_SLOT_REGEX = re.compile(r'(\d+_)?mat_(statistics|preconditioner)_\d+')

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('momentum', 0.9, 'Momentum parameter.')
    p.Define('start_preconditioning_steps', 1000,
             'When to start approximate full matrix preconditioning.')
    p.Define('initial_accumulator_value', 0.0, 'Initial accumulator value.')
    p.Define('block_size', 4096, 'Block size for partitioning.')
    p.Define('block_partition_threshold_size', 1000000, 'Threshold for block partitioning.')
    p.Define('max_any_dim', 8192, 'Max dimension before skipping preconditioning altogether.')
    p.Define('matrix_epsilon', 1e-6, 'Minimum eigen value used to improve the conditioning.')
    p.Define('second_moment_averaging', 1.0,
             '1.0 means sum of squares; less than 1.0 is an RMSProp-style moving average.')
    p.Define('fallback_to_diagonal_dim', 4096,
             'Axes larger than this get no preconditioner.')
    p.Define('statistics_computation_frequency', 1, 'How often to compute statistics.')
    p.Define('exponent_multiplier', 1.0, 'Multiplier of the inverse-root exponent.')
    p.Define('preconditioning_compute_steps', 1,
             'How often (steps) the inverse roots are recomputed.')
    p.Define('synchronous_preconditioning', True, 'Kept for parity: see async_preconditioning.')
    p.Define('async_preconditioning', False,
             'Solve the inverse roots on the low-priority side stream of '
             '`preconditioner_captain` and step with the last finished ones.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self._partition_info = PartitionConfig(p.block_partition_threshold_size, p.block_size)
    self._metadata: Dict[str, PartitionMetadata] = {}

  # -- shape rules (ref :233-264) -----------------------------------------------------
  def _FallbackToDiagonalForShape(self, shape) -> bool:
    p = self.params
    if len(shape) <= 1:
      return True
    if any(d > p.max_any_dim for d in shape):
      return True
    return all(d == 1 for d in shape)

  def _PreconditionerAvailableForDims(self, shape):
    p = self.params
    return [d <= p.fallback_to_diagonal_dim and d != 1 for d in shape]

  @staticmethod
  def _StatKey(dim_index, partition_index, num_partitions):
    base = 'mat_statistics_%d' % dim_index
    return base if num_partitions == 1 else '%d_%s' % (partition_index, base)

  @staticmethod
  def _PrecondKey(dim_index, partition_index, num_partitions):
    base = 'mat_preconditioner_%d' % dim_index
    return base if num_partitions == 1 else '%d_%s' % (partition_index, base)

  def _Blocks(self, tensor):
    return TensorPartitioner.partition_tensor(tensor, self._partition_info)

  def _EnsureMatrixSlots(self, var):
    """Creates the statistics / preconditioner slots of `var` (ref `_create_slots` :324).
    Preconditioners start as zeros like the reference: with grafting a zero preconditioned
    step falls back to multiplier 1 (i.e. contributes nothing) until the first solve lands."""
    key = optimizer._VarKey(var)   # pylint: disable=protected-access
    if key in self._metadata:
      return
    self._metadata[key] = TensorPartitioner.partition_metadata(var, self._partition_info)
    blocks = self._Blocks(var)
    for bi, blk in enumerate(blocks):
      avail = self._PreconditionerAvailableForDims(blk.shape)
      for i, d in enumerate(blk.shape):
        if avail[i]:
          self._Slot(var, self._StatKey(i, bi, len(blocks)), shape=[d, d], dtype=torch.float32)
          self._Slot(var, self._PrecondKey(i, bi, len(blocks)), shape=[d, d],
                     dtype=torch.float32)

  # -- statistics (ref :465) ----------------------------------------------------------
  def _UpdateStatistics(self, var, blocks):
    p = self.params
    n = len(blocks)
    for bi, g in enumerate(blocks):
      avail = self._PreconditionerAvailableForDims(g.shape)
      rank = g.dim()
      gf = g.float()
      for i in range(rank):
        if not avail[i]:
          continue
        axes = [a for a in range(rank) if a != i]
        new_stat = torch.tensordot(gf, gf, dims=(axes, axes))
        stat = self._Slot(var, self._StatKey(i, bi, n))
        if p.second_moment_averaging == 1.0:
          stat.add_(new_stat)
        else:
          stat.mul_(p.second_moment_averaging).add_(new_stat,
                                                    alpha=1.0 - p.second_moment_averaging)

  # -- inverse roots (ref :367-444) ---------------------------------------------------
  def _InversePthRoot(self, stat, exponent):
    """stat^{exponent·multiplier} with exponent = −1/(2·rank)."""
    p = self.params
    root = -1.0 / (exponent * p.exponent_multiplier)
    if abs(root - round(root)) < 1e-6 and round(root) >= 1:
      fn = (matrix_functions.inverse_pth_root_no_sync if stat.is_cuda
            else matrix_functions.inlined_matrix_inverse_pth_root)
      return fn(stat, int(round(root)), ridge_epsilon=p.matrix_epsilon)
    # generalised (non-integer) exponents: symmetric eigendecomposition (ref :274)
    d = stat.shape[0]
    s, u = torch.linalg.eigh(stat.double() + torch.eye(d, dtype=torch.float64,
                                                       device=stat.device) * p.matrix_epsilon)
    s = s.clamp_min(p.matrix_epsilon).pow(exponent * p.exponent_multiplier)
    return ((u * s.unsqueeze(0)) @ u.t()).float()

  def _ComputePreconditioners(self, var, blocks, step):
    p = self.params
    n = len(blocks)
    vkey = optimizer._VarKey(var)   # pylint: disable=protected-access
    for bi, g in enumerate(blocks):
      avail = self._PreconditionerAvailableForDims(g.shape)
      rank_p = sum(avail)
      for i in range(g.dim()):
        if not avail[i]:
          continue
        stat = self._Slot(var, self._StatKey(i, bi, n))
        pre = self._Slot(var, self._PrecondKey(i, bi, n))
        exponent = -1.0 / (2.0 * rank_p)
        if p.async_preconditioning:
          from lingvo_b200.core import preconditioner_captain   # pylint: disable=g-import-not-at-top
          cap = preconditioner_captain.GetCaptain()
          ckey = 'P_%d_D_%d_%s' % (bi, i, vkey)
          if step % p.preconditioning_compute_steps == 0:
            cap.InsertGradientStatistics(ckey, stat, -1.0 / (exponent * p.exponent_multiplier),
                                         step)
          done, ok = cap.GetPreconditioner(ckey)
          if ok:
            pre.copy_(done)
        elif step % p.preconditioning_compute_steps == 0:
          pre.copy_(self._InversePthRoot(stat, exponent))

  # -- preconditioned gradient (ref :536) ---------------------------------------------
  def _PreconditionedRawGrad(self, var, blocks):
    n = len(blocks)
    out = []
    for bi, g in enumerate(blocks):
      avail = self._PreconditionerAvailableForDims(g.shape)
      rank = g.dim()
      pg = g.float()
      if rank == 2 and all(avail):
        pg = self._Slot(var, self._PrecondKey(0, bi, n)) @ pg @ self._Slot(
            var, self._PrecondKey(1, bi, n))
      else:
        # rotate through the axes: contract axis 0 with the preconditioner (the new axis lands
        # last) or just move axis 0 to the end — after `rank` rounds the layout is restored
        for i in range(rank):
          if avail[i]:
            pg = torch.tensordot(pg, self._Slot(var, self._PrecondKey(i, bi, n)),
                                 dims=([0], [0]))
          else:
            pg = pg.permute(*range(1, rank), 0)
      out.append(pg)
    key = optimizer._VarKey(var)   # pylint: disable=protected-access
    return TensorPartitioner.reform_tensor(out, self._metadata[key].num_splits_per_dim)

  def _Update(self, lr, variables, grads):
    p = self.params
    step = int(self._step_count)          # == global step of the reference (0-based)
    run_nondiagonal = step >= p.start_preconditioning_steps
    if p.start_preconditioning_steps > 0:
      warmup = min(1.0, max((step - p.start_preconditioning_steps) /
                            float(p.start_preconditioning_steps), 0.0))
    else:
      warmup = 1.0
    run_stats = step % max(1, p.statistics_computation_frequency) == 0
    lr_t = lr if isinstance(lr, torch.Tensor) else float(lr)
    for v, g in zip(variables, optimizer._F32(grads, variables)):   # pylint: disable=protected-access
      fallback = self._FallbackToDiagonalForShape(v.shape)
      blocks = None
      if not fallback:
        self._EnsureMatrixSlots(v)
        blocks = self._Blocks(g)
        if run_stats:
          self._UpdateStatistics(v, blocks)
      acc = self._Slot(v, 'accumulator', init=p.initial_accumulator_value)
      acc.addcmul_(g, g)
      diag = g * torch.rsqrt(acc + 1e-30)
      if p.momentum > 0.0:
        gbar = self._Slot(v, 'momentum')
        gbar.mul_(p.momentum).add_(diag, alpha=1.0 - p.momentum)
        diag = gbar
      update = diag
      if not fallback:
        self._ComputePreconditioners(v, blocks, step)
        if run_nondiagonal:
          pg = self._PreconditionedRawGrad(v, blocks).to(g.dtype)
          if p.momentum > 0.0:
            pbar = self._Slot(v, 'precond_grad_momentum')
            pbar.mul_(p.momentum).add_(pg, alpha=1.0 - p.momentum)
            pg = pbar
          pn = pg.float().norm()
          dn = diag.float().norm()
          mult = torch.where(pn > 0, dn.clamp_min(1e-30) / pn.clamp_min(1e-30),
                             torch.ones_like(pn))
          update = warmup * (pg * mult.to(pg.dtype)) + (1.0 - warmup) * diag
        elif p.momentum > 0.0:
          self._Slot(v, 'precond_grad_momentum')        # slot exists from step 0 (ckpt layout)
      if isinstance(lr_t, torch.Tensor):
        v.sub_(update * lr_t.to(update.dtype))
      else:
        v.add_(update, alpha=-lr_t)

  # Checkpoints name matrix slots dynamically: accept them by pattern on restore.
  def LoadOptimizerSlots(self, tensors):
    used = super().LoadOptimizerSlots(tensors)
    seen = set(used)
    for key, t in tensors.items():
      if key in seen:
        continue
      base, _, suffix = key.rpartition('/')
      if self.EXTRA_SLOT_REGEX.fullmatch(suffix):
        dst = self._slots.setdefault(base + '/var', {})
        if suffix in dst:
          dst[suffix].copy_(t.to(dst[suffix].device))
        else:
          dst[suffix] = t.clone()
        used.append(key)
    return used
