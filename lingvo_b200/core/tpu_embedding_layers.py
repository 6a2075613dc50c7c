"""Large-table embeddings with their own sparse optimizers
(ref `lingvo/core/tpu_embedding_layers{,_v1,_v2}.py`, `tpu_embedding_manager.py`).

On TPU these tables live in the embedding hardware with dedicated
SGD/Adagrad/Adam/FTRL optimizers fed by "send gradients" ops. The H100 equivalent:
tables are row-sharded across ranks (`index % world == rank`), lookups are an
all-to-all of ids + rows over NVLink, and the table optimizer is applied **sparsely**
(only to the rows touched in the step) right after backward, outside the dense
optimizer — so a 100M-row table never pays a dense update.
"""

from __future__ import annotations

import torch
import torch.distributed as dist

from lingvo_b200.core import base_layer
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.core.py_utils import WeightInit
from lingvo_b200.core.py_utils import WeightParams


class _TableOptimizer(base_layer.BaseLayer):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('clip_weight_min', None, 'Clip table values.')
    p.Define('clip_weight_max', None, 'Clip table values.')
    p.Define('clip_gradient_min', None, 'Clip gradients.')
    p.Define('clip_gradient_max', None, 'Clip gradients.')
    p.Define('weight_decay_factor', None, 'Weight decay.')
    p.name = 'table_optimizer'
    return p

  def CreateSlots(self, table):
    return {}

  def Apply(self, lr, table, slots, rows, grads):
    raise NotImplementedError

  def _Clip(self, g):
    p = self.params
    if p.clip_gradient_min is not None or p.clip_gradient_max is not None:
      g = g.clamp(p.clip_gradient_min, p.clip_gradient_max)
    return g

  def _Post(self, table, rows):
    p = self.params
    if p.clip_weight_min is not None or p.clip_weight_max is not None:
      table[rows] = table[rows].clamp(p.clip_weight_min, p.clip_weight_max)


class TPUEmbeddingSGDOptimizer(_TableOptimizer):

  def Apply(self, lr, table, slots, rows, grads):
    table.index_add_(0, rows, -lr * self._Clip(grads))
    self._Post(table, rows)


class TPUEmbeddingAdagradOptimizer(_TableOptimizer):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('initial_accumulator', 0.1, 'Initial accumulator value.')
    p.Define('use_gradient_accumulation', True, 'Kept for parity.')
    return p

  def CreateSlots(self, table):
    return {'accumulator': torch.full_like(table, self.params.initial_accumulator)}

  def Apply(self, lr, table, slots, rows, grads):
    g = self._Clip(grads)
    acc = slots['accumulator']
    acc.index_add_(0, rows, g * g)
    table.index_add_(0, rows, -lr * g / acc[rows].sqrt())
    self._Post(table, rows)


class TPUEmbeddingAdamOptimizer(_TableOptimizer):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('lazy_adam', True, 'Only touched rows are updated.')
    p.Define('beta1', 0.9, 'β1.')
    p.Define('beta2', 0.999, 'β2.')
    p.Define('epsilon', 1e-8, 'ε.')
    p.Define('sum_inside_sqrt', True, 'Kept for parity.')
    return p

  def CreateSlots(self, table):
    return {'m': torch.zeros_like(table), 'v': torch.zeros_like(table),
            'step': torch.zeros((), device=table.device)}

  def Apply(self, lr, table, slots, rows, grads):
    p = self.params
    g = self._Clip(grads)
    slots['step'] += 1
    t = float(slots['step'])
    m, v = slots['m'], slots['v']
    m[rows] = p.beta1 * m[rows] + (1 - p.beta1) * g
    v[rows] = p.beta2 * v[rows] + (1 - p.beta2) * g * g
    lr_t = lr * (1 - p.beta2 ** t) ** 0.5 / (1 - p.beta1 ** t)
    table[rows] = table[rows] - lr_t * m[rows] / (v[rows].sqrt() + p.epsilon)
    self._Post(table, rows)


class TPUEmbeddingFTRLOptimizer(_TableOptimizer):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('learning_rate_power', -0.5, 'Learning-rate power.')
    p.Define('initial_accumulator_value', 0.1, 'Initial accumulator.')
    p.Define('l1_regularization_strength', 0.0, 'L1.')
    p.Define('l2_regularization_strength', 0.0, 'L2.')
    return p

  def CreateSlots(self, table):
    return {'accumulator': torch.full_like(table, self.params.initial_accumulator_value),
            'linear': torch.zeros_like(table)}

  def Apply(self, lr, table, slots, rows, grads):
    p = self.params
    g = self._Clip(grads)
    acc, lin = slots['accumulator'], slots['linear']
    a0 = acc[rows]
    a1 = a0 + g * g
    pw = -p.learning_rate_power
    sigma = (a1 ** pw - a0 ** pw) / lr
    lin[rows] = lin[rows] + g - sigma * table[rows]
    acc[rows] = a1
    quad = a1 ** pw / lr + 2 * p.l2_regularization_strength
    l1 = p.l1_regularization_strength
    z = lin[rows]
    table[rows] = torch.where(z.abs() > l1, -(z - torch.sign(z) * l1) / quad, torch.zeros_like(z))


class TPUEmbeddingTable(base_layer.BaseLayer):
  """One row-sharded table (ref v1 :300)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_size', 0, 'Rows.')
    p.Define('embedding_dim', 0, 'Columns.')
    p.Define('input_keys', None, 'Input features looked up in this table.')
    p.Define('combiner', 'sum', 'sum | mean | sqrtn | None (sequence).')
    p.Define('max_sequence_length', None, 'For combiner=None.')
    p.Define('num_tpu_hosts', 0, 'Kept for parity.')
    p.Define('optimizer', None, 'Table optimizer (defaults to the layer-level one).')
    p.Define('learning_rate', 0.0, 'Table learning rate.')
    p.Define('lr_schedule', None, 'LR schedule layer params.')
    p.Define('inference_use_merged_variable', False, 'Kept for parity.')
    p.Define('inference_variable_dtype', None, 'Kept for parity.')
    p.Define('inference_auxiliary_variable_specs', None, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.vocab_size > 0 and p.embedding_dim > 0 and p.input_keys
    self._world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    self._rank = dist.get_rank() if self._world > 1 else 0
    self._local_rows = -(-p.vocab_size // self._world)
    self.CreateChild('optimizer', p.optimizer or TPUEmbeddingSGDOptimizer.Params())
    if p.lr_schedule is not None:
      self.CreateChild('schedule', p.lr_schedule)
    self._slots = None
    self._pending = []
    self._pending_grads = []         # (local rows, gradient rows) received from other ranks
    self.gradient_multiplier = 1.0   # set by the layer's gradient-multiplier schedule

  def _CreateLayerVariables(self):
    p = self.params
    w = self.CreateVariable('var', WeightParams([self._local_rows, p.embedding_dim],
                                                p.params_init, p.dtype), trainable=False)
    del w

  @property
  def table(self):
    return self.vars['var'].data

  def Lookup(self, ids):
    """ids (any shape, global row ids; −1 = missing) → embeddings `[..., D]` with grad
    hooks that feed the sparse optimizer. With several ranks the table is row-sharded
    (`row % world` owns row, stored at `row // world`): ids travel to their owners and rows
    come back in two all-to-alls; the backward sends the row gradients to the owners, which
    queue them for their sparse optimizer."""
    p = self.params
    flat = ids.reshape(-1)
    valid = flat >= 0
    rows = flat.clamp_min(0)
    if self._world > 1:
      # a differentiable anchor makes autograd call the backward (ids are integers)
      anchor = torch.zeros((), device=self.table.device, requires_grad=torch.is_grad_enabled())
      emb = _ShardedLookup.apply(self, rows, anchor)
      out = emb * valid.unsqueeze(-1).to(emb.dtype)
      return out.reshape(*ids.shape, p.embedding_dim)
    emb = self.table[rows].detach().clone().requires_grad_(True)
    out = emb * valid.unsqueeze(-1).to(emb.dtype)
    if torch.is_grad_enabled():
      self._pending.append((rows, emb))
    return out.reshape(*ids.shape, p.embedding_dim)

  # -- cross-rank exchange ------------------------------------------------------------
  def _ExchangePlan(self, rows):
    """Sorts the requested global rows by owner and exchanges the per-owner counts."""
    w = self._world
    owner = rows % w
    order = torch.argsort(owner, stable=True)
    send_ids = rows[order]
    send_counts = torch.bincount(owner, minlength=w)
    recv_counts = torch.empty_like(send_counts)
    dist.all_to_all_single(recv_counts, send_counts)
    return order, send_ids, send_counts.tolist(), recv_counts.tolist()

  def _FetchRows(self, rows):
    order, send_ids, sc, rc = self._ExchangePlan(rows)
    req = torch.empty(sum(rc), dtype=send_ids.dtype, device=send_ids.device)
    dist.all_to_all_single(req, send_ids.contiguous(), rc, sc)
    local = req // self._world
    reply = self.table[local].contiguous()
    got = torch.empty(len(send_ids), reply.shape[1], dtype=reply.dtype, device=reply.device)
    dist.all_to_all_single(got, reply, sc, rc)
    out = torch.empty_like(got)
    out[order] = got
    return out, (order, sc, rc, local)

  def _ReturnGrads(self, grad, plan):
    order, sc, rc, local = plan
    send = grad[order].contiguous()
    recv = torch.empty(sum(rc), grad.shape[1], dtype=grad.dtype, device=grad.device)
    dist.all_to_all_single(recv, send, rc, sc)
    self._pending_grads.append((local, recv))

  def ApplyGradients(self, global_step=0):
    """Applies the sparse optimizer to every row looked up since the last call."""
    p = self.params
    if self._slots is None:
      self._slots = self.optimizer.CreateSlots(self.table)
    lr = p.learning_rate
    if p.lr_schedule is not None:
      lr = lr * float(self.schedule.Value(global_step))
    with torch.no_grad():
      todo = [(rows, emb.grad) for rows, emb in self._pending if emb.grad is not None]
      todo += self._pending_grads
      for rows, grad in todo:
        uniq, inv = torch.unique(rows, return_inverse=True)
        g = torch.zeros(uniq.shape[0], grad.shape[1], device=grad.device, dtype=grad.dtype)
        g.index_add_(0, inv, grad)
        if self.gradient_multiplier != 1.0:
          g = g * self.gradient_multiplier
        self.optimizer.Apply(lr, self.table, self._slots, uniq, g)
    self._pending = []
    self._pending_grads = []


class _ShardedLookup(torch.autograd.Function):
  """Row fetch from a row-sharded table; the backward routes row gradients to the owners."""

  @staticmethod
  def forward(ctx, table_layer, rows, anchor):
    del anchor
    emb, plan = table_layer._FetchRows(rows)   # pylint: disable=protected-access
    ctx.layer, ctx.plan = table_layer, plan
    return emb

  @staticmethod
  def backward(ctx, grad):
    ctx.layer._ReturnGrads(grad.contiguous(), ctx.plan)   # pylint: disable=protected-access
    return None, None, None


class TPUEmbeddingLayer(base_layer.BaseLayer):
  """A set of tables + feature → table routing (ref v1 :600)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_tpu_hosts', 0, 'Kept for parity.')
    p.Define('tables', None, 'List of TPUEmbeddingTable params.')
    p.Define('pipeline_execution_with_tensor_core', False, 'Kept for parity.')
    p.Define('batch_size', 0, 'Kept for parity.')
    p.Define('optimizer', TPUEmbeddingAdagradOptimizer.Params(), 'Default table optimizer.')
    p.Define('learning_rate', 0.0, 'Default learning rate.')
    p.Define('lr_schedule', None, 'Default LR schedule.')
    p.Define('partition_strategy', 'div', 'Kept for parity.')
    p.Define('gradient_multiplier_schedule', None,
             'Schedule params: table gradients are multiplied by its value at the step.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    tables = []
    for tp in p.tables:
      tp = tp.Copy()
      tp.optimizer = tp.optimizer or p.optimizer.Copy()
      tp.learning_rate = tp.learning_rate or p.learning_rate
      tp.lr_schedule = tp.lr_schedule or p.lr_schedule
      tables.append(tp)
    self.CreateChildren('tables', tables)
    if p.gradient_multiplier_schedule is not None:
      self.CreateChild('gradient_multiplier_schedule', p.gradient_multiplier_schedule)
    self._route = {}
    for t in self.tables:
      for k in t.params.input_keys:
        self._route[k] = t

  def EmbLookup(self, theta, ids_map):
    """ids_map: key → `[B, L]` ids (−1 padded) → key → combined `[B, D]` (or `[B, L, D]`)."""
    del theta
    out = NestedMap()
    for k, ids in ids_map.items():
      t = self._route[k]
      emb = t.Lookup(ids)
      comb = t.params.combiner
      if comb is None:
        out[k] = emb
        continue
      n = (ids >= 0).sum(-1, keepdim=True).clamp_min(1).to(emb.dtype)
      s = emb.sum(-2)
      out[k] = s if comb == 'sum' else (s / n if comb == 'mean' else s / n.sqrt())
    return out

  def ApplyGradients(self, global_step=0):
    mult = 1.0
    if self.params.gradient_multiplier_schedule is not None:
      mult = float(self.gradient_multiplier_schedule.Value(global_step))
    for t in self.tables:
      t.gradient_multiplier = mult
      t.ApplyGradients(global_step)
