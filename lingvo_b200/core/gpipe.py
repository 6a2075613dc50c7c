"""GPipe-style pipelining layers (ref `lingvo/core/gpipe.py`).

* `FeatureExtractionLayer` (ref :107) — a sequence of sub-layers that can also
  fetch/forward cached activations.
* `PartitionSequentialLayers` (ref :179) — FLOP-balanced split of a sequential
  stack into `num_partitions` cells using each layer's `FPropMeta`.
* `SeqLayer` / `PipeliningLayer` (ref :251, :324) — run `cell_tpl[i]` as
  pipeline stage i over `num_micro_batches` micro-batches.

The reference pipelines inside one TF graph with `recurrent.StackedRecurrent`
(Send/Recv between devices of one process). On H100 each GPU is its own
process, so stages live on different ranks and activations/gradients move as
NCCL point-to-point transfers over NVLink — that engine is
`lingvo_b200.parallel.pp.PipelineEngine`. When all stages are in this process
(the default, and the CPU tests) `PipeliningLayer.FProp` runs the same
micro-batch schedule locally, which is numerically identical.
"""

from __future__ import annotations

import torch

from lingvo_b200.core import base_layer
from lingvo_b200.core import builder_layers
from lingvo_b200.core import py_utils
from lingvo_b200.core import tshape
from lingvo_b200.core.nested_map import NestedMap

_OVERWRITE_GLOBAL_STEP = [None]


def GetOverWriteGlobalStep(graph=None):
  """Per-micro-batch global step override used for step seeds (ref :46)."""
  del graph
  gs = _OVERWRITE_GLOBAL_STEP[0]
  return gs if gs is not None else py_utils.GetGlobalStep()


def SetOverWriteGlobalStep(tensor, graph=None):
  del graph
  _OVERWRITE_GLOBAL_STEP[0] = tensor


def GenerateStepSeedPair(p, unused_global_step=None, op_seed=None):
  """Step seed that differs per micro-batch (ref :65)."""
  return py_utils.GenerateStepSeedPair(p, op_seed=op_seed)


def _ToTuple(x):
  return x if isinstance(x, tuple) else (tuple(x) if isinstance(x, list) else (x,))


class FeatureExtractionLayer(base_layer.BaseLayer):
  """Sequential sub-layers + activation fetch/forward (ref :107)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('variable_name_prefix', '', 'Prefix for sub-layer names.')
    p.Define('sub', [], 'List of sub-layer params.')
    p.Define('num_act_inputs', 0, 'Trailing args that are forwarded untouched.')
    p.Define('num_act_outputs', 0, 'Forwarded + fetched activations.')
    p.Define('act_fetch_layers', [], 'Sub-layers whose `.activation` is appended.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.num_act_outputs == p.num_act_inputs + len(p.act_fetch_layers or [])
    self._seq = []
    for sub in p.sub:
      assert sub.name
      sub = sub.Copy()
      sub.name = p.variable_name_prefix + sub.name
      self.CreateChild(sub.name, sub)
      self._seq.append(sub.name)

  def FProp(self, theta, *args):
    p = self.params
    assert len(args) > p.num_act_inputs
    out_args = args[:-p.num_act_inputs] if p.num_act_inputs > 0 else args
    extra = tuple(args[-p.num_act_inputs:]) if p.num_act_inputs > 0 else ()
    for name in self._seq:
      out_args = self.children[name].FProp(theta[name], *_ToTuple(out_args))
    for fetch in (p.act_fetch_layers or []):
      act = self.children[fetch].activation
      if isinstance(act, (tuple, list)):
        act = act[0]
      extra += (act,)
    if extra:
      out_args = _ToTuple(out_args) + extra
    return out_args

  @classmethod
  def FPropMeta(cls, p, *args):
    seq_args = args[:-p.num_act_inputs] if p.num_act_inputs > 0 else args
    extra = tuple(args[-p.num_act_inputs:]) if p.num_act_inputs > 0 else ()
    total = 0
    fetched = {}
    for sub in p.sub:
      meta = sub.cls.FPropMeta(sub, *seq_args)
      if sub.name in (p.act_fetch_layers or []):
        fetched[sub.name] = meta.out_shapes[0]
      total += meta.flops
      seq_args = meta.out_shapes
    for f in p.act_fetch_layers or []:
      extra += (fetched[f],)
    return NestedMap(flops=total, out_shapes=tuple(seq_args) + extra)


def PartitionSequentialLayers(params, num_partitions, *shapes):
  """Splits a sequential stack into `num_partitions` FLOP-balanced cells (ref :179).

  Layer i goes to partition floor(cumulative_cost_fraction(i) · P).
  """

  def _Flatten(p):
    if isinstance(p, list):
      return p
    if p.cls not in (builder_layers.SequentialLayer, FeatureExtractionLayer):
      return [p.Copy()]
    subs = []
    for _ in range(p.repeat if 'repeat' in p else 1):
      for s in p.sub:
        subs += _Flatten(s)
    return subs

  subs = _Flatten(params)
  assert len(shapes) == 1
  total, histo = 0, []
  cur = shapes
  for i, s in enumerate(subs):
    s.name = 'cell_%03d' % i
    meta = s.cls.FPropMeta(s, *cur)
    total += meta.flops
    histo.append(total)
    cur = meta.out_shapes
  pct = [float(x) / max(total, 1) for x in histo]
  parts = [[] for _ in range(num_partitions)]
  for i, s in enumerate(subs):
    j = min(int(pct[i] * num_partitions), num_partitions - 1)
    parts[j].append(s)
  return [FeatureExtractionLayer.Params().Set(name='d%d' % i, sub=pa)
          for i, pa in enumerate(parts)]


class SeqLayer(base_layer.BaseLayer):
  """`before_tpl` layers, then `cell_tpl[i]` placed on split i (ref :251)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('before_tpl', [], 'Layers that run before the pipelined cells.')
    p.Define('cell_tpl', [], 'List of FeatureExtractionLayer params (one per stage).')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.name
    self._before_names, self._cell_names = [], []
    for l in p.before_tpl:
      self.CreateChild(l.name, l)
      self._before_names.append(l.name)
    for l in p.cell_tpl:
      self.CreateChild(l.name, l)
      self._cell_names.append(l.name)

  @property
  def num_stages(self):
    return len(self._cell_names)

  def _RunBefore(self, theta, args):
    for name in self._before_names:
      args = _ToTuple(self.children[name].FProp(theta[name], *args))
    return args

  def _RunCells(self, theta, args, first=0, last=None):
    names = self._cell_names[first:last]
    for name in names:
      args = _ToTuple(self.children[name].FProp(theta[name], *args))
    return args

  def FProp(self, theta, *args):
    args = self._RunBefore(theta, _ToTuple(args))
    out = self._RunCells(theta, args)
    return out[0] if len(out) == 1 else out


class PipeliningLayer(SeqLayer):
  """Micro-batched pipeline over the cells (ref :324).

  FProp splits every tensor argument along `batch_dim` into
  `num_micro_batches`, runs each micro-batch through all stages and
  concatenates the results. With a `parallel.pp.PipelineEngine` attached
  (`AttachEngine`) this rank only executes its own stage and the engine moves
  activations / gradients between ranks.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_micro_batches', 1, 'Number of micro-batches.')
    p.Define('micro_batch_size', None, 'Alternative to num_micro_batches.')
    p.Define('batch_dim', 0, 'Batch dimension of the inputs.')
    p.Define('state_dtype', None, 'Kept for parity.')
    p.Define('nested_map_fprop', False, 'Args/returns are NestedMaps.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self._engine = None

  def AttachEngine(self, engine):
    self._engine = engine

  def _CalculateOutputShapes(self, input_shapes):
    """Output shapes of every cell from `FPropMeta` (ref :339)."""
    p = self.params
    shapes = tuple(s if s is None or isinstance(s, tshape.Shape) else tshape.Shape(list(s))
                   for s in input_shapes)
    outs = []
    for tpl in p.cell_tpl:
      shapes = tpl.cls.FPropMeta(tpl, *shapes).out_shapes
      outs.append(shapes)
    return outs

  def _NumMicro(self, args):
    p = self.params
    if p.micro_batch_size:
      for a in args:
        if isinstance(a, torch.Tensor):
          return max(a.shape[p.batch_dim] // p.micro_batch_size, 1)
    return p.num_micro_batches

  def _Split(self, x, n):
    p = self.params
    if isinstance(x, torch.Tensor) and x.dim() > p.batch_dim:
      return list(x.chunk(n, p.batch_dim))
    if isinstance(x, NestedMap):
      parts = [self._Split(v, n) for v in x.Flatten()]
      return [x.Pack([pp[i] for pp in parts]) for i in range(n)]
    return [x] * n

  def _Concat(self, xs):
    p = self.params
    if isinstance(xs[0], torch.Tensor):
      return torch.cat(xs, p.batch_dim) if xs[0].dim() > 0 else torch.stack(xs).mean()
    if isinstance(xs[0], NestedMap):
      flats = [x.Flatten() for x in xs]
      return xs[0].Pack([self._Concat([f[i] for f in flats])
                         for i in range(len(flats[0]))])
    return xs[0]

  def FProp(self, theta, *args):
    args = self._RunBefore(theta, _ToTuple(args))
    n = self._NumMicro(args)
    split = [self._Split(a, n) for a in args]
    micro_in = [tuple(s[i] for s in split) for i in range(n)]
    if self._engine is not None:
      outs = self._engine.Forward(self, theta, micro_in)
    else:
      outs = []
      step0 = py_utils.GetGlobalStep()
      for i, mi in enumerate(micro_in):
        SetOverWriteGlobalStep(step0 * n + i if isinstance(step0, int) else None)
        outs.append(self._RunCells(theta, mi))
      SetOverWriteGlobalStep(None)
    merged = tuple(self._Concat([o[k] for o in outs]) for k in range(len(outs[0])))
    return merged[0] if len(merged) == 1 else merged
