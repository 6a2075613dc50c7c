"""`Learner`: loss → gradients → adjust/clip/skip → optimizer.

Contract per reference `lingvo/core/learner.py` (`Apply` :177-239,
`_ComputeLossesAndGradients` :268-351, `AdjustGradients`/`ScaleGradients`
:353-500 — L1/L2 via gradient adjust, global-norm clip, clip-to-zero,
NaN/Inf ⇒ grad_scale = 0 step skip — and eval metrics :170-175, :462-495).

H100-first: gradients come from autograd. When the task's data-parallel
engine (`parallel/dp.py`) owns the variables, the engine's bucketed
reduce-scatter / fused scale+Adam path is invoked through
`self.grad_sync`, and the scalar bookkeeping (norms, NaN check) is done on
device without host syncs except for the returned metrics.
"""

from __future__ import annotations

import re
from typing import Dict, Optional, Tuple

import torch

from lingvo_b200.core import base_layer
from lingvo_b200.core import optimizer
from lingvo_b200.core import fault_injection
from lingvo_b200.core import py_utils
from lingvo_b200.core import schedule
from lingvo_b200.core import summary_utils
from lingvo_b200.core.nested_map import NestedMap


def _EpAllReduce(t):
  """Sums a small device tensor over the expert-parallel group (no-op without EP)."""
  import torch.distributed as dist  # pylint: disable=g-import-not-at-top
  if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
    return t
  from lingvo_b200.parallel import mesh as mesh_lib  # pylint: disable=g-import-not-at-top
  ctx = mesh_lib.Get()
  engines = list(getattr(ctx, '_ep_engines', {}).values())
  if not engines:
    return t
  t = t.clone()
  dist.all_reduce(t, group=engines[0].group)
  return t


class Learner(base_layer.BaseLayer):
  """Optimizes one (or a combination of) loss(es) over a set of variables."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('l2_regularizer_weight', None, 'L2 regularization weight or None.')
    p.Define('loss_name', None,
             'Name(s) of the loss(es) to optimize; defaults to learner name.')
    p.Define('gradient_combiner', None,
             'GradientCombiner params for multi-loss learners.')
    p.Define('l1_regularizer_weight', None, 'L1 regularization weight or None.')
    p.Define('learning_rate', 0.0, 'Learning rate to use.')
    p.Define('clip_gradient_norm_to_value', 0.0,
             'Clip gradients by global norm to this value (0 = off).')
    p.Define('clip_gradient_single_norm_to_value', 0.0,
             'Clip each gradient tensor norm to this value (0 = off).')
    p.Define('grad_norm_to_clip_to_zero', 0.0,
             'Zero all gradients if the global norm exceeds this value.')
    p.Define('grad_norm_tracker', None, 'Params for GradNormTracker.')
    p.Define('optimizer', optimizer.Adam.Params(), 'Params for the optimizer.')
    p.Define('lr_schedule', schedule.ContinuousSchedule.Params(),
             'Learning rate decay schedule.')
    p.Define('bprop_variable_filter', None,
             'Only backprop variables whose names match (re.search).')
    p.Define('bprop_variable_exclusion', None,
             'Do not backprop variables whose names match (re.search).')
    p.Define('grad_aggregation_method', None, 'Kept for parity.')
    p.Define('gate_gradients', False, 'Kept for parity.')
    p.Define('colocate_gradients_with_ops', True, 'Kept for parity.')
    p.Define('skip_zero_gradients', None, 'None|"variable"|"weight".')
    p.Define('scale_gradients', True,
             'Whether to apply gradient adjustment and scaling.')
    p.Define('learner_use_variable_scope', True, 'Kept for ckpt compat.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self._var_grads = None
    self._eval_metrics: Dict[str, Tuple[torch.Tensor, torch.Tensor]] = {}
    if p.grad_norm_tracker:
      self.CreateChild('grad_norm_tracker', p.grad_norm_tracker)
    self.CreateChild('lr_schedule', p.lr_schedule)
    self.CreateChild('optimizer', p.optimizer)
    if isinstance(p.loss_name, (list, tuple)):
      assert p.gradient_combiner
      self.CreateChild('gradient_combiner', p.gradient_combiner)
    else:
      assert p.gradient_combiner is None
    # Optional hook installed by the data-parallel engine: fn(var_grads)->var_grads
    self.grad_sync = None

  def GetVarGrads(self):
    return self._var_grads

  def GetTrainableVariables(self, vmap: NestedMap) -> NestedMap:
    p = self.params
    return py_utils.GetTrainableVariables(p.name, p.bprop_variable_filter,
                                          p.bprop_variable_exclusion, vmap)

  def LearningRate(self) -> float:
    p = self.params
    return float(p.learning_rate) * float(self.lr_schedule.Value())

  def ApplyPostTrainingLoop(self):
    """Forwards the end-of-loop hook to the optimizer (ref :216)."""
    return self.optimizer.ApplyPostTrainingLoop()

  def ComputeLosses(self, metrics):
    """The loss tensor(s) named by `loss_name` (default: the learner's name), in order
    (ref :283)."""
    p = self.params
    names = p.loss_name or p.name
    names = [names] if not isinstance(names, (list, tuple)) else list(names)
    out = []
    for name in names:
      item = metrics.get(name, None)
      if item is None:
        raise ValueError('Loss %s not found in metrics %s' % (name, list(metrics.keys())))
      out.append(item[0] if isinstance(item, (tuple, list)) else item)
    return out

  # ------------------------------------------------------------------ apply --
  def Apply(self, metrics, vmap: NestedMap, gradient_mask=None,
            gradient_adjuster=None, retain_graph=False):
    """Computes updates on `vmap` to optimize the loss(es) in `metrics`.

    Returns (losses, eval_metrics). Variables are updated in place.
    """
    p = self.params
    losses, var_grads, eval_metrics = self._ComputeLossesAndGradients(
        metrics, vmap, retain_graph=retain_graph)
    fused_update = getattr(self, 'fused_update', None)
    if fused_update is not None:
      # ZeRO path: reduce-scatter + clip + Adam on the master shard + all-gather of the
      # new bf16 weights happen inside the engine (parallel/zero.py); nothing else to do.
      lr = self.LearningRate()
      gnorm = fused_update.Apply(lr, var_grads,
                                 clip_norm=float(p.clip_gradient_norm_to_value or 0.0))
      eval_metrics['grad_norm/all'] = (gnorm.reshape(()).float(), torch.tensor(1.0))
      self._AddScalar(eval_metrics, 'learning_rate', lr)
      self._var_grads = var_grads
      return losses, {self._Key(k): v for k, v in eval_metrics.items()}
    if self.grad_sync is not None:
      var_grads = self.grad_sync(var_grads)
    if 'tpu_embedding_var_grads' in var_grads:
      del var_grads['tpu_embedding_var_grads']
    defer = (self.optimizer.supports_grad_scale and
             not p.clip_gradient_single_norm_to_value)
    self._deferred_scale = None
    var_grads, stats = self.AdjustGradients(
        var_grads, gradient_mask=gradient_mask,
        gradient_adjuster=gradient_adjuster, defer_scale=defer)
    eval_metrics.update(stats)
    self._var_grads = var_grads
    lr = self.LearningRate()
    self._AddScalar(eval_metrics, 'learning_rate', lr)
    self._AddScalar(eval_metrics, 'lr_schedule', float(self.lr_schedule.Value()))
    if self._deferred_scale is not None:
      self.optimizer.Apply(lr, var_grads, grad_scale=self._deferred_scale)
    else:
      self.optimizer.Apply(lr, var_grads)
    return losses, {self._Key(k): v for k, v in eval_metrics.items()}

  def _Key(self, name: str) -> str:
    return '%s/%s' % (name, self.params.name)

  @staticmethod
  def _AddScalar(metrics, name, value):
    metrics[name] = (torch.as_tensor(value, dtype=torch.float32),
                     torch.tensor(1.0))

  def _ComputeLossesAndGradients(self, metrics, vmap, retain_graph=False):
    p = self.params
    vmap = self.GetTrainableVariables(vmap)
    for v in vmap.Flatten():
      if not v.dtype.is_floating_point and not v.dtype.is_complex:
        raise ValueError('Cannot differentiate non-float variable %s' %
                         getattr(v, 'var_name', v))
    loss_names = p.loss_name or p.name
    single = not isinstance(loss_names, (list, tuple))
    names = [loss_names] if single else list(loss_names)
    losses, per_loss = [], {}
    eval_metrics = {}
    for i, name in enumerate(names):
      item = metrics.get(name, None)
      if item is None:
        raise ValueError('Loss %s not found in metrics %s' %
                         (name, list(metrics.keys())))
      loss = item[0] if isinstance(item, (tuple, list)) else item
      injector = fault_injection.Get()
      if injector is not None:
        loss = injector.OnLoss(py_utils.GetGlobalStep(), loss)
      losses.append(loss)
      keep = retain_graph or i < len(names) - 1
      per_loss[name] = NestedMap(
          loss_metric=item,
          grads=self.optimizer.ComputeGradients(
              loss, vmap, skip_zero_gradients=p.skip_zero_gradients,
              retain_graph=keep))
    if single:
      var_grads = per_loss[names[0]].grads
    else:
      var_grads, eval_metrics = self.gradient_combiner.Combine(vmap, per_loss)
    injector = fault_injection.Get()
    if injector is not None:
      var_grads = injector.OnGradients(py_utils.GetGlobalStep(), var_grads)
    return losses, var_grads, eval_metrics

  # ------------------------------------------------------- adjust and scale --
  def AdjustGradients(self, var_grads: NestedMap, gradient_mask=None,
                      gradient_adjuster=None, defer_scale=False):
    """L2/L1 adjust → mask → scale(clip / zero / NaN-skip) (:353-432)."""
    p = self.params
    stats = {}
    if p.l2_regularizer_weight is not None:
      l2_loss, var_grads = py_utils.AdjustGradientsWithLpLoss(
          var_grads, p.l2_regularizer_weight, p=2.0)
      self._AddScalar(stats, 'l2_loss', l2_loss)
    if p.l1_regularizer_weight is not None:
      l1_loss, var_grads = py_utils.AdjustGradientsWithLpLoss(
          var_grads, p.l1_regularizer_weight, p=1.0)
      self._AddScalar(stats, 'l1_loss', l1_loss)
    if gradient_mask:
      def mask(vg):
        m = gradient_mask.get(getattr(vg.var, 'var_name', None))
        if m is None:
          return vg
        return py_utils.VarGrad(vg.var, vg.grad * m.to(vg.grad.dtype))
      var_grads = var_grads.Transform(
          lambda vg: mask(vg) if isinstance(vg, py_utils.VarGrad) else vg)
    if p.scale_gradients:
      scaled = self.ScaleGradients(var_grads, gradient_adjuster,
                                   defer_scale=defer_scale)
      var_grads = scaled.final_var_grads
      stats.update(scaled.stats)
    return var_grads, stats

  def ScaleGradients(self, var_grads: NestedMap, gradient_adjuster=None,
                     defer_scale=False):
    """Returns NestedMap(final_var_grads, grad_scale, stats) (:395-500)."""
    p = self.params
    leaves = [vg for vg in var_grads.Flatten()
              if isinstance(vg, py_utils.VarGrad)]
    dev = leaves[0].grad.device if leaves else torch.device('cpu')
    stats = {}
    # Optimizers with a fused two-phase step hand back Σg² of the variables they own as a
    # by-product of their statistics pass; only the remaining gradients are reduced here.
    pre_sumsq, handled = None, set()
    pre_fn = getattr(self.optimizer, 'PreGradStats', None)
    is_ep = lambda v: bool(getattr(v, 'expert_parallel', False))
    is_tp = lambda v: getattr(v, 'tp_shard', None) is not None
    has_tp = any(is_tp(vg.var) for vg in leaves)
    if (pre_fn is not None and defer_scale and gradient_adjuster is None and
        dev.type == 'cuda' and not has_tp):
      pre_sumsq, handled = pre_fn([(vg.var, vg.grad) for vg in leaves])
    # Tensor-parallel shards: every TP rank holds a different slice, so their Σg² is summed
    # over the TP group (replicated variables carry identical gradients on all TP ranks).
    tp_leaves = [vg for vg in leaves if is_tp(vg.var)]
    tp_sumsq = None
    if tp_leaves:
      from lingvo_b200.parallel import mesh as mesh_lib   # pylint: disable=g-import-not-at-top
      from lingvo_b200.parallel import tp_layers   # pylint: disable=g-import-not-at-top
      handled = set(handled) | {id(vg.var) for vg in tp_leaves}
      tp_sumsq = tp_layers.AllReduceScalar(
          py_utils.SumSquared([vg.grad for vg in tp_leaves]).to(dev).reshape(1),
          mesh_lib.TensorParallel())
    rest = [vg.grad for vg in leaves if id(vg.var) not in handled and not is_ep(vg.var)]
    rest_ep = [vg.grad for vg in leaves if id(vg.var) not in handled and is_ep(vg.var)]
    grad_sumsq = py_utils.SumSquared(rest).to(dev) if rest else torch.zeros((), device=dev)
    if pre_sumsq is not None:
      grad_sumsq = grad_sumsq + pre_sumsq.reshape(())
    if tp_sumsq is not None:
      grad_sumsq = grad_sumsq + tp_sumsq.reshape(())
    # Σg² of expert-parallel variables: every rank holds different experts, so the global
    # norm needs the sum over the EP group (one 4-byte all-reduce).
    ep_sumsq = getattr(self.optimizer, '_pre_ep_sumsq', None) if pre_sumsq is not None else None
    if rest_ep:
      extra = py_utils.SumSquared(rest_ep).to(dev).reshape(1)
      ep_sumsq = extra if ep_sumsq is None else ep_sumsq + extra
    if ep_sumsq is not None:
      ep_sumsq = _EpAllReduce(ep_sumsq)
      grad_sumsq = grad_sumsq + ep_sumsq.reshape(())
    all_grad_norm = torch.sqrt(grad_sumsq)
    # Σw²: variables stepped by the fused Adafactor carry it from their last update
    # (no extra pass over the fp32 masters); the rest are reduced directly.
    carried, direct = [], []
    if dev.type == 'cuda':
      from lingvo_b200.ops import optim as fused_optim  # pylint: disable=g-import-not-at-top
      pre_w = getattr(self.optimizer, '_pre_var_sumsq', None) if pre_sumsq is not None else None
      if pre_w is not None:
        carried.append(pre_w[0])
      for vg in leaves:
        if pre_w is not None and id(vg.var) in pre_w[1]:
          continue
        c = fused_optim.carried_sumsq(vg.var)
        (carried if c is not None else direct).append(c if c is not None else vg.var.detach())
    else:
      direct = [vg.var.detach() for vg in leaves]
    var_sumsq = py_utils.SumSquared(direct).to(dev) if direct else torch.zeros((), device=dev)
    if carried:
      var_sumsq = var_sumsq + torch.cat(carried).sum()
    all_var_norm = torch.sqrt(var_sumsq)
    self._AddScalar(stats, 'grad_norm/all', all_grad_norm)
    self._AddScalar(stats, 'var_norm/all', all_var_norm)
    grad_norm_is_nan_or_inf = ~torch.isfinite(all_grad_norm)
    # An Inf/NaN entry always surfaces in the global norm, so one reduction
    # replaces the reference's separate per-tensor check.
    has_nan_or_inf = grad_norm_is_nan_or_inf
    self._AddScalar(stats, 'has_nan_or_inf', has_nan_or_inf.float())
    self._AddScalar(stats, 'grad_norm_is_nan_or_inf',
                    grad_norm_is_nan_or_inf.float())
    grad_scale = torch.ones((), device=dev)
    if p.clip_gradient_norm_to_value:
      assert not p.clip_gradient_single_norm_to_value
      grad_scale = torch.clamp(
          p.clip_gradient_norm_to_value / all_grad_norm, max=1.0)
    if self.params.grad_norm_tracker:
      grad_scale = grad_scale * self.grad_norm_tracker.FPropDefaultTheta(
          all_grad_norm, has_nan_or_inf)
    if p.grad_norm_to_clip_to_zero:
      grad_scale = torch.where(all_grad_norm > p.grad_norm_to_clip_to_zero,
                               torch.zeros_like(grad_scale), grad_scale)
    grad_scale = torch.where(has_nan_or_inf, torch.zeros_like(grad_scale),
                             grad_scale)
    self._AddScalar(stats, 'grad_scale_all', grad_scale)

    if gradient_adjuster is not None:
      var_grads = gradient_adjuster(var_grads)

    if p.clip_gradient_single_norm_to_value:
      final = py_utils.ApplyGradNormClipping(
          var_grads, p.clip_gradient_single_norm_to_value)
      bad = has_nan_or_inf

      def zero_bad(vg):
        if not isinstance(vg, py_utils.VarGrad):
          return vg
        return py_utils.VarGrad(vg.var, torch.where(
            bad, torch.zeros_like(vg.grad), vg.grad))
      final = final.Transform(zero_bad)
    elif defer_scale:
      # The optimizer kernels fold grad_scale (0 ⇒ skip) into the update.
      self._deferred_scale = grad_scale.float().reshape(1)
      final = var_grads
    else:
      def scale(vg):
        if not isinstance(vg, py_utils.VarGrad):
          return vg
        s = grad_scale.to(vg.grad.dtype)
        # where() instead of mul so NaN·0 cannot leak through.
        g = torch.where(s == 0, torch.zeros_like(vg.grad), vg.grad * s)
        return py_utils.VarGrad(vg.var, g)
      final = var_grads.Transform(scale)
    return NestedMap(final_var_grads=final, grad_scale=grad_scale, stats=stats)


def ExtractLearnerFromLegacyParams(tp, cls=Learner):
  """Builds Learner params from `task.train` legacy knobs (reference :526)."""
  lp = cls.Params()
  lp.name = 'loss'
  for k, v in tp.IterParams():
    if k not in lp:
      continue
    if k in ('name', 'cls', 'dtype', 'fprop_dtype', 'random_seed', 'vn',
             'params_init', 'is_inference', 'inference_driver_name',
             'skip_lp_regularization', 'device_mesh',
             'weight_split_dims_mapping', 'activation_split_dims_mapping'):
      continue
    lp.Set(**{k: v.Copy() if hasattr(v, 'Copy') else v})
  return lp
