"""Optimizers.

Catalogue and update rules follow reference `lingvo/core/optimizer.py`
(`Base.Apply` :99, slot checkpoint naming :170-196, `CompositeOptimizer`,
`SGD/Momentum/RMSProp/Adagrad/AdaDelta/Adam(ParamsA/B)/AdamV2`, `Accumulator`
:507, `DynamicAccumulator` :575, `DistributedShampoo` :689, `AdaGraft` :803,
`XLAShardingAdafactor` :905-1275, `GradientAggregationOptimizer` :1276).

H100-first design: an optimizer is a layer owning *slot tensors* keyed by the
variable's checkpoint name (`<var>/Adam`, `<var>/Adam_1`, …, the TF names, so
checkpoints keep the reference layout). `Apply(lr, var_grads)` updates the
Parameters in place under `no_grad`; on CUDA the dense rules run as
multi-tensor (`torch._foreach_*`) launches or as the fused sm_90a kernels in
`lingvo_b200.ops.optim` (Adam / Adafactor), and the data-parallel runtime
(`parallel/dp.py`) fuses reduce-scatter + the same Adam math over a flat shard.
"""

from __future__ import annotations

import contextlib
import math
import re
from typing import Dict, List, Optional, Tuple

import torch

from lingvo_b200 import ops
from lingvo_b200.core import base_layer
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap


def _VarKey(var) -> str:
  name = getattr(var, 'var_name', None)
  if name is None:
    name = 'var_%x' % id(var)
  return name[:-len('/var')] + '/var' if name.endswith('/var') else name


def _Pairs(var_grads) -> List[Tuple[torch.nn.Parameter, torch.Tensor]]:
  if isinstance(var_grads, NestedMap):
    leaves = [vg for vg in var_grads.Flatten()
              if isinstance(vg, py_utils.VarGrad)]
  else:
    leaves = list(var_grads)
  return [(vg.var, vg.grad) for vg in leaves if vg.grad is not None]


def GetLrValue(lr_or_callable):
  """A learning rate given as a number or as a zero-arg callable (ref :29)."""
  return lr_or_callable() if callable(lr_or_callable) else lr_or_callable


class Base(base_layer.BaseLayer):
  """Base class for all optimizers."""

  # slot name → checkpoint suffix (TF slot naming)
  SLOT_SUFFIX: Dict[str, str] = {}
  # Slot names saved under their own name (no TF alias) that must also be restored.
  EXTRA_SLOT_NAMES: tuple = ()
  # Host-side integer/float counters that are part of the optimizer state.
  COUNTER_ATTRS: tuple = ()

  @classmethod
  def Params(cls):
    p = super().Params()
    p.name = cls.__name__
    p.Define('use_bf16_gradients_ar', False,
             'Reduce gradients across replicas in bf16.')
    p.Define('skip_zero_gradients', None, 'See py_utils.SkipZeroGradients.')
    p.Define('clear_variable_scope', False, 'Kept for parity.')
    p.Define('add_summary_in_apply', True, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self._slots: Dict[str, Dict[str, torch.Tensor]] = {}
    self._scalars: Dict[str, float] = {}
    self._step_count = 0

  # ------------------------------------------------------------------ slots --
  def _Slot(self, var, name: str, init=None, shape=None, dtype=None):
    key = _VarKey(var)
    slots = self._slots.setdefault(key, {})
    if name not in slots:
      shape = list(var.shape) if shape is None else list(shape)
      dtype = dtype or (var.dtype if var.dtype.is_floating_point
                        else torch.float32)
      if init is None or init == 0:
        slots[name] = torch.zeros(shape, dtype=dtype, device=var.device)
      else:
        slots[name] = torch.full(shape, float(init), dtype=dtype,
                                 device=var.device)
    return slots[name]

  def GetOptimizerSlots(self) -> Dict[str, torch.Tensor]:
    """Checkpoint-key → slot tensor (TF names, reference :170-196)."""
    out = {}
    for key, slots in self._slots.items():
      base = key[:-len('/var')] if key.endswith('/var') else key
      for sname, t in slots.items():
        out['%s/%s' % (base, self.SLOT_SUFFIX.get(sname, sname))] = t
    for k, v in self._scalars.items():
      out[k] = torch.tensor(v, dtype=torch.float32)
    out['%s/step_count' % self.params.name] = torch.tensor(
        self._step_count, dtype=torch.int64)
    for attr in self.COUNTER_ATTRS:
      out['%s/%s' % (self.params.name, attr.strip('_'))] = torch.tensor(
          float(getattr(self, attr)), dtype=torch.float64)
    return out

  def LoadOptimizerSlots(self, tensors: Dict[str, torch.Tensor]) -> List[str]:
    """Restores slots from a checkpoint-key map; returns the keys consumed."""
    used = []
    inv = {v: k for k, v in self.SLOT_SUFFIX.items()}
    pending = {}
    for key, t in tensors.items():
      if key == '%s/step_count' % self.params.name:
        self._step_count = int(t.item())
        used.append(key)
        continue
      if key in self._scalars or key in self._ScalarNames():
        self._scalars[key] = float(t.item())
        used.append(key)
        continue
      hit = False
      for attr in self.COUNTER_ATTRS:
        if key == '%s/%s' % (self.params.name, attr.strip('_')):
          cur = getattr(self, attr)
          setattr(self, attr, type(cur)(t.item()))
          used.append(key)
          hit = True
      if hit:
        continue
      base, _, suffix = key.rpartition('/')
      sname = inv.get(suffix)
      if sname is None and suffix in self.EXTRA_SLOT_NAMES:
        sname = suffix
      if sname is None:
        continue
      pending.setdefault(base + '/var', {})[sname] = (key, t)
    for vkey, slots in pending.items():
      dst = self._slots.setdefault(vkey, {})
      for sname, (key, t) in slots.items():
        if sname in dst:
          dst[sname].copy_(t.to(dst[sname].device))
        else:
          dst[sname] = t.clone()
        used.append(key)
    return used

  def _ScalarNames(self) -> List[str]:
    return []

  def to(self, device=None, dtype=None):  # pylint: disable=invalid-name
    for slots in self._slots.values():
      for k in list(slots):
        slots[k] = slots[k].to(device)
    return self

  def GetOptimizer(self, lr):
    """The object that applies updates at learning rate `lr` (ref :116): the optimizer
    layer itself, bound to `lr` through `apply_gradients(var_grad)`."""
    outer = self

    class _Bound:
      learning_rate = lr

      @staticmethod
      def apply_gradients(var_grad, grad_scale=None):   # pylint: disable=invalid-name
        return outer.Apply(lr, var_grad, grad_scale=grad_scale)

    return _Bound()

  def GetLrScheduleValue(self, lr_schedule=None, step=None):
    """Value of a learning-rate schedule layer at the current (or given) step."""
    if lr_schedule is None:
      return 1.0
    return float(lr_schedule.Value() if step is None else lr_schedule.Value(step))

  def ApplyPostTrainingLoop(self):
    """Work an optimizer defers to the end of a device training loop (e.g. Shampoo's
    preconditioner refresh); nothing for first-order optimizers (ref :215)."""
    return None

  @staticmethod
  def VarReuseForSlotVars():
    import contextlib  # pylint: disable=g-import-not-at-top
    return contextlib.nullcontext()

  # ------------------------------------------------------------------ apply --
  def ComputeGradients(self, loss, vmap, *args, **kwargs):
    return py_utils.ComputeGradients(loss, vmap, *args, **kwargs)

  # Optimizers whose kernels fold `grad_scale` (clip / NaN-skip factor, a
  # device scalar) into the update avoid a full pass over the gradients.
  supports_grad_scale = False

  def Apply(self, lr, var_grad, grad_scale=None):
    """Applies one update with learning rate `lr` (python float or tensor)."""
    pairs = _Pairs(var_grad)
    if not pairs:
      return
    lr = float(lr) if not isinstance(lr, torch.Tensor) else lr
    variables = [v for v, _ in pairs]
    grads = [g for _, g in pairs]
    self._refreshed = set()
    with torch.no_grad():
      if grad_scale is not None:
        grad_scale = grad_scale.reshape(())     # 0-dim: never broadcasts scalar grads up
      if grad_scale is not None and not self.supports_grad_scale:
        grads = [torch.where(grad_scale == 0, torch.zeros_like(g),
                             g * grad_scale.to(g.dtype)) for g in grads]
        grad_scale = None
      self._grad_scale = grad_scale
      self._Update(lr, variables, grads)
      py_utils.RefreshComputeCopies(
          [v for v in variables if id(v) not in self._refreshed])
    self._step_count += 1

  def _Update(self, lr, variables, grads):
    raise NotImplementedError()

  def AddSummary(self, lr, optimizer, var_grad):
    from lingvo_b200.core import summary_utils
    summary_utils.scalar('%s_lr' % self.params.name.lower(), lr)

  def FProp(self, theta, *args):
    raise NotImplementedError('Optimizers are applied with Apply()')


def _ScaledF32(pairs, grad_scale):
  """fp32 (variable-dtype) gradients of `pairs`, times the optional device scalar."""
  grads = _F32([g for _, g in pairs], [v for v, _ in pairs])
  if grad_scale is None:
    return grads
  gs = grad_scale.reshape(())
  return [torch.where(gs == 0, torch.zeros_like(g), g * gs.to(g.dtype)) for g in grads]


def _F32(grads, like):
  return [g.to(v.dtype) if g.dtype != v.dtype else g
          for g, v in zip(grads, like)]


class SGD(Base):
  """w -= lr * g."""

  def _Update(self, lr, variables, grads):
    grads = _F32(grads, variables)
    torch._foreach_add_(variables, grads, alpha=-float(lr))


class Momentum(Base):
  """TF MomentumOptimizer: acc = m·acc + g; w -= lr·acc (nesterov optional)."""

  SLOT_SUFFIX = {'momentum': 'Momentum'}

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('alpha', 0.9, 'The damping factor in the momentum optimizer.')
    p.Define('use_nesterov', False, 'True iff use Nesterov')
    return p

  def _Update(self, lr, variables, grads):
    p = self.params
    grads = _F32(grads, variables)
    accs = [self._Slot(v, 'momentum') for v in variables]
    torch._foreach_mul_(accs, p.alpha)
    torch._foreach_add_(accs, grads)
    if p.use_nesterov:
      upd = torch._foreach_mul(accs, p.alpha)
      torch._foreach_add_(upd, grads)
      torch._foreach_add_(variables, upd, alpha=-float(lr))
    else:
      torch._foreach_add_(variables, accs, alpha=-float(lr))


class RMSProp(Base):
  """TF RMSPropOptimizer (optionally centered)."""

  SLOT_SUFFIX = {'rms': 'RMSProp', 'mom': 'RMSProp_1', 'mg': 'RMSProp_2'}

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('decay', 0.9, 'Discounting factor for the history.')
    p.Define('momentum', 0.9, 'Momentum in RMSProp.')
    p.Define('epsilon', 1.0, 'Epsilon term for RMSProp.')
    p.Define('centered', False, 'Normalise by the estimated variance.')
    return p

  def _Update(self, lr, variables, grads):
    p = self.params
    for v, g in zip(variables, _F32(grads, variables)):
      ms = self._Slot(v, 'rms', init=1.0)
      mom = self._Slot(v, 'mom')
      ms.mul_(p.decay).addcmul_(g, g, value=1 - p.decay)
      denom = ms
      if p.centered:
        mg = self._Slot(v, 'mg')
        mg.mul_(p.decay).add_(g, alpha=1 - p.decay)
        denom = ms - mg * mg
      mom.mul_(p.momentum).add_(g / torch.sqrt(denom + p.epsilon),
                                alpha=float(lr))
      v.sub_(mom)


class Adagrad(Base):

  SLOT_SUFFIX = {'acc': 'Adagrad'}

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('initial_accumulator_value', 1.0, 'Initial accumulator value.')
    return p

  def _Update(self, lr, variables, grads):
    p = self.params
    for v, g in zip(variables, _F32(grads, variables)):
      acc = self._Slot(v, 'acc', init=p.initial_accumulator_value)
      acc.addcmul_(g, g)
      v.addcdiv_(g, acc.sqrt(), value=-float(lr))


class AdaDelta(Base):

  SLOT_SUFFIX = {'acc': 'Adadelta', 'acc_update': 'Adadelta_1'}

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('decay', 0.95, 'Discounting factor for the history.')
    p.Define('epsilon', 1e-8, 'Epsilon term for AdaDelta.')
    return p

  def _Update(self, lr, variables, grads):
    p = self.params
    for v, g in zip(variables, _F32(grads, variables)):
      acc = self._Slot(v, 'acc')
      accu = self._Slot(v, 'acc_update')
      acc.mul_(p.decay).addcmul_(g, g, value=1 - p.decay)
      upd = torch.sqrt(accu + p.epsilon) / torch.sqrt(acc + p.epsilon) * g
      accu.mul_(p.decay).addcmul_(upd, upd, value=1 - p.decay)
      v.add_(upd, alpha=-float(lr))


class Adam(Base):
  """TF AdamOptimizer: lr_t = lr·sqrt(1-β2^t)/(1-β1^t); w -= lr_t·m/(√v+ε)."""

  SLOT_SUFFIX = {'m': 'Adam', 'v': 'Adam_1'}
  supports_grad_scale = True

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('beta1', 0.9, 'Beta1 for Adam.')
    p.Define('beta2', 0.999, 'Beta2 for Adam.')
    p.Define('epsilon', 1e-6, 'Epsilon for Adam.')
    p.Define('fused', True, 'Use the fused sm_90a multi-tensor kernel on CUDA.')
    return p

  @classmethod
  def ParamsA(cls):
    """Transformer paper (beta2 .997)."""
    return cls.Params().Set(beta1=0.9, beta2=0.997, epsilon=1e-9)

  @classmethod
  def ParamsB(cls):
    """Tensor2tensor settings."""
    return cls.Params().Set(beta1=0.9, beta2=0.98, epsilon=1e-9)

  def _ScalarNames(self):
    return ['beta1_power', 'beta2_power']

  def _Update(self, lr, variables, grads):
    p = self.params
    t = self._step_count + 1
    b1p, b2p = p.beta1**t, p.beta2**t
    self._scalars['beta1_power'] = b1p * p.beta1
    self._scalars['beta2_power'] = b2p * p.beta2
    lr_t = float(lr) * math.sqrt(1 - b2p) / (1 - b1p)
    ms = [self._Slot(v, 'm') for v in variables]
    vs = [self._Slot(v, 'v') for v in variables]
    if p.fused and ops.use_cuda_kernels(variables[0]):
      from lingvo_b200.ops import optim
      optim.multi_tensor_adam(variables, grads, ms, vs, lr_t, p.beta1,
                              p.beta2, p.epsilon,
                              grad_scale_t=self._grad_scale)
      for v in variables:
        self._refreshed.add(id(v))
      return
    if getattr(self, '_grad_scale', None) is not None:
      gs = self._grad_scale
      grads = [torch.where(gs == 0, torch.zeros_like(g), g * gs.to(g.dtype))
               for g in grads]
    grads = _F32(grads, variables)
    torch._foreach_mul_(ms, p.beta1)
    torch._foreach_add_(ms, grads, alpha=1 - p.beta1)
    torch._foreach_mul_(vs, p.beta2)
    torch._foreach_addcmul_(vs, grads, grads, value=1 - p.beta2)
    denom = torch._foreach_sqrt(vs)
    torch._foreach_add_(denom, p.epsilon)
    torch._foreach_addcdiv_(variables, ms, denom, value=-lr_t)


class AdamV2(Adam):
  """Keras-style Adam (same math; epsilon inside the bias-corrected step)."""

  SLOT_SUFFIX = {'m': 'm', 'v': 'v'}


class Accumulator(Base):
  """Accumulates grads for N steps then applies the wrapped optimizer (:507)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('optimizer_tpl', Adam.Params(), 'Params for the wrapped optimizer.')
    p.Define('accum_steps', 5, 'Number of gradient accumulation steps.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self.CreateChild('_opt', self.params.optimizer_tpl)
    self._accum_count = 0

  SLOT_SUFFIX = {'grad_accum': 'grad_accumulator'}
  COUNTER_ATTRS = ('_accum_count',)

  def Apply(self, lr, var_grad, grad_scale=None):
    p = self.params
    pairs = _Pairs(var_grad)
    with torch.no_grad():
      accs = [self._Slot(v, 'grad_accum') for v, _ in pairs]
      torch._foreach_add_(accs, _ScaledF32(pairs, grad_scale))
    self._accum_count += 1
    if self._accum_count % p.accum_steps != 0:
      return
    with torch.no_grad():
      avg = torch._foreach_div(accs, float(p.accum_steps))
    self._opt.Apply(lr, [py_utils.VarGrad(v, g)
                         for (v, _), g in zip(pairs, avg)])
    with torch.no_grad():
      torch._foreach_zero_(accs)
    self._step_count += 1

  def GetOptimizerSlots(self):
    out = super().GetOptimizerSlots()
    out.update(self._opt.GetOptimizerSlots())
    return out

  def LoadOptimizerSlots(self, tensors):
    return super().LoadOptimizerSlots(tensors) + self._opt.LoadOptimizerSlots(
        tensors)


class DynamicAccumulator(Accumulator):
  """Accumulates until `accum_weight_threshold` total weight is seen (:575)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('accum_weight_threshold', 1.0, 'Apply when weight sum ≥ this.')
    return p

  COUNTER_ATTRS = ('_accum_count', '_weight')

  def __init__(self, params):
    super().__init__(params)
    self._weight = 0.0

  def ApplyWeighted(self, lr, var_grad, weight: float, grad_scale=None):
    pairs = _Pairs(var_grad)
    with torch.no_grad():
      accs = [self._Slot(v, 'grad_accum') for v, _ in pairs]
      torch._foreach_add_(accs, _ScaledF32(pairs, grad_scale), alpha=float(weight))
    self._weight += float(weight)
    if self._weight < self.params.accum_weight_threshold:
      return
    with torch.no_grad():
      avg = torch._foreach_div(accs, self._weight)
    self._opt.Apply(lr, [py_utils.VarGrad(v, g)
                         for (v, _), g in zip(pairs, avg)])
    with torch.no_grad():
      torch._foreach_zero_(accs)
    self._weight = 0.0
    self._step_count += 1

  def Apply(self, lr, var_grad, grad_scale=None):
    self.ApplyWeighted(lr, var_grad, 1.0, grad_scale=grad_scale)


class GradientAggregation(Base):
  """Micro-batch accumulation with a *deferred* cross-replica sum (:1276).

  Grads of `num_micro_batches` consecutive Apply calls are summed locally; the
  all-reduce (via `reduce_fn`) happens once, right before the wrapped
  optimizer's apply — the H100 analogue of `GradientAggregationOptimizer`.
  """

  SLOT_SUFFIX = {'grad_accum': 'grad_accum'}
  COUNTER_ATTRS = ('_count',)

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('optimizer_tpl', Adam.Params(), 'Wrapped optimizer.')
    p.Define('num_micro_batches', 1, 'Micro batches per apply.')
    p.Define('apply_crs_to_grad', False, 'All-reduce accumulated grads.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self.CreateChild('_opt', self.params.optimizer_tpl)
    self._count = 0
    self.reduce_fn = None

  def GetOptimizerSlots(self):
    out = super().GetOptimizerSlots()
    out.update(self._opt.GetOptimizerSlots())
    return out

  def LoadOptimizerSlots(self, tensors):
    return super().LoadOptimizerSlots(tensors) + self._opt.LoadOptimizerSlots(tensors)

  def Apply(self, lr, var_grad, grad_scale=None):
    p = self.params
    pairs = _Pairs(var_grad)
    if p.num_micro_batches <= 1:
      if grad_scale is not None:
        var_grad = [py_utils.VarGrad(v, g) for (v, _), g in zip(
            pairs, _ScaledF32(pairs, grad_scale))]
      self._opt.Apply(lr, var_grad)
      return
    with torch.no_grad():
      accs = [self._Slot(v, 'grad_accum') for v, _ in pairs]
      torch._foreach_add_(accs, _ScaledF32(pairs, grad_scale))
    self._count += 1
    if self._count % p.num_micro_batches:
      return
    with torch.no_grad():
      avg = torch._foreach_div(accs, float(p.num_micro_batches))
      if p.apply_crs_to_grad and self.reduce_fn is not None:
        avg = [self.reduce_fn(g) for g in avg]
    self._opt.Apply(lr, [py_utils.VarGrad(v, g)
                         for (v, _), g in zip(pairs, avg)])
    with torch.no_grad():
      torch._foreach_zero_(accs)
    self._step_count += 1


def _ReduceRms(x):
  return torch.sqrt(torch.mean(x.float().square()))


class XLAShardingAdafactor(Base):
  """Adafactor as used by the GShard LMs (reference :905-1275).

  g² + ε1 → factored row/col EMAs (two largest dims, both ≥
  `min_dim_size_to_factor`) or full `v`; x = g·rsqrt(v̂); RMS-clip to
  `clipping_threshold`; scale by max(RMS(w), ε2)·lr; optional β1; assign_sub.
  """

  SLOT_SUFFIX = {'m': 'Adafactor_m', 'vr': 'Adafactor_vr', 'vc': 'Adafactor_vc',
                 'v': 'Adafactor_v'}
  supports_grad_scale = True

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('beta1', 0, 'Beta1 of Adam. Can be zero.')
    p.Define('beta2', 0.999, 'Beta2 of Adam.')
    p.Define('multiply_by_parameter_scale', True,
             'update_scale = max(RMS(w), eps2)·lr when True else lr.')
    p.Define('clipping_threshold', None, '≥1.0 or None for no update clipping.')
    p.Define('factored', True, 'Factor the second-moment estimator.')
    p.Define('decay_exponent_pow', None, 'decay = 1-(t-offset+1)^-pow if set.')
    p.Define('decay_exponent_offset', 0, 'Start step of the decay schedule.')
    p.Define('min_dim_size_to_factor', 128, 'Only factor dims ≥ this.')
    p.Define('cond_is_finite', False, 'Skip the update if stats are not finite.')
    p.Define('epsilon1', 1e-30, 'Regularization constant for squared gradient.')
    p.Define('epsilon2', 1e-3, 'Regularization constant for parameter scale.')
    p.Define('fused', True, 'Use the fused sm_90a kernel on CUDA.')
    p.Define('num_update_streams', 8,
             'Factored variables are spread round-robin over this many CUDA streams, so that '
             'the latency-bound kernels of small tensors overlap (also inside a captured '
             'graph, where the streams become parallel branches). ≤1: single stream.')
    p.name = 'Adafactor'
    return p

  class _Fan:
    """Fork/join helper: `with fan.On(i):` runs on side stream i % n (after everything already
    queued on the caller's stream); `Join()` makes the caller's stream wait for all of them."""

    def __init__(self, streams):
      self._streams = streams
      self._used = set()
      if streams:
        self._main = torch.cuda.current_stream(streams[0].device)
        self._fork = torch.cuda.Event()
        self._fork.record(self._main)

    def On(self, i):
      if not self._streams:
        return contextlib.nullcontext()
      k = i % len(self._streams)
      s = self._streams[k]
      if k not in self._used:
        s.wait_event(self._fork)
        self._used.add(k)
      return torch.cuda.stream(s)

    def Slot(self, i):
      return 1 + i % len(self._streams) if self._streams else 0

    def Join(self):
      for k in sorted(self._used):
        self._main.wait_stream(self._streams[k])
      self._used.clear()

  def _UpdateFan(self, device):
    n = int(self.params.num_update_streams or 0)
    if n <= 1 or device.type != 'cuda':
      return self._Fan([])
    if getattr(self, '_side_streams', None) is None:
      self._side_streams = [torch.cuda.Stream(device=device) for _ in range(n)]
    return self._Fan(self._side_streams)

  def _FactoredDims(self, shape):
    p = self.params
    if not p.factored or len(shape) < 2:
      return None
    order = sorted(((s, i) for i, s in enumerate(shape)), key=lambda d: -d[0])
    if order[1][0] < p.min_dim_size_to_factor:
      return None
    return order[0][1], order[1][1]

  def DecayRate(self, step: Optional[int] = None) -> float:
    p = self.params
    t = float(py_utils.GetGlobalStep() if step is None else step)
    if p.decay_exponent_pow:
      return 1.0 - (t - p.decay_exponent_offset + 1.0)**(-p.decay_exponent_pow)
    t = t + 1.0
    return p.beta2 * (1.0 - p.beta2**(t - 1.0)) / (1.0 - p.beta2**t)

  def _FusedModule(self, var):
    if self.params.fused and ops.use_cuda_kernels(var):
      from lingvo_b200.ops import optim
      return optim
    return None

  def _FusedEligible(self, var, dims):
    p = self.params
    return (dims is not None and var.dim() >= 2 and not p.beta1 and not p.cond_is_finite and
            sorted(dims) == [var.dim() - 2, var.dim() - 1] and var.shape[-1] % 8 == 0 and
            var.is_contiguous())

  def _SlotIndex(self, idx, device):
    """Device index tensor of `idx`, built once per variable set: the first (eager) steps
    create it, so a captured step never copies it from the host."""
    cache = self.__dict__.setdefault('_slot_index_cache', {})
    key = (tuple(idx), str(device))
    if key not in cache:
      cache[key] = torch.tensor(idx, dtype=torch.long, device=device)
    return cache[key]

  def PreGradStats(self, var_grad_pairs):
    """Phase A of the fused step for every eligible variable. The same pass that builds the
    factored second-moment sums also yields Σg² — the learner gets the global gradient
    norm without a separate sweep over the gradients.

    Returns (device scalar Σg² over the handled variables, set of handled var ids)."""
    p = self.params
    self._pre = {}
    fused = self._FusedModule(var_grad_pairs[0][0]) if var_grad_pairs else None
    if fused is None:
      return None, set()
    total = torch.zeros(1, dtype=torch.float32, device=var_grad_pairs[0][0].device)
    # Expert-parallel variables differ across ranks: their Σg² is accumulated separately so
    # that the learner can all-reduce just that scalar for the true global norm.
    total_ep = torch.zeros(1, dtype=torch.float32, device=total.device)
    any_ep = False
    handled = set()
    small = []
    self._pre_var_sumsq = None
    self._pre_ep_sumsq = None
    fan = self._UpdateFan(total.device)
    # One Σg² slot per variable (the stats kernels of different side streams never share an
    # accumulator), summed below in variable order: the norm is the same on every run.
    parts = torch.zeros(len(var_grad_pairs), dtype=torch.float32, device=total.device)
    dense_idx, ep_idx = [], []
    for k, (var, grad) in enumerate(var_grad_pairs):
      dims = self._FactoredDims(list(var.shape))
      if grad.device == var.device and self._SmallEligible(var, grad, dims):
        small.append((var, grad))
        continue
      if not self._FusedEligible(var, dims) or grad.device != var.device:
        continue
      is_ep = bool(getattr(var, 'expert_parallel', False))
      any_ep = any_ep or is_ep
      with fan.On(len(handled)):
        fresh = fused.adafactor_stats(var, grad, dims[0], dims[1],
                                      bool(p.multiply_by_parameter_scale),
                                      parts[k:k + 1], fan.Slot(len(handled)))
      (ep_idx if is_ep else dense_idx).append(k)
      self._pre[id(var)] = (grad.data_ptr(), fresh)
      handled.add(id(var))
    fan.Join()
    if dense_idx:
      total = total + parts.index_select(0, self._SlotIndex(dense_idx, parts.device)).sum().reshape(1)
    if ep_idx:
      total_ep = total_ep + parts.index_select(0, self._SlotIndex(ep_idx, parts.device)).sum().reshape(1)
    if any_ep:
      self._pre_ep_sumsq = total_ep
    if small:
      # all small variables: Σg² and Σw² with one launch (instead of one reduction each)
      acc = torch.zeros(2, dtype=torch.float32, device=total.device)
      self._UpdateSmallFused(fused, 0.0, 0.0, small, sumsq_out=acc)
      total = total + acc[0:1]
      ids = {id(v) for v, _ in small}
      handled |= ids
      self._pre_var_sumsq = (acc[1:2], ids)
    return total, handled

  # -- device-resident hyper-parameters (CUDA-graph capture) ------------------------
  graph_capturable = True

  def EnableDeviceHyper(self, device):
    """After this, the fused kernels read (lr, decay) from a device tensor that
    `SetHyper` refreshes before every (graph) step; nothing step-dependent is baked
    into a kernel argument."""
    self._hyper = torch.zeros(2, dtype=torch.float32, device=device)
    self._hyper_host = torch.zeros(2, dtype=torch.float32).pin_memory()

  def SetHyper(self, lr, step=None):
    self._hyper_host[0] = float(lr)
    self._hyper_host[1] = self.DecayRate(step)
    self._hyper.copy_(self._hyper_host, non_blocking=True)

  def _SmallEligible(self, var, grad, dims):
    p = self.params
    return (dims is None and not p.beta1 and not p.cond_is_finite and var.is_contiguous() and
            grad.dtype in (torch.float32, torch.bfloat16) and var.dtype == torch.float32)

  def _UpdateSmallFused(self, fused, lr, decay, small, sumsq_out=None):
    """All non-factored variables in one multi-tensor launch (`sumsq_out`: only reduce
    Σg² / Σw² into it — the pre-pass that feeds global gradient clipping)."""
    p = self.params
    rows = []
    for var, grad in small:
      v = self._Slot(var, 'v')
      g = grad if grad.is_contiguous() else grad.contiguous()
      compute = getattr(var, 'compute', None)
      rows.append((var.data.data_ptr(), g.data_ptr(), v.data_ptr(),
                   compute.data.data_ptr() if compute is not None else 0, var.numel(),
                   1 if g.dtype == torch.bfloat16 else 0))
      self._small_keepalive = getattr(self, '_small_keepalive', [])
      self._small_keepalive.append(g)
      if compute is not None and sumsq_out is None:
        self._refreshed.add(id(var))
    if getattr(self, '_small_table', None) is None:
      self._small_table = fused.SmallVarTable(small[0][0].device)
    table = self._small_table.Build(rows)
    if sumsq_out is not None:
      fused.small_sumsq(table, sumsq_out)
      return
    fused.adafactor_small(table, lr, decay, p.epsilon1, p.epsilon2,
                          p.clipping_threshold or 0.0, bool(p.multiply_by_parameter_scale),
                          self._grad_scale, getattr(self, '_hyper', None))
    self._small_keepalive = self._small_keepalive[-2 * len(small):]

  def _Update(self, lr, variables, grads):
    p = self.params
    decay = self.DecayRate()
    fused = self._FusedModule(variables[0])
    hyper = getattr(self, '_hyper', None)
    pre = getattr(self, '_pre', {})
    self._pre = {}
    small = []
    factored = []
    for var, grad in zip(variables, grads):
      dims = self._FactoredDims(list(var.shape))
      if fused is not None and self._SmallEligible(var, grad, dims):
        small.append((var, grad))
        continue
      if fused is not None and self._FusedEligible(var, dims):
        d0, d1 = dims
        vr_shape = [s for i, s in enumerate(var.shape) if i != d0]
        vc_shape = [s for i, s in enumerate(var.shape) if i != d1]
        # Slots are created (zero-filled) here, on the caller's stream, *before* the side
        # streams fork: anything enqueued after the fork would race with them.
        factored.append((var, grad, d0, d1, self._Slot(var, 'vr', shape=vr_shape),
                         self._Slot(var, 'vc', shape=vc_shape)))
        continue
      if self._grad_scale is not None:
        gs = self._grad_scale
        grad = torch.where(gs == 0, torch.zeros_like(grad),
                           grad * gs.to(grad.dtype))
      self._UpdateOne(var, grad, dims, float(lr), decay)
    fan = self._UpdateFan(variables[0].device) if factored else None
    for i, (var, grad, d0, d1, vr, vc) in enumerate(factored):
      done = pre.get(id(var))
      with fan.On(i):
        if done is not None and done[0] == grad.data_ptr():
          fresh = done[1]                       # statistics already in the scratch
        else:
          fresh = fused.adafactor_stats(var, grad, d0, d1, bool(p.multiply_by_parameter_scale),
                                        None, fan.Slot(i))
        fused.adafactor_update(var, grad, vr, vc, d0, d1, float(lr), decay, p.epsilon1,
                               p.epsilon2, p.clipping_threshold or 0.0,
                               bool(p.multiply_by_parameter_scale), self._grad_scale, fresh,
                               hyper)
      if getattr(var, 'compute', None) is not None:
        self._refreshed.add(id(var))
    if fan is not None:
      fan.Join()
    if small:
      self._UpdateSmallFused(fused, float(lr), decay, small)

  def _UpdateOne(self, var, grad, dims, lr, decay):
    p = self.params
    g = grad.to(var.dtype)
    g2 = g * g + p.epsilon1
    mix = 1.0 - decay
    if p.multiply_by_parameter_scale:
      update_scale = torch.clamp(_ReduceRms(var), min=p.epsilon2) * lr
    else:
      update_scale = lr
    finite = True
    new_slots = {}
    if dims is not None:
      d0, d1 = dims
      vr_shape = [s for i, s in enumerate(var.shape) if i != d0]
      vc_shape = [s for i, s in enumerate(var.shape) if i != d1]
      vr = self._Slot(var, 'vr', shape=vr_shape)
      vc = self._Slot(var, 'vc', shape=vc_shape)
      new_vr = vr * decay + g2.mean(dim=d0) * mix
      new_vc = vc * decay + g2.mean(dim=d1) * mix
      new_slots = {'vr': (vr, new_vr), 'vc': (vc, new_vc)}
      long_term_mean = new_vr.mean(dim=-1, keepdim=True)
      r_factor = torch.rsqrt(new_vr / long_term_mean)
      c_factor = torch.rsqrt(new_vc)
      x = g * r_factor.unsqueeze(d0) * c_factor.unsqueeze(d1)
    else:
      v = self._Slot(var, 'v')
      new_v = v * decay + g2 * mix
      new_slots = {'v': (v, new_v)}
      x = g * torch.rsqrt(new_v)
    if p.clipping_threshold is not None:
      x = x / torch.clamp(_ReduceRms(x) / p.clipping_threshold, min=1.0)
    sub = x * update_scale
    if p.beta1:
      m = self._Slot(var, 'm')
      new_m = m * p.beta1 + sub * (1.0 - p.beta1)
      new_slots['m'] = (m, new_m)
      sub = new_m
    if p.cond_is_finite:
      finite = bool(torch.isfinite(sub).all()) and all(
          bool(torch.isfinite(n).all()) for _, n in new_slots.values())
    if finite:
      for old, new in new_slots.values():
        old.copy_(new)
      var.sub_(sub.to(var.dtype))


Adafactor = XLAShardingAdafactor


class XLAShardingAdafactorOptimizer(torch.optim.Optimizer):
  """The same Adafactor as a plain `torch.optim.Optimizer` (ref :905, the raw optimizer the
  `XLAShardingAdafactor` layer wraps): for code that drives its own training loop.
  `learning_rate` / `decay_rate` may be numbers or zero-arg callables evaluated every step.
  Runs the fused sm_90a kernels on CUDA parameters, the eager formulation elsewhere."""

  def __init__(self, params, multiply_by_parameter_scale=True, learning_rate=None,
               decay_rate=None, beta1=0.0, clipping_threshold=1.0, factored=True,
               epsilon1=1e-30, epsilon2=1e-3, min_dim_size_to_factor=128, use_locking=False,
               cond_is_finite=False, name='Adafactor'):
    del use_locking
    assert learning_rate is not None and decay_rate is not None
    super().__init__(list(params), dict(name=name))
    self._learning_rate, self._decay_rate = learning_rate, decay_rate
    decay_of = self

    class _Impl(XLAShardingAdafactor):
      def DecayRate(self, step=None):   # pylint: disable=invalid-name
        return float(GetLrValue(decay_of._decay_rate))   # pylint: disable=protected-access

    self._impl = _Impl.Params().Set(
        name=name, beta1=beta1, multiply_by_parameter_scale=multiply_by_parameter_scale,
        clipping_threshold=clipping_threshold, factored=factored, epsilon1=epsilon1,
        epsilon2=epsilon2, min_dim_size_to_factor=min_dim_size_to_factor,
        cond_is_finite=cond_is_finite).Instantiate()

  def slots(self):   # pylint: disable=invalid-name
    return self._impl._slots   # pylint: disable=protected-access

  @torch.no_grad()
  def step(self, closure=None):   # pylint: disable=invalid-name
    loss = None
    if closure is not None:
      with torch.enable_grad():
        loss = closure()
    pairs = [py_utils.VarGrad(p, p.grad) for g in self.param_groups for p in g['params']
             if p.grad is not None]
    self._impl.Apply(float(GetLrValue(self._learning_rate)), pairs)
    return loss


class XLAShardingAdafactorAccuGrad(XLAShardingAdafactor):
  """Adafactor + N-step gradient accumulation in slots (reference :1300)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_micro_batches', 1, 'Accumulate this many applies.')
    return p

  SLOT_SUFFIX = dict(XLAShardingAdafactor.SLOT_SUFFIX, grad_accum='grad_accum')
  COUNTER_ATTRS = ('_count',)

  def __init__(self, params):
    super().__init__(params)
    self._count = 0

  def PreGradStats(self, *args, **kwargs):
    """Micro-batch gradients are not the gradients the update sees: no fused pre-pass."""
    if self.params.num_micro_batches <= 1:
      return super().PreGradStats(*args, **kwargs)
    return None, set()

  def Apply(self, lr, var_grad, grad_scale=None):
    n = self.params.num_micro_batches
    if n <= 1:
      return super().Apply(lr, var_grad, grad_scale=grad_scale)
    pairs = _Pairs(var_grad)
    with torch.no_grad():
      accs = [self._Slot(v, 'grad_accum') for v, _ in pairs]
      # The clip / NaN-skip factor applies to *this* micro-batch's gradients.
      torch._foreach_add_(accs, _ScaledF32(pairs, grad_scale))
    self._count += 1
    if self._count % n:
      return None
    with torch.no_grad():
      avg = torch._foreach_div(accs, float(n))
    super().Apply(lr, [py_utils.VarGrad(v, g)
                       for (v, _), g in zip(pairs, avg)])
    with torch.no_grad():
      torch._foreach_zero_(accs)
    return None


class CompositeOptimizer(Base):
  """regex → (optimizer, lr) dispatch (reference CompositeOptimizer)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('optimizer_map', None,
             'Dict regex → (optimizer params, learning rate). Must contain '
             '"default_optimizer".')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.optimizer_map and 'default_optimizer' in p.optimizer_map
    self._regex = []
    subs = []
    for i, (regex, (opt_p, lr)) in enumerate(p.optimizer_map.items()):
      subs.append(opt_p.Copy().Set(name='%s_%d' % (opt_p.name or 'opt', i)))
      self._regex.append((regex, i, lr))
    self.CreateChildren('_opts', subs)

  def Apply(self, lr, var_grad):
    pairs = _Pairs(var_grad)
    buckets: Dict[int, List] = {}
    default_idx = [i for r, i, _ in self._regex if r == 'default_optimizer'][0]
    for v, g in pairs:
      name = getattr(v, 'var_name', '')
      hits = [i for r, i, _ in self._regex
              if r != 'default_optimizer' and re.match(r, name)]
      if len(hits) > 1:
        raise Exception('Variable {} is matched {} times by regex {}'.format(
            name, len(hits), [r for r, _, _ in self._regex]))
      idx = hits[0] if hits else default_idx
      buckets.setdefault(idx, []).append(py_utils.VarGrad(v, g))
    for idx, vgs in buckets.items():
      sub_lr = [l for _, i, l in self._regex if i == idx][0]
      sub_lr = sub_lr if sub_lr is not None else lr
      if hasattr(sub_lr, 'Value'):
        sub_lr = sub_lr.Value()
      self._opts[idx].Apply(sub_lr, vgs)
    self._step_count += 1

  def GetOptimizerSlots(self):
    out = {}
    for o in self._opts:
      out.update(o.GetOptimizerSlots())
    return out

  def LoadOptimizerSlots(self, tensors):
    used = []
    for o in self._opts:
      used += o.LoadOptimizerSlots(tensors)
    return used


# Shampoo and AdaGraft live in their own modules (as in the reference) and import this one;
# `optimizer.DistributedShampoo` / `optimizer.AdaGraft` resolve lazily (PEP 562) so either
# import order works.
def __getattr__(name):
  if name in ('AdaGraft', 'AdaGraftOptimizer'):
    from lingvo_b200.core import adagraft  # pylint: disable=g-import-not-at-top
    return getattr(adagraft, name)
  if name == 'DistributedShampoo':
    from lingvo_b200.core import distributed_shampoo  # pylint: disable=g-import-not-at-top
    return distributed_shampoo.DistributedShampoo
  raise AttributeError('module %r has no attribute %r' % (__name__, name))
