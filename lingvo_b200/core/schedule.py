"""Learning-rate (and other step-driven) schedules.

Same catalogue and formulas as reference `lingvo/core/schedule.py` (:25-998):
every schedule is a layer with `Value(step=None) -> float`.

H100-first difference: the global step lives on the host, so a schedule value
is a *python float* computed with `math` — no device op, no sync. The value is
handed to the fused optimizer kernels as a scalar argument.
"""

from __future__ import annotations

import math

from lingvo_b200.core import base_layer
from lingvo_b200.core import py_utils


def _Step(step):
  s = py_utils.GetGlobalStep() if step is None else step
  if hasattr(s, 'item'):
    s = s.item()
  return s


def _PiecewiseConstant(x, boundaries, values):
  """values[i] for boundaries[i-1] <= x < boundaries[i]."""
  idx = 0
  for b in boundaries:
    if x >= b:
      idx += 1
  return values[idx]


def _TrainerSplits(layer, num_splits):
  """`num_splits_per_client` from the trainer's perspective (sync mode)."""
  if num_splits and num_splits > 0:
    return num_splits
  cp = layer.cluster.params.Copy()
  cp.task = 0
  assert cp.mode == 'sync', 'this schedule only makes sense for sync training'
  cp.job = 'trainer_client'
  return cp.Instantiate().num_splits_per_client


class BaseSchedule(base_layer.BaseLayer):
  """Base class for schedules."""

  def GetStep(self, step=None):
    return _Step(step)

  def Value(self, step=None):
    return self.FProp(self.theta, step)

  def FProp(self, theta, step=None):
    raise NotImplementedError()


class Constant(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('value', 1., 'The constant value.')
    return p

  def Value(self, step=None):
    return float(self.params.value)


class ConstantOne(Constant):
  pass


class PiecewiseConstantSchedule(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('boundaries', None, 'Boundaries at which learning rate drops.')
    p.Define('values', None, 'Values in each interval.')
    return p

  def Value(self, step=None):
    p = self.params
    return float(_PiecewiseConstant(_Step(step), p.boundaries, p.values))


class PolynomialSchedule(BaseSchedule):
  """y0 → y1 between x0 and x1 following ratio**power."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('power', 1, 'Polynomial power.')
    p.Define('start', (0, 1.), '(x0, y0)')
    p.Define('limit', (1, 1.), '(x1, y1)')
    p.Define('origin', 'start', 'Origin of the polynomial: "start"|"limit".')
    return p

  def Value(self, step=None):
    p = self.params
    x = float(_Step(step))
    (x0, y0), (x1, y1) = p.start, p.limit
    if x0 >= x1:
      raise ValueError(f'{x0} must be < {x1}')
    if x < x0:
      return float(y0)
    if x >= x1:
      return float(y1)
    ratio = (x - x0) / (x1 - x0)
    if p.origin == 'start':
      f = ratio**p.power
    elif p.origin == 'limit':
      f = 1 - (1 - ratio)**p.power
    else:
      raise ValueError('Invalid parameter origin: %s' % p.origin)
    return float(y0 + f * (y1 - y0))


class LinearSchedule(PolynomialSchedule):

  @classmethod
  def Params(cls):
    return super().Params().Set(power=1)


class ExponentialSchedule(BaseSchedule):
  """Linear in log-space between (x0,y0) and (x1,y1)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('start', (0, 1.), '(x0, y0)')
    p.Define('limit', (1, 0.5), '(x1, y1)')
    return p

  def __init__(self, params):
    super().__init__(params)
    (x0, y0), (x1, y1) = self.params.start, self.params.limit
    assert x0 < x1, '%s must be < %s' % (x0, x1)
    assert y0 > 0 and y1 > 0
    self.CreateChild('linear', LinearSchedule.Params().Set(
        start=(x0, math.log(y0)), limit=(x1, math.log(y1))))

  def Value(self, step=None):
    return math.exp(self.linear.Value(step))


class ContinuousSchedule(BaseSchedule):
  """Exponential decay with a half-life after `start_step`."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('initial_value', 1.0, 'Initial decay value.')
    p.Define('start_step', 400000, 'Starts to decay from this step.')
    p.Define('half_life_steps', 100000, 'Halve every this many steps.')
    p.Define('min', 0.01, 'Minimum relative learning rate.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('exp', ExponentialSchedule.Params().Set(
        start=(p.start_step, 1.0),
        limit=(p.start_step + p.half_life_steps * math.log(p.min) /
               math.log(0.5), p.min)))

  def Value(self, step=None):
    return self.params.initial_value * self.exp.Value(step)


class LinearRampupDecaySchedule(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('peak', 1, 'Number of steps at peak learning rate.')
    p.Define('end', 2, 'Number of steps at end of learning rate schedule.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('rampup_schedule', LinearSchedule.Params().Set(
        start=(0, 0.0), limit=(p.peak, 1.0)))
    self.CreateChild('decay_schedule', LinearSchedule.Params().Set(
        start=(p.peak, 1.0), limit=(p.end, 0.0)))

  def Value(self, step=None):
    return min(self.rampup_schedule.Value(step),
               self.decay_schedule.Value(step))


class AnnealingSchedule(BaseSchedule):
  """y = max(factor**step, lower_bound)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('init', None, 'start value.')
    p.Define('lower_bound', None, 'lower bound value.')
    p.Define('factor', None, 'Annealing factor.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.init and p.lower_bound and p.factor and 0 < p.factor <= 1

  def Value(self, step=None):
    p = self.params
    return max(p.factor**float(_Step(step)), p.lower_bound)


class StepwiseExponentialSchedule(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('decay', 0.99, 'Decay factor.')
    p.Define('num_steps_per_decay', 1000, 'Number of steps between decays.')
    return p

  def Value(self, step=None):
    p = self.params
    return p.decay**(int(_Step(step)) // p.num_steps_per_decay)


class CombinedMinimumSchedule(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('schedules', [LinearSchedule.Params()], 'Schedules to combine.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self.CreateChildren('schedules', self.params.schedules)

  def Value(self, step=None):
    return min(s.Value(step) for s in self.schedules)


class TransformerSchedule(BaseSchedule):
  """d^-0.5 · min((t+1)·(w·r)^(decay-1), (t+start+1)^decay) (:305-342)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('warmup_steps', 4000, 'Linear warm-up length.')
    p.Define('model_dim', 512, 'Model dimension.')
    p.Define('worker_replicas', 1, 'Number of worker replicas.')
    p.Define('decay_end', None, 'Ends the decay at this step.')
    p.Define('decay_factor', -0.5, 'Decay exponent after warmup.')
    p.Define('start_step', 0, 'Translate the function left in the step axis.')
    p.Define('cyclical_step', None, 'If set, the cycle restarts at this step.')
    return p

  def Value(self, step=None):
    p = self.params
    t = _Step(step)
    if p.cyclical_step is not None:
      t = t % p.cyclical_step
    t = float(t)
    warm = float(p.warmup_steps * p.worker_replicas)
    if p.decay_end is not None:
      t = min(t, float(p.decay_end))
    return p.model_dim**-0.5 * min((t + 1) * warm**(p.decay_factor - 1.0),
                                   (t + p.start_step + 1)**p.decay_factor)


class TransformerMLPerfSchedule(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('warmup_steps', 4000, 'Linear warm-up length.')
    p.Define('warmup_init_fraction', 0., 'Fraction of peak at step 0.')
    p.Define('model_dim', 512, 'Model dimension.')
    return p

  def Value(self, step=None):
    p = self.params
    t = float(_Step(step))
    w = float(p.warmup_steps)
    f0 = float(p.warmup_init_fraction)
    lin = min(1.0, f0 + (1. - f0) * t / w)
    return p.model_dim**-0.5 * lin / math.sqrt(max(t, w))


class TransformerScheduleNoWarmUp(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('decay_start', 4000, 'It is used to estimate peak-lr.')
    p.Define('decay_end', None, 'Ends the learning rate decay at this step.')
    p.Define('model_dim', 512, 'Model dimension.')
    p.Define('worker_replicas', 1, 'Number of worker replicas.')
    return p

  def Value(self, step=None):
    p = self.params
    warm = float(p.decay_start * p.worker_replicas)
    t = float(_Step(step))
    if p.decay_end is not None:
      t = min(t, float(p.decay_end))
    return p.model_dim**-0.5 * min(min(t + 1, (t + 1)**-0.5), warm**-0.5)


class LinearRampupExponentialDecayScaledByNumSplitSchedule(BaseSchedule):
  """min of {warm-up ramp, plateau=splits, exp decay to `min`, cap} (:416)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('warmup', 300, 'Warm-up steps (per split).')
    p.Define('warmup_init', 1.0, 'Initial value of the warm-up phase.')
    p.Define('decay_start', 70000, 'Starts the decay at decay_start-th step.')
    p.Define('decay_end', 100000, 'Ends the decay at decay_end-th step.')
    p.Define('min', 0.01, 'After decay_end, the multiplier stays at min.')
    p.Define('max', 1e8, 'The schedule is never larger than this value.')
    p.Define('num_splits', 0, 'Overrides num_splits_per_client if non-zero.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    splits = _TrainerSplits(self, p.num_splits)
    warmup_end = p.warmup * splits
    decay_start = max(warmup_end + 1.0, p.decay_start / splits)
    peak = 1.0 * splits
    decay_end = max(decay_start + 1.0, p.decay_end / splits)
    schedules = [
        LinearSchedule.Params().Set(start=(warmup_end, peak),
                                    limit=(decay_start, peak)),
        ExponentialSchedule.Params().Set(start=(decay_start, peak),
                                         limit=(decay_end, p.min)),
        LinearSchedule.Params().Set(start=(0, p.max), limit=(decay_end, p.max)),
    ]
    if warmup_end > 0.0:
      schedules.insert(0, LinearSchedule.Params().Set(
          start=(0., p.warmup_init), limit=(warmup_end, peak)))
    self.CreateChild('combine', CombinedMinimumSchedule.Params().Set(
        schedules=schedules))

  def Value(self, step=None):
    return self.combine.Value(step)


class LinearRampupExponentialDecay(
    LinearRampupExponentialDecayScaledByNumSplitSchedule):

  @classmethod
  def Params(cls):
    return super().Params().Set(num_splits=1)


class LinearRampupSqrtDecay(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('peak', 1.0, 'The peak value of the schedule.')
    p.Define('warmup_steps', 4000, 'Linear warm-up length.')
    return p

  def Value(self, step=None):
    p = self.params
    t = float(max(_Step(step), 1))
    w = float(p.warmup_steps)
    return p.peak * min(t / w, math.sqrt(w / t))


class LinearRampupSqrtDecayByBatchSizeAndReplicas(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('warmup_examples', 256 * 2**20, 'Warm-up length in examples.')
    p.Define('batch_size', None, 'Per-replica batch size.')
    p.Define('num_replicas', None, 'Worker replicas; None ⇒ from cluster.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.batch_size > 0
    self._num_replicas = p.num_replicas or _TrainerSplits(self, 0)
    assert self._num_replicas > 0

  def Value(self, step=None):
    p = self.params
    t = float(_Step(step))
    w = p.warmup_examples / (p.batch_size * self._num_replicas)
    return min((t + 1) * w**-1.5, (t + 1)**-0.5)


class LinearRampupPiecewiseConstantSchedule(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('boundaries', [], 'Boundaries at which learning rate changes.')
    p.Define('lrs', [], 'A list of learning rate multipliers.')
    p.Define('num_splits', 0, 'Overrides num_splits if non-zero.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert len(p.boundaries) >= 2 and len(p.boundaries) == len(p.lrs)
    splits = float(_TrainerSplits(self, p.num_splits))
    assert splits >= 1
    boundaries = [b / splits for b in p.boundaries]
    lrs = [v * splits for v in p.lrs]
    self.CreateChild('combine', CombinedMinimumSchedule.Params().Set(schedules=[
        LinearSchedule.Params().Set(start=(0., 0.),
                                    limit=(boundaries[0], lrs[0])),
        PiecewiseConstantSchedule.Params().Set(boundaries=boundaries,
                                               values=[1e8] + lrs),
    ]))

  def Value(self, step=None):
    return self.combine.Value(step)


class CosineSchedule(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('initial_value', 1.0, 'Initial decay value.')
    p.Define('final_value', 0., 'Final decay value.')
    p.Define('total_steps', 0, 'Number of steps to reach full decay.')
    p.Define('cyclical', False, 'Restart at the end of the cycle if True.')
    p.Define('half_cycle', True, 'Cyclical only: angle reset period is pi.')
    return p

  def Value(self, step=None):
    p = self.params
    assert p.total_steps > 0
    gap = p.initial_value - p.final_value
    total = int(p.total_steps)
    t = _Step(step)
    if p.cyclical:
      rel = t % total if p.half_cycle else t
    else:
      rel = min(t, total)
    return p.final_value + 0.5 * gap * (1 + math.cos(math.pi * float(rel) /
                                                     p.total_steps))


class LinearRampupCosineSchedule(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('warmup_init', 0, 'The initial lr value of the warm-up phase.')
    p.Define('warmup_steps', 0, 'Number of warm up steps.')
    p.Define('initial_value', 1.0, 'Initial decay value.')
    p.Define('final_value', 0., 'Final decay value.')
    p.Define('total_steps', 0, 'Number of steps to reach full decay.')
    p.Define('cyclical', False, 'Restart at the end of the cycle if True.')
    p.Define('num_splits', 1, '<=0 ⇒ num_splits_per_client.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    splits = _TrainerSplits(self, p.num_splits)
    self.CreateChild('combine', CombinedMinimumSchedule.Params().Set(schedules=[
        LinearSchedule.Params().Set(
            start=(0., p.warmup_init * splits),
            limit=(p.warmup_steps // splits, p.initial_value * splits)),
        CosineSchedule.Params().Set(
            initial_value=p.initial_value * splits,
            final_value=p.final_value * splits,
            total_steps=p.total_steps // splits, cyclical=p.cyclical),
    ]))

  def Value(self, step=None):
    return self.combine.Value(step)


class EmaDecaySchedule(BaseSchedule):
  """min((1+t)/(10+t), ema_decay)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('ema_decay', 0.9999, 'The EMA decay parameter.')
    return p

  def Value(self, step=None):
    x = float(_Step(step))
    return min((1.0 + x) / (10.0 + x), self.params.ema_decay)


class DevBasedSchedule(BaseSchedule):
  """Decays when a dev metric stops improving (reads MetricHistory) (:728)."""

  @classmethod
  def Params(cls):
    from lingvo_b200.core import early_stop
    p = super().Params()
    p.Define('metric_history', early_stop.MetricHistory.Params(),
             'Metric history params (file the evaler writes).')
    p.Define('tolerance', 0.0, 'Minimum significant difference in metric.')
    p.Define('window', 10000, 'Steps without improvement before decaying.')
    p.Define('decay', 0.5, 'Decay factor.')
    p.Define('min_factor', 0.01, 'Minimum learning rate multiplier.')
    return p

  def __init__(self, params):
    from lingvo_b200.core import early_stop
    super().__init__(params)
    self._metric_history = early_stop.MetricHistory(self.params.metric_history)
    self._cur_factor = 1.0
    self._ref_step = 0

  def Value(self, step=None):
    from lingvo_b200.core import early_stop
    p = self.params
    best_step, last_step = early_stop.BestStep(
        self._metric_history.hist_file, p.tolerance,
        self._metric_history.params.minimize)
    ref = max(self._ref_step, best_step)
    f = self._cur_factor
    new_f = f if last_step - ref < p.window else max(p.min_factor, f * p.decay)
    self._ref_step = ref if new_f == f else last_step
    self._cur_factor = new_f
    return new_f


class PiecewiseSchedule(BaseSchedule):
  """Sub-schedule i runs on [boundaries[i-1], boundaries[i]) with relative step."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('boundaries', None, 'Boundaries between subschedules.')
    p.Define('schedules', None, 'len(boundaries)+1 sub-schedules.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    prev = 0
    for b in p.boundaries:
      if b < prev:
        raise ValueError('Invalid boundary %s < %s' % (b, prev))
      prev = b
    if len(p.schedules) != len(p.boundaries) + 1:
      raise ValueError('len(schedules) != len(boundaries) + 1: %s vs %s' %
                       (len(p.schedules), len(p.boundaries)))
    self.CreateChildren('schedules', p.schedules)

  def Value(self, step=None):
    p = self.params
    cur = int(_Step(step))
    starts = [0] + list(p.boundaries)
    vals = [s.Value(max(0, cur - st)) for st, s in zip(starts, self.schedules)]
    return _PiecewiseConstant(cur, p.boundaries, vals)


class SqrtDecay(BaseSchedule):
  """multiplier · rsqrt(max(t − offset, warmup_steps)) (GShard LMs, :904)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('warmup_steps', 10000, 'Number of warm up steps.')
    p.Define('multiplier', 1.0, 'Multiplier.')
    p.Define('offset', 0.0, 'Offset.')
    return p

  def Value(self, step=None):
    p = self.params
    t = float(_Step(step))
    return p.multiplier / math.sqrt(max(t - p.offset, p.warmup_steps))


class SqrtDecayToZero(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('warmup_steps', 10000.0, 'Number of warmup steps. Must be > 0.')
    p.Define('starting_lr', 0.01, 'LR during warmup.')
    p.Define('final_steps', 100000.0, 'Steps at which LR decays to 0.')
    return p

  def Value(self, step=None):
    p = self.params
    t = float(_Step(step))
    scale = p.starting_lr * math.sqrt(p.warmup_steps * p.final_steps) / (
        math.sqrt(p.final_steps) - math.sqrt(p.warmup_steps))
    shift = scale / math.sqrt(p.final_steps)
    return scale / math.sqrt(max(t, p.warmup_steps)) - shift


class CycleSchedule(BaseSchedule):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('schedules', None, 'A list of sub-schedules.')
    p.Define('steps', None, 'The number of steps to run each sub-schedule.')
    p.Define('pass_absolute_step', True, 'Pass absolute step to sub-schedules.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    if len(p.schedules) != len(p.steps):
      raise ValueError('len(schedules) != len(steps): %s vs %s' %
                       (len(p.schedules), len(p.steps)))
    self.CreateChildren('schedules', p.schedules)
    bounds = [0]
    for s in p.steps:
      bounds.append(bounds[-1] + s)
    self._period = bounds[-1]
    self._boundaries = bounds[1:-1]

  def Value(self, step=None):
    t = int(_Step(step))
    rel = t % self._period
    sub = t if self.params.pass_absolute_step else rel
    vals = [s.Value(sub) for s in self.schedules]
    return _PiecewiseConstant(rel, self._boundaries, vals)


class InverseSigmoid(BaseSchedule):
  """k / (k + exp(t / k))."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('k', None, 'k >= 1, the greater k is, the slower it decays.')
    return p

  def __init__(self, params):
    super().__init__(params)
    if not self.params.k or self.params.k < 1:
      raise ValueError(f'Param k invalid: {self.params.k}')

  def Value(self, step=None):
    k = self.params.k
    return k / (k + math.exp(min(float(_Step(step)) / k, 700.0)))
