"""Host-side evaluation metrics (reference `lingvo/core/metrics.py`).

`BaseMetric` / `AverageMetric` / `F1Metric` / `MCCMetric` / `CorpusBleuMetric`
/ `AUCMetric` / `CorrelationMetric` / `SamplingMetric` / `MultiClassAUCMetric`
/ `AverageKeyedCustomMetric` and a device-side accumulator
(`DeviceEvalMetrics`, the H100 analogue of `TpuEvalMetrics` :258-384: metric
(value, weight) pairs are accumulated on the GPU across loop steps and only
synced to host once per eval program).
"""

from __future__ import annotations

import collections
import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from lingvo_b200.core import hyperparams


def CreateScalarSummary(name: str, simple_value: float):
  from lingvo_b200.utils import tfevents
  return tfevents.ScalarValue(name, simple_value)


class BaseMetric:
  """Base class for aggregating statistics to compute a metric."""

  def Update(self, *args, **kwargs):
    raise NotImplementedError()

  @property
  def value(self):
    raise NotImplementedError()

  def Summary(self, name: str):
    return CreateScalarSummary(name, self.value)


class ConstantMetric(BaseMetric):

  def __init__(self):
    self._value = 0.0

  def Update(self, value):
    self._value = value

  @property
  def value(self):
    return self._value


class AverageMetric(BaseMetric):
  """Weighted average."""

  def __init__(self):
    self._total_value = 0.0
    self._total_weight = 0.0

  def Update(self, value, weight=1.0):
    if weight < 0.0:
      raise ValueError('weight must be non-negative, got %s' % weight)
    self._total_value += float(value) * float(weight)
    self._total_weight += float(weight)

  def GetTotalValue(self):
    return self._total_value

  def SetTotalValue(self, val):
    self._total_value = val

  total_value = property(GetTotalValue, SetTotalValue)

  def GetTotalWeight(self):
    return self._total_weight

  def SetTotalWeight(self, val):
    self._total_weight = val

  total_weight = property(GetTotalWeight, SetTotalWeight)

  @property
  def value(self):
    return (self._total_value / self._total_weight
            if self._total_weight > 0 else 0.0)


class UniqueAverageMetric(AverageMetric):
  """Average over unique keys; asserts values are consistent per key."""

  def __init__(self, mismatch_is_error=True):
    super().__init__()
    self._map = {}
    self._mismatch_is_error = mismatch_is_error

  def Update(self, key, value, weight=1.0):
    if key in self._map:
      if self._mismatch_is_error and self._map[key] != (value, weight):
        raise ValueError('Conflicting value for key %s' % key)
      return
    self._map[key] = (value, weight)
    super().Update(value, weight)

  @property
  def num_keys(self):
    return len(self._map)


class F1Metric(BaseMetric):

  def __init__(self):
    self._true_pos = 0.0
    self._false_pos = 0.0
    self._false_neg = 0.0

  def UpdateTruePositive(self, count=1.0):
    self._true_pos += count

  def UpdateFalsePositive(self, count=1.0):
    self._false_pos += count

  def UpdateFalseNegative(self, count=1.0):
    self._false_neg += count

  @property
  def value(self):
    if self._true_pos + self._false_pos > 0:
      precision = self._true_pos / (self._true_pos + self._false_pos)
    else:
      precision = 0.0
    if self._true_pos + self._false_neg > 0:
      recall = self._true_pos / (self._true_pos + self._false_neg)
    else:
      recall = 0.0
    if precision + recall > 0:
      return 2.0 * precision * recall / (precision + recall)
    return 0.0


class MCCMetric(F1Metric):
  """Matthews correlation coefficient."""

  def __init__(self):
    super().__init__()
    self._true_neg = 0.0

  def UpdateTrueNegative(self, count=1.0):
    self._true_neg += count

  @property
  def value(self):
    tp, fp, fn, tn = self._true_pos, self._false_pos, self._false_neg, self._true_neg
    num = tp * tn - fp * fn
    den = math.sqrt((tp + fp) * (tp + fn) * (tn + fp) * (tn + fn))
    return num / den if den > 0 else 0.0


def _Ngrams(tokens: Sequence[str], n: int):
  return collections.Counter(
      tuple(tokens[i:i + n]) for i in range(len(tokens) - n + 1))


class CorpusBleuMetric(BaseMetric):
  """Corpus-level BLEU-4 with brevity penalty."""

  def __init__(self, separator_type=None, max_order: int = 4):
    self._max_order = max_order
    self._matches = [0] * max_order
    self._possible = [0] * max_order
    self._ref_len = 0
    self._hyp_len = 0
    self._separator_type = separator_type

  def _Split(self, s: str) -> List[str]:
    if self._separator_type == 'wpm':
      s = s.replace(' ', '').replace('▁', ' ')
    return s.split()

  def Update(self, ref_str: str, hyp_str: str):
    ref, hyp = self._Split(ref_str), self._Split(hyp_str)
    self._ref_len += len(ref)
    self._hyp_len += len(hyp)
    for n in range(1, self._max_order + 1):
      r, h = _Ngrams(ref, n), _Ngrams(hyp, n)
      self._matches[n - 1] += sum((r & h).values())
      self._possible[n - 1] += max(len(hyp) - n + 1, 0)

  @property
  def unsegmenter(self):
    return None

  @property
  def value(self):
    if self._hyp_len == 0 or min(self._possible) == 0:
      return 0.0
    precisions = []
    smooth = 1.0
    for m, p in zip(self._matches, self._possible):
      if m > 0:
        precisions.append(m / p)
      else:
        smooth *= 2
        precisions.append(1.0 / (smooth * p))
    geo = math.exp(sum(math.log(x) for x in precisions) / self._max_order)
    ratio = self._hyp_len / max(self._ref_len, 1)
    bp = 1.0 if ratio >= 1.0 else math.exp(1 - 1.0 / max(ratio, 1e-9))
    return geo * bp


def _CurvePng(xs, ys, size=256):
  """Polyline through (xs, ys) ∈ [0,1]² on a white `size`×`size` canvas with a light 0.25
  grid; y grows upwards. Dependency-free stand-in for the matplotlib curve plot."""
  from lingvo_b200.utils import tfevents  # pylint: disable=g-import-not-at-top
  img = np.full((size, size), 255, np.uint8)
  for g in (0.25, 0.5, 0.75):
    k = int(round(g * (size - 1)))
    img[k, :] = 224
    img[:, k] = 224
  img[[0, -1], :] = 128
  img[:, [0, -1]] = 128
  xs = np.clip(np.asarray(xs, np.float64), 0.0, 1.0) * (size - 1)
  ys = (1.0 - np.clip(np.asarray(ys, np.float64), 0.0, 1.0)) * (size - 1)
  for i in range(len(xs) - 1):
    n = int(max(abs(xs[i + 1] - xs[i]), abs(ys[i + 1] - ys[i]))) + 2
    cx = np.round(np.linspace(xs[i], xs[i + 1], n)).astype(int)
    cy = np.round(np.linspace(ys[i], ys[i + 1], n)).astype(int)
    img[cy, cx] = 0
  return tfevents.EncodePng(img)


class AUCMetric(BaseMetric):
  """ROC-AUC or PR-AUC over accumulated (label, prob[, weight])."""

  def __init__(self, mode='roc', samples=-1):
    assert mode in ('roc', 'pr')
    self._mode = mode
    self._label, self._prob, self._weight = [], [], []
    self._samples = samples

  def Update(self, label, prob, weight=None):
    self._label += list(label)
    self._prob += list(prob)
    self._weight += list(weight) if weight is not None else [1.0] * len(label)
    if self._samples > 0:
      self._label = self._label[-self._samples:]
      self._prob = self._prob[-self._samples:]
      self._weight = self._weight[-self._samples:]

  def _Sorted(self):
    y = np.asarray(self._label, dtype=np.float64)
    s = np.asarray(self._prob, dtype=np.float64)
    w = np.asarray(self._weight, dtype=np.float64)
    if y.size == 0 or (y * w).sum() == 0 or ((1 - y) * w).sum() == 0:
      return None
    order = np.argsort(-s, kind='mergesort')
    y, s, w = y[order], s[order], w[order]
    tp = np.cumsum(y * w)
    fp = np.cumsum((1 - y) * w)
    last = np.r_[np.where(np.diff(s))[0], y.size - 1]
    return tp[last], fp[last], s[last]

  def _PrCurve(self):
    """(precision, recall, thresholds) in sklearn's order: thresholds ascending, recall
    descending, with the final (precision=1, recall=0) point appended."""
    st = self._Sorted()
    if st is None:
      return np.array([1.0]), np.array([0.0]), np.array([])
    tp, fp, th = st
    precision = tp / np.maximum(tp + fp, 1e-12)
    recall = tp / tp[-1]
    stop = int(np.searchsorted(tp, tp[-1]))      # first threshold reaching full recall
    sl = slice(stop, None, -1)
    return np.r_[precision[sl], 1.0], np.r_[recall[sl], 0.0], th[sl]

  def Curve(self):
    """(xs, ys, axis labels) of the curve the AUC integrates: (FPR, TPR) for 'roc',
    (recall, precision) for 'pr'."""
    if self._mode == 'pr':
      precision, recall, _ = self._PrCurve()
      return recall, precision, ('Recall', 'Precision')
    st = self._Sorted()
    if st is None:
      return np.array([0.0, 1.0]), np.array([0.0, 1.0]), ('False Positive Rate',
                                                           'True Positive Rate')
    tp, fp, _ = st
    return (np.r_[0.0, fp / fp[-1]], np.r_[0.0, tp / tp[-1]],
            ('False Positive Rate', 'True Positive Rate'))

  def Summary(self, name):
    """The scalar AUC plus an image of the curve under the same tag (ref :533). With
    matplotlib the plot has a grid / axis labels; without, the curve is rasterised on a unit
    square by `_CurvePng`."""
    from lingvo_b200.core import plot  # pylint: disable=g-import-not-at-top
    from lingvo_b200.utils import tfevents  # pylint: disable=g-import-not-at-top
    xs, ys, labels = self.Curve()

    def _Setter(fig, axes):
      ticks = np.arange(0, 1.05, 0.05)
      axes.grid(visible=True)
      axes.set_xlabel(labels[0])
      axes.set_xticks(ticks)
      axes.set_ylabel(labels[1])
      axes.set_yticks(ticks)
      fig.tight_layout()

    png = plot.Curve(name=name, figsize=(12, 12), xs=xs, ys=ys, setter=_Setter)
    if png is None:
      png = _CurvePng(xs, ys)
    return tfevents.ImageValue(name, png) + CreateScalarSummary(name, self.value)

  @property
  def value(self):
    st = self._Sorted()
    if st is None:
      return 0.0
    tp, fp, _ = st
    if self._mode == 'roc':
      tpr = np.r_[0.0, tp / tp[-1]]
      fpr = np.r_[0.0, fp / fp[-1]]
      return float(np.trapezoid(tpr, fpr))
    precision = tp / np.maximum(tp + fp, 1e-12)
    recall = tp / tp[-1]
    return float(np.sum(np.diff(np.r_[0.0, recall]) * precision))

  def _PrecisionAtRecall(self, recall):
    """Precision at the highest threshold whose recall is still ≥ `recall` (ref :552)."""
    assert self._mode == 'pr'
    p, r, t = self._PrCurve()
    last_p = 0.0
    for pp, rr, _ in zip(p, r, t):
      if rr >= recall:
        last_p = pp
    return float(last_p)

  def _RecallAtPrecision(self, precision):
    """Recall at the lowest threshold whose precision reaches `precision` (ref :564)."""
    assert self._mode == 'pr'
    p, r, t = self._PrCurve()
    for pp, rr, _ in zip(p, r, t):
      if pp >= precision:
        return float(rr)
    return 0.0


class PrecisionAtRecall(AUCMetric):
  """Precision of the PR curve at a recall threshold (ref :576)."""

  def __init__(self, recall_threshold, samples=-1):
    super().__init__(mode='pr', samples=samples)
    self._recall_threshold = recall_threshold

  @property
  def value(self):
    return self._PrecisionAtRecall(self._recall_threshold)


class RecallAtPrecision(AUCMetric):
  """Recall of the PR curve at a precision threshold (ref :587)."""

  def __init__(self, precision_threshold, samples=-1):
    super().__init__(mode='pr', samples=samples)
    self._precision_threshold = precision_threshold

  @property
  def value(self):
    return self._RecallAtPrecision(self._precision_threshold)


class MultiClassAUCMetric(BaseMetric):

  def __init__(self, num_classes, mode='roc', samples=-1):
    self._metrics = [AUCMetric(mode, samples) for _ in range(num_classes)]

  def Update(self, labels, probs, weights=None):
    labels, probs = np.asarray(labels), np.asarray(probs)
    for c, m in enumerate(self._metrics):
      m.Update(labels[:, c], probs[:, c],
               None if weights is None else np.asarray(weights)[:, c])

  @property
  def value(self):
    return float(np.mean([m.value for m in self._metrics]))


def _Ranks(x):
  """Average ranks (ties share the mean rank), as scipy.stats.rankdata."""
  x = np.asarray(x, np.float64)
  order = np.argsort(x, kind='mergesort')
  ranks = np.empty(x.size, np.float64)
  sx = x[order]
  i = 0
  while i < x.size:
    j = i
    while j + 1 < x.size and sx[j + 1] == sx[i]:
      j += 1
    ranks[order[i:j + 1]] = 0.5 * (i + j) + 1.0
    i = j + 1
  return ranks


def _Correlation(mode, target, pred):
  """pearson | spearman | kendalltau (tau-b) of two sequences; NaN when undefined."""
  t, p = np.asarray(target, np.float64), np.asarray(pred, np.float64)
  if t.size < 2:
    return float('nan')
  if mode == 'kendalltau':
    dt = np.sign(t[:, None] - t[None, :])
    dp = np.sign(p[:, None] - p[None, :])
    iu = np.triu_indices(t.size, 1)
    dt, dp = dt[iu], dp[iu]
    denom = np.sqrt(float((dt != 0).sum()) * float((dp != 0).sum()))
    return float((dt * dp).sum() / denom) if denom > 0 else float('nan')
  if mode == 'spearman':
    t, p = _Ranks(t), _Ranks(p)
  if t.std() == 0 or p.std() == 0:
    return float('nan')
  return float(np.corrcoef(t, p)[0, 1])


class CorrelationMetric(BaseMetric):
  """Pearson / Spearman / Kendall-tau correlation of accumulated (target, pred) (ref :652)."""

  def __init__(self, mode='pearson'):
    assert mode in ('pearson', 'spearman', 'kendalltau')
    self._mode = mode
    self._t, self._p = [], []

  def Update(self, target, pred):
    self._t += list(target)
    self._p += list(pred)

  @property
  def value(self):
    c = _Correlation(self._mode, self._t, self._p)
    return float(0.0 if np.isnan(c) else c)


class AverageKeyedCorrelationMetric(BaseMetric):
  """Correlation computed per key, averaged over keys (ref :700); keys whose correlation is
  undefined (a single example, constant values) are skipped when `bypass_nan`."""

  def __init__(self, mode='pearson', bypass_nan=True):
    assert mode in ('pearson', 'spearman', 'kendalltau')
    self._mode = mode
    self._bypass_nan = bypass_nan
    self._target = collections.defaultdict(list)
    self._pred = collections.defaultdict(list)

  def Update(self, key, target, pred):
    self._target[key] += list(target)
    self._pred[key] += list(pred)

  @property
  def value(self):
    results = []
    for k in self._target:
      c = _Correlation(self._mode, self._target[k], self._pred[k])
      if not self._bypass_nan or not np.isnan(c):
        results.append(c)
    if results:
      return float(np.mean(results))
    return 0.0 if self._bypass_nan else float('nan')


class ConfigurableMetric(BaseMetric):
  """A metric constructed from Params (ref :67)."""

  @classmethod
  def Params(cls):
    return hyperparams.InstantiableParams(cls)

  def __init__(self, params):
    self.params = params


class SamplingMetric(ConfigurableMetric):
  """Keeps a uniform sample of `num_samples` decoded outputs; subclasses turn them into a
  summary in `_CreateSummary` (ref :764). Accepts Params or (legacy) a plain sample count."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_samples', 8, 'The number of samples to store uniformly.')
    return p

  def __init__(self, params=8):
    if not isinstance(params, hyperparams.Params):
      params = self.Params().Set(num_samples=int(params))
    super().__init__(params)
    self._NewSampler()
    self._summary = None

  def _NewSampler(self):
    from lingvo_b200.core import py_utils  # pylint: disable=g-import-not-at-top
    self._sampler = py_utils.UniformSampler(num_samples=self.params.num_samples, seed=0)

  @property
  def samples(self):
    return self._sampler.samples

  def Update(self, decoded_outputs, *args, **kwargs):
    self._sampler.Add(decoded_outputs if not (args or kwargs)
                      else ((decoded_outputs,) + args, kwargs))
    self._summary = None

  @property
  def value(self):
    return 0

  def Summary(self, name):
    if self._summary is None:
      self._summary = self._CreateSummary(name)
      self._NewSampler()
    return self._summary

  def _CreateSummary(self, name):
    return CreateScalarSummary(name, float(len(self.samples)))


class AverageKeyedCustomMetric(BaseMetric):
  """Groups values by key; value = mean over keys of fn(values)."""

  def __init__(self, fn=np.mean):
    self._fn = fn
    self._vals = collections.defaultdict(list)

  def Update(self, key, value):
    self._vals[key].append(value)

  @property
  def value(self):
    if not self._vals:
      return 0.0
    return float(np.mean([self._fn(v) for v in self._vals.values()]))


class GroupPairAUCMetric(AUCMetric):
  """AUC over all pairs of items with different targets inside each group (ref :810): pair
  (i, j) is a binary example with label `target[i] > target[j]` and probability
  `sigmoid(logits[i] - logits[j])`. Groups are the *contiguous* runs of equal `group_ids`."""

  def UpdateRaw(self, group_ids, target, logits, weight=None, ignore_ids=None):
    if ignore_ids is not None:
      keep = np.asarray(ignore_ids) == 0
      group_ids = np.asarray(group_ids)[keep].tolist()
      target = np.asarray(target)[keep].tolist()
      logits = np.asarray(logits)[keep].tolist()
      if weight is not None:
        weight = np.asarray(weight)[keep].tolist()
    assert self._samples <= 0
    n = len(target)
    s = 0
    for e in range(1, n + 1):
      if e < n and group_ids[e] == group_ids[s]:
        continue
      for i in range(s, e):
        for j in range(i + 1, e):
          if target[i] == target[j]:
            continue
          self._label.append(1 if target[i] > target[j] else 0)
          self._prob.append(1.0 / (1.0 + math.exp(-(logits[i] - logits[j]))))
          self._weight.append(min(1.0, weight[i] + weight[j]) if weight is not None
                              and len(weight) else 1.0)
      s = e


class DeviceEvalMetrics:
  """Accumulates {name: (value, weight)} on device across steps.

  Equivalent of reference `TpuEvalMetrics` (:258-384): one fused
  `value·weight` / `weight` accumulator tensor pair, finalised (and optionally
  all-reduced across ranks) once per program run.
  """

  def __init__(self, max_metrics: int = 256):
    self._names: List[str] = []
    self._acc: Optional[torch.Tensor] = None  # [n, 2] (sum v·w, sum w)
    self._max_metrics = int(max_metrics)
    self._metrics = None
    self._initial_values = [torch.zeros((), dtype=torch.float32)
                            for _ in range(2 * self._max_metrics)]

  # -- loop-carried form (ref :288-384): a flat [v0·w0, w0, v1·w1, w1, …] list of scalars that
  # a device loop threads through its iterations.
  @property
  def initial_values(self):
    return self._initial_values

  @property
  def metrics(self):
    return self._metrics

  def PackStepMetricsForAccumulation(self, metric_dict, step_args):
    """This step's (value·weight, weight) pairs in sorted-name order, followed by the
    untouched tail of `step_args`."""
    n = len(metric_dict)
    assert n <= self._max_metrics, 'Increase max_metrics to >= %d' % n
    self._metrics = metric_dict
    ret = []
    for _, (value, weight) in sorted(metric_dict.items()):
      weight = torch.as_tensor(weight, dtype=torch.float32).detach()
      value = torch.as_tensor(value, dtype=torch.float32).detach() * weight
      assert value.numel() == 1 and weight.numel() == 1, (value.shape, weight.shape)
      ret += [value.reshape(()), weight.reshape(())]
    return ret + list(step_args)[len(ret):]

  def FinalizeMetrics(self, loop_carried_metrics, group=None):
    """Sums the carried scalars over the ranks (one fused all-reduce) and returns the flat
    [avg0, total_weight0, avg1, …] list."""
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    n = 2 * len(self._metrics)
    dev = next((x.device for x in loop_carried_metrics[:n] if x.is_cuda), None)
    flat = torch.stack([torch.as_tensor(x, dtype=torch.float32).to(dev or 'cpu')
                        for x in loop_carried_metrics[:n]])
    if dist.is_available() and dist.is_initialized():
      dist.all_reduce(flat, group=group)
    pairs = flat.reshape(-1, 2)
    avg = torch.where(pairs[:, 1] > 0, pairs[:, 0] / pairs[:, 1].clamp(min=1e-30),
                      torch.zeros_like(pairs[:, 0]))
    out = torch.stack([avg, pairs[:, 1]], 1).reshape(-1)
    return list(out.unbind(0))

  def PackMetricsValues(self, values):
    """Stores fetched host values back as {name: (value, weight)}."""
    vals = [float(v) for v in values]
    for i, k in enumerate(sorted(self._metrics.keys())):
      self._metrics[k] = (vals[2 * i], vals[2 * i + 1])

  @classmethod
  def ToAverageMetric(cls, value, weight=1.0) -> AverageMetric:
    m = AverageMetric()
    m.total_weight = weight
    m.total_value = weight * value
    return m

  def ToAverageMetrics(self) -> Dict[str, AverageMetric]:
    return {name: self.ToAverageMetric(value, weight)
            for name, (value, weight) in self._metrics.items()}

  def Update(self, metrics: Dict[str, Tuple[torch.Tensor, torch.Tensor]]):
    if not self._names:
      self._names = list(metrics.keys())
    vals, wts = [], []
    dev = None
    for k in self._names:
      v, w = metrics[k]
      v = torch.as_tensor(v, dtype=torch.float32)
      w = torch.as_tensor(w, dtype=torch.float32)
      if v.is_cuda:
        dev = v.device
      vals.append(v.detach().reshape(()))
      wts.append(w.detach().reshape(()))
    if dev is not None:
      vals = [v.to(dev) for v in vals]
      wts = [w.to(dev) for w in wts]
    v, w = torch.stack(vals).float(), torch.stack(wts).float()
    cur = torch.stack([v * w, w], dim=1)
    self._acc = cur if self._acc is None else self._acc + cur

  def AllReduce(self, group=None):
    import torch.distributed as dist
    if self._acc is not None and dist.is_available() and dist.is_initialized():
      dist.all_reduce(self._acc, group=group)

  def Finalize(self) -> Dict[str, Tuple[float, float]]:
    if self._acc is None:
      return {}
    acc = self._acc.cpu()
    out = {}
    for i, k in enumerate(self._names):
      s, w = float(acc[i, 0]), float(acc[i, 1])
      out[k] = (s / w if w > 0 else 0.0, w)
    return out

  def Reset(self):
    self._acc = None


TpuEvalMetrics = DeviceEvalMetrics


class DeviceVariableMetrics:
  """Fixed-capacity twin of `DeviceEvalMetrics` (ref `TpuVariableMetrics` :386): `2 *
  max_metrics` persistent device scalars (Σ value·weight, Σ weight per metric, metrics in
  sorted-name order) that a CUDA-graph-captured eval step can add into without reallocating;
  `FinalizeMetricsWithStructure` all-reduces them over the ranks and packs the averages back
  into the caller's dict structure."""

  def __init__(self, max_metrics: int, strategy=None, device=None):
    del strategy
    self._max_metrics = int(max_metrics)
    self._vars = torch.zeros(2 * self._max_metrics, dtype=torch.float32, device=device)

  @property
  def variables(self):
    return [self._vars[i] for i in range(self._vars.numel())]

  def ResetState(self):
    self._vars.zero_()

  def AccumulateStepMetrics(self, metric_dict):
    n = len(metric_dict)
    assert n <= self._max_metrics, 'Increase max_metrics to >= %d' % n
    dev = self._vars.device
    vw, w = [], []
    for _, (value, weight) in sorted(metric_dict.items()):
      value = torch.as_tensor(value, dtype=torch.float32, device=dev).reshape(())
      weight = torch.as_tensor(weight, dtype=torch.float32, device=dev).reshape(())
      vw.append(value.detach() * weight.detach())
      w.append(weight.detach())
    upd = torch.stack([torch.stack(vw), torch.stack(w)], 1).reshape(-1)
    self._vars[:2 * n] += upd

  def FinalizeMetricsWithStructure(self, structure, group=None):
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    acc = self._vars.clone()
    if dist.is_available() and dist.is_initialized():
      dist.all_reduce(acc, group=group)
    pairs = acc.reshape(-1, 2)
    out = {}
    for i, k in enumerate(sorted(structure)):
      vw, w = pairs[i, 0], pairs[i, 1]
      out[k] = (torch.where(w > 0, vw / w.clamp(min=1e-30), torch.zeros_like(vw)), w)
    return out if type(structure) is dict else type(structure)(out)   # pylint: disable=unidiomatic-typecheck


TpuVariableMetrics = DeviceVariableMetrics
