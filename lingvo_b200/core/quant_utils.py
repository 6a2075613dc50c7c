"""Quantization-aware training: `QuantizableLayer`, quantization domains and clipping schedules.

Capability parity with reference `lingvo/core/quant_utils.py`:
  * `QDistribution` (:29) — known activation distributions,
  * `QuantizableLayer` (:62) — the layer mixin whose `QWeight / QAct / QRAct / QMatmul /
    QEinsum / QConv1D / QConv2D / *Aqt*` hooks and `fns.q*` wrappers layers call
    unconditionally (identities without a qdomain, so float models pay nothing),
  * `QDomain` (:748) — the no-op domain and the interface,
  * `FakeQDomain` (:1082) — natural-range activations (tanh/softmax/relu/… ranges),
  * clipping-cap schedules `BaseClippingCapSchedule` (:1138), `IdentityClippingCapSchedule`
    (:1228), `LinearClippingCapSchedule` (:1246), `FakeQuantizationSchedule` (:1316),
  * `SymmetricScheduledClipQDomain` (:1530), `PassiveAsymQDomain` (:1606) with its counted
    min/max accumulator (:1582).

H100 notes. Everything here is elementwise device work with *no host synchronisation*:
ranges are 0-d device tensors (batch min/max, EMA state variables), the delayed-start and
clip→quantize switches are `torch.where` on values derived from the global step, and the
fake-quant op itself is a single fused expression with a straight-through gradient — so a
quantization-aware step captures into a CUDA graph like any other (the global step enters
through `py_utils.GetGlobalStep()`, which is a device tensor inside a step context).
"""

from __future__ import annotations

import enum
from typing import Iterable, Optional

import numpy as np
import torch
import torch.nn.functional as F

from lingvo_b200.core import base_layer
from lingvo_b200.core import hyperparams
from lingvo_b200.core import py_utils
from lingvo_b200.core import summary_utils


class QDistribution(str, enum.Enum):
  """Distribution of a tensor handed to a QDomain (ref :29)."""
  SYMMETRIC = 'symmetric'
  POSITIVE = 'positive'
  LOG_SOFTMAX = 'log_softmax'
  PADDING = 'padding'
  RANDOM_UNIFORM = 'random_uniform'
  RELU = 'relu'
  RELU6 = 'relu6'
  SIGMOID = 'sigmoid'
  SOFTMAX = 'softmax'
  TANH = 'tanh'

  @classmethod
  def IsPositive(cls, dist: 'QDistribution') -> bool:
    # (the reference lists TANH here too; kept for behavioural parity)
    return dist in (cls.POSITIVE, cls.PADDING, cls.RANDOM_UNIFORM, cls.RELU, cls.RELU6,
                    cls.SIGMOID, cls.SOFTMAX, cls.TANH)


# ---------------------------------------------------------------------------------------
# The fake-quant primitive.
# ---------------------------------------------------------------------------------------
def _AsTensor(v, like):
  if isinstance(v, torch.Tensor):
    return v.to(device=like.device, dtype=torch.float32)
  return torch.tensor(float(v), dtype=torch.float32, device=like.device)


def FakeQuantWithMinMax(x, min_v, max_v, num_bits=8, narrow_range=False):
  """`fake_quant_with_min_max_vars` semantics: the [min, max] range is first *nudged* so that
  0.0 is exactly representable, then x is clamped to the nudged range and rounded to one of
  2^bits (−1 if narrow) levels. Gradient: identity inside the nudged range, 0 outside
  (straight-through). min/max may be python numbers or 0-d tensors (no host sync)."""
  xf = x.float()
  lo, hi = _AsTensor(min_v, x), _AsTensor(max_v, x)
  qmin = 1.0 if narrow_range else 0.0
  qmax = float(2**num_bits - 1)
  scale = (hi - lo) / (qmax - qmin)
  safe = torch.where(scale > 0, scale, torch.ones_like(scale))
  zp = qmin - lo / safe
  nudged_zp = torch.clamp(torch.floor(zp + 0.5), qmin, qmax)
  nudged_lo = (qmin - nudged_zp) * safe
  nudged_hi = (qmax - nudged_zp) * safe
  clamped = torch.maximum(torch.minimum(xf, nudged_hi), nudged_lo)
  q = torch.floor((clamped - nudged_lo) / safe + 0.5) * safe + nudged_lo
  out = clamped + (q - clamped).detach()
  # a degenerate (empty) range quantizes everything to zero, like the TF op
  out = torch.where(scale > 0, out, torch.zeros_like(out))
  return out.to(x.dtype)


def FakeQuant(x, min_v, max_v, bits=8, narrow=False):
  """Back-compat alias of `FakeQuantWithMinMax`."""
  return FakeQuantWithMinMax(x, min_v, max_v, num_bits=bits, narrow_range=narrow)


def _StepF32(like=None):
  """Global step as a float32 0-d tensor (device tensor inside graph-captured steps)."""
  gs = py_utils.GetGlobalStep()
  if isinstance(gs, torch.Tensor):
    return gs.to(torch.float32)
  dev = like.device if isinstance(like, torch.Tensor) else 'cpu'
  return torch.tensor(float(gs), dtype=torch.float32, device=dev)


class _Fns:
  """Attribute view over a layer's function library (`layer.fns.qadd(...)`)."""

  def __init__(self, table):
    self._table = table

  def __getattr__(self, name):
    try:
      return self._table[name]
    except KeyError:
      raise AttributeError(name) from None

  def __getitem__(self, name):
    return self._table[name]

  def __contains__(self, name):
    return name in self._table

  def __dir__(self):
    return sorted(self._table)


# ---------------------------------------------------------------------------------------
# QuantizableLayer
# ---------------------------------------------------------------------------------------
class QuantizableLayer(base_layer.BaseLayer):
  """Layer base with quantization tags (ref :62).

  Tags: `QWeight(w)` for weights, `QAct(name, act)` for tracked intermediate activations,
  `QRAct(act, dist)` for activations with a natural range. `p.qdomain.<name>` associates
  QDomain params with the layer; 'default' is used for any domain left as None.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('qdomain', hyperparams.Params(), 'Container for quantization domains.')
    p.qdomain.Define('default', None, 'Default quantization domain.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self._all_names = set()
    self._act_name_to_qdomain_name = {}
    self._weight_name_to_qdomain_name = {}
    self._qdomains = {}
    for qdname, qdparams in p.qdomain.IterParams():
      if qdparams is None:
        self._qdomains[qdname] = None
        continue
      if not issubclass(qdparams.cls, QDomain):
        raise TypeError('Expected p.qdomain.%s to extend QDomain, but got %s' %
                        (qdname, qdparams.cls))
      child = 'qdomain_' + qdname
      self.CreateChild(child, qdparams.Copy().Set(name=child))
      self._qdomains[qdname] = self.children[child]
    self._AddQuantizationFunctions()

  @property
  def fns(self):
    return _Fns(self._private_fns)

  # -- tracking ----------------------------------------------------------------------
  def TrackQActs(self, *act_names: str, shape: Optional[Iterable[int]] = None,
                 feature_axes: Optional[Iterable[int]] = None, domain: str = 'default'):
    """Declares activation names (ref :177); the domain allocates its range state."""
    for act_name in act_names:
      if act_name in self._all_names:
        raise ValueError("act_name='%s' is already tracked for this layer." % act_name)
      self._all_names.add(act_name)
      self._act_name_to_qdomain_name[act_name] = domain
    qd = self._GetQDomain(domain)
    if qd is not None:
      qd.TrackQActs(*act_names, shape=shape, feature_axes=feature_axes)

  def TrackQTensor(self, *t_names, **kwargs):
    """Older spelling of `TrackQActs`."""
    return self.TrackQActs(*t_names, domain=kwargs.get('domain', 'default'))

  def TrackQWeight(self, weight_name, shape=None, feature_axis=-1, domain: str = 'default', *,
                   tensor_split_dims_mapping=None, device_mesh=None,
                   legacy_aqt_weight_name=None):
    """Declares a weight that the AQT hooks will quantize (ref :209)."""
    if weight_name in self._all_names:
      raise ValueError("weight_name='%s' is already tracked for this layer." % weight_name)
    self._all_names.add(weight_name)
    self._weight_name_to_qdomain_name[weight_name] = domain
    qd = self._GetQDomain(domain)
    if qd is not None:
      qd.TrackQWeight(weight_name, shape, feature_axis, tensor_split_dims_mapping,
                      device_mesh, legacy_aqt_weight_name)

  # -- tags --------------------------------------------------------------------------
  def QAct(self, act_name, act, eval_only=False):
    if act_name not in self._act_name_to_qdomain_name:
      raise ValueError("The given act_name='%s' must first be tracked using TrackQActs. "
                       'Expected one of %s' % (act_name, sorted(self._act_name_to_qdomain_name)))
    qd = self._GetQDomain(self._act_name_to_qdomain_name[act_name])
    return act if qd is None else qd.QuantizeAct(act_name, act, eval_only=eval_only)

  QTensor = QAct

  def QTensorMulti(self, t_name, *ts):
    return tuple(self.QAct(t_name, t) for t in ts)

  def QWeight(self, w, domain: str = 'default'):
    qd = self._GetQDomain(domain)
    return qd.QuantizeWeight(w) if qd is not None else w

  def QRAct(self, act, dist: QDistribution, domain: str = 'default'):
    qd = self._GetQDomain(domain)
    return act if qd is None else qd.QRAct(act, dist)

  # convenience spellings used across the layer library
  def QRTanh(self, x, domain='default'):
    return self.QRAct(torch.tanh(x), QDistribution.TANH, domain)

  def QRSigmoid(self, x, domain='default'):
    return self.QRAct(torch.sigmoid(x), QDistribution.SIGMOID, domain)

  def QRRelu(self, x, domain='default'):
    return self.QRAct(torch.relu(x), QDistribution.RELU, domain)

  def QRSoftmax(self, logits, dim=-1, domain='softmax'):
    return self.QRAct(torch.softmax(logits, dim=dim), QDistribution.SOFTMAX, domain)

  def QRPadding(self, paddings, domain='default'):
    return self.QRAct(paddings, QDistribution.PADDING, domain)

  def _ValidateArgName(self, op_arg_name, name):
    if name is not None and name not in self._all_names:
      raise ValueError("Expected %s='%s' to be None or one of %s. Use TrackQActs or "
                       'TrackQWeight to create it' % (op_arg_name, name, sorted(self._all_names)))

  def QMatmul(self, lhs, rhs, *, lhs_name=None, rhs_name=None,
              lhs_dist=QDistribution.SYMMETRIC, rhs_dist=QDistribution.SYMMETRIC,
              ensure2d=False, qdomain='default', **op_kwargs):
    self._ValidateArgName('lhs_name', lhs_name)
    self._ValidateArgName('rhs_name', rhs_name)
    qd = self._GetQDomain(qdomain)
    if qd is None:
      return torch.matmul(lhs, rhs)
    return qd.QMatmul(lhs, rhs, lhs_name=lhs_name, rhs_name=rhs_name, lhs_dist=lhs_dist,
                      rhs_dist=rhs_dist, ensure2d=ensure2d, **op_kwargs)

  def QEinsum(self, equation, lhs, rhs, *, lhs_name=None, rhs_name=None,
              lhs_dist=QDistribution.SYMMETRIC, rhs_dist=QDistribution.SYMMETRIC,
              qdomain='default'):
    self._ValidateArgName('lhs_name', lhs_name)
    self._ValidateArgName('rhs_name', rhs_name)
    qd = self._GetQDomain(qdomain)
    if qd is None:
      return torch.einsum(equation, lhs, rhs)
    return qd.QEinsum(equation, lhs, rhs, lhs_name=lhs_name, rhs_name=rhs_name,
                      lhs_dist=lhs_dist, rhs_dist=rhs_dist)

  def QConv1D(self, inputs, filters, strides, padding, *, inputs_name=None, filters_name=None,
              inputs_dist=QDistribution.SYMMETRIC, filters_dist=QDistribution.SYMMETRIC,
              qdomain='default'):
    """inputs [B, T, Cin], filters [K, Cin, Cout] (TF layouts)."""
    self._ValidateArgName('inputs_name', inputs_name)
    self._ValidateArgName('filters_name', filters_name)
    qd = self._GetQDomain(qdomain) or _NOOP
    return qd.QConv1D(inputs, filters, strides, padding, inputs_name=inputs_name,
                      filters_name=filters_name, inputs_dist=inputs_dist,
                      filters_dist=filters_dist)

  def QConv2D(self, inputs, filters, strides, padding, *, inputs_name=None, filters_name=None,
              inputs_dist=QDistribution.SYMMETRIC, filters_dist=QDistribution.SYMMETRIC,
              is_depthwise=False, qdomain='default'):
    """inputs [B, H, W, Cin], filters [KH, KW, Cin, Cout | mult] (TF layouts)."""
    self._ValidateArgName('inputs_name', inputs_name)
    self._ValidateArgName('filters_name', filters_name)
    qd = self._GetQDomain(qdomain) or _NOOP
    return qd.QConv2D(inputs, filters, strides, padding, inputs_name=inputs_name,
                      filters_name=filters_name, inputs_dist=inputs_dist,
                      filters_dist=filters_dist, is_depthwise=is_depthwise)

  # -- AQT-style (scale → round → clip, rescale the output) ------------------------
  def _ValidateWeight(self, w_name):
    if w_name not in self._weight_name_to_qdomain_name:
      raise ValueError("The given w_name='%s' must first be tracked using TrackQWeight. "
                       'Expected one of %s' %
                       (w_name, sorted(self._weight_name_to_qdomain_name)))
    return self._GetQDomain(self._weight_name_to_qdomain_name[w_name])

  def ToAqtWeight(self, w_name, w, feature_axis=-1, expected_scale_shape=None):
    qd = self._ValidateWeight(w_name)
    if qd is None:
      return w
    return qd.ToAqtWeight(w_name, w, feature_axis=feature_axis,
                          expected_scale_shape=expected_scale_shape)

  def FromAqtWeight(self, w_name, out, merge_feature_axes=False):
    qd = self._ValidateWeight(w_name)
    return out if qd is None else qd.FromAqtWeight(w_name, out, merge_feature_axes)

  def ToAqtInputs(self, w_name, act, weight, w_feature_axis=-1,
                  act_distribution=QDistribution.SYMMETRIC, w_expected_scale_shape=None):
    qd = self._ValidateWeight(w_name)
    if qd is None:
      return act, weight
    return qd.ToAqtInputs(w_name, act=act, weight=weight, w_feature_axis=w_feature_axis,
                          act_distribution=act_distribution,
                          w_expected_scale_shape=w_expected_scale_shape)

  def FromAqtMatmul(self, w_name, output):
    qd = self._ValidateWeight(w_name)
    return output if qd is None else qd.FromAqtMatmul(w_name, output)

  def ToAqtConv(self, w_name, act, weight, w_feature_axis=-1,
                act_distribution=QDistribution.SYMMETRIC, w_expected_scale_shape=None):
    qd = self._ValidateWeight(w_name)
    if qd is None:
      return act, weight
    return qd.ToAqtConv(w_name, act=act, weight=weight, w_feature_axis=w_feature_axis,
                        act_distribution=act_distribution,
                        w_expected_scale_shape=w_expected_scale_shape)

  def FromAqtConv(self, w_name, output, *, is_depthwise=False):
    qd = self._ValidateWeight(w_name)
    return output if qd is None else qd.FromAqtConv(w_name, output, is_depthwise=is_depthwise)

  def ToAqtActActInputs(self, act_lhs, act_rhs, *, act_lhs_distribution=QDistribution.SYMMETRIC,
                        act_rhs_distribution=QDistribution.SYMMETRIC, domain='default'):
    qd = self._GetQDomain(domain)
    if qd is None:
      return act_lhs, act_rhs
    return qd.ToAqtActActInputs(act_lhs=act_lhs, act_rhs=act_rhs,
                                act_lhs_distribution=act_lhs_distribution,
                                act_rhs_distribution=act_rhs_distribution)

  def FromAqtActActMatmul(self, output, domain='default'):
    qd = self._GetQDomain(domain)
    return output if qd is None else qd.FromAqtActActMatmul(output)

  # -- domain lookup -----------------------------------------------------------------
  def _GetQDomain(self, domain: str):
    qd = self._qdomains.get(domain)
    return qd if qd is not None else self._qdomains.get('default')

  _QDomain = _GetQDomain

  def GetQDomainParams(self, domain: str = 'default'):
    p = self.params
    qdparams = p.qdomain.Get(domain) if domain in p.qdomain else None
    return p.qdomain.default if qdparams is None else qdparams

  # -- fns library (ref :707-744) ---------------------------------------------------
  def _AddQuantizationFunctions(self):

    def WrapOp(op_name, op, dist=None):

      def Wrapped(*op_args, qout_name=None, qdomain='default', **op_kwargs):
        if qout_name is None and dist is None:
          raise ValueError('Quantized op "%s" requires qout_name to be set.' % op_name)
        op_kwargs.pop('name', None)
        y = op(*op_args, **op_kwargs)
        if qout_name is not None:
          return self.QAct(qout_name, y)
        return self.QRAct(y, dist, qdomain)

      self.AddFunction(op_name, Wrapped)

    def Conv1D(x, w, stride=1, padding='SAME'):
      return _NOOP.QConv1D(x, w, stride, padding, inputs_name=None, filters_name=None)

    # dynamic-range ops: the output range is tracked by name
    WrapOp('qadd', torch.add)
    WrapOp('qsubtract', torch.sub)
    WrapOp('qmultiply', torch.mul)
    WrapOp('qlog', torch.log)
    WrapOp('qmatmul', lambda a, b: torch.matmul(a.reshape(-1, a.shape[-1]), b).reshape(
        *a.shape[:-1], b.shape[-1]))
    WrapOp('qbatchmatmul', torch.matmul)
    WrapOp('qconv1d', Conv1D)
    # natural-range ops
    WrapOp('qtanh', torch.tanh, dist=QDistribution.TANH)
    WrapOp('qsigmoid', torch.sigmoid, dist=QDistribution.SIGMOID)
    WrapOp('qsoftmax', lambda x, dim=-1: torch.softmax(x, dim=dim), dist=QDistribution.SOFTMAX)
    WrapOp('qlogsigmoid', F.logsigmoid, dist=QDistribution.LOG_SOFTMAX)
    WrapOp('qlogsoftmax', lambda x, dim=-1: torch.log_softmax(x, dim=dim),
           dist=QDistribution.LOG_SOFTMAX)
    WrapOp('qrelu', torch.relu, dist=QDistribution.RELU)
    WrapOp('qrelu6', F.relu6, dist=QDistribution.RELU6)
    WrapOp('qrandom_uniform', lambda shape, **kw: torch.rand(*shape, **kw),
           dist=QDistribution.RANDOM_UNIFORM)


# ---------------------------------------------------------------------------------------
# Domains
# ---------------------------------------------------------------------------------------
def _TfPad1D(x, k, stride, padding):
  if padding == 'SAME':
    t = x.shape[-1]
    total = max((-(-t // stride) - 1) * stride + k - t, 0)
    return F.pad(x, (total // 2, total - total // 2))
  return x


class QDomain(base_layer.BaseLayer):
  """Base quantization domain; doubles as the no-op domain (ref :748)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.name = 'qdomain'
    return p

  def __init__(self, params):
    super().__init__(params)
    self.all_names = set()
    self.act_names = set()
    self.weight_names = set()

  @property
  def bits(self):
    """Bits of this domain, None if unquantized."""
    return None

  def QuantizeWeight(self, w):
    return w

  def QRAct(self, act, dist: QDistribution):
    del dist
    return act

  def QuantizeAct(self, act_name: str, act, eval_only: bool = False):
    return act

  def QuantizeConstantRange(self, t, min_value, max_value):
    """A true-constant range not used arithmetically (e.g. paddings)."""
    return t

  def QuantizeNaturalRange(self, t, min_value, max_value):
    return t

  def QMatmul(self, lhs, rhs, *, lhs_name=None, rhs_name=None,
              lhs_dist=QDistribution.SYMMETRIC, rhs_dist=QDistribution.SYMMETRIC,
              out_name=None, ensure2d=False, **op_kwargs):
    del lhs_name, rhs_name, lhs_dist, rhs_dist, out_name, ensure2d, op_kwargs
    return torch.matmul(lhs, rhs)

  def QEinsum(self, equation, lhs, rhs, *, lhs_name=None, rhs_name=None,
              lhs_dist=QDistribution.SYMMETRIC, rhs_dist=QDistribution.SYMMETRIC):
    del lhs_name, rhs_name, lhs_dist, rhs_dist
    return torch.einsum(equation, lhs, rhs)

  def QConv1D(self, inputs, filters, strides, padding, *, inputs_name=None, filters_name=None,
              inputs_dist=QDistribution.SYMMETRIC, filters_dist=QDistribution.SYMMETRIC):
    del inputs_name, filters_name, inputs_dist, filters_dist
    stride = strides if isinstance(strides, int) else int(strides[0])
    x = _TfPad1D(inputs.transpose(1, 2), filters.shape[0], stride, padding)
    return F.conv1d(x, filters.permute(2, 1, 0), stride=stride).transpose(1, 2)

  def QConv2D(self, inputs, filters, strides, padding, *, inputs_name=None, filters_name=None,
              inputs_dist=QDistribution.SYMMETRIC, filters_dist=QDistribution.SYMMETRIC,
              is_depthwise=False):
    del inputs_name, filters_name, inputs_dist, filters_dist
    if isinstance(strides, int):
      strides = (strides, strides)
    strides = tuple(strides)[-3:-1] if len(strides) == 4 else tuple(strides)
    kh, kw, cin, cout = filters.shape
    x = inputs.permute(0, 3, 1, 2)
    if padding == 'SAME':
      h, w = x.shape[-2:]
      ph = max((-(-h // strides[0]) - 1) * strides[0] + kh - h, 0)
      pw = max((-(-w // strides[1]) - 1) * strides[1] + kw - w, 0)
      x = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
    if is_depthwise:
      wt = filters.permute(2, 3, 0, 1).reshape(cin * cout, 1, kh, kw)
      y = F.conv2d(x, wt, stride=strides, groups=cin)
    else:
      y = F.conv2d(x, filters.permute(3, 2, 0, 1), stride=strides)
    return y.permute(0, 2, 3, 1)

  # AQT hooks: no-ops for domains that emulate quantization with fake-quant ops
  def ToAqtWeight(self, w_name, w, feature_axis, expected_scale_shape=None):
    del w_name, feature_axis, expected_scale_shape
    return w

  def FromAqtWeight(self, w_name, out, merge_feature_axes=False):
    del w_name, merge_feature_axes
    return out

  def ToAqtInputs(self, w_name, act, weight, w_feature_axis,
                  act_distribution=QDistribution.SYMMETRIC, w_expected_scale_shape=None):
    del w_name, w_feature_axis, act_distribution, w_expected_scale_shape
    return act, weight

  def FromAqtMatmul(self, w_name, output):
    del w_name
    return output

  def ToAqtConv(self, w_name, act, weight, w_feature_axis,
                act_distribution=QDistribution.SYMMETRIC, w_expected_scale_shape=None):
    del w_name, w_feature_axis, act_distribution, w_expected_scale_shape
    return act, weight

  def FromAqtConv(self, w_name, output, *, is_depthwise=False):
    del w_name, is_depthwise
    return output

  def ToAqtActActInputs(self, act_lhs, act_rhs, act_lhs_distribution=QDistribution.SYMMETRIC,
                        act_rhs_distribution=QDistribution.SYMMETRIC):
    del act_lhs_distribution, act_rhs_distribution
    return act_lhs, act_rhs

  def FromAqtActActMatmul(self, output):
    return output

  def TrackQActs(self, *act_names: str, shape=None, feature_axes=None):
    for act_name in act_names:
      if act_name in self.all_names:
        raise ValueError("act_name '%s' is already tracked for this qdomain." % act_name)
      self.all_names.add(act_name)
      self.act_names.add(act_name)

  def TrackQWeight(self, weight_name, shape, feature_axis, tensor_split_dims_mapping=None,
                   device_mesh=None, legacy_aqt_weight_name=None):
    if weight_name in self.all_names:
      raise ValueError("weight_name '%s' is already tracked for this qdomain." % weight_name)
    self.all_names.add(weight_name)
    self.weight_names.add(weight_name)

  def FProp(self, theta, x):
    return x


_NOOP = QDomain(QDomain.Params().Set(name='noop_qdomain'))


class FakeQDomain(QDomain):
  """Base of the fake-quant domains: maps known distributions to natural ranges (ref :1082)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('narrow_to_asym_bit_depth', True,
             'Narrow the softmax / tanh upper bound by one quantum (TFLite convention).')
    p.Define('log_softmax_range', None,
             'Manual (min, max) for log-softmax activations, or None.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    if not (p.log_softmax_range is None or len(p.log_softmax_range) == 2):
      raise ValueError('p.log_softmax_range=%s should be None or a sequence of two numbers' %
                       (p.log_softmax_range,))

  def _MaybeNarrowToAsymBitDepth(self, qmin, qmax):
    if self.params.narrow_to_asym_bit_depth:
      qrange = qmax - qmin
      qmax = qmin + qrange * (2**self.bits - 1) / (2**self.bits)
    return qmin, qmax

  def QRAct(self, act, dist: QDistribution):
    p = self.params
    dist = QDistribution(dist)
    if dist == QDistribution.LOG_SOFTMAX:
      if p.log_softmax_range is None:
        raise ValueError('p.log_softmax_range must be set to quantize a log-softmax '
                         'activation without a tracked output name')
      return self.QuantizeNaturalRange(act, *p.log_softmax_range)
    if dist == QDistribution.PADDING:
      return self.QuantizeConstantRange(act, 0.0, 1.0)
    if dist in (QDistribution.RELU, QDistribution.SIGMOID, QDistribution.RANDOM_UNIFORM):
      return self.QuantizeNaturalRange(act, 0.0, 1.0)
    if dist == QDistribution.RELU6:
      return self.QuantizeNaturalRange(act, 0.0, 6.0)
    if dist == QDistribution.SOFTMAX:
      return self.QuantizeNaturalRange(act, *self._MaybeNarrowToAsymBitDepth(0.0, 1.0))
    if dist == QDistribution.TANH:
      return self.QuantizeNaturalRange(act, *self._MaybeNarrowToAsymBitDepth(-1.0, 1.0))
    raise ValueError('cannot quantize act with dist=%s to a known range' % dist)


# ---------------------------------------------------------------------------------------
# Clipping-cap schedules
# ---------------------------------------------------------------------------------------
class BaseClippingCapSchedule(base_layer.BaseLayer):
  """Interface of a clipping-cap schedule (ref :1138)."""

  @property
  def is_quantized(self):
    return False

  @property
  def bits(self):
    return None

  def GetEndRange(self):
    """The ideal final (min, max), before bit-depth adjustment."""
    raise NotImplementedError('Abstract method: GetEndRange')

  def GetQuantizedEndRange(self):
    assert not self.is_quantized
    return self.GetEndRange()

  def ApplyConstantClip(self, x, min_value, max_value):
    raise NotImplementedError('Abstract method: ApplyConstantClip')

  def GetState(self, theta):
    """Opaque float32 state tensor for `ApplyClippingWithState`."""
    raise NotImplementedError('Abstract method: GetState')

  def ApplyClipping(self, theta, x, **kwargs):
    return self.ApplyClippingWithState(self.GetState(theta), x, **kwargs)

  def ApplyClippingWithState(self, state, x):
    raise NotImplementedError('Abstract method: ApplyClippingWithState')


class IdentityClippingCapSchedule(BaseClippingCapSchedule):
  """A schedule that never clips (ref :1228)."""

  def GetEndRange(self):
    info = torch.finfo(self.params.dtype if isinstance(self.params.dtype, torch.dtype)
                       else torch.float32)
    return (info.min, info.max)

  def ApplyConstantClip(self, x, min_value, max_value):
    return x

  def GetState(self, theta):
    return torch.zeros([1], dtype=torch.float32)

  def ApplyClippingWithState(self, state, x):
    return x


class LinearClippingCapSchedule(BaseClippingCapSchedule):
  """Cap decays linearly from start_cap to end_cap over [start_step, end_step] (ref :1246)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.name = 'CCSchedule'
    p.Define('start_step', 0, 'Step at which the cap starts narrowing.')
    p.Define('end_step', 15000, 'Step at which the cap reaches end_cap.')
    p.Define('start_cap', 8.0, 'Clipping range at the start of training.')
    p.Define('end_cap', 1.0, 'Clipping range towards the end of training.')
    return p

  def ApplyConstantClip(self, x, min_value, max_value):
    return torch.clamp(x, min_value, max_value)

  def GetState(self, theta):
    return self._Value()

  def ApplyClippingWithState(self, state, x):
    cap = state.to(device=x.device, dtype=x.dtype)
    return torch.maximum(torch.minimum(x, cap), -cap)

  def GetEndRange(self):
    return (-self.params.end_cap, self.params.end_cap)

  def _Value(self):
    p = self.params
    step = _StepF32()
    span = float(p.end_step - p.start_step)
    ratio = torch.clamp(step - p.start_step, max=span) / span
    cap = ratio * p.end_cap + (1.0 - ratio) * p.start_cap
    return torch.where(step < p.start_step, torch.full_like(cap, float(p.start_cap)), cap)

  def Value(self, step=None):
    """Python-float cap at `step` (host-side inspection / summaries)."""
    if step is None:
      return float(self._Value())
    with py_utils.GlobalStepContext(int(step)):
      return float(self._Value())


class FakeQuantizationSchedule(BaseClippingCapSchedule):
  """Clip-then-quantize schedule (ref :1316): the cap ramps start_cap → end_cap over
  [clip_start_step, clip_end_step]; from quant_start_step on, values are fake-quantized to
  `bits` inside the (bit-depth adjusted) cap instead of only clipped."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.name = 'FQSchedule'
    p.Define('clip_start_step', 0, 'Step at which the cap starts narrowing.')
    p.Define('clip_end_step', 15000, 'Step at which the cap reaches end_cap.')
    p.Define('quant_start_step', 15000, 'Step at which quantization starts.')
    p.Define('start_cap', 8.0, 'Default clipping/quant start cap.')
    p.Define('end_cap', 1.0, 'Default clipping/quant end cap.')
    p.Define('bits', 8, 'Default quantized bit depth.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.quant_start_step >= p.clip_end_step, 'quant_start_step must be >= clip_end_step'

  @property
  def is_quantized(self):
    return True

  @property
  def bits(self):
    return self.params.bits

  def GetEndRange(self):
    p = self.params
    return (-p.end_cap, p.end_cap)

  def GetQuantizedEndRange(self, end_cap=None, bits=None):
    p = self.params
    return self._GetQuantizedRangeForCap(p.end_cap if end_cap is None else end_cap,
                                         p.bits if bits is None else bits)

  def ApplyConstantClip(self, x, min_value, max_value):
    return FakeQuantWithMinMax(x, min_value, max_value, num_bits=self.params.bits)

  def GetState(self, theta):
    """[clip_ratio, fq_ratio]: clip_ratio < 0 before clip_start_step (no clipping yet),
    rises to 1 at clip_end_step; fq_ratio is −1 before quant_start_step, +1 after."""
    p = self.params
    if p.is_inference:
      return torch.zeros([1], dtype=torch.float32)
    step = _StepF32()
    span = float(p.clip_end_step - p.clip_start_step)
    clip_ratio = torch.clamp(step - p.clip_start_step, max=span) / max(1.0, span)
    fq_ratio = torch.where(step < p.quant_start_step, -torch.ones_like(step),
                           torch.ones_like(step))
    return torch.stack([clip_ratio, fq_ratio])

  @staticmethod
  def _GetQuantizedRangeForCap(current_cap, bits):
    dt_max = 2**(bits - 1)            # 8 bit → 128: the positive side has one level less
    return -current_cap, current_cap * (dt_max - 1) / dt_max

  def _GetCurrentMinMax(self, state, start_cap, end_cap, bits, fixate_to_end_state=False):
    if fixate_to_end_state:
      current_cap = end_cap
    else:
      clip_ratio = state[0]
      current_cap = clip_ratio * end_cap + (1.0 - clip_ratio) * start_cap
    return self._GetQuantizedRangeForCap(current_cap, bits)

  def ApplyClippingWithState(self, state, x, start_cap=None, end_cap=None, bits=None):
    p = self.params
    start_cap = p.start_cap if start_cap is None else start_cap
    end_cap = p.end_cap if end_cap is None else end_cap
    bits = p.bits if bits is None else bits
    if p.is_inference:
      lo, hi = self._GetCurrentMinMax(state, start_cap, end_cap, bits, fixate_to_end_state=True)
      return FakeQuantWithMinMax(x, lo, hi, num_bits=bits)
    state = state.to(x.device)
    lo, hi = self._GetCurrentMinMax(state, start_cap, end_cap, bits)
    lo, hi = lo.detach(), hi.detach()
    clipped = torch.where(state[0] >= 0.0,
                          torch.maximum(torch.minimum(x, hi.to(x.dtype)), lo.to(x.dtype)), x)
    quantized = FakeQuantWithMinMax(x, lo, hi, num_bits=bits)
    return torch.where(state[1] <= 0.0, clipped, quantized)

  def Value(self, step=None):
    """(cap, quantizing?) as python values at `step` — host-side inspection."""
    p = self.params
    ctx = py_utils.GlobalStepContext(int(step)) if step is not None else None
    if ctx is not None:
      ctx.__enter__()
    try:
      st = self.GetState(self.theta)
      ratio = max(float(st[0]), 0.0)
      return ratio * p.end_cap + (1.0 - ratio) * p.start_cap, bool(float(st[1]) > 0)
    finally:
      if ctx is not None:
        ctx.__exit__(None, None, None)


# ---------------------------------------------------------------------------------------
# Concrete domains
# ---------------------------------------------------------------------------------------
class SymmetricScheduledClipQDomain(FakeQDomain):
  """Symmetric scheduled clipping via a clipping-cap schedule (ref :1530); suited to layers
  known to tolerate operating inside fixed ranges (LSTM cells)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('cc_schedule', FakeQuantizationSchedule.Params(), 'Quantization clipping schedule.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self.CreateChild('cc_schedule', self.params.cc_schedule)

  @property
  def bits(self):
    return self.cc_schedule.bits

  def QuantizeWeight(self, w):
    return self.cc_schedule.ApplyClipping(self.cc_schedule.theta, w)

  def QuantizeNaturalRange(self, t, min_value, max_value):
    return self.cc_schedule.ApplyClipping(self.cc_schedule.theta, t)

  def QuantizeConstantRange(self, t, min_value, max_value):
    return torch.clamp(t, min_value, max_value)

  def QuantizeAct(self, act_name, act, eval_only=False):
    if eval_only and not self.do_eval:
      return act
    return self.cc_schedule.ApplyClipping(self.cc_schedule.theta, act)


class _CountedMinMaxAccumulator(base_layer.Accumulator):
  """[count, min, max]; every update adds to the count and widens min/max (ref :1582)."""

  def __init__(self, dtype=torch.float32, device='cpu'):
    super().__init__()
    self.dtype = dtype if isinstance(dtype, torch.dtype) else torch.float32
    self.device = device

  def DefaultValue(self):
    return torch.zeros([3], dtype=self.dtype, device=self.device)

  def Update(self, new_value):
    if self.is_disabled:
      return
    self.device = new_value.device
    state0 = self.GetValue().to(new_value.device)
    self.SetValue(torch.stack([state0[0] + new_value[0],
                               torch.minimum(state0[1], new_value[1]),
                               torch.maximum(state0[2], new_value[2])]))


class PassiveAsymQDomain(FakeQDomain):
  """Passive asymmetric quantization (ref :1606; arXiv:1712.05877): batch min/max drive the
  training-time fake-quant; an EMA of them is recorded in `<act>_min/_max` state variables
  after every step and used at eval / inference time."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('bits', 8, 'Default quantized bit depth.')
    p.Define('ema_decay', 0.99, 'Moving average decay.')
    p.Define('default_min', -1.0, 'Initial minimum of a tracked activation.')
    p.Define('default_max', 1.0, 'Initial maximum of a tracked activation.')
    p.Define('quantize_weight_epsilon', 0.0,
             'Weights ranges are widened to at least ±epsilon (prevents an empty range).')
    p.Define('delay_start_steps', 0,
             'Training-time quantization starts after this many steps (0 = immediately, '
             '-1 = never). Eval is not affected.')
    p.Define('freeze', False, 'Freeze the recorded ranges.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self._qvars = {}

  @property
  def bits(self):
    return self.params.bits

  def _MaybeFakeQuant(self, inputs, min_v, max_v, num_bits):
    p = self.params
    if p.delay_start_steps != 0 and not self.do_eval:
      if p.delay_start_steps == -1:
        return inputs
      q = FakeQuantWithMinMax(inputs, min_v, max_v, num_bits=num_bits)
      step = _StepF32(inputs).to(inputs.device)
      return torch.where(step >= p.delay_start_steps, q, inputs)
    return FakeQuantWithMinMax(inputs, min_v, max_v, num_bits=num_bits)

  def QuantizeWeight(self, w):
    p = self.params
    wd = w.detach().float()
    w_min = torch.clamp(wd.min(), max=-p.quantize_weight_epsilon)
    w_max = torch.clamp(wd.max(), min=p.quantize_weight_epsilon)
    quant_w = self._MaybeFakeQuant(w, w_min, w_max, num_bits=p.bits)
    if self.do_eval:
      return quant_w
    return torch.where(torch.isnan(quant_w), w, quant_w)

  def QuantizeNaturalRange(self, t, min_value, max_value):
    return self._MaybeFakeQuant(t, min_value, max_value, num_bits=self.params.bits)

  def QuantizeConstantRange(self, t, min_value, max_value):
    return self._MaybeFakeQuant(t, min_value, max_value, num_bits=self.params.bits)

  def TrackQActs(self, *act_names, shape=None, feature_axes=None):
    super().TrackQActs(*act_names, shape=shape, feature_axes=feature_axes)
    p = self.params
    for act_name in act_names:
      self.RegisterAccumulator(self._GetAccumulatorNameForTensor(act_name),
                               _CountedMinMaxAccumulator(p.dtype))
      for suffix, init in (('min', p.default_min), ('max', p.default_max)):
        name = self._GetQStateVarName(act_name, suffix)
        assert name not in self._qvars, 'QState var already exists: %s' % name
        self.CreateVariable(
            name, py_utils.WeightParams((), py_utils.WeightInit.Constant(init), p.dtype),
            trainable=False)
        self._qvars[name] = name

  def _GetAccumulatorNameForTensor(self, act_name):
    return 'qact_%s' % act_name

  @staticmethod
  def _GetQStateVarName(act_name, suffix):
    return '%s_%s' % (act_name, suffix)

  def _GetQStateVar(self, act_name, suffix):
    return self.vars[self._qvars[self._GetQStateVarName(act_name, suffix)]]

  def QuantizeAct(self, act_name, act, eval_only=False):
    p = self.params
    if self.do_eval:
      return self._MaybeFakeQuant(act, self._GetQStateVar(act_name, 'min').data,
                                  self._GetQStateVar(act_name, 'max').data, num_bits=p.bits)
    ad = act.detach().float()
    batch_min = torch.clamp(ad.min(), max=0.0)
    batch_max = torch.clamp(ad.max(), min=0.0)
    acc = self._private_accumulators[self._GetAccumulatorNameForTensor(act_name)]
    acc.Update(torch.stack([torch.ones_like(batch_min), batch_min, batch_max]))
    if eval_only:
      return act
    quant_act = self._MaybeFakeQuant(act, batch_min, batch_max, num_bits=p.bits)
    return torch.where(torch.isnan(quant_act), act, quant_act)

  def PostTrainingStepUpdate(self):
    super().PostTrainingStepUpdate()
    if self.params.freeze or self.do_eval:
      return
    for act_name in sorted(self.act_names):
      self._RecordTensor(act_name)
      self._SummarizeTensor(act_name)

  def _RecordTensor(self, act_name):
    """EMA-folds the accumulated [count, min, max] into the state variables (ref :1803)."""
    p = self.params
    acc = self._private_accumulators[self._GetAccumulatorNameForTensor(act_name)]
    cur = acc.GetValue()
    acc.Reset()
    min_var = self._GetQStateVar(act_name, 'min')
    max_var = self._GetQStateVar(act_name, 'max')
    cur = cur.to(min_var.device)
    seen = cur[0] > 0
    with torch.no_grad():
      zero = torch.zeros_like(min_var.data)
      dmin = torch.where(seen, (1.0 - p.ema_decay) * (min_var.data - cur[1]), zero)
      dmax = torch.where(seen, (1.0 - p.ema_decay) * (max_var.data - cur[2]), zero)
      min_var.data.copy_(torch.clamp(min_var.data - dmin, max=0.0))
      max_var.data.copy_(torch.clamp(max_var.data - dmax, min=0.0))

  def _SummarizeTensor(self, act_name):
    summary_utils.scalar('%s/%s_min' % (self.path, act_name),
                         self._GetQStateVar(act_name, 'min').data)
    summary_utils.scalar('%s/%s_max' % (self.path, act_name),
                         self._GetQStateVar(act_name, 'max').data)


def GetQuantizedNumpyRange(bits, cap):
  """Host helper: the representable values of a symmetric `bits` grid with cap `cap`."""
  lo, hi = FakeQuantizationSchedule._GetQuantizedRangeForCap(cap, bits)  # pylint: disable=protected-access
  return np.linspace(lo, hi, 2**bits)
