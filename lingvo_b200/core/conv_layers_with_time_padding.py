"""Padding-aware conv layers over `[B, T, F, C]` (ref
`lingvo/core/conv_layers_with_time_padding.py`).

Every layer takes `(inputs [B,T,F,C], paddings [B,T])`, zeroes padded frames
before convolving, and returns `(outputs, out_paddings)` where the output
padding is the max-pool of the input padding over the conv window (ref :76,
:150). Causal variants pad `(k−1)·dilation` frames on the left only (ref :119)
and support `StreamStep` with a `(k−1)·dilation`-frame rolling context.

NHWC activations are kept as-is (channels-last is what cuDNN/our depthwise
kernel want on H100); weights keep the reference's `[h, w, in, out]` layout.
"""

from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from lingvo_b200.core import base_layer
from lingvo_b200.core import bn_layers
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.core.py_utils import WeightInit
from lingvo_b200.core.py_utils import WeightParams


def ComputeConvOutputShape(in_shape, t_stride, f_stride, outc=None,
                           padding='SAME'):
  """[B,T,F,C] → output shape under SAME/VALID (ref :36)."""
  n, t, f, c = in_shape
  def _Out(x, s):
    if x is None:
      return None
    return -(-x // s) if padding == 'SAME' else x // s
  return [n, _Out(t, t_stride), _Out(f, f_stride), outc if outc is not None else c]


def _ComputeConvOutputPaddingV2(paddings, window, stride, padding_algorithm='SAME'):
  """Output frame is padding iff its window's *centre-aligned* input is (ref :150)."""
  if stride == 1 and padding_algorithm == 'SAME':
    return paddings
  b, t = paddings.shape
  if padding_algorithm == 'SAME':
    out_t = -(-t // stride)
    total = max((out_t - 1) * stride + window - t, 0)
    left = total // 2
    centre = torch.arange(out_t, device=paddings.device) * stride - left + (window - 1) // 2
  else:
    out_t = max((t - window) // stride + 1, 0)
    centre = torch.arange(out_t, device=paddings.device) * stride + (window - 1) // 2
  valid = (centre >= 0) & (centre < t)
  idx = centre.clamp(0, max(t - 1, 0))
  out = paddings[:, idx]
  return torch.where(valid.unsqueeze(0), out, torch.ones_like(out))


def ComputeConvOutputPadding(paddings, window, stride, padding_algorithm='SAME',
                             v2_padding=False):
  """out_padding[i] = 1 iff any input frame in window i is padding (ref :76)."""
  if v2_padding:
    return _ComputeConvOutputPaddingV2(paddings, window, stride, padding_algorithm)
  if stride == 1:
    return paddings
  t = paddings.shape[1]
  pad_len = -(-t // stride) * stride - t
  p = F.pad(paddings.float(), (0, pad_len), value=1.0).unsqueeze(1)
  if padding_algorithm == 'SAME':
    out_t = -(-p.shape[-1] // stride)
    total = max((out_t - 1) * stride + window - p.shape[-1], 0)
    p = F.pad(p, (total // 2, total - total // 2), value=0.0)
  out = F.max_pool1d(p, window, stride)
  return out.squeeze(1).to(paddings.dtype)


def ComputeExplicitPaddingForCausalConv(filter_shape, dilation_rate):
  """(left, right) explicit time padding of a causal conv (ref :119)."""
  return ((filter_shape[0] - 1) * dilation_rate[0], 0)


class BaseConv2DLayerWithPadding(base_layer.BaseLayer):
  """Shared params/FProp of the padding-aware convs (ref :233)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('filter_shape', (0, 0, 0, 0), '[time, freq, in, out|multiplier].')
    p.Define('filter_stride', (1, 1), '(time, freq) stride.')
    p.Define('dilation_rate', (1, 1), '(time, freq) dilation.')
    p.Define('weight_norm', False, 'Weight normalisation (g·w/‖w‖).')
    p.Define('bias', False, 'Add a bias.')
    p.Define('bias_init', WeightInit.Constant(0.0), 'Bias init.')
    p.Define('partial_conv', False, 'Rescale near sequence boundaries (1811.11718).')
    p.Define('v2_padding', False, 'Correct padding for strided convs.')
    p.Define('is_causal', False, 'Left-only time padding.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.name and len(p.filter_shape) == 4
    assert all(x > 0 for x in p.filter_shape), p.filter_shape

  # subclass hooks
  @classmethod
  def OutputChannels(cls, p):
    raise NotImplementedError

  @property
  def output_channels(self):
    return self.OutputChannels(self.params)

  @property
  def input_channels(self):
    return self.params.filter_shape[2]

  def _WeightShape(self):
    return list(self.params.filter_shape)

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w', WeightParams(self._WeightShape(), p.params_init, p.dtype))
    if p.weight_norm:
      self.CreateVariable('g', WeightParams([self.output_channels],
                                            WeightInit.Constant(0.0), p.dtype))
    if p.bias:
      self.CreateVariable('b', WeightParams([self.output_channels], p.bias_init, p.dtype))

  def _GetWeight(self, theta):
    p = self.params
    w = theta.w
    if p.weight_norm:
      wn = F.normalize(w.float().reshape(-1, w.shape[-1]) if not self._depthwise
                       else w.float().reshape(w.shape[0] * w.shape[1], -1), dim=0)
      w = (wn.reshape(w.shape) * (1.0 + theta.g.float().reshape(
          [1, 1, -1, p.filter_shape[3]] if self._depthwise else [-1]))).to(w.dtype)
    return w

  _depthwise = False

  def _TimePad(self):
    """(left, right) SAME or causal padding along time."""
    p = self.params
    k = (p.filter_shape[0] - 1) * p.dilation_rate[0]
    if p.is_causal:
      return k, 0
    return k // 2, k - k // 2

  def _FreqPad(self, f):
    p = self.params
    s = p.filter_stride[1]
    k = (p.filter_shape[1] - 1) * p.dilation_rate[1] + 1
    total = max((-(-f // s) - 1) * s + k - f, 0)
    return total // 2, total - total // 2

  def _Conv(self, x_nchw, w):
    raise NotImplementedError

  def _ApplyConv(self, theta, inputs):
    """inputs [B,T,F,C] already masked → [B,T',F',Cout]."""
    p = self.params
    w = self._GetWeight(theta).to(inputs.dtype)
    t, f = inputs.shape[1], inputs.shape[2]
    x = inputs.permute(0, 3, 1, 2)                      # NCHW view of NHWC data
    tl, tr = self._TimePad()
    if p.filter_stride[0] > 1 and not p.is_causal:
      # SAME with stride: total padding depends on T.
      s = p.filter_stride[0]
      k = (p.filter_shape[0] - 1) * p.dilation_rate[0] + 1
      total = max((-(-t // s) - 1) * s + k - t, 0)
      tl, tr = total // 2, total - total // 2
    fl, fr = self._FreqPad(f)
    x = F.pad(x, (fl, fr, tl, tr))
    y = self._Conv(x, w)
    if p.bias:
      y = y + theta.b.to(y.dtype).view(1, -1, 1, 1)
    return y.permute(0, 2, 3, 1)

  def FProp(self, theta, inputs, paddings):
    p = self.params
    inputs = self._CastToFPropDtype(inputs)
    mask = (1.0 - paddings.to(inputs.dtype)).unsqueeze(-1).unsqueeze(-1)
    x = inputs * mask
    out = self._ApplyConv(theta, x)
    window = (p.filter_shape[0] - 1) * p.dilation_rate[0] + 1 if p.v2_padding else p.filter_shape[0]
    if p.is_causal and p.filter_stride[0] == 1:
      out_pad = paddings
    else:
      out_pad = ComputeConvOutputPadding(paddings, window, p.filter_stride[0],
                                         'SAME', p.v2_padding)
    if p.partial_conv:
      ones = mask.expand(-1, -1, 1, 1)
      k = p.filter_shape[0]
      tl, tr = self._TimePad()
      cnt = F.avg_pool1d(F.pad(ones.reshape(ones.shape[0], 1, -1), (tl, tr)), k,
                         p.filter_stride[0])
      out = out / cnt.clamp_min(1.0 / k).reshape(out.shape[0], -1, 1, 1).to(out.dtype)
    out = out * (1.0 - out_pad.to(out.dtype)).unsqueeze(-1).unsqueeze(-1)
    return out, out_pad

  # -- streaming (causal, stride 1 in time) ----------------------------------------
  def zero_state(self, batch_size):
    p = self.params
    assert p.is_causal, 'StreamStep needs a causal layer'
    ctx = (p.filter_shape[0] - 1) * p.dilation_rate[0]
    dev, dt = self.Device(), py_utils.FPropDtype(p)
    return NestedMap(context=torch.zeros(batch_size, ctx, 1, self.input_channels,
                                         device=dev, dtype=dt))

  def StreamStep(self, theta, inputs, paddings, state0):
    """inputs [B, Q, F=1, C] → (outputs, paddings, state1)."""
    p = self.params
    assert p.is_causal and p.filter_stride[0] == 1
    x = inputs * (1.0 - paddings.to(inputs.dtype)).unsqueeze(-1).unsqueeze(-1)
    ctx_len = state0.context.shape[1]
    cat = torch.cat([state0.context.to(x.dtype), x], 1)
    w = self._GetWeight(theta).to(x.dtype)
    y = self._Conv(cat.permute(0, 3, 1, 2), w)
    if p.bias:
      y = y + theta.b.to(y.dtype).view(1, -1, 1, 1)
    y = y.permute(0, 2, 3, 1)
    state1 = NestedMap(context=cat[:, -ctx_len:] if ctx_len else cat[:, :0])
    return y, paddings, state1

  @classmethod
  def FPropMeta(cls, p, inputs, paddings):
    b, t, f, _ = inputs
    oc = cls.OutputChannels(p)
    flops = b * t * f * p.filter_shape[0] * p.filter_shape[1] * p.filter_shape[2] * oc * 2
    return NestedMap(flops=flops, out_shapes=(inputs, paddings))


class Conv2DLayerWithPadding(BaseConv2DLayerWithPadding):
  """Dense conv2d (ref :425)."""

  @classmethod
  def OutputChannels(cls, p):
    return p.filter_shape[3]

  def _Conv(self, x, w):
    p = self.params
    return F.conv2d(x, w.permute(3, 2, 0, 1), stride=tuple(p.filter_stride),
                    dilation=tuple(p.dilation_rate))


class CausalConv2DLayerWithPadding(Conv2DLayerWithPadding):
  """Conv2d that never looks ahead in time (ref :506). Frequency kernel must be 1."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.is_causal = True
    return p

  def __init__(self, params):
    super().__init__(params)
    assert self.params.filter_shape[1] == 1, 'Only 1d causal convolution is supported.'


class DepthwiseConv2DLayer(BaseConv2DLayerWithPadding):
  """Depthwise conv; filter `[h, w, in, multiplier]` (ref :608)."""

  _depthwise = True

  @classmethod
  def OutputChannels(cls, p):
    return p.filter_shape[2] * p.filter_shape[3]

  def _Conv(self, x, w):
    p = self.params
    h, wd, cin, mult = w.shape
    wt = w.permute(2, 3, 0, 1).reshape(cin * mult, 1, h, wd)
    return F.conv2d(x, wt, stride=tuple(p.filter_stride),
                    dilation=tuple(p.dilation_rate), groups=cin)


class CausalDepthwiseConv2DLayer(DepthwiseConv2DLayer):
  """Causal depthwise conv with streaming support (ref :717)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.is_causal = True
    return p

  def __init__(self, params):
    super().__init__(params)
    assert self.params.filter_shape[1] == 1, 'Only 1d causal convolution is supported.'


class ChunkwiseDepthwiseConv2DLayer(DepthwiseConv2DLayer):
  """Depthwise conv that does not cross chunk boundaries (ref :846)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('chunk_size', 0, 'Chunk length in frames.')
    return p

  def FProp(self, theta, inputs, paddings):
    p = self.params
    b, t, f, c = inputs.shape
    cs = p.chunk_size
    pad_t = -(-t // cs) * cs - t
    x = F.pad(inputs, (0, 0, 0, 0, 0, pad_t))
    pd = F.pad(paddings, (0, pad_t), value=1.0)
    n = x.shape[1] // cs
    y, yp = super().FProp(theta, x.reshape(b * n, cs, f, c), pd.reshape(b * n, cs))
    return y.reshape(b, n * cs, f, -1)[:, :t], yp.reshape(b, n * cs)[:, :t]


class NormalizedDepthwiseConv2DLayer(DepthwiseConv2DLayer):
  """Lightweight conv: weights softmax-normalised over time, tiled over
  channels, optional DropConnect (ref :903)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('dropconnect_prob', 0.0, 'DropConnect probability.')
    p.Define('deterministic_dropout', False, 'Kept for parity.')
    p.Define('temperature', 1.0, 'Softmax temperature.')
    p.Define('weight_tiling_factor', 1, 'Times the weights are tiled over channels.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.filter_shape[1] == 1 and p.temperature > 0.0

  @classmethod
  def OutputChannels(cls, p):
    return p.filter_shape[2] * p.filter_shape[3] * p.weight_tiling_factor

  @property
  def input_channels(self):
    p = self.params
    return p.filter_shape[2] * p.weight_tiling_factor

  def _GetWeight(self, theta):
    p = self.params
    w = torch.softmax(theta.w.float() / p.temperature, 0)
    if p.dropconnect_prob > 0.0 and not self.do_eval:
      w = F.dropout(w, p.dropconnect_prob, training=True)
    return w.repeat(1, 1, p.weight_tiling_factor, 1).to(theta.w.dtype)


class CausalNormalizedDepthwiseConv2DLayer(NormalizedDepthwiseConv2DLayer):
  """Causal lightweight conv (ref :981)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.is_causal = True
    return p


class ConvBatchNormLayer(bn_layers.BatchNormLayer):
  """BN over `[B,T,F,C]` with `[B,T]` paddings (ref :989)."""

  def FProp(self, theta, inputs, paddings):
    pad = paddings.unsqueeze(-1).unsqueeze(-1)
    return super().FProp(theta, inputs, pad), paddings


class PaddingLayer(base_layer.BaseLayer):
  """Zeroes padded frames (ref :1004)."""

  def FProp(self, theta, inputs, paddings):
    mask = (1.0 - paddings.to(inputs.dtype)).reshape(
        paddings.shape + (1,) * (inputs.dim() - 2))
    return inputs * mask, paddings


class GlobalPoolingLayer(base_layer.BaseLayer):
  """Padding-aware global AVG/MAX pooling over time and frequency (ref :1012)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('pooling_type', 'MAX', 'AVG or MAX.')
    return p

  def FProp(self, theta, inputs, paddings):
    p = self.params
    b, t, f, c = inputs.shape
    if paddings is None:
      mask = torch.ones(b, t, 1, 1, device=inputs.device, dtype=inputs.dtype)
    else:
      mask = (1.0 - paddings.to(inputs.dtype)).view(b, t, 1, 1)
    if p.pooling_type == 'AVG':
      tot = (inputs * mask).sum((1, 2), keepdim=True)
      out = tot / (mask.sum((1, 2), keepdim=True) * f).clamp_min(1e-8)
    else:
      neg = torch.finfo(inputs.dtype).min
      out = inputs.masked_fill(mask == 0, neg).amax((1, 2), keepdim=True)
      out = torch.where(out == neg, torch.zeros_like(out), out)
    out_pad = None
    if paddings is not None:
      out_pad = paddings.min(1, keepdim=True).values
    return out, out_pad
