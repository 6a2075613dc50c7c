"""Common layers.

Catalogue follows reference `lingvo/core/layers.py` (63 classes, SURVEY §2.4).
Activations are NHWC / `[batch, time, …, channels]` like the reference;
`paddings` are `[batch, time]` floats (1 = padded). Each layer cites the
reference line it mirrors. Compute is PyTorch with the sm_90a kernels
(`lingvo_b200.ops`: wgmma GEMM with fused bias/activation, fused
LayerNorm, fused softmax-xent) swapped in on CUDA bf16 paths.
"""

from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

from lingvo_b200 import ops
from lingvo_b200.core import activations
from lingvo_b200.core import base_layer
from lingvo_b200.core import bn_layers
from lingvo_b200.core import py_utils
from lingvo_b200.core import quant_utils
from lingvo_b200.core import summary_utils
from lingvo_b200.core.nested_map import NestedMap

BatchNormLayer = bn_layers.BatchNormLayer
BatchNormLayerNoPadding = bn_layers.BatchNormLayerNoPadding
CategoricalBN = bn_layers.CategoricalBN
GroupNormLayer = bn_layers.GroupNormLayer
WeightInit = py_utils.WeightInit
WeightParams = py_utils.WeightParams


def _Pad2(padding):
  return padding


def _ConvOutSize(size, k, stride, padding, dilation=1):
  if size is None:
    return None
  eff = (k - 1) * dilation + 1
  if padding == 'SAME':
    return -(-size // stride)
  return max(-(-(size - eff + 1) // stride), 0)


def _SamePad(size, k, stride, dilation=1):
  eff = (k - 1) * dilation + 1
  out = -(-size // stride)
  total = max((out - 1) * stride + eff - size, 0)
  return total // 2, total - total // 2


def ComputeConvOutputPadding(paddings, window, stride, padding_algorithm='SAME',
                             v2_padding=False):
  """Paddings `[B, T]` after a time-strided conv/pool (reference conv_util)."""
  if stride == 1 and padding_algorithm == 'SAME':
    return paddings
  b, t = paddings.shape
  p = paddings.reshape(b, 1, t).float()
  if padding_algorithm == 'SAME':
    lo, hi = _SamePad(t, window, stride)
    p = F.pad(p, (lo, hi), value=1.0)
    out = F.max_pool1d(-p, window, stride).neg() if False else None
    # A frame is padding iff its *first* (stride-aligned) input frame is.
    idx = torch.arange(0, t, stride, device=paddings.device)
    return paddings[:, idx]
  out_t = _ConvOutSize(t, window, stride, 'VALID')
  idx = torch.arange(0, out_t, device=paddings.device) * stride + (window - 1)
  return paddings[:, idx.clamp(max=t - 1)]


class IdentityLayer(base_layer.BaseLayer):
  """Identity (reference :148)."""

  def FProp(self, theta, inputs, *args):
    if isinstance(inputs, NestedMap):
      inputs = inputs.DeepCopy()
    return (inputs,) + args if args else inputs

  @classmethod
  def FPropMeta(cls, p, inputs, *args):
    return NestedMap(flops=0, out_shapes=(inputs,) + args)


class BaseConv2DLayer(quant_utils.QuantizableLayer):
  """Base of 2-D convolution layers (reference :182-683).

  filter_shape = (h, w, in, out); inputs `[B, T, F, C]`; optional BN
  (padding-aware), bias, activation, weight-norm, causal convolution in time,
  and `conv_last` ordering.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('filter_shape', (0, 0, 0, 0), '(height, width, in, out).')
    p.Define('filter_stride', (1, 1), '(height/time stride, width stride).')
    p.Define('dilation_rate', (1, 1), 'Atrous dilation.')
    p.Define('activation', 'RELU', 'Activation applied after normalisation.')
    p.Define('bias', False, 'Apply a bias before activation.')
    p.Define('batch_norm', True, 'Apply BN.')
    p.Define('bn_decay', 0.999, 'BN moving-average decay.')
    p.Define('bn_fold_weights', None, 'Fold BN into the weights (quant).')
    p.Define('causal_convolution', False, 'Left-pad time so no look-ahead.')
    p.Define('conv_last', False, 'BN → act → conv instead of conv → BN → act.')
    p.Define('weight_norm', False, 'Weight normalisation.')
    p.Define('disable_activation_quantization', False, 'Kept for parity.')
    p.Define('v2_padding', False, 'Padding mode of reference conv_util.')
    p.Define('padding_algorithm', 'SAME', 'SAME|VALID.')
    p.Define('batch_norm_params', None, 'Override BN layer params.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.name
    assert len(p.filter_shape) == 4 and len(p.filter_stride) == 2
    assert all(x > 0 for x in p.filter_shape)
    if p.batch_norm:
      bn = (p.batch_norm_params.Copy() if p.batch_norm_params is not None
            else bn_layers.BatchNormLayer.Params().Set(decay=p.bn_decay))
      bn.Set(dim=self._BNDim(), name=p.name + '_bn')
      self.CreateChild('bn', bn)

  def _BNDim(self):
    return self.output_channels if not self.params.conv_last else (
        self.params.filter_shape[2])

  @property
  def output_channels(self):
    return self.params.filter_shape[-1]

  @property
  def input_channels(self):
    return self.params.filter_shape[-2]

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w', WeightParams(
        shape=list(p.filter_shape), init=p.params_init, dtype=p.dtype,
        collections=[self.__class__.__name__ + '_vars']))
    if p.bias:
      self.CreateVariable('b', WeightParams(
          shape=[self.output_channels], init=WeightInit.Constant(0.0),
          dtype=p.dtype, collections=[self.__class__.__name__ + '_vars']))
    if p.weight_norm:
      self.CreateVariable('g', WeightParams(
          shape=[self.output_channels], init=WeightInit.Constant(0.0),
          dtype=p.dtype, collections=[self.__class__.__name__ + '_vars']))

  def OutShape(self, in_shape):
    """[B, H, W, C] → conv output shape (None dims preserved)."""
    p = self.params
    b, h, w, _ = in_shape
    pad = 'SAME' if (p.padding_algorithm == 'SAME' or p.causal_convolution) \
        else 'VALID'
    return [b, _ConvOutSize(h, p.filter_shape[0], p.filter_stride[0], pad,
                            p.dilation_rate[0]),
            _ConvOutSize(w, p.filter_shape[1], p.filter_stride[1], pad,
                         p.dilation_rate[1]), self.output_channels]

  def _GetWeight(self, theta):
    p = self.params
    w = theta.w
    if p.weight_norm:
      w = F.normalize(w.reshape(-1, w.shape[-1]), dim=0).reshape(w.shape) * (
          theta.g + 1.0).reshape([1] * (w.dim() - 1) + [-1])
    return self.QWeight(w)

  def _EvaluateConvKernel(self, inputs, w):
    """inputs NHWC, w (h, w, in/groups·…, out) → NHWC."""
    raise NotImplementedError()

  def _Conv(self, inputs, w, groups=1):
    p = self.params
    x = inputs.permute(0, 3, 1, 2)
    kh, kw = w.shape[0], w.shape[1]
    dh, dw = p.dilation_rate
    sh, sw = p.filter_stride
    if p.causal_convolution:
      assert dh == 1 or sh == 1
      wl, wr = _SamePad(x.shape[3], kw, sw, dw)
      x = F.pad(x, (wl, wr, (kh - 1) * dh, 0))
    elif p.padding_algorithm == 'SAME':
      hl, hr = _SamePad(x.shape[2], kh, sh, dh)
      wl, wr = _SamePad(x.shape[3], kw, sw, dw)
      x = F.pad(x, (wl, wr, hl, hr))
    wt = w.permute(3, 2, 0, 1)
    y = F.conv2d(x, wt.to(x.dtype), None, stride=(sh, sw), dilation=(dh, dw),
                 groups=groups)
    return y.permute(0, 2, 3, 1)

  def _ApplyBiasAct(self, theta, out):
    p = self.params
    if p.bias:
      out = out + theta.b.to(out.dtype)
    return out

  def FProp(self, theta, inputs, paddings=None):
    """Returns (out, out_paddings) when paddings given, else (out, None)."""
    p = self.params
    inputs = self._CastToFPropDtype(inputs)
    b, t = inputs.shape[0], inputs.shape[1]
    if paddings is None:
      conv_pad = None
    else:
      conv_pad = ComputeConvOutputPadding(
          paddings, p.filter_shape[0], p.filter_stride[0],
          'SAME' if (p.padding_algorithm == 'SAME' or p.causal_convolution)
          else 'VALID')
      inputs = py_utils.ApplyPadding(paddings, inputs)
    w = self._GetWeight(theta)
    act = activations.GetFn(p.activation)
    if p.conv_last:
      out = inputs
      if p.batch_norm:
        out = self.bn.FProp(theta.bn, out,
                            None if paddings is None else
                            paddings.reshape(b, t, 1, 1))
      out = act(out)
      out = self._EvaluateConvKernel(out, w)
      out = self._ApplyBiasAct(theta, out)
    else:
      out = self._EvaluateConvKernel(inputs, w)
      out = self._ApplyBiasAct(theta, out)
      if p.batch_norm:
        bn_pad = None if conv_pad is None else conv_pad.reshape(
            out.shape[0], out.shape[1], 1, 1)
        out = self.bn.FProp(theta.bn, out, bn_pad)
      out = act(out)
    if conv_pad is not None:
      out = py_utils.ApplyPadding(conv_pad, out)
    return out, conv_pad

  @classmethod
  def FPropMeta(cls, p, inputs, paddings=None):
    b, h, w, c = inputs
    fh, fw, ic, oc = p.filter_shape
    sh, sw = p.filter_stride
    oh = _ConvOutSize(h, fh, sh, 'SAME')
    ow = _ConvOutSize(w, fw, sw, 'SAME')
    from lingvo_b200.core import tshape
    out = tshape.Shape([b, oh, ow, oc])
    flops = b * oh * ow * fh * fw * ic * oc * 2
    return NestedMap(flops=flops, out_shapes=(out,) if paddings is None
                     else (out, paddings))


class Conv2DLayer(BaseConv2DLayer):
  """Plain 2-D convolution (reference :684)."""

  def _EvaluateConvKernel(self, inputs, w):
    return self._Conv(inputs, w)


ConvLayer = Conv2DLayer


class ConvNN2DLayer(BaseConv2DLayer):
  """tf.nn.convolution flavour (same maths here) (reference :699)."""

  def _EvaluateConvKernel(self, inputs, w):
    return self._Conv(inputs, w)


class DepthwiseConv2DLayer(BaseConv2DLayer):
  """Depthwise conv: filter (h, w, in, channel_multiplier) (reference :724)."""

  @property
  def output_channels(self):
    fs = self.params.filter_shape
    return fs[2] * fs[3]

  def _EvaluateConvKernel(self, inputs, w):
    kh, kw, cin, mult = w.shape
    # TF depthwise: out channel index = in * mult + m.
    w2 = w.reshape(kh, kw, 1, cin * mult)
    return self._Conv(inputs, w2, groups=cin)


class SeparableConv2DLayer(Conv2DLayer):
  """Depthwise followed by pointwise (reference :771)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('depth_multiplier', 1, 'Depthwise channel multiplier.')
    p.Define('depthwise_tpl', DepthwiseConv2DLayer.Params().Set(
        activation='NONE', batch_norm=False), 'Depthwise template.')
    return p

  def __init__(self, params):
    params = params.Copy()
    fs = params.filter_shape
    dw = params.depthwise_tpl.Copy().Set(
        filter_shape=(fs[0], fs[1], fs[2], params.depth_multiplier),
        filter_stride=params.filter_stride, dilation_rate=params.dilation_rate,
        causal_convolution=params.causal_convolution,
        padding_algorithm=params.padding_algorithm, name='depthwise_conv')
    self._orig_filter_shape = tuple(fs)
    params.filter_shape = (1, 1, fs[2] * params.depth_multiplier, fs[3])
    params.filter_stride = (1, 1)
    params.dilation_rate = (1, 1)
    self._dw_params = dw
    super().__init__(params)
    self.CreateChild('depthwise_conv', dw)

  def FProp(self, theta, inputs, paddings=None):
    mid, mid_pad = self.depthwise_conv.FProp(theta.depthwise_conv, inputs,
                                             paddings)
    return super().FProp(theta, mid, mid_pad)


class DeconvLayer(base_layer.BaseLayer):
  """Transposed 2-D convolution (reference :46)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('filter_shape', (0, 0, 0, 0), '(h, w, out_channels, in_channels).')
    p.Define('filter_stride', (0, 0), 'Strides.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w', WeightParams(list(p.filter_shape), p.params_init,
                                          p.dtype))
    self.CreateVariable('b', WeightParams([p.filter_shape[-2]],
                                          WeightInit.Constant(0.0), p.dtype))

  def OutShape(self, in_shape):
    p = self.params
    return [in_shape[0], in_shape[1] * p.filter_stride[0],
            in_shape[2] * p.filter_stride[1], p.filter_shape[2]]

  def FProp(self, theta, inputs):
    p = self.params
    x = inputs.permute(0, 3, 1, 2)
    w = theta.w.permute(3, 2, 0, 1)  # (in, out, h, w)
    sh, sw = p.filter_stride
    kh, kw = p.filter_shape[:2]
    y = F.conv_transpose2d(x, w.to(x.dtype), theta.b.to(x.dtype),
                           stride=(sh, sw))
    oh, ow = inputs.shape[1] * sh, inputs.shape[2] * sw
    ph, pw = (y.shape[2] - oh) // 2, (y.shape[3] - ow) // 2
    y = y[:, :, ph:ph + oh, pw:pw + ow]
    return y.permute(0, 2, 3, 1)


class Conv2DLayerNoPadding(base_layer.BaseLayer):
  """2-D conv without padding tensors (reference :5981)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('filter_shape', (0, 0, 0, 0), '(h, w, in, out).')
    p.Define('filter_stride', (0, 0), '(stride_h, stride_w).')
    p.Define('padding', 'SAME', 'SAME|VALID')
    p.Define('use_bias', False, 'Add bias.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w', WeightParams(list(p.filter_shape), p.params_init,
                                          p.dtype))
    if p.use_bias:
      self.CreateVariable('b', WeightParams([p.filter_shape[-1]],
                                            WeightInit.Constant(0.0), p.dtype))

  def FProp(self, theta, x):
    p = self.params
    xi = x.permute(0, 3, 1, 2)
    if p.padding == 'SAME':
      hl, hr = _SamePad(xi.shape[2], p.filter_shape[0], p.filter_stride[0])
      wl, wr = _SamePad(xi.shape[3], p.filter_shape[1], p.filter_stride[1])
      xi = F.pad(xi, (wl, wr, hl, hr))
    y = F.conv2d(xi, theta.w.permute(3, 2, 0, 1).to(xi.dtype),
                 theta.b.to(xi.dtype) if p.use_bias else None,
                 stride=tuple(p.filter_stride))
    return y.permute(0, 2, 3, 1)

  @classmethod
  def FPropMeta(cls, p, inputs):
    b, h, w, c = inputs
    fh, fw, ic, oc = p.filter_shape
    sh, sw = p.filter_stride
    oh = _ConvOutSize(h, fh, sh, p.padding)
    ow = _ConvOutSize(w, fw, sw, p.padding)
    from lingvo_b200.core import tshape
    return NestedMap(flops=b * oh * ow * fh * fw * ic * oc * 2,
                     out_shapes=(tshape.Shape([b, oh, ow, oc]),))


class ProjectionLayer(quant_utils.QuantizableLayer):
  """y = act(BN(x·w + b)) (reference :845-1417).

  On CUDA/bf16 without BN the GEMM + bias + activation run as ONE wgmma
  kernel (`ops.gemm.linear`).
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Depth of the input.')
    p.Define('output_dim', 0, 'Depth of the output.')
    p.Define('activation', 'RELU', 'Activation function.')
    p.Define('batch_norm', None, 'Whether to use BN (None ⇒ False).')
    p.Define('has_bias', False, 'Whether to use bias.')
    p.Define('bias_init', 0.0, 'Initial bias value.')
    p.Define('affine_last', False, 'BN → act → affine instead.')
    p.Define('weight_norm', False, 'Weight normalisation.')
    p.Define('bn_fold_weights', None, 'Fold BN into weights.')
    p.Define('bn_params', bn_layers.BatchNormLayer.Params().Set(decay=0.999),
             'BN params.')
    p.Define('apply_pruning', False, 'Kept for parity (pruning masks).')
    p.Define('pruning_hparams_dict', None, 'Kept for parity.')
    p.Define('use_einsum', True, 'Kept for parity.')
    p.Define('use_blocked_matmul', False, 'Kept for parity.')
    p.Define('block_dim', 1024, 'Kept for parity.')
    p.Define('use_block_diagonal_matmul', False, 'Block-diagonal weight.')
    p.Define('bd_num_blocks', 1, 'Number of diagonal blocks.')
    p.Define('use_bd_mix', False, 'Mix blocks after block-diag matmul.')
    p.Define('weight', None, 'External weight tensor (tied).')
    p.Define('xla_num_partitions', None, 'Kept for parity.')
    p.Define('w_dtype', None, 'Weight dtype override.')
    p.Define('enable_vn', False, 'Apply variational noise to w.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.name
    assert p.input_dim > 0 and p.output_dim > 0
    assert activations.IsSupported(p.activation)
    self.TrackQActs(self.output_qt_name)
    if p.batch_norm:
      bn = p.bn_params.Copy()
      bn.name = p.name + '_bn'
      bn.dim = p.input_dim if p.affine_last else p.output_dim
      self.CreateChild('bn', bn)

  def _CreateLayerVariables(self):
    p = self.params
    wdt = p.w_dtype or p.dtype
    coll = [self.__class__.__name__ + '_vars']
    if p.weight is None:
      if p.use_block_diagonal_matmul:
        shape = [p.bd_num_blocks, p.input_dim // p.bd_num_blocks,
                 p.output_dim // p.bd_num_blocks]
      else:
        shape = [p.input_dim, p.output_dim]
      self.CreateVariable('w', WeightParams(shape, p.params_init, wdt, coll))
      if p.use_block_diagonal_matmul and p.use_bd_mix:
        self.CreateVariable('mix_kernel', WeightParams(
            [p.bd_num_blocks, p.bd_num_blocks], WeightInit.Gaussian(0.1), wdt,
            coll))
    if p.has_bias:
      self.CreateVariable('b', WeightParams(
          [p.output_dim], WeightInit.Constant(scale=p.bias_init), p.dtype, coll))
    if p.weight_norm:
      self.CreateVariable('g', WeightParams(
          [p.output_dim], WeightInit.Constant(0.0), p.dtype, coll))

  @classmethod
  def NumOutputNodes(cls, p):
    return p.output_dim

  @property
  def output_qt_name(self):
    return 'activation'

  def _GetWeights(self, theta):
    p = self.params
    w = theta.w if p.weight is None else p.weight
    if p.enable_vn:
      w = py_utils.AddVN(p, w)
    if p.weight_norm:
      w = F.normalize(w, dim=0) * (theta.g.to(w.dtype) + 1.0)
    return self.QWeight(w)

  def FProp(self, theta, inputs, paddings=None):
    p = self.params
    inputs = self._CastToFPropDtype(inputs)
    w = self._GetWeights(theta)
    b = theta.b if p.has_bias else None
    if paddings is not None:
      paddings = paddings.reshape(list(inputs.shape[:-1]) + [1]) if (
          paddings.numel() == inputs.numel() // inputs.shape[-1]) else paddings
    act = p.activation

    def affine(x, fuse_act):
      if p.use_block_diagonal_matmul:
        y = py_utils.BlockDiagonalMatmul(x, w.to(x.dtype), p.bd_num_blocks)
        if p.use_bd_mix:
          shp = list(y.shape)
          yb = y.reshape(shp[:-1] + [p.bd_num_blocks, -1])
          y = torch.einsum('...bd,bc->...cd', yb,
                           theta.mix_kernel.to(y.dtype)).reshape(shp)
        if b is not None:
          y = y + b.to(y.dtype)
        return activations.GetFn(act)(y) if fuse_act else y
      if (fuse_act and ops.use_cuda_kernels(x, w) and
          x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and
          act in ('NONE', 'RELU') and w.shape[0] % 8 == 0 and
          w.shape[1] % 8 == 0):
        from lingvo_b200.ops import gemm
        return gemm.linear(x, w, b, act=act)
      y = torch.matmul(x, w.to(x.dtype))
      if b is not None:
        y = y + b.to(y.dtype)
      return activations.GetFn(act)(y) if fuse_act else y

    if p.affine_last:
      out = inputs
      if p.batch_norm:
        out = self.bn.FProp(theta.bn, out, paddings)
      out = activations.GetFn(act)(out)
      out = affine(out, fuse_act=False)
    else:
      if p.batch_norm:
        out = affine(inputs, fuse_act=False)
        out = self.bn.FProp(theta.bn, out, paddings)
        out = activations.GetFn(act)(out)
      else:
        out = affine(inputs, fuse_act=True)
    out = self.QAct(self.output_qt_name, out)
    if paddings is not None:
      out = py_utils.ApplyPadding(paddings, out)
    return out

  @classmethod
  def FPropMeta(cls, p, inputs, paddings=None):
    dim_in = inputs[-1]
    other = inputs.num_elements() / dim_in
    flops = 2 * other * p.input_dim * p.output_dim
    if p.has_bias:
      flops += other * p.output_dim
    flops += other * p.output_dim * activations.GetFlops(p.activation)
    from lingvo_b200.core import tshape
    out = tshape.Shape(inputs[:-1] + [p.output_dim])
    return NestedMap(flops=flops, out_shapes=(out,))


class FCLayer(ProjectionLayer):
  """Fully-connected layer (projection with bias) (reference :1586)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.batch_norm = False
    p.has_bias = True
    return p


class MultitaskProjectionEinsumLayer(quant_utils.QuantizableLayer):
  """Per-task projection weights selected by task id (reference :1418)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Depth of the input.')
    p.Define('output_dim', 0, 'Depth of the output.')
    p.Define('num_tasks', 0, 'Number of tasks.')
    p.Define('activation', 'RELU', 'Activation.')
    p.Define('has_bias', False, 'Use bias.')
    p.Define('bias_init', 0.0, 'Bias init.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w', WeightParams(
        [p.num_tasks, p.input_dim, p.output_dim], p.params_init, p.dtype))
    if p.has_bias:
      self.CreateVariable('b', WeightParams(
          [p.num_tasks, p.output_dim], WeightInit.Constant(p.bias_init),
          p.dtype))

  def FProp(self, theta, inputs, tasks, paddings=None):
    p = self.params
    out = py_utils.MultiTaskProjection(theta.w.to(inputs.dtype),
                                       theta.b.to(inputs.dtype) if p.has_bias
                                       else None, inputs, tasks)
    out = activations.GetFn(p.activation)(out)
    if paddings is not None:
      out = py_utils.ApplyPadding(paddings, out)
    return out


class FeedForwardNet(quant_utils.QuantizableLayer):
  """A stack of projection layers (reference :1597)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Depth of the input to the network.')
    p.Define('hidden_layer_dims', [], 'Depth of the hidden layer outputs.')
    p.Define('projection', ProjectionLayer.Params(), 'Projection template.')
    p.Define('dropout', None, 'Dropout params (single or list).')
    p.Define('batch_norm', False, 'BN per layer (bool or list).')
    p.Define('activation', 'RELU', 'Activation per layer (str or list).')
    p.Define('weight_norm', False, 'Weight norm.')
    p.Define('skip_connections', None, 'None|"ResNet"|"DenseNet" or list.')
    p.Define('bn_fold_weights', None, 'Kept for parity.')
    p.Define('has_bias', None, 'Bias per layer (None ⇒ not BN).')
    p.Define('memory_augmentation', None, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.name
    n = len(p.hidden_layer_dims)
    bn = p.batch_norm if isinstance(p.batch_norm, (list, tuple)) else [p.batch_norm] * n
    act = p.activation if isinstance(p.activation, (list, tuple)) else [p.activation] * n
    dropout = p.dropout
    if dropout is None:
      dropout = DropoutLayer.Params()
    dropouts = dropout if isinstance(dropout, (list, tuple)) else [dropout.Copy() for _ in range(n)]
    skips = p.skip_connections
    self._skip = skips if isinstance(skips, (list, tuple)) else [skips] * n
    self._layer_dims = [p.input_dim] + list(p.hidden_layer_dims)
    proj, drop = [], []
    in_dim = p.input_dim
    for i in range(n):
      out_dim = p.hidden_layer_dims[i]
      has_bias = (not bn[i]) if p.has_bias is None else (
          p.has_bias[i] if isinstance(p.has_bias, (list, tuple)) else p.has_bias)
      proj.append(p.projection.Copy().Set(
          name='%s_%d' % (p.name, i) if False else 'proj_%d' % i,
          batch_norm=bn[i], has_bias=has_bias, activation=act[i],
          weight_norm=p.weight_norm, input_dim=in_dim, output_dim=out_dim))
      drop.append(dropouts[i].Copy().Set(name='dropout_%d' % i))
      if self._skip[i] == 'DenseNet':
        in_dim = in_dim + out_dim
      else:
        in_dim = out_dim
    self.CreateChildren('fc', proj)
    self.CreateChildren('dropout', drop)

  def FProp(self, theta, inputs, paddings=None):
    out = inputs
    for i in range(len(self.fc)):
      prev = out
      out = self.fc[i].FProp(theta.fc[i], out, paddings)
      out = self.dropout[i].FProp(theta.dropout[i], out)
      if self._skip[i] == 'ResNet' and prev.shape[-1] == out.shape[-1]:
        out = out + prev
      elif self._skip[i] == 'DenseNet':
        out = torch.cat([prev, out], dim=-1)
    return out

  @classmethod
  def FPropMeta(cls, p, inputs, paddings=None):
    flops = 0
    in_dim = inputs[-1]
    other = inputs.num_elements() / in_dim
    for d in p.hidden_layer_dims:
      flops += 5 * other * in_dim * d
      in_dim = d
    from lingvo_b200.core import tshape
    return NestedMap(flops=flops,
                     out_shapes=(tshape.Shape(inputs[:-1] + [in_dim]),))


class MultitaskFeedForwardNet(base_layer.BaseLayer):
  """Stack of per-task projections (reference :1850)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input depth.')
    p.Define('hidden_layer_dims', [], 'Hidden dims.')
    p.Define('num_tasks', 0, 'Number of tasks.')
    p.Define('activation', 'RELU', 'Activation (str or list).')
    p.Define('dropout', None, 'Dropout params.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    n = len(p.hidden_layer_dims)
    act = p.activation if isinstance(p.activation, (list, tuple)) else [p.activation] * n
    layers, d = [], p.input_dim
    for i, h in enumerate(p.hidden_layer_dims):
      layers.append(MultitaskProjectionEinsumLayer.Params().Set(
          name='fc_%d' % i, input_dim=d, output_dim=h, num_tasks=p.num_tasks,
          activation=act[i], has_bias=True))
      d = h
    self.CreateChildren('fc', layers)
    self.CreateChildren('dropout', [
        (p.dropout or DropoutLayer.Params()).Copy().Set(name='do_%d' % i)
        for i in range(n)])

  def FProp(self, theta, inputs, tasks, paddings=None):
    out = inputs
    for i in range(len(self.fc)):
      out = self.fc[i].FProp(theta.fc[i], out, tasks, paddings)
      out = self.dropout[i].FProp(theta.dropout[i], out)
    return out


class StackingOverTime(base_layer.BaseLayer):
  """Stacks `left+1+right` frames with a stride (reference :2006)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('left_context', 0, 'Frames stacked from the left.')
    p.Define('right_context', 0, 'Frames stacked from the right.')
    p.Define('stride', 1, 'Output stride.')
    p.Define('pad_with_left_frame', False, 'Pad left with the first frame.')
    p.Define('pad_with_right_frame', False, 'Pad right with the last frame.')
    p.Define('padding_reduce_option', 'reduce_min', 'reduce_min|reduce_max.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.left_context >= 0 and p.right_context >= 0 and p.stride >= 1
    assert p.padding_reduce_option in ('reduce_min', 'reduce_max')

  @property
  def window_size(self):
    return self.params.left_context + self.params.right_context + 1

  def _Stack(self, x, pad_left_frame=False, pad_right_frame=False, pad_val=0.0):
    """x [B, T, D] → [B, ceil(T/stride), D*window]."""
    p = self.params
    if p.left_context == 0 and p.right_context == 0:
      return x[:, ::p.stride]
    b, t, d = x.shape
    left = (x[:, :1].expand(b, p.left_context, d) if pad_left_frame
            else torch.full((b, p.left_context, d), pad_val, dtype=x.dtype,
                            device=x.device))
    right = (x[:, -1:].expand(b, p.right_context, d) if pad_right_frame
             else torch.full((b, p.right_context, d), pad_val, dtype=x.dtype,
                             device=x.device))
    xp = torch.cat([left, x, right], dim=1)
    win = xp.unfold(1, self.window_size, 1)          # [B, T, D, W]
    win = win.permute(0, 1, 3, 2).reshape(b, t, self.window_size * d)
    return win[:, ::p.stride]

  def FProp(self, inputs, paddings=None):
    """inputs [B, T, D], paddings [B, T, 1] → (stacked, out_paddings)."""
    p = self.params
    if paddings is None:
      paddings = torch.zeros(inputs.shape[0], inputs.shape[1], 1,
                             dtype=inputs.dtype, device=inputs.device)
    out = self._Stack(inputs, p.pad_with_left_frame, p.pad_with_right_frame)
    sp = self._Stack(paddings, pad_val=1.0)
    if p.padding_reduce_option == 'reduce_min':
      out_pad = sp.amin(dim=2, keepdim=True)
    else:
      out_pad = sp.amax(dim=2, keepdim=True)
    out = out * (1.0 - out_pad).to(out.dtype)
    return out, out_pad

  def Unstack(self, stacked):
    """Inverse for stride == window (reference :2230)."""
    p = self.params
    if p.stride == 1 and self.window_size == 1:
      return stacked
    assert p.stride == self.window_size
    b, t, dw = stacked.shape
    d = dw // self.window_size
    out = stacked.reshape(b, t * self.window_size, d)
    return out[:, p.left_context:]

  def __call__(self, *args, **kwargs):
    return self.FProp(*args, **kwargs)


class PoolingLayer(quant_utils.QuantizableLayer):
  """2-D max/avg pooling with paddings (reference :2285)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('window_shape', (0, 0), '(height, width).')
    p.Define('window_stride', (0, 0), '(height, width) strides.')
    p.Define('pooling_type', 'MAX', 'MAX|AVG.')
    p.Define('padding_algorithm', 'SAME', 'SAME|VALID.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.name
    assert len(p.window_shape) == 2 and len(p.window_stride) == 2
    assert all(x > 0 for x in p.window_shape)
    assert all(x > 0 for x in p.window_stride)
    assert p.pooling_type in ['MAX', 'AVG']

  def OutShape(self, in_shape):
    p = self.params
    b, h, w, c = in_shape
    return [b, _ConvOutSize(h, p.window_shape[0], p.window_stride[0],
                            p.padding_algorithm),
            _ConvOutSize(w, p.window_shape[1], p.window_stride[1],
                         p.padding_algorithm), c]

  def FProp(self, theta, inputs, paddings=None):
    p = self.params
    x = inputs.permute(0, 3, 1, 2)
    kh, kw = p.window_shape
    sh, sw = p.window_stride
    if paddings is not None:
      x = x * (1.0 - paddings.reshape(paddings.shape[0], 1, -1, 1).to(x.dtype))
    neg = torch.finfo(x.dtype).min if p.pooling_type == 'MAX' else 0.0
    if p.padding_algorithm == 'SAME':
      hl, hr = _SamePad(x.shape[2], kh, sh)
      wl, wr = _SamePad(x.shape[3], kw, sw)
      if hl or hr or wl or wr:
        if p.pooling_type == 'AVG':
          ones = torch.ones_like(x[:, :1])
          cnt = F.avg_pool2d(F.pad(ones, (wl, wr, hl, hr)), (kh, kw), (sh, sw))
          y = F.avg_pool2d(F.pad(x, (wl, wr, hl, hr)), (kh, kw), (sh, sw)) / cnt
          x = None
        else:
          x = F.pad(x, (wl, wr, hl, hr), value=neg)
    if x is not None:
      y = (F.max_pool2d(x, (kh, kw), (sh, sw)) if p.pooling_type == 'MAX'
           else F.avg_pool2d(x, (kh, kw), (sh, sw)))
    out = y.permute(0, 2, 3, 1)
    if paddings is None:
      return out
    out_pad = ComputeConvOutputPadding(paddings, kh, sh, p.padding_algorithm)
    return py_utils.ApplyPadding(out_pad, out), out_pad

  @classmethod
  def FPropMeta(cls, p, inputs, paddings=None):
    b, h, w, c = inputs
    from lingvo_b200.core import tshape
    oh = _ConvOutSize(h, p.window_shape[0], p.window_stride[0], 'SAME')
    ow = _ConvOutSize(w, p.window_shape[1], p.window_stride[1], 'SAME')
    out = tshape.Shape([b, oh, ow, c])
    return NestedMap(flops=out.num_elements() * p.window_shape[0] *
                     p.window_shape[1], out_shapes=(out,))


class BlurPoolLayer(base_layer.BaseLayer):
  """Anti-aliased downsampling in time (reference :2410)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('blur_filter', 'B5', 'B5|B7.')
    p.Define('subsample_type', '1D', '1D|2D.')
    p.Define('input_channels', None, 'Number of input channels.')
    return p

  def FProp(self, theta, inputs, paddings):
    p = self.params
    k = {'B5': [1., 4., 6., 4., 1.], 'B7': [1., 6., 15., 20., 15., 6., 1.]}[
        p.blur_filter]
    k = torch.tensor(k, dtype=inputs.dtype, device=inputs.device)
    k = k / k.sum()
    b, t, f, c = inputs.shape
    x = py_utils.ApplyPadding(paddings, inputs).permute(0, 3, 2, 1).reshape(
        b * c * f, 1, t)
    stride = 2
    lo, hi = _SamePad(t, k.numel(), stride)
    y = F.conv1d(F.pad(x, (lo, hi)), k.reshape(1, 1, -1), stride=stride)
    y = y.reshape(b, c, f, -1).permute(0, 3, 2, 1)
    if p.subsample_type == '2D':
      y = F.avg_pool2d(y.permute(0, 3, 1, 2), (1, 2), (1, 2)).permute(0, 2, 3, 1)
    out_pad = paddings[:, ::stride]
    return py_utils.ApplyPadding(out_pad, y), out_pad


# ------------------------------------------------------------------ embedding --
class SingleShardEmbeddingLayer(base_layer.BaseLayer):
  """Embedding lookup, single table (reference :2505)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_size', 0, 'Num tokens in vocab.')
    p.Define('embedding_dim', 0, 'Depth of the output.')
    p.Define('scale_sqrt_depth', False, 'Scale activations by sqrt(dim).')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.vocab_size > 0 and p.embedding_dim > 0 and p.name

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('emb_var', WeightParams(
        [p.vocab_size, p.embedding_dim], p.params_init, p.dtype,
        [self.__class__.__name__ + '_vars']))

  def EmbLookupDefaultTheta(self, ids):
    return self.EmbLookup(self.theta, ids)

  def EmbLookup(self, theta, ids):
    p = self.params
    out = F.embedding(ids.long(), theta.emb_var)
    if p.scale_sqrt_depth:
      out = out * (p.embedding_dim**0.5)
    return out

  def FProp(self, theta, ids):
    return self.EmbLookup(theta, ids)


class EmbeddingLayer(base_layer.BaseLayer):
  """Vocab-sharded embedding (reference :2585).

  `max_num_shards` variables `var_i` hold the rows `i, i+S, …` ("mod"
  sharding like tf.nn.embedding_lookup); lookups gather from the owning shard.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_size', 0, 'Depth of the input.')
    p.Define('embedding_dim', 0, 'Depth of the output.')
    p.Define('max_num_shards', 0, 'Num param shards.')
    p.Define('on_ps', True, 'Kept for parity.')
    p.Define('scale_sqrt_depth', False, 'Scale by sqrt(dim).')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.vocab_size > 0 and p.embedding_dim > 0 and p.max_num_shards > 0
    self._ids_per_shard = int(math.ceil(p.vocab_size / p.max_num_shards))
    self._actual_shards = int(math.ceil(p.vocab_size / self._ids_per_shard))

  @property
  def actual_shards(self):
    return self._actual_shards

  def _CreateLayerVariables(self):
    p = self.params
    for i in range(self._actual_shards):
      self.CreateVariable('var_%d' % i, WeightParams(
          [self._ids_per_shard, p.embedding_dim], p.params_init, p.dtype,
          [self.__class__.__name__ + '_vars']))

  def _Table(self, theta):
    # mod-sharded rows interleaved back into [V, D]
    shards = [theta['var_%d' % i] for i in range(self._actual_shards)]
    tbl = torch.stack(shards, dim=1).reshape(-1, self.params.embedding_dim)
    return tbl

  def EmbLookupDefaultTheta(self, ids):
    return self.EmbLookup(self.theta, ids)

  def EmbLookup(self, theta, ids):
    p = self.params
    s = self._actual_shards
    ids = ids.long()
    if s == 1:
      out = F.embedding(ids, theta.var_0)
    else:
      out = F.embedding(ids, self._Table(theta))
    if p.scale_sqrt_depth:
      out = out * (p.embedding_dim**0.5)
    return out

  def FProp(self, theta, ids):
    return self.EmbLookup(theta, ids)


class SimpleEmbeddingLayer(quant_utils.QuantizableLayer):
  """Embedding via gather or one-hot matmul (reference :2679)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_size', 0, 'Depth of the input.')
    p.Define('embedding_dim', 0, 'Depth of the output.')
    p.Define('use_matmul', False, 'One-hot matmul instead of gather.')
    p.Define('fprop_mode', None, 'None|matmul|loop|gather.')
    p.Define('use_3d_weight_tensor', False, 'Kept for parity.')
    p.Define('apply_pruning', False, 'Kept for parity.')
    p.Define('scale_sqrt_depth', False, 'Scale by sqrt(dim).')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.vocab_size > 0 and p.embedding_dim > 0

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('wm', WeightParams(
        [p.vocab_size, p.embedding_dim], p.params_init, p.dtype,
        [self.__class__.__name__ + '_vars']))

  def EmbLookupDefaultTheta(self, ids):
    return self.EmbLookup(self.theta, ids)

  def EmbLookup(self, theta, ids):
    p = self.params
    w = self.QWeight(theta.wm)
    if p.use_matmul or p.fprop_mode == 'matmul':
      oh = F.one_hot(ids.long(), p.vocab_size).to(w.dtype)
      out = torch.matmul(oh, w)
    else:
      out = F.embedding(ids.long(), w)
    if p.scale_sqrt_depth:
      out = out * (p.embedding_dim**0.5)
    return out

  def FProp(self, theta, ids):
    return self.EmbLookup(theta, ids)


class EinsumEmbeddingLayer(base_layer.BaseLayer):
  """Embedding with optional [V, N, H] reshaped weight (reference :3018)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_size', 0, 'Vocab size.')
    p.Define('embedding_dim', 0, 'Embedding dim.')
    p.Define('scale_sqrt_depth', False, 'Scale by sqrt(dim).')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('wm', WeightParams([p.vocab_size, p.embedding_dim],
                                           p.params_init, p.dtype))

  def EmbLookup(self, theta, ids):
    p = self.params
    out = F.embedding(ids.long(), theta.wm)
    return out * (p.embedding_dim**0.5) if p.scale_sqrt_depth else out

  def FProp(self, theta, ids):
    return self.EmbLookup(theta, ids)


class OneHotEmbeddingLayer(base_layer.BaseLayer):
  """ids → one-hot (optionally uncertain / smoothed) (reference :3088)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_size', 0, 'Depth of the input.')
    p.Define('embedding_dim', 0, 'Must equal vocab_size.')
    p.Define('uncertainty', 0.0, 'Mass spread uniformly over other ids.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.vocab_size > 1 and p.embedding_dim == p.vocab_size

  def EmbLookupDefaultTheta(self, ids):
    return self.EmbLookup(self.theta, ids)

  def EmbLookup(self, theta, ids):
    p = self.params
    low = p.uncertainty / (p.vocab_size - 1)
    oh = F.one_hot(ids.long().squeeze(-1) if ids.dim() > 1 and
                   ids.shape[-1] == 1 else ids.long(), p.vocab_size)
    return oh.to(self.fprop_dtype) * (1.0 - p.uncertainty - low) + low

  def FProp(self, theta, ids):
    return self.EmbLookup(theta, ids)


class PositionalEmbeddingLayer(base_layer.BaseLayer):
  """Sinusoidal timing signal (reference :3143)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('min_timescale', 1, 'Start of the geometric index.')
    p.Define('max_timescale', 10000, 'End of the geometric index.')
    p.Define('embedding_dim', 0, 'Dimension of the embedding.')
    p.Define('trainable_scaling', False, 'Learn a scale for the signal.')
    p.Define('trainable_scaling_init', 1.0, 'Initial scale value.')
    return p

  def __init__(self, params):
    super().__init__(params)
    assert self.params.embedding_dim % 2 == 0 or True

  def _CreateLayerVariables(self):
    p = self.params
    if p.trainable_scaling:
      self.CreateVariable('scale', WeightParams(
          [1], WeightInit.Constant(0.0), p.dtype))

  def _PosEmbeddingsFromPositions(self, theta, position):
    """position [B, T] → [B, T, D]."""
    p = self.params
    num_timescales = p.embedding_dim // 2
    log_inc = math.log(float(p.max_timescale) / float(p.min_timescale)) / max(
        num_timescales - 1, 1)
    inv = p.min_timescale * torch.exp(
        torch.arange(num_timescales, dtype=torch.float32,
                     device=position.device) * -log_inc)
    scaled = position.float().unsqueeze(-1) * inv
    signal = torch.cat([torch.sin(scaled), torch.cos(scaled)], dim=-1)
    if p.embedding_dim % 2:
      signal = F.pad(signal, (0, 1))
    if p.trainable_scaling:
      signal = signal * (p.trainable_scaling_init + theta.scale.float())
    return signal.to(self.fprop_dtype)

  def FProp(self, theta, seq_length):
    pos = torch.arange(seq_length, device=py_utils.CurrentDevice()).unsqueeze(0)
    if 'scale' in theta:
      pos = pos.to(theta.scale.device)
    return self._PosEmbeddingsFromPositions(theta, pos)[0]

  def FPropWithPosition(self, theta, position_tensor):
    return self._PosEmbeddingsFromPositions(theta, position_tensor)


class LearnablePositionalEmbeddingLayer(base_layer.BaseLayer):
  """Learned absolute positions (reference :3296)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('embedding_dim', 0, 'Dimension of the embedding.')
    p.Define('max_pos', 512, 'Maximum position.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w', WeightParams([p.max_pos, p.embedding_dim],
                                          p.params_init, p.dtype))

  def FProp(self, theta, seq_length):
    return theta.w[:seq_length]

  def FPropWithPosition(self, theta, position_tensor):
    return F.embedding(position_tensor.long(), theta.w)


class RelativePositionalEmbeddingLayer(base_layer.BaseLayer):
  """Clipped relative-position embedding table (reference :3380)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('radius', None, 'Relative distance is clipped to [-r, r].')
    p.Define('dim', None, 'Dimension of embedding.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    if not isinstance(p.radius, int) or p.radius <= 0:
      raise ValueError('params.radius must be a positive int, got %s' % p.radius)
    if not isinstance(p.dim, int) or p.dim <= 0:
      raise ValueError('params.dim must be a positive int, got %s' % p.dim)

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w', WeightParams([2 * p.radius + 1, p.dim],
                                          p.params_init, p.dtype))

  def FProp(self, theta, relative_distance):
    p = self.params
    d = relative_distance.clamp(-p.radius, p.radius) + p.radius
    return F.embedding(d.long(), theta.w)


class SinusoidalPositionalEmbeddingLayer(base_layer.BaseLayer):
  """sin/cos interleaved positional embedding (reference :3433)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('embedding_dim', 0, 'Dimension of the embedding.')
    return p

  def FPropWithPosition(self, theta, position):
    p = self.params
    d = p.embedding_dim
    inv = torch.exp(torch.arange(0, d, 2, dtype=torch.float32,
                                 device=position.device) * (-math.log(10000.0) / d))
    ang = position.float().unsqueeze(-1) * inv
    out = torch.stack([torch.sin(ang), torch.cos(ang)], dim=-1).reshape(
        list(position.shape) + [-1])[..., :d]
    return out.to(self.fprop_dtype)

  def FProp(self, theta, seq_length):
    return self.FPropWithPosition(
        theta, torch.arange(seq_length, device=py_utils.CurrentDevice())
        .unsqueeze(0))[0]


class RotaryPositionalEmbeddingLayer(PositionalEmbeddingLayer):
  """RoPE, half-split rotate (reference :3476; SURVEY K8)."""

  def _Rotate(self, inputs, position):
    """inputs [B, T, N, H] (or [B, T, H]); position [B, T] or None."""
    p = self.params
    h = inputs.shape[-1]
    assert h == p.embedding_dim, (h, p.embedding_dim)
    half = h // 2
    frac = torch.arange(half, dtype=torch.float32, device=inputs.device) * 2.0 / h
    timescale = p.min_timescale * (p.max_timescale / p.min_timescale)**frac
    if position is None:
      position = torch.arange(inputs.shape[1], dtype=torch.float32,
                              device=inputs.device).unsqueeze(0)
    ang = position.float().unsqueeze(-1) / timescale     # [B, T, half]
    while ang.dim() < inputs.dim():
      ang = ang.unsqueeze(-2)
    sin, cos = torch.sin(ang), torch.cos(ang)
    x = inputs.float()
    a, b = x[..., :half], x[..., half:]
    out = torch.cat([a * cos - b * sin, b * cos + a * sin], dim=-1)
    return out.to(inputs.dtype)

  def FProp(self, theta, inputs, position=None):
    return self._Rotate(inputs, position)


# -------------------------------------------------------------------- softmax --
class SoftmaxLayer(quant_utils.QuantizableLayer):
  """Base class for softmax layers (reference :3559)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Dimension of the input.')
    p.Define('num_classes', 0, 'Total number of target classes.')
    p.Define('logits_abs_max', None, 'Clip logits to ±this (hard).')
    p.Define('logits_soft_max', 0.0, 'Soft cap: max·tanh(logits/max).')
    p.Define('chunk_size', 0, 'Compute xent in row chunks to save memory.')
    return p

  def Logits(self, **unused):
    raise NotImplementedError('GetLogits is not implemented.')

  def XentLossFromLogits(self, **unused):
    raise NotImplementedError()

  def XentLoss(self, *args, **kwargs):
    return self.FProp(self.theta, *args, **kwargs)

  def _FProp2D(self, theta, inputs, class_weights, class_ids=None,
               class_probabilities=None):
    raise NotImplementedError('_FProp2D is not implemented.')

  def FProp(self, theta, inputs, class_weights, class_ids=None,
            class_probabilities=None):
    """inputs [..., D]; class_weights [...]; class_ids [...] → xent NestedMap."""
    p = self.params
    if isinstance(inputs, (list, tuple)):
      inputs = inputs[0] if len(inputs) == 1 else torch.cat(inputs, -1)
    lead = list(inputs.shape[:-1])
    x2 = inputs.reshape(-1, inputs.shape[-1])
    w2 = class_weights.reshape(-1, 1)
    ids2 = class_ids.reshape(-1, 1) if class_ids is not None else None
    pr2 = (class_probabilities.reshape(-1, p.num_classes)
           if class_probabilities is not None else None)
    out = self._FProp2D(theta, x2, w2, ids2, pr2)
    def unflat(t, tail):
      return t.reshape(lead + tail) if t is not None else None
    if out.get('logits') is not None:
      out.logits = unflat(out.logits, [p.num_classes])
    if out.get('log_probs') is not None:
      out.log_probs = unflat(out.log_probs, [p.num_classes])
    out.per_example_argmax = unflat(out.per_example_argmax, [])
    out.per_example_xent = unflat(out.per_example_xent, [])
    out.per_example_weight = unflat(out.per_example_weight, [])
    return out


def _CapLogits(logits, abs_max, soft_max):
  if abs_max is not None:
    logits = torch.clamp(logits, -abs_max, abs_max)
  if soft_max and soft_max > 0.0:
    logits = soft_max * torch.tanh(logits / soft_max)
  return logits


class SimpleFullSoftmax(SoftmaxLayer):
  """Full softmax (optionally sampled) (reference :3697).

  Weights `weight_i` / `bias_i` per shard, each `[D, C/num_shards]` (or
  `[C/num_shards, D]` with `use_num_classes_major_weight`). With
  `num_sampled > 0` training uses sampled softmax (log-uniform candidates).
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_sampled', 0, 'Number of samples for sampled softmax.')
    p.Define('num_shards', 1, 'Number of weight shards along the class dim.')
    p.Define('apply_pruning', False, 'Kept for parity.')
    p.Define('pruning_hparams_dict', None, 'Kept for parity.')
    p.Define('use_num_classes_major_weight', False, 'Weights are [C, D].')
    p.Define('use_bias', True, 'Whether to use bias.')
    p.Define('bias_init', 0, 'Bias init.')
    p.Define('label_smoothing', 0.0, 'Uniform label smoothing.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.name
    assert p.num_classes % p.num_shards == 0
    assert p.input_dim > 0 and p.num_classes > 0
    self.TrackQTensor('inputs', 'logits')

  def _CreateLayerVariables(self):
    p = self.params
    per = p.num_classes // p.num_shards
    shape = [per, p.input_dim] if p.use_num_classes_major_weight else [
        p.input_dim, per]
    coll = [self.__class__.__name__ + '_vars']
    for i in range(p.num_shards):
      self.CreateVariable('weight_%d' % i, WeightParams(
          shape, p.params_init, p.dtype, coll))
    if p.use_bias:
      for i in range(p.num_shards):
        self.CreateVariable('bias_%d' % i, WeightParams(
            [per], WeightInit.Constant(scale=p.bias_init), p.dtype, coll))

  def _GetInputs(self, inputs):
    if isinstance(inputs, (list, tuple)):
      assert len(inputs) == 1
      return inputs[0]
    return inputs

  def _ConcatWeights(self, theta):
    """→ ([D, C] weights, [C] bias or None)."""
    p = self.params
    ws = [theta['weight_%d' % i] for i in range(p.num_shards)]
    if p.use_num_classes_major_weight:
      ws = [w.t() for w in ws]
    w = ws[0] if len(ws) == 1 else torch.cat(ws, dim=1)
    b = None
    if p.use_bias:
      bs = [theta['bias_%d' % i] for i in range(p.num_shards)]
      b = bs[0] if len(bs) == 1 else torch.cat(bs, dim=0)
    return self.QWeight(w), b

  def _LogitsUsingConcatenatedWeights(self, theta, inputs):
    p = self.params
    inputs = self.QTensor('inputs', inputs)
    w, b = self._ConcatWeights(theta)
    logits = torch.matmul(inputs, w.to(inputs.dtype))
    if b is not None:
      logits = logits + b.to(logits.dtype)
    logits = _CapLogits(logits, p.logits_abs_max, p.logits_soft_max)
    return self.QTensor('logits', logits)

  def Logits(self, theta, inputs):
    inputs = self._GetInputs(inputs)
    return self._LogitsUsingConcatenatedWeights(theta, inputs)

  def SimpleLogits(self, theta, inputs):
    return self.Logits(theta, inputs)

  def _XentLossByChunk(self, theta, activation, class_ids):
    """Memory-lean xent: logits are computed per row chunk and recomputed in
    the backward pass (reference `_XentLossByChunk`)."""
    p = self.params
    n = activation.shape[0]
    chunk = p.chunk_size
    from torch.utils.checkpoint import checkpoint
    w, b = self._ConcatWeights(theta)

    def one(act, ids):
      logits = torch.matmul(act, w.to(act.dtype))
      if b is not None:
        logits = logits + b.to(logits.dtype)
      logits = _CapLogits(logits, p.logits_abs_max, p.logits_soft_max).float()
      xent = F.cross_entropy(logits, ids.reshape(-1).long(), reduction='none',
                             label_smoothing=p.label_smoothing)
      return xent, logits.argmax(-1)

    xs, am = [], []
    for s in range(0, n, chunk):
      x, a = checkpoint(one, activation[s:s + chunk], class_ids[s:s + chunk],
                        use_reentrant=False)
      xs.append(x)
      am.append(a)
    return torch.cat(xs), torch.cat(am)

  def _SampledXent(self, theta, inputs, class_ids):
    """Sampled softmax with log-uniform candidates + logQ correction."""
    p = self.params
    w, b = self._ConcatWeights(theta)
    n = inputs.shape[0]
    c = p.num_classes
    gen = torch.Generator(device=inputs.device)
    gen.manual_seed(py_utils.GenerateStepSeedPair(p)[1] + 17)
    u = torch.rand(p.num_sampled, generator=gen, device=inputs.device)
    sampled = (torch.exp(u * math.log(c + 1.0)) - 1.0).long().clamp(max=c - 1)
    def logq(ids):
      idf = ids.float()
      prob = (torch.log(idf + 2.0) - torch.log(idf + 1.0)) / math.log(c + 1.0)
      return torch.log(-torch.expm1(p.num_sampled * torch.log1p(-prob)))
    true = class_ids.reshape(-1).long()
    wt = w.to(inputs.dtype)
    true_logits = (inputs * wt[:, true].t()).sum(-1).float()
    samp_logits = torch.matmul(inputs, wt[:, sampled]).float()
    if b is not None:
      true_logits = true_logits + b[true].float()
      samp_logits = samp_logits + b[sampled].float()
    true_logits = true_logits - logq(true)
    samp_logits = samp_logits - logq(sampled)
    hit = sampled.unsqueeze(0) == true.unsqueeze(1)
    samp_logits = samp_logits.masked_fill(hit, -1e9)
    logits = torch.cat([true_logits.unsqueeze(1), samp_logits], dim=1)
    xent = F.cross_entropy(logits, torch.zeros(n, dtype=torch.long,
                                               device=inputs.device),
                           reduction='none')
    return xent

  def _FProp2D(self, theta, inputs, class_weights, class_ids=None,
               class_probabilities=None):
    p = self.params
    inputs = self._CastToFPropDtype(self._GetInputs(inputs))
    per_example_argmax = None
    logits = None
    log_probs = None
    if (p.num_sampled > 0 and not self.do_eval and class_ids is not None):
      per_example_xent = self._SampledXent(theta, inputs, class_ids)
      per_example_argmax = torch.zeros_like(class_ids.reshape(-1))
    elif p.chunk_size and class_ids is not None:
      per_example_xent, per_example_argmax = self._XentLossByChunk(
          theta, inputs, class_ids)
    else:
      fused = None
      if (class_ids is not None and ops.use_cuda_kernels(inputs) and
          inputs.dtype == torch.bfloat16 and p.logits_abs_max is None and
          not p.logits_soft_max and not p.label_smoothing):
        from lingvo_b200.ops import xent as xent_ops
        w, b = self._ConcatWeights(theta)
        fused = xent_ops.linear_xent(inputs, w, b, class_ids.reshape(-1))
      if fused is not None:
        per_example_xent, per_example_argmax, logits = fused
      else:
        logits = self.Logits(theta, inputs)
        lf = logits.float()
        log_probs = F.log_softmax(lf, dim=-1)
        if class_probabilities is not None:
          per_example_xent = -(class_probabilities.float() * log_probs).sum(-1)
        else:
          per_example_xent = F.nll_loss(log_probs, class_ids.reshape(-1).long(),
                                        reduction='none')
          if p.label_smoothing:
            per_example_xent = (1 - p.label_smoothing) * per_example_xent + (
                p.label_smoothing * -log_probs.mean(-1))
        per_example_argmax = lf.argmax(-1)
    cw = class_weights.reshape(-1).float()
    total_xent = (per_example_xent * cw).sum()
    total_weight = cw.sum()
    return NestedMap(
        logits=logits, log_probs=log_probs,
        per_example_argmax=per_example_argmax,
        per_example_xent=per_example_xent, per_example_weight=cw,
        total_xent=total_xent, total_weight=total_weight,
        avg_xent=total_xent / torch.clamp(total_weight, min=1e-8) if False else
        total_xent / torch.where(total_weight > 0, total_weight,
                                 torch.ones_like(total_weight)))

  def XentLossFromLogits(self, theta, logits, class_weights, class_ids=None,
                         class_probabilities=None):
    lf = logits.float()
    log_probs = F.log_softmax(lf, dim=-1)
    if class_probabilities is not None:
      xent = -(class_probabilities.float() * log_probs).sum(-1)
    else:
      xent = -torch.gather(log_probs, -1, class_ids.long().unsqueeze(-1)
                           ).squeeze(-1)
    cw = class_weights.float()
    total_xent = (xent * cw).sum()
    total_weight = cw.sum()
    return NestedMap(logits=logits, log_probs=log_probs,
                     per_example_argmax=lf.argmax(-1), per_example_xent=xent,
                     per_example_weight=cw, total_xent=total_xent,
                     total_weight=total_weight,
                     avg_xent=total_xent / torch.clamp(total_weight, min=1e-8))


class SimpleFullSigmoidCrossEntropy(SimpleFullSoftmax):
  """Sigmoid xent over independent classes (reference :4130)."""

  def _FProp2D(self, theta, inputs, class_weights, class_ids=None,
               class_probabilities=None):
    p = self.params
    logits = self.Logits(theta, self._GetInputs(inputs))
    if class_probabilities is None:
      class_probabilities = F.one_hot(class_ids.reshape(-1).long(),
                                      p.num_classes).float()
    xent = F.binary_cross_entropy_with_logits(
        logits.float(), class_probabilities.float(), reduction='none').sum(-1)
    cw = class_weights.reshape(-1).float()
    tx, tw = (xent * cw).sum(), cw.sum()
    return NestedMap(logits=logits, log_probs=F.logsigmoid(logits.float()),
                     per_example_argmax=logits.argmax(-1),
                     per_example_xent=xent, per_example_weight=cw,
                     total_xent=tx, total_weight=tw,
                     avg_xent=tx / torch.clamp(tw, min=1e-8))


class FocalFullSoftmax(SimpleFullSoftmax):
  """Focal-loss softmax (reference :4184)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('focal_loss_alpha', None, 'Per-class weights.')
    p.Define('focal_loss_gamma', None, 'Focusing parameter.')
    return p

  def _FProp2D(self, theta, inputs, class_weights, class_ids=None,
               class_probabilities=None):
    p = self.params
    logits = self.Logits(theta, self._GetInputs(inputs))
    xent = py_utils.SoftmaxCrossEntropyFocalLoss(
        logits, None if class_ids is None else class_ids.reshape(-1),
        class_probabilities, p.focal_loss_alpha, p.focal_loss_gamma)
    cw = class_weights.reshape(-1).float()
    tx, tw = (xent * cw).sum(), cw.sum()
    return NestedMap(logits=logits,
                     log_probs=F.log_softmax(logits.float(), -1),
                     per_example_argmax=logits.argmax(-1),
                     per_example_xent=xent, per_example_weight=cw,
                     total_xent=tx, total_weight=tw,
                     avg_xent=tx / torch.clamp(tw, min=1e-8))


class Scones(SimpleFullSoftmax):
  """SCONES: per-class sigmoids with pos/neg weighting (reference :4221)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('pos_weight', 1.0, 'Weight of positive classes.')
    return p

  def _FProp2D(self, theta, inputs, class_weights, class_ids=None,
               class_probabilities=None):
    p = self.params
    logits = self.Logits(theta, self._GetInputs(inputs)).float()
    if class_probabilities is None:
      class_probabilities = F.one_hot(class_ids.reshape(-1).long(),
                                      p.num_classes).float()
    ls = F.logsigmoid(logits)
    lns = F.logsigmoid(-logits)
    xent = -(p.pos_weight * class_probabilities * ls +
             (1 - class_probabilities) * lns).sum(-1)
    cw = class_weights.reshape(-1).float()
    tx, tw = (xent * cw).sum(), cw.sum()
    return NestedMap(logits=logits, log_probs=ls,
                     per_example_argmax=logits.argmax(-1),
                     per_example_xent=xent, per_example_weight=cw,
                     total_xent=tx, total_weight=tw,
                     avg_xent=tx / torch.clamp(tw, min=1e-8))


class SingleShardFullSoftmax(SoftmaxLayer):
  """Full softmax with a single [D, C] weight (reference :4494)."""

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    lin = builder_linear = None
    self.CreateChild('linear', ProjectionLayer.Params().Set(
        input_dim=p.input_dim, output_dim=p.num_classes, batch_norm=False,
        has_bias=False, activation='NONE', name='linear'))
    self.CreateChild('bias', BiasLayerSimple.Params().Set(
        dims=p.num_classes, name='bias'))

  def Logits(self, theta, inputs):
    if isinstance(inputs, (list, tuple)):
      inputs = inputs[0]
    p = self.params
    logits = self.bias.FProp(theta.bias, self.linear.FProp(theta.linear, inputs))
    return _CapLogits(logits, p.logits_abs_max, p.logits_soft_max)

  def DenseWeights(self, theta):
    """NestedMap(wm `[D, C]`, b `[C]`) — the dense view of the softmax weights (ref :4523)."""
    return NestedMap(wm=theta.linear.w, b=theta.bias.b)

  def XentLossByChunk(self, theta, activation, class_ids, class_probabilities=None):
    """Per-example (xent, argmax) with the `[chunk, C]` logits of ONE row chunk alive at a
    time: every chunk is rematerialised in the backward pass (ref :4583). The number of rows
    must be a multiple of `chunk_size`."""
    from torch.utils.checkpoint import checkpoint   # pylint: disable=g-import-not-at-top
    p = self.params
    n, chunk = activation.shape[0], p.chunk_size
    assert chunk > 0 and n % chunk == 0, (n, chunk)

    def One(act, ids, probs):
      logits = self.Logits(theta, act).float()
      if probs is not None:
        xent = -(probs.float() * F.log_softmax(logits, -1)).sum(-1)
      else:
        xent = F.cross_entropy(logits, ids.reshape(-1).long(), reduction='none')
      return xent, logits.argmax(-1)

    xs, am = [], []
    for s in range(0, n, chunk):
      ids = None if class_ids is None else class_ids[s:s + chunk]
      probs = None if class_probabilities is None else class_probabilities[s:s + chunk]
      x, a = checkpoint(One, activation[s:s + chunk], ids, probs, use_reentrant=False)
      xs.append(x)
      am.append(a)
    return torch.cat(xs), torch.cat(am)

  def _FProp2D(self, theta, inputs, class_weights, class_ids=None,
               class_probabilities=None):
    p = self.params
    if p.chunk_size:
      if isinstance(inputs, (list, tuple)):
        inputs = inputs[0]
      xent, amax = self.XentLossByChunk(
          theta, inputs, None if class_ids is None else class_ids.reshape(-1),
          class_probabilities)
      cw = class_weights.reshape(-1).float()
      tx, tw = (xent * cw).sum(), cw.sum()
      return NestedMap(logits=None, log_probs=None, per_example_argmax=amax,
                       per_example_xent=xent, per_example_weight=cw, total_xent=tx,
                       total_weight=tw, avg_xent=tx / torch.clamp(tw, min=1e-8))
    logits = self.Logits(theta, inputs)
    return SimpleFullSoftmax.XentLossFromLogits(
        self, theta, logits, class_weights.reshape(-1),
        None if class_ids is None else class_ids.reshape(-1),
        class_probabilities)


class BiasLayerSimple(base_layer.BaseLayer):
  """y = x + b."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('dims', 0, 'Depth of the input.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('b', WeightParams([p.dims], WeightInit.Constant(0.0),
                                          p.dtype))

  def FProp(self, theta, inputs):
    return inputs + theta.b.to(inputs.dtype)


class SingleShardSharedEmbeddingSoftmax(SingleShardFullSoftmax):
  """Softmax whose weight doubles as the embedding table (reference :4725)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_size', 0, 'Num tokens in vocab.')
    p.Define('embedding_dim', 0, 'Depth of the output.')
    p.Define('scale_sqrt_depth', False, 'Scale by sqrt(dim).')
    p.Define('emb_with_matmul', False, 'One-hot matmul lookup.')
    return p

  def __init__(self, params):
    params = params.Copy()
    if params.vocab_size:
      params.num_classes = params.vocab_size
    if params.embedding_dim:
      params.input_dim = params.embedding_dim
    super().__init__(params)

  def EmbLookupDefaultTheta(self, ids):
    return self.EmbLookup(self.theta, ids)

  def EmbLookup(self, theta, ids):
    p = self.params
    w = theta.linear.w  # [D, V]
    out = F.embedding(ids.long(), w.t())
    if p.scale_sqrt_depth:
      out = out * (p.input_dim**0.5)
    return out


class SharedSoftmaxLayer(base_layer.BaseLayer):
  """Softmax + embedding sharing one weight (reference :4403)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('softmax', SimpleFullSoftmax.Params(), 'Softmax params.')
    p.Define('vocab_size', 0, 'Vocab size.')
    p.Define('embedding_dim', 0, 'Embedding dim.')
    p.Define('scale_sqrt_depth', False, 'Scale by sqrt(dim).')
    p.Define('input_dim', 0, 'Softmax-side name of embedding_dim (either may be set).')
    p.Define('num_classes', 0, 'Softmax-side name of vocab_size (either may be set).')
    p.Define('num_shards', 1, 'Kept for the softmax interface; the weight is one shard.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self._dim = p.embedding_dim or p.input_dim
    self._vocab = p.vocab_size or p.num_classes
    sp = p.softmax.Copy().Set(name='softmax', input_dim=self._dim, num_classes=self._vocab,
                              num_shards=1, use_num_classes_major_weight=True)
    self.CreateChild('softmax', sp)

  def EmbLookup(self, theta, ids):
    p = self.params
    out = F.embedding(ids.long(), theta.softmax.weight_0)
    return out * (self._dim**0.5) if p.scale_sqrt_depth else out

  def Logits(self, theta, inputs):
    return self.softmax.Logits(theta.softmax, inputs)

  def FProp(self, theta, *args, **kwargs):
    return self.softmax.FProp(theta.softmax, *args, **kwargs)


class EinsumSoftmax(base_layer.BaseLayer):
  """Softmax on [..., D] with [D, C] weight via einsum (reference :4252)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('num_classes', 0, 'Classes.')
    p.Define('use_bias', True, 'Use bias.')
    p.Define('label_smoothing', 0.0, 'Label smoothing.')
    p.Define('z_loss_coef', 0.0, 'z-loss coefficient.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w', WeightParams([p.input_dim, p.num_classes],
                                          p.params_init, p.dtype))
    if p.use_bias:
      self.CreateVariable('b', WeightParams([p.num_classes],
                                            WeightInit.Constant(0.0), p.dtype))

  def Logits(self, theta, inputs):
    y = torch.matmul(inputs, theta.w.to(inputs.dtype))
    return y + theta.b.to(y.dtype) if self.params.use_bias else y

  def FProp(self, theta, inputs, class_weights, class_ids=None,
            class_probabilities=None):
    p = self.params
    logits = self.Logits(theta, inputs).float()
    log_probs = F.log_softmax(logits, -1)
    if class_probabilities is None:
      class_probabilities = F.one_hot(class_ids.long(), p.num_classes).float()
      if p.label_smoothing:
        class_probabilities = class_probabilities * (1 - p.label_smoothing) + (
            p.label_smoothing / p.num_classes)
    xent = -(class_probabilities * log_probs).sum(-1)
    if p.z_loss_coef:
      xent = xent + p.z_loss_coef * torch.logsumexp(logits, -1)**2
    cw = class_weights.float()
    tx, tw = (xent * cw).sum(), cw.sum()
    return NestedMap(logits=logits, log_probs=log_probs,
                     per_example_argmax=logits.argmax(-1),
                     per_example_xent=xent, per_example_weight=cw,
                     total_xent=tx, total_weight=tw,
                     avg_xent=tx / torch.clamp(tw, min=1e-8))


class ConvSoftmax(quant_utils.QuantizableLayer):
  """A softmax implemented as a 1x1 conv over time (reference :4784)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('hidden_dim', 0, 'Bottleneck dim (0 = none).')
    p.Define('num_classes', 0, 'Classes.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    d = p.input_dim
    if p.hidden_dim:
      self.CreateVariable('w_proj', WeightParams([1, p.input_dim, p.hidden_dim],
                                                 p.params_init, p.dtype))
      d = p.hidden_dim
    self.CreateVariable('w', WeightParams([1, d, p.num_classes],
                                          p.params_init, p.dtype))
    self.CreateVariable('b', WeightParams([p.num_classes],
                                          WeightInit.Constant(0.0), p.dtype))

  def Logits(self, theta, inputs):
    p = self.params
    x = inputs
    if p.hidden_dim:
      x = torch.matmul(x, theta.w_proj[0].to(x.dtype))
    return torch.matmul(x, theta.w[0].to(x.dtype)) + theta.b.to(x.dtype)


# -------------------------------------------------------------------- dropout --
class DropoutLayer(base_layer.BaseLayer):
  """Dropout (reference :4842); `noise_shape` broadcast dims supported."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('keep_prob', 1.0, 'Keep probability.')
    p.Define('noise_shape', None, 'Shape of the random keep/drop flags.')
    p.Define('noise_shape_broadcast_dims', None, 'Dims with shared noise.')
    p.Define('dropout_at_eval', False, 'Apply dropout in eval too.')
    return p

  def _Dropout(self, theta, inputs, noise_shape):
    p = self.params
    if noise_shape is None:
      return F.dropout(inputs, 1.0 - p.keep_prob, training=True)
    keep = torch.rand(noise_shape, device=inputs.device) < p.keep_prob
    return inputs * keep.to(inputs.dtype) / p.keep_prob

  @classmethod
  def NumOutputNodes(cls, p):
    return None

  def FProp(self, theta, inputs):
    p = self.params
    if not self.do_eval or p.dropout_at_eval:
      if isinstance(p.keep_prob, (int, float)) and p.keep_prob == 1.0:
        return inputs
      noise_shape = p.noise_shape
      if p.noise_shape_broadcast_dims:
        noise_shape = list(inputs.shape)
        for d in p.noise_shape_broadcast_dims:
          noise_shape[d] = 1
      return self._Dropout(theta, inputs, noise_shape)
    return inputs

  @classmethod
  def FPropMeta(cls, p, inputs, *args):
    return NestedMap(flops=inputs.num_elements() * 10, out_shapes=(inputs,))


class DeterministicDropoutLayer(DropoutLayer):
  """Dropout keyed by (global_step, step_seed) (reference :4916)."""

  def _Dropout(self, theta, inputs, noise_shape):
    return py_utils.DeterministicDropout(
        inputs, self.params.keep_prob,
        py_utils.GenerateStepSeedPair(self.params), noise_shape=noise_shape)


# ------------------------------------------------------------------ layernorm --
class LayerNorm(base_layer.BaseLayer):
  """Layer normalisation (reference :4927).

  scale stored as `(1 + scale)` unless `direct_scale`; `bias`/`center`
  switches. bf16 inputs on CUDA take the fused sm_90a kernel (`ops.norm.layer_norm`);
  every other input is normalised in fp32 and keeps its dtype.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Depth of the input to the network.')
    p.Define('epsilon', 1e-6, 'Tiny value to guard rsqrt.')
    p.Define('use_fused_layernorm', False, 'Kept for parity (always fused here).')
    p.Define('direct_scale', False, 'Scale var holds the scale (init 1).')
    p.Define('bias', True, 'Whether to use bias.')
    p.Define('center', True, 'Subtract the mean.')
    p.Define('use_defun', True, 'Kept for parity.')
    p.Define('use_batch_norm_backend', False, 'Kept for parity.')
    p.Define('trainable_scale_and_bias', True, 'Scale/bias are trainable.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.name
    assert p.input_dim > 0

  def _CreateLayerVariables(self):
    p = self.params
    coll = [self.__class__.__name__ + '_vars', py_utils._SKIP_LP_COLLECTION]  # pylint: disable=protected-access
    if p.bias:
      self.CreateVariable('bias', WeightParams(
          [p.input_dim], WeightInit.Constant(0.0), p.dtype, coll),
          trainable=p.trainable_scale_and_bias)
    self.CreateVariable('scale', WeightParams(
        [p.input_dim], WeightInit.Constant(1.0 if p.direct_scale else 0.0),
        p.dtype, coll), trainable=p.trainable_scale_and_bias)

  def _GetScaleAndBias(self, theta):
    p = self.params
    scale = theta.scale if p.direct_scale else 1.0 + theta.scale
    bias = theta.bias if p.bias else None
    return scale, bias

  def FProp(self, theta, inputs):
    p = self.params
    inputs = self._CastToFPropDtype(inputs)
    scale, bias = self._GetScaleAndBias(theta)
    if (inputs.dtype == torch.bfloat16 and ops.use_cuda_kernels(inputs) and
        inputs.shape[-1] % 8 == 0):
      from lingvo_b200.ops import norm
      return norm.layer_norm(inputs, scale, bias, p.epsilon, center=p.center)
    x = inputs.float()
    if p.center:
      mean = x.mean(-1, keepdim=True)
      x = x - mean
    var = (x * x).mean(-1, keepdim=True)
    y = x * torch.rsqrt(var + p.epsilon) * scale.float()
    if bias is not None:
      y = y + bias.float()
    return y.to(inputs.dtype)

  @classmethod
  def NumOutputNodes(cls, p):
    return p.input_dim

  @classmethod
  def FPropMeta(cls, p, inputs):
    return NestedMap(flops=inputs.num_elements() * 10, out_shapes=(inputs,))


class ReshapedLayerNorm(LayerNorm):
  """LayerNorm over the last two dims of [..., N, H] (reference :5099)."""

  def FProp(self, theta, inputs):
    shp = inputs.shape
    flat = inputs.reshape(list(shp[:-2]) + [shp[-2] * shp[-1]])
    return super().FProp(theta, flat).reshape(shp)


class CategoricalLayerNorm(LayerNorm):
  """LayerNorm with per-class scale/bias (reference :5151)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_classes', 1, 'Number of privatized copies of LN params.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    coll = [py_utils._SKIP_LP_COLLECTION]  # pylint: disable=protected-access
    for i in range(p.num_classes):
      self.CreateVariable('bias_%d' % i, WeightParams(
          [p.input_dim], WeightInit.Constant(0.0), p.dtype, coll))
      self.CreateVariable('scale_%d' % i, WeightParams(
          [p.input_dim], WeightInit.Constant(0.0), p.dtype, coll))
    self._class_index = 0

  def SetClassIndex(self, idx):
    self._class_index = idx

  def _GetScaleAndBias(self, theta):
    i = self._class_index
    if isinstance(i, torch.Tensor):
      i = int(i.item())
    return 1.0 + theta['scale_%d' % i], theta['bias_%d' % i]


# ------------------------------------------------------------- small layers --
class ConvSetLayer(quant_utils.QuantizableLayer):
  """Parallel convs with different kernels, concatenated (reference :5203)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('cnn_tpl', ConvLayer.Params().Set(filter_stride=(1, 1)),
             'Conv layer template.')
    p.Define('filter_shapes', [(0, 0, 0, 0)], 'Filter shapes of the set.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    filters = sorted(set(p.filter_shapes))
    self.CreateChildren('conv_set', [
        p.cnn_tpl.Copy().Set(name='%s_%d' % (p.name, i), filter_shape=f)
        for i, f in enumerate(filters)])

  def FProp(self, theta, inputs, paddings):
    outs, out_pad = [], None
    for i, conv in enumerate(self.conv_set):
      o, out_pad = conv.FProp(theta.conv_set[i], inputs, paddings)
      outs.append(o)
    return torch.cat(outs, dim=-1), out_pad


class UniformLabelSmoother(base_layer.BaseLayer):
  """Uniform label smoothing (reference :5383)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_classes', 0, 'Number of classes.')
    p.Define('uncertainty', 0.1, 'Uncertainty of correct label.')
    p.Define('uncertainty_larger', 0.1, 'Uncertainty for EOS etc.')
    p.Define('token_id_uncertainty_larger', None, 'Id with larger uncertainty.')
    return p

  def FProp(self, theta, target_paddings, target_labels, target_ids):
    p = self.params
    low = p.uncertainty / (p.num_classes - 1)
    oh = F.one_hot(target_labels.long(), p.num_classes).float()
    out = oh * (1.0 - p.uncertainty - low) + low
    if p.token_id_uncertainty_larger is not None:
      low2 = p.uncertainty_larger / (p.num_classes - 1)
      alt = oh * (1.0 - p.uncertainty_larger - low2) + low2
      is_larger = (target_ids == p.token_id_uncertainty_larger).unsqueeze(-1)
      out = torch.where(is_larger, alt, out)
    return out


class LocalizedLabelSmoother(base_layer.BaseLayer):
  """Smooths one-hot labels with the labels of neighbouring *time steps* (reference :5305):
  at time t the target is `onehot[t] + Σ_i weights[i] · onehot[t + offsets[i]]`, renormalised.
  Offsets reaching outside the sequence contribute nothing, and neither do padded positions
  (nor the last valid label, so EOS is not made more probable elsewhere)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_classes', 0, 'Number of classes.')
    p.Define('offsets', [], 'Time offsets (e.g. [-2, -1, 1, 2]).')
    p.Define('weights', [], 'Weight of the smoothing at the corresponding offset.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.num_classes > 0
    assert len(p.offsets) == len(p.weights)
    assert p.name

  def FProp(self, theta, target_paddings, target_labels, target_ids):
    """paddings / labels / ids `[B, T]` → distribution `[B, T, num_classes]`."""
    del target_ids
    p = self.params
    probs = F.one_hot(target_labels.long(), p.num_classes).to(py_utils.FPropDtype(p))
    seq_len = probs.shape[1]
    lo = -min(list(p.offsets) + [0])
    hi = max(list(p.offsets) + [0])
    padded = F.pad(probs, (0, 0, lo, hi))
    # weights shifted left by one: the last valid position (EOS) never leaks to neighbours
    cw = F.pad(1.0 - target_paddings[:, 1:].to(probs.dtype), (lo, hi + 1)).unsqueeze(-1)
    out = probs
    for off, w in zip(p.offsets, p.weights):
      s = off + lo
      out = out + padded[:, s:s + seq_len] * cw[:, s:s + seq_len] * w
    return out / out.sum(-1, keepdim=True)


class HighwaySkipLayer(base_layer.BaseLayer):
  """Highway: y = t·x̃ + (1-t)·x (reference :5461)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dimension.')
    p.Define('batch_norm', False, 'BN in the projections.')
    p.Define('carry_bias_init', 1.0, 'Carry gate bias init.')
    p.Define('couple_carry_transform_gates', False, 'c = 1 - t.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    carry = ProjectionLayer.Params().Set(
        batch_norm=p.batch_norm, has_bias=True, activation='SIGMOID',
        input_dim=p.input_dim, output_dim=p.input_dim,
        bias_init=p.carry_bias_init, name='%s_carry_gate' % p.name)
    self.CreateChild('carry_gate', carry)
    if not p.couple_carry_transform_gates:
      self.CreateChild('transform_gate', carry.Copy().Set(
          bias_init=-p.carry_bias_init, name='%s_transform_gate' % p.name))

  def FProp(self, theta, x, transformed_x, paddings=None):
    p = self.params
    carry = self.carry_gate.FProp(theta.carry_gate, x, paddings)
    t = (1.0 - carry if p.couple_carry_transform_gates else
         self.transform_gate.FProp(theta.transform_gate, x, paddings))
    return transformed_x * t + x * carry


class GatingLayer(base_layer.BaseLayer):
  """g = σ(W[a;b]); out = g·a + (1-g)·b (reference :5533)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('has_bias', False, 'Use bias.')
    p.Define('carry_bias_init', 0.0, 'Bias init.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('carry_gate', ProjectionLayer.Params().Set(
        batch_norm=False, has_bias=p.has_bias, activation='SIGMOID',
        input_dim=p.input_dim * 2, output_dim=p.input_dim,
        bias_init=p.carry_bias_init, name='carry'))

  def FProp(self, theta, x, y, paddings=None):
    carry = self.carry_gate.FProp(theta.carry_gate, torch.cat([x, y], -1),
                                  paddings)
    return x * carry + y * (1.0 - carry)


class GradNormTracker(base_layer.BaseLayer):
  """Tracks log-grad-norm moments and rejects outliers (reference :5590)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('decay', 0.995, 'Decay of the moving moments.')
    p.Define('grad_norm_lower_cap', 1e-2, 'Lower cap of grad norm.')
    p.Define('clip_threshold', 4.0, 'Std-devs above the mean to reject.')
    p.Define('grad_norm_clip_cap_min', 0.0, 'Never clip below this norm.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self._log_mean = 0.0
    self._log_mean_sq = 0.0
    self._total_weight = 0.0
    self._total_rejections = 0.0

  def FProp(self, theta, grad_norm, has_nan=None):
    """Returns grad_scale ∈ {0, 1}."""
    p = self.params
    gn = float(grad_norm)
    if has_nan is not None and bool(has_nan):
      return torch.zeros((), device=grad_norm.device if isinstance(
          grad_norm, torch.Tensor) else None)
    gn = max(gn, p.grad_norm_lower_cap)
    lg = math.log(gn)
    tw = max(self._total_weight, 1e-6)
    mean = self._log_mean / tw
    var = max(self._log_mean_sq / tw - mean * mean, 0.0)
    std = math.sqrt(var)
    cap = math.exp(mean + std * p.clip_threshold)
    cap = max(cap, p.grad_norm_clip_cap_min)
    reject = self._total_weight > 0.75 and gn > cap
    if not reject:
      self._log_mean = self._log_mean * p.decay + lg * (1 - p.decay)
      self._log_mean_sq = self._log_mean_sq * p.decay + lg * lg * (1 - p.decay)
      self._total_weight = self._total_weight * p.decay + (1 - p.decay)
    else:
      self._total_rejections += 1
    dev = grad_norm.device if isinstance(grad_norm, torch.Tensor) else None
    return torch.tensor(0.0 if reject else 1.0, device=dev)


class WeightedSumLayer(base_layer.BaseLayer):
  """Softmax-weighted (or global) sum of N tensors (reference :5705)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_sources', 0, 'Number of input sources to combine.')
    p.Define('weighted_merger_dropout_prob', 0.1, 'Dropout on merge weights.')
    p.Define('weighted_merger_softmax', True, 'Softmax the weights.')
    p.Define('global_weight_scale', 1.0, 'Scale of the sum.')
    p.Define('minimal_prob', 0.0, 'Floor for each weight.')
    p.Define('add_weight_summaries', False, 'Emit summaries.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.num_sources > 0
    self.CreateChild('weighted_merger_dropout', DropoutLayer.Params().Set(
        keep_prob=1.0 - p.weighted_merger_dropout_prob, name='dropout'))

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('sum_weight', WeightParams(
        [p.num_sources], WeightInit.Constant(1.0 / p.num_sources), p.dtype))

  def FProp(self, theta, inputs):
    p = self.params
    w = theta.sum_weight.float()
    if p.weighted_merger_softmax:
      w = torch.softmax(w, 0)
      if p.minimal_prob > 0:
        w = torch.clamp(w, min=p.minimal_prob)
        w = w / w.sum()
    w = self.weighted_merger_dropout.FProp(theta.weighted_merger_dropout, w)
    out = sum(x * w[i].to(x.dtype) for i, x in enumerate(inputs))
    return out * p.global_weight_scale


class GatedAverageLayer(base_layer.BaseLayer):
  """Input-conditioned softmax gating of N vectors (reference :5793)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_nodes', 0, 'Depth of each input.')
    p.Define('num_inputs', 0, 'Number of inputs.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('gm', WeightParams(
        [p.num_nodes * p.num_inputs, p.num_inputs], p.params_init, p.dtype))

  def FProp(self, theta, inputs):
    cat = torch.cat(inputs, dim=-1)
    gates = torch.softmax(torch.matmul(cat, theta.gm.to(cat.dtype)).float(), -1)
    stacked = torch.stack(inputs, dim=-1)
    return (stacked * gates.unsqueeze(-2).to(stacked.dtype)).sum(-1)


class LHUCLayer(base_layer.BaseLayer):
  """Learning hidden unit contribution: y = 2σ(w)·x (reference :5857)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Depth of the input.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w', WeightParams([p.input_dim],
                                          WeightInit.Constant(0.0), p.dtype))

  def FProp(self, theta, inp):
    return 2.0 * torch.sigmoid(theta.w.to(inp.dtype)) * inp


class ResidualAdapterLayer(base_layer.BaseLayer):
  """LN → down-proj → ReLU → up-proj → + residual (reference :5895)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('bottleneck_dim', 0, 'Bottleneck dim.')
    p.Define('ln_tpl', LayerNorm.Params(), 'LN template.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('ln', p.ln_tpl.Copy().Set(input_dim=p.input_dim, name='ln'))
    self.CreateChild('layers', FeedForwardNet.Params().Set(
        name='layers', input_dim=p.input_dim,
        hidden_layer_dims=[p.bottleneck_dim, p.input_dim],
        activation=['RELU', 'NONE'], has_bias=True,
        params_init=WeightInit.Gaussian(0.001)))

  def FProp(self, theta, x, paddings=None):
    h = self.ln.FProp(theta.ln, x)
    return x + self.layers.FProp(theta.layers, h, paddings)


class FetchLayer(base_layer.BaseLayer):
  """Records intermediate activations by name (reference :6077)."""

  def __init__(self, params):
    super().__init__(params)
    self._activations = None
    self._gradients = None

  @classmethod
  def FPropMeta(cls, p, *args):
    return NestedMap(flops=0, out_shapes=args)

  def _ReturnSingleValueOrList(self, lst):
    assert lst is not None
    return lst[0] if len(lst) == 1 else lst

  @property
  def activation(self):
    return self._ReturnSingleValueOrList(self._activations)

  @property
  def gradient(self):
    return self._ReturnSingleValueOrList(self._gradients)

  def FProp(self, theta, *args):
    self._activations = list(args)
    self._gradients = [None] * len(args)
    out = []
    for i, a in enumerate(args):
      if isinstance(a, torch.Tensor) and a.requires_grad:
        def hook(g, i=i):
          self._gradients[i] = g
        a.register_hook(hook)
      out.append(a)
    return tuple(out) if len(out) > 1 else out[0]


class GluLayer(base_layer.BaseLayer):
  """Gated linear unit block with residual (reference :6124)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('output_dim', 0, 'Output dim (0 ⇒ input dim).')
    p.Define('ln_tpl', LayerNorm.Params(), 'LN template.')
    p.Define('dense_tpl', FCLayer.Params().Set(activation='NONE'), 'Dense tpl.')
    p.Define('activation', 'RELU', 'Non-linearity before the gate.')
    p.Define('dropout_tpl', DropoutLayer.Params(), 'Dropout.')
    p.Define('apply_residual', True, 'Residual connection.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    od = p.output_dim or p.input_dim
    if p.apply_residual:
      assert od == p.input_dim
    self.CreateChild('layer_norm', p.ln_tpl.Copy().Set(
        name='ln', input_dim=p.input_dim))
    self.CreateChildren('dense', [
        p.dense_tpl.Copy().Set(name='dense_%d' % i, input_dim=p.input_dim,
                               output_dim=od) for i in range(2)])
    self.CreateChild('dropout', p.dropout_tpl.Copy().Set(name='dropout'))

  def FProp(self, theta, inputs, paddings):
    p = self.params
    x = self.layer_norm.FProp(theta.layer_norm, inputs)
    a = activations.GetFn(p.activation)(self.dense[0].FProp(theta.dense[0], x))
    g = torch.sigmoid(self.dense[1].FProp(theta.dense[1], x))
    out = self.dropout.FProp(theta.dropout, a * g)
    if p.apply_residual:
      out = out + inputs
    return py_utils.ApplyPadding(paddings, out) if paddings is not None else out


class MultitaskAdapterBaseLayer(quant_utils.QuantizableLayer):
  """Base of per-task residual adapters (reference :6205)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_tasks', 0, 'Number of tasks.')
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('bottleneck_dim', 0, 'Bottleneck dim.')
    p.Define('layer_norm_tpl', LayerNorm.Params(), 'LN template.')
    p.Define('projection_params_init', None, 'Init for projections.')
    p.Define('data_format', 'TBC', 'TBC|BTC.')
    p.Define('clip_task_ids', False, 'Clip task ids into range.')
    return p


class MultitaskAdapterLayer(MultitaskAdapterBaseLayer):
  """Adapters with task-embedded weights (reference :6249)."""

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    init = p.projection_params_init or WeightInit.Gaussian(0.01)
    self.CreateChild('down_proj_w', EmbeddingLayer.Params().Set(
        vocab_size=p.num_tasks, embedding_dim=p.input_dim * p.bottleneck_dim,
        max_num_shards=1, params_init=init, name='down_proj_w'))
    self.CreateChild('down_proj_b', EmbeddingLayer.Params().Set(
        vocab_size=p.num_tasks, embedding_dim=p.bottleneck_dim,
        max_num_shards=1, params_init=WeightInit.Constant(0.0),
        name='down_proj_b'))
    self.CreateChild('up_proj_w', EmbeddingLayer.Params().Set(
        vocab_size=p.num_tasks, embedding_dim=p.bottleneck_dim * p.input_dim,
        max_num_shards=1, params_init=init, name='up_proj_w'))
    self.CreateChild('up_proj_b', EmbeddingLayer.Params().Set(
        vocab_size=p.num_tasks, embedding_dim=p.input_dim,
        max_num_shards=1, params_init=WeightInit.Constant(0.0),
        name='up_proj_b'))
    self.CreateChild('layer_norm', p.layer_norm_tpl.Copy().Set(
        input_dim=p.input_dim, name='ln'))

  def FProp(self, theta, inputs, tasks):
    """inputs [T,B,D] (TBC) or [B,T,D]; tasks [B] (or matching [T,B])."""
    p = self.params
    if p.clip_task_ids:
      tasks = tasks.clamp(0, p.num_tasks - 1)
    x = inputs if p.data_format == 'BTC' else inputs.transpose(0, 1)
    if tasks.dim() == 2:
      tasks = tasks[:, 0] if p.data_format == 'BTC' else tasks[0]
    b = x.shape[0]
    dw = self.down_proj_w.EmbLookup(theta.down_proj_w, tasks).reshape(
        b, p.input_dim, p.bottleneck_dim)
    db = self.down_proj_b.EmbLookup(theta.down_proj_b, tasks).unsqueeze(1)
    uw = self.up_proj_w.EmbLookup(theta.up_proj_w, tasks).reshape(
        b, p.bottleneck_dim, p.input_dim)
    ub = self.up_proj_b.EmbLookup(theta.up_proj_b, tasks).unsqueeze(1)
    h = self.layer_norm.FProp(theta.layer_norm, x)
    h = torch.relu(torch.bmm(h, dw.to(h.dtype)) + db.to(h.dtype))
    h = torch.bmm(h, uw.to(h.dtype)) + ub.to(h.dtype)
    out = x + h
    return out if p.data_format == 'BTC' else out.transpose(0, 1)


class MultitaskAdapterEinsumLayer(MultitaskAdapterBaseLayer):
  """Adapters with stacked [num_tasks, …] weights (reference :6386)."""

  def _CreateLayerVariables(self):
    p = self.params
    init = p.projection_params_init or WeightInit.Gaussian(0.01)
    self.CreateVariable('down_w', WeightParams(
        [p.num_tasks, p.input_dim, p.bottleneck_dim], init, p.dtype))
    self.CreateVariable('down_b', WeightParams(
        [p.num_tasks, p.bottleneck_dim], WeightInit.Constant(0.0), p.dtype))
    self.CreateVariable('up_w', WeightParams(
        [p.num_tasks, p.bottleneck_dim, p.input_dim], init, p.dtype))
    self.CreateVariable('up_b', WeightParams(
        [p.num_tasks, p.input_dim], WeightInit.Constant(0.0), p.dtype))

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('layer_norm', p.layer_norm_tpl.Copy().Set(
        input_dim=p.input_dim, name='ln'))

  def FProp(self, theta, inputs, tasks):
    p = self.params
    if p.clip_task_ids:
      tasks = tasks.clamp(0, p.num_tasks - 1)
    x = inputs if p.data_format == 'BTC' else inputs.transpose(0, 1)
    if tasks.dim() == 2:
      tasks = tasks[:, 0] if p.data_format == 'BTC' else tasks[0]
    h = self.layer_norm.FProp(theta.layer_norm, x)
    h = torch.relu(py_utils.MultiTaskProjection(
        theta.down_w.to(h.dtype), theta.down_b.to(h.dtype), h, tasks))
    h = py_utils.MultiTaskProjection(theta.up_w.to(h.dtype),
                                     theta.up_b.to(h.dtype), h, tasks)
    out = x + h
    return out if p.data_format == 'BTC' else out.transpose(0, 1)


class CCTGatingNetwork(quant_utils.QuantizableLayer):
  """Conditional-computation gating network (reference :6565)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('hidden_layer_dim', 0, 'Hidden dim.')
    p.Define('num_outputs', 0, 'Number of gates.')
    p.Define('noise_std', 1.0, 'Training noise std.')
    p.Define('noise_warmup_steps', 1.0, 'Noise warm-up steps.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('gating_layer', FeedForwardNet.Params().Set(
        name='gating_layer', input_dim=p.input_dim,
        hidden_layer_dims=[p.hidden_layer_dim, p.num_outputs],
        activation=['RELU', 'NONE'], has_bias=True))

  def FProp(self, theta, inputs, paddings=None):
    p = self.params
    logits = self.gating_layer.FProp(theta.gating_layer, inputs, paddings)
    if self.do_eval:
      return (logits > 0).to(inputs.dtype)
    step = float(py_utils.GetGlobalStep())
    std = p.noise_std * min(1.0, step / max(p.noise_warmup_steps, 1.0))
    return torch.sigmoid(logits + torch.randn_like(logits) * std)


class CondScaleShiftFFNLayer(base_layer.BaseLayer):
  """FFN producing conditional (scale, shift) (reference :6623)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('output_dim', 0, 'Output dim (scale & shift each).')
    p.Define('ffn', FeedForwardNet.Params(), 'Shared FFN.')
    p.Define('fc_out', FCLayer.Params(), 'Output FC.')
    p.Define('scale_fn', 'NONE', 'Activation on scale.')
    p.Define('shift_fn', 'NONE', 'Activation on shift.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    ffn = p.ffn.Copy().Set(name='ffn', input_dim=p.input_dim)
    self.CreateChild('ffn', ffn)
    hid = ffn.hidden_layer_dims[-1] if ffn.hidden_layer_dims else p.input_dim
    self.CreateChild('fc_out', p.fc_out.Copy().Set(
        name='fc_out', input_dim=hid, output_dim=2 * p.output_dim,
        activation='NONE'))

  def FProp(self, theta, inputs, paddings=None):
    p = self.params
    h = self.ffn.FProp(theta.ffn, inputs, paddings)
    out = self.fc_out.FProp(theta.fc_out, h, paddings)
    scale, shift = torch.chunk(out, 2, dim=-1)
    return (activations.GetFn(p.scale_fn)(scale),
            activations.GetFn(p.shift_fn)(shift))


class StatisticalPoolingLayer(base_layer.BaseLayer):
  """Mean (+std) pooling over time (reference :6694)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('has_stddev', True, 'Concatenate stddev.')
    p.Define('epsilon', 1e-6, 'Stability epsilon.')
    p.Define('float_var_floor', 1e-6, 'Variance floor.')
    return p

  def FProp(self, features, paddings):
    """features [B, T, D], paddings [B, T] → [B, D or 2D]."""
    p = self.params
    mask = (1.0 - paddings.float()).unsqueeze(-1)
    x = features.float() * mask
    cnt = torch.clamp(mask.sum(1), min=1.0)
    mean = x.sum(1) / cnt
    if not p.has_stddev:
      return mean.to(features.dtype)
    var = (((features.float() - mean.unsqueeze(1))**2) * mask).sum(1) / cnt
    std = torch.sqrt(torch.clamp(var, min=p.float_var_floor) + p.epsilon)
    return torch.cat([mean, std], -1).to(features.dtype)

  def __call__(self, *a, **k):
    return self.FProp(*a, **k)


class PerFrameStatisticalPoolingLayer(base_layer.BaseLayer):
  """Causal / windowed per-frame mean (+std) (reference :6997)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('has_stddev', True, 'Concatenate stddev.')
    p.Define('left_context', -1, 'Frames to the left (-1 = all).')
    p.Define('right_context', 0, 'Frames to the right.')
    p.Define('epsilon', 1e-6, 'Epsilon.')
    return p

  def FProp(self, features, paddings):
    p = self.params
    mask = (1.0 - paddings.float()).unsqueeze(-1)
    x = features.float() * mask
    b, t, d = x.shape
    def wsum(v):
      c = torch.cumsum(v, 1)
      c0 = F.pad(c, (0, 0, 1, 0))
      idx = torch.arange(t, device=v.device)
      hi = (idx + p.right_context).clamp(max=t - 1) + 1
      lo = torch.zeros_like(idx) if p.left_context < 0 else (
          idx - p.left_context).clamp(min=0)
      return c0[:, hi] - c0[:, lo]
    cnt = torch.clamp(wsum(mask), min=1.0)
    mean = wsum(x) / cnt
    if not p.has_stddev:
      return mean.to(features.dtype)
    var = torch.clamp(wsum(x * x) / cnt - mean * mean, min=0.0)
    return torch.cat([mean, torch.sqrt(var + p.epsilon)], -1).to(features.dtype)

  def __call__(self, *a, **k):
    return self.FProp(*a, **k)


class LSHMemoryRankKOneHotTaskLayer(base_layer.BaseLayer):
  """LSH-bucketed per-task memory lookup (reference :6749, simplified hash)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('output_dim', 0, 'Output dim.')
    p.Define('num_tasks', 1, 'Number of tasks.')
    p.Define('num_hash_bits', 8, 'Hash bits ⇒ 2^bits buckets.')
    p.Define('rank', 1, 'Rank of the per-bucket update.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('hash_proj', WeightParams(
        [p.input_dim, p.num_hash_bits], WeightInit.Gaussian(1.0), p.dtype),
        trainable=False)
    self.CreateVariable('memory', WeightParams(
        [p.num_tasks, 2**p.num_hash_bits, p.rank, p.output_dim],
        WeightInit.Gaussian(0.01), p.dtype))

  def FProp(self, theta, inputs, tasks=None):
    p = self.params
    bits = (torch.matmul(inputs.float(), theta.hash_proj.float()) > 0).long()
    pw = 2**torch.arange(p.num_hash_bits, device=inputs.device)
    bucket = (bits * pw).sum(-1)
    t = torch.zeros_like(bucket) if tasks is None else tasks.long().reshape(
        [-1] + [1] * (bucket.dim() - 1)).expand_as(bucket)
    return theta.memory[t, bucket].sum(-2).to(inputs.dtype)


class LSHTaskWithMultiplierLayer(LSHMemoryRankKOneHotTaskLayer):
  """LSH memory producing a multiplicative gate (reference :6896)."""

  def FProp(self, theta, inputs, tasks=None):
    mem = super().FProp(theta, inputs, tasks)
    return inputs * (1.0 + mem) if mem.shape[-1] == inputs.shape[-1] else mem


class MaskedLmDataAugmenter(base_layer.BaseLayer):
  """BERT-style masking of input ids (reference :7175)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_size', 0, 'Vocab size.')
    p.Define('mask_prob', 0.12, 'Probability a token is masked.')
    p.Define('random_prob', 0.015, 'Probability replaced by a random token.')
    p.Define('same_prob', 0.015, 'Probability kept but predicted.')
    p.Define('mask_token_id', -1, 'Id of the [MASK] token.')
    return p

  def FProp(self, theta, inputs, paddings):
    """→ (augmented_ids, augmented_pos mask)."""
    p = self.params
    assert p.vocab_size > 0 and p.mask_token_id >= 0
    gen = torch.Generator(device=inputs.device)
    a, b = py_utils.GenerateStepSeedPair(p)
    gen.manual_seed((a * 1000003 + b) % (2**31 - 1))
    u = torch.rand(inputs.shape, generator=gen, device=inputs.device)
    total = p.mask_prob + p.random_prob + p.same_prob
    valid = paddings < 0.5
    is_mask = (u < p.mask_prob) & valid
    is_rand = (u >= p.mask_prob) & (u < p.mask_prob + p.random_prob) & valid
    is_same = (u >= p.mask_prob + p.random_prob) & (u < total) & valid
    rnd = torch.randint(0, p.vocab_size, inputs.shape, generator=gen,
                        device=inputs.device, dtype=inputs.dtype)
    out = torch.where(is_mask, torch.full_like(inputs, p.mask_token_id), inputs)
    out = torch.where(is_rand, rnd, out)
    pos = (is_mask | is_rand | is_same).float()
    return out, pos


def Conv2DFlops(inputs, filter_shape, stride, padding):
  """Multiply-adds ×2 of a conv2d: `inputs` shape [B, H, W, …], filter [fh, fw, ic, oc],
  stride (sh, sw), padding 'SAME' | 'VALID' (reference :5950)."""
  b, h, w = int(inputs[0]), int(inputs[1]), int(inputs[2])
  fh, fw, ic, oc = [int(x) for x in filter_shape]
  sh, sw = stride
  ceil_div = lambda x, y: (x + y - 1) // y
  if padding == 'SAME':
    oh, ow = ceil_div(h, sh), ceil_div(w, sw)
  else:
    assert padding == 'VALID'
    oh, ow = ceil_div(h - fh + 1, sh), ceil_div(w - fw + 1, sw)
  return b * oh * ow * fh * fw * ic * oc * 2
