"""Model builder base with composition helpers.

Reference `lingvo/core/builder.py:37-374`: `Base.Params` (fprop_dtype,
device_mesh, split mappings, deterministic_dropout) and the composition
methods `_Rep/_Seq/_Graph/_Id/_Arg/_Par/_Fn/_Save/_AddFetches/_Rematerialize/
_BatchParallel/_PrintShape/_CreateNestedMap/_Dropout/_Linear/_Bias/_Add…`.
"""

from __future__ import annotations

import numpy as np
import torch

from lingvo_b200.core import activations
from lingvo_b200.core import builder_layers
from lingvo_b200.core import hyperparams
from lingvo_b200.core import layers
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap


class Base:
  """Model builder with commonly used layers."""

  @classmethod
  def Params(cls):
    p = hyperparams.InstantiableParams(cls)
    p.Define('deterministic_dropout', False, 'Use deterministic dropout.')
    p.Define('dtype', torch.float32, 'Variable dtype.')
    p.Define('fprop_dtype', None, 'Activations dtype (bf16 on H100).')
    p.Define('device_mesh', None, 'np.ndarray device mesh.')
    p.Define('weight_split_dims_mapping', None, 'Default weight sharding.')
    p.Define('activation_split_dims_mapping', None, 'Default act sharding.')
    return p

  @property
  def params(self):
    return self._params

  def __init__(self, params):
    self._params = params.Copy()
    p = self._params
    if p.device_mesh is not None:
      p.device_mesh = np.array(p.device_mesh)

  def _Layer(self, p, name):
    p.name = name
    bp = self.params
    if 'fprop_dtype' in p and bp.fprop_dtype is not None:
      p.fprop_dtype = bp.fprop_dtype
    return p

  # ------------------------------------------------------------ composition --
  def _Rep(self, name, repeat, *subs):
    """Sequentially repeats `subs` `repeat` times (stacked variables)."""
    return builder_layers.SequentialLayer.Params().Set(
        name=name, repeat=repeat, sub=list(subs))

  def _Seq(self, name, *subs):
    return self._Rep(name, 1, *subs)

  def _Graph(self, name, input_endpoints, output_endpoints, *signature_sub):
    return builder_layers.GraphLayer.Params().Set(
        name=name, input_endpoints=list(input_endpoints),
        output_endpoints=list(output_endpoints), sub=list(signature_sub))

  def _Id(self, name):
    return self._Seq(name)

  def _Identity(self, name):
    return layers.IdentityLayer.Params().Set(name=name)

  def _Arg(self, name, index):
    return builder_layers.ArgIndexLayer.Params().Set(name=name, idx=[index])

  def _Par(self, name, *subs):
    def merge(xs):
      rets = []
      for x in xs:
        rets += list(x)
      return tuple(rets)
    return builder_layers.ParallelLayer.Params().Set(
        name=name, sub=list(subs), merge=merge)

  def _Fn(self, name, fn, fn_out=None, fn_flops=None):
    def fn_meta(*shapes):
      flops = fn_flops(*shapes) if fn_flops else sum(
          s.size() if hasattr(s, 'size') else 0 for s in shapes)
      outs = fn_out(*shapes) if fn_out else shapes
      if not isinstance(outs, tuple):
        outs = (outs,)
      return NestedMap(flops=flops, out_shapes=outs)
    return builder_layers.FnLayer.Params().Set(name=name, fn=fn,
                                               fn_meta=fn_meta)

  def _Save(self, name):
    return layers.FetchLayer.Params().Set(name=name)

  def _AddFetches(self, name, body, fetches):
    return builder_layers.BranchLayer.Params().Set(name=name, body=body,
                                                   fetches=fetches)

  def _Rematerialize(self, name, body):
    return builder_layers.RematerializationLayer.Params().Set(name=name,
                                                              body=body)

  def _BatchParallel(self, name, sub):
    return builder_layers.BatchParallelLayer.Params().Set(name=name, sub=sub)

  def _PrintShape(self, name):
    return builder_layers.PrintShapeLayer.Params().Set(name=name)

  def _CreateNestedMap(self, name, keys):
    return builder_layers.CreateNestedMapLayer.Params().Set(name=name,
                                                            keys=keys)

  # ------------------------------------------------------------ basic layers --
  def _BN(self, name, dims):
    return layers.BatchNormLayer.Params().Set(name=name, dim=dims, decay=0.99)

  def _LN(self, name, dims, use_fused_layernorm=False):
    return self._Layer(layers.LayerNorm.Params().Set(input_dim=dims), name)

  def _Dropout(self, name, keep_prob, noise_shape_broadcast_dims=None):
    cls = (layers.DeterministicDropoutLayer if self.params.deterministic_dropout
           else layers.DropoutLayer)
    return cls.Params().Set(
        name=name, keep_prob=keep_prob,
        noise_shape_broadcast_dims=noise_shape_broadcast_dims)

  def _Linear(self, name, idims, odims, device_mesh=None,
              weight_split_dims_mapping=None, qdomain=None):
    p = builder_layers.LinearLayer.Params().Set(
        input_dims=idims, output_dims=odims,
        device_mesh=device_mesh if device_mesh is not None
        else self.params.device_mesh,
        weight_split_dims_mapping=weight_split_dims_mapping)
    return self._Layer(p, name)

  def _Bias(self, name, dims, device_mesh=None, weight_split_dims_mapping=None):
    return self._Layer(builder_layers.BiasLayer.Params().Set(
        dims=dims, device_mesh=device_mesh,
        weight_split_dims_mapping=weight_split_dims_mapping), name)

  def _Activation(self, name, fn='RELU'):
    return activations.ActivationLayer.Params().Set(name=name, activation=fn)

  def _FC(self, name, idims, odims, act='RELU'):
    return self._Seq(name, self._Linear('linear', idims, odims),
                     self._Bias('bias', odims), self._Activation('act', fn=act))

  def _MLP(self, name, dims, act='RELU'):
    l = []
    for n, (i, o) in enumerate(zip(dims[:-1], dims[1:])):
      l += [self._FC('l%03d' % n, i, o, act)]
    return self._Seq(name, *l)

  def _Conv2D(self, name, filter_shape, filter_stride):
    return layers.Conv2DLayerNoPadding.Params().Set(
        name=name, filter_shape=filter_shape, filter_stride=filter_stride)

  def _Reshape(self, name, shape):
    return builder_layers.ReshapeLayer.Params().Set(name=name, shape=shape)

  def _Add(self, name, residual_weight=1.0):
    return self._Fn(name, fn=lambda x, y: x + residual_weight * y,
                    fn_out=lambda x, y: x)

  def _Embedding(self, name, vocab_size, embedding_dim):
    return layers.SimpleEmbeddingLayer.Params().Set(
        name=name, vocab_size=vocab_size, embedding_dim=embedding_dim)
