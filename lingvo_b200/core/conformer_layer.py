"""Conformer blocks (ref `lingvo/core/conformer_layer.py`).

`LConvLayer` (ref :35): LN → linear(2d) → GLU → depthwise conv1d(k) →
BN/GroupNorm/LN → Swish → linear → dropout → +residual.
`ConformerLayer` (ref :471): ½·FFN → MHSA / LConv (order configurable) →
½·FFN → final LN, with streaming (`StreamStep`) for causal configs.

H100 path of the conv module: the three memory-bound stages in the middle
(GLU gate, padding mask, depthwise conv) run as ONE kernel
(`ops.conv.glu_dwconv1d`) that reads the `[B,T,2D]` projection once and writes
`[B,T,D]` once; LN/GroupNorm + Swish follow in the fused norm kernel.
"""

from __future__ import annotations

import torch
import torch.nn.functional as F

from lingvo_b200.core import activations
from lingvo_b200.core import base_layer
from lingvo_b200.core import batch_major_attention as attention_lib
from lingvo_b200.core import bn_layers
from lingvo_b200.core import conv_layers_with_time_padding as conv_lib
from lingvo_b200.core import hyperparams as hparams_lib
from lingvo_b200.core import layers
from lingvo_b200.core import layers_with_attention
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap


class LConvLayer(base_layer.BaseLayer):
  """Lightweight conv module of the Conformer (ref :35)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', None, 'Input (== output) dim.')
    p.Define('kernel_size', None, 'Depthwise conv kernel size.')
    p.Define('conv_activation', 'SWISH', 'Activation after normalisation.')
    p.Define('is_causal', False, 'Causal depthwise conv.')
    p.Define('glu_activation', 'NONE', 'Activation of the GLU gate input.')
    p.Define('dropout_prob', 0., 'Dropout probability.')
    p.Define('ln_tpl', layers.LayerNorm.Params(), 'Input LN.')
    p.Define('linear_start_tpl', layers.FCLayer.Params(), 'Linear start.')
    p.Define('depthwise_conv_tpl', conv_lib.DepthwiseConv2DLayer.Params(),
             'Depthwise conv template.')
    p.Define('conv_norm_layer_tpl', bn_layers.BatchNormLayer.Params(), 'Norm after conv.')
    p.Define('linear_end_tpl', layers.FCLayer.Params(), 'Linear end.')
    p.Define('dropout_tpl', layers.DropoutLayer.Params(), 'Residual dropout.')
    p.Define('split_act_gated_linear_start', False, 'Two separate start projections.')
    p.linear_start_tpl.Set(activation='NONE', has_bias=True)
    p.linear_end_tpl.Set(activation='NONE', has_bias=True)
    return p

  @classmethod
  def CommonParams(cls, input_dim=None, kernel_size=None, is_causal=False,
                   conv_activation='SWISH', dropout_prob=0.):
    p = cls.Params().Set(input_dim=input_dim, kernel_size=kernel_size,
                         is_causal=is_causal, conv_activation=conv_activation,
                         dropout_prob=dropout_prob)
    if is_causal:
      p.depthwise_conv_tpl = conv_lib.CausalDepthwiseConv2DLayer.Params()
    return p

  @classmethod
  def SetFPropDtype(cls, p, dtype):
    p.fprop_dtype = dtype
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    d = p.input_dim
    self.CreateChild('ln', p.ln_tpl.Copy().Set(input_dim=d))
    if p.split_act_gated_linear_start:
      self.CreateChild('linear_start_act', p.linear_start_tpl.Copy().Set(
          input_dim=d, output_dim=d))
      self.CreateChild('linear_start_gated', p.linear_start_tpl.Copy().Set(
          input_dim=d, output_dim=d))
    else:
      self.CreateChild('linear_start', p.linear_start_tpl.Copy().Set(
          input_dim=d, output_dim=2 * d))
    conv_tpl = p.depthwise_conv_tpl
    if p.is_causal and not issubclass(conv_tpl.cls, conv_lib.CausalDepthwiseConv2DLayer) \
        and not conv_tpl.is_causal:
      conv_tpl = conv_lib.CausalDepthwiseConv2DLayer.Params()
    self.CreateChild('depthwise_conv1d', conv_tpl.Copy().Set(
        filter_shape=(p.kernel_size, 1, d, 1)))
    norm = p.conv_norm_layer_tpl.Copy()
    if 'dim' in norm:
      norm.dim = d
    elif 'input_dim' in norm:
      norm.input_dim = d
    self.CreateChild('norm', norm)
    self.CreateChild('linear_end', p.linear_end_tpl.Copy().Set(input_dim=d, output_dim=d))
    self.CreateChild('dropout', p.dropout_tpl.Copy().Set(keep_prob=1. - p.dropout_prob))

  def _GLU(self, gated, act):
    p = self.params
    return activations.GetFn(p.glu_activation)(act) * torch.sigmoid(gated)

  def _Normalize(self, theta, x, paddings):
    """x [B,T,D] → normalised, dispatching on the norm layer's calling convention."""
    n = self.norm
    if isinstance(n, bn_layers.GroupNormLayer):
      y = n.FProp(theta.norm, x.unsqueeze(2), paddings)
      y = y[0] if isinstance(y, tuple) else y
      return y.squeeze(2)
    if isinstance(n, bn_layers.BatchNormLayer):
      return n.FProp(theta.norm, x, paddings.unsqueeze(-1))
    return n.FProp(theta.norm, x)

  def _Start(self, theta, inputs):
    p = self.params
    if p.split_act_gated_linear_start:
      act = self.linear_start_act.FProp(theta.linear_start_act, inputs)
      gated = self.linear_start_gated.FProp(theta.linear_start_gated, inputs)
      return gated, act
    proj = self.linear_start.FProp(theta.linear_start, inputs)
    gated, act = proj.chunk(2, -1)
    return gated, act

  def FProp(self, theta, inputs, paddings):
    """inputs [B,T,D], paddings [B,T] → (outputs [B,T,D], paddings)."""
    p = self.params
    inputs = self._CastToFPropDtype(inputs)
    residual = inputs
    x = self.ln.FProp(theta.ln, inputs)
    from lingvo_b200.ops import conv as conv_ops  # pylint: disable=g-import-not-at-top
    conv = self.depthwise_conv1d
    fused = (not p.split_act_gated_linear_start and p.glu_activation == 'NONE' and
             conv_ops.glu_dwconv1d_supported(x, conv))
    if fused:
      proj = self.linear_start.FProp(theta.linear_start, x)          # [B,T,2D]
      w = conv._GetWeight(theta.depthwise_conv1d).reshape(p.kernel_size, p.input_dim)  # pylint: disable=protected-access
      x = conv_ops.glu_dwconv1d(proj, w, paddings, causal=conv.params.is_causal)
    else:
      gated, act = self._Start(theta, x)
      x = self._GLU(gated, act)
      x, paddings = conv.FProp(theta.depthwise_conv1d, x.unsqueeze(2), paddings)
      x = x.squeeze(2)
    x = self._Normalize(theta, x, paddings)
    x = activations.GetFn(p.conv_activation)(x)
    x = self.linear_end.FProp(theta.linear_end, x)
    x = self.dropout.FProp(theta.dropout, x)
    return x + residual, paddings

  @classmethod
  def SetCanonicalShardingParams(cls, params):
    """Canonical 2-D mesh sharding: projections split [data, model], activations on the
    feature axis (ref :133)."""
    assert params.device_mesh is not None and params.device_mesh.ndim >= 2
    params.weight_split_dims_mapping = NestedMap(df=[0, 1], hwim=[-1, -1, 1, -1], fd=[1, 0])
    params.activation_split_dims_mapping = NestedMap(blf=[0, -1, 1], bld=[1, -1, -1])

  def _ApplyActivation(self, inputs, act_name):
    return inputs if act_name == 'NONE' else activations.GetFn(act_name)(inputs)

  def _NormalizeStep(self, theta, x, paddings, state0, state1):
    """Streaming normalisation (ref :361): a cumulative GroupNorm carries its running
    statistics in `norm_state`; BatchNorm (eval statistics) and LayerNorm are stateless."""
    n = self.norm
    if isinstance(n, bn_layers.GroupNormLayer) and n.params.cumulative:
      y, paddings, state1.norm_state = n.StreamStep(theta.norm, x.unsqueeze(2), paddings,
                                                    state0.norm_state)
      return y.squeeze(2), paddings
    return self._Normalize(theta, x, paddings), paddings

  def zero_state(self, batch_size):
    st = NestedMap(conv_state=self.depthwise_conv1d.zero_state(batch_size))
    if isinstance(self.norm, bn_layers.GroupNormLayer) and self.norm.params.cumulative:
      st.norm_state = self.norm.zero_state(batch_size)
    return st

  def StreamStep(self, theta, inputs, paddings, state0):
    """Causal streaming step over a chunk `[B, Q, D]`."""
    p = self.params
    assert p.is_causal
    residual = inputs
    x = self.ln.FProp(theta.ln, inputs)
    gated, act = self._Start(theta, x)
    x = self._GLU(gated, act)
    x, paddings, conv_state1 = self.depthwise_conv1d.StreamStep(
        theta.depthwise_conv1d, x.unsqueeze(2), paddings, state0.conv_state)
    x = x.squeeze(2)
    state1 = NestedMap(conv_state=conv_state1)
    x, paddings = self._NormalizeStep(theta, x, paddings, state0, state1)
    x = self._ApplyActivation(x, p.conv_activation)
    x = self.linear_end.FProp(theta.linear_end, x)
    return x + residual, paddings, state1


def _AttenCtxIsSet(atten_context):
  return atten_context is not None and atten_context >= 0


def GShardMoELayerParams(num_devices, num_experts, num_groups=None,
                         per_expert_capacity_dim=None):
  """MoE builder params used inside a Conformer FFN slot (ref :449)."""
  from lingvo_b200.core import gshard_builder  # pylint: disable=g-import-not-at-top
  return gshard_builder.MoEBuilder.Params().Set(
      num_devices=num_devices, e_dim=num_experts,
      num_groups=num_groups or num_devices, c_dim=per_expert_capacity_dim or 0)


def _PGet(params, name, default=None):
  return params.Get(name) if name in params else default


class ConformerLayer(base_layer.BaseLayer):
  """Conformer block (ref :471)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', None, 'Input dim.')
    p.Define('is_causal', False, 'Causal conv + limited right context attention.')
    p.Define('layer_order', 'mhsa_before_conv',
             'mhsa | conv | mhsa_before_conv | conv_before_mhsa.')
    p.Define('dropout_prob', None, 'Dropout of the inner components.')
    p.Define('fflayer_start_tpl',
             layers_with_attention.TransformerFeedForwardLayer.Params(), 'First FFN.')
    p.Define('trans_atten_tpl', attention_lib.TransformerAttentionLayer.Params(),
             'Self-attention sub-layer.')
    p.Define('lconv_tpl', LConvLayer.Params(), 'Conv module (None: omitted).')
    p.Define('fflayer_end_tpl',
             layers_with_attention.TransformerFeedForwardLayer.Params(), 'Second FFN.')
    p.Define('fflayer_weight_sharing', False, 'Second FFN shares the first one\'s weights.')
    p.Define('fflayer_task_ids', '', 'Kept for parity.')
    p.Define('final_ln_tpl', layers.LayerNorm.Params(), 'Final LN.')
    p.Define('adapter_tpl', None, 'Optional adapter layer.')
    p.Define('adapter_pos', 'block_sequential', 'Kept for parity.')
    p.Define('remat', False, 'Rematerialise the block in backward.')
    p.Define('list_regex_dtypes', [], 'Kept for parity.')
    p.Define('allow_attention_summaries', False, 'Kept for parity.')
    p.Define('moe_expert_id_field_name', 'language_id', 'Kept for parity.')
    return p

  @classmethod
  def ConfigFFLayer(cls, tpl, input_dim, hidden_dim, activation, residual_weight,
                    dropout_prob):
    return tpl.Copy().Set(
        input_dim=input_dim, hidden_dim=hidden_dim, activation=activation,
        residual_weight=residual_weight, residual_dropout_prob=dropout_prob,
        relu_dropout_prob=dropout_prob)

  @classmethod
  def _ConfigSelfAttenContext(cls, left, right, *, use_relative_atten,
                              atten_chunk_size=None, query_stride=1,
                              relative_pos_emb_dim=None):
    """Chooses the attention class for the requested context (ref :740-820)."""
    common = dict(enable_value_proj=True, enable_per_dim_scale=True, use_bias=True)
    if atten_chunk_size is not None:
      cls_ = attention_lib.ChunkwiseSelfAttention
      tpl = cls_.Params().Set(chunk_size=atten_chunk_size, left_context=left or 0,
                              right_context=right or 0, **common)
    elif not _AttenCtxIsSet(left) and not _AttenCtxIsSet(right):
      if use_relative_atten:
        tpl = attention_lib.MultiHeadedAttentionXL.Params().Set(
            rel_pos_emb_dim=relative_pos_emb_dim, **common)
      else:
        tpl = attention_lib.MultiHeadedAttention.Params().Set(**common)
    else:
      if use_relative_atten:
        tpl = attention_lib.LocalSelfAttentionXL.Params().Set(
            left_context=left, right_context=right,
            rel_pos_emb_dim=relative_pos_emb_dim, **common)
      else:
        tpl = attention_lib.LocalSelfAttention.Params().Set(
            left_context=left, right_context=right, **common)
    tpl.query_stride = query_stride
    return tpl

  @classmethod
  def CommonParams(cls, input_dim, atten_num_heads=None, atten_local_context=None,
                   atten_left_context=None, atten_right_context=None,
                   atten_chunk_size=None, atten_logit_cap=0.0, use_relative_atten=None,
                   kernel_size=None, fflayer_hidden_dim=None, fflayer_activation=None,
                   fflayer_residual_weight=None, layer_order='mhsa_before_conv',
                   dropout_prob=0., conv_norm_layer_tpl=None, fprop_dtype=None,
                   is_causal=False, lconv_tpl=None, trans_atten_tpl=None,
                   fflayer_start_tpl=None, fflayer_end_tpl=None, query_stride=1,
                   fflayer_weight_sharing=False):
    assert input_dim
    if layer_order != 'conv':
      assert atten_num_heads or trans_atten_tpl
    if layer_order != 'mhsa':
      assert kernel_size
    if _AttenCtxIsSet(atten_local_context):
      assert not _AttenCtxIsSet(atten_left_context)
      assert not _AttenCtxIsSet(atten_right_context)
      atten_left_context = atten_local_context + 1
      atten_right_context = atten_local_context
    if is_causal and trans_atten_tpl is None:
      assert atten_right_context is not None
    p = cls.Params().Set(input_dim=input_dim, is_causal=is_causal,
                         layer_order=layer_order, dropout_prob=dropout_prob,
                         fflayer_weight_sharing=fflayer_weight_sharing)
    ff = dict(input_dim=input_dim, hidden_dim=fflayer_hidden_dim or 4 * input_dim,
              activation=fflayer_activation or 'SWISH',
              residual_weight=0.5 if fflayer_residual_weight is None
              else fflayer_residual_weight, dropout_prob=dropout_prob)
    base_ff = layers_with_attention.TransformerFeedForwardLayer.Params()
    p.fflayer_start_tpl = fflayer_start_tpl or cls.ConfigFFLayer(base_ff, **ff)
    p.fflayer_end_tpl = fflayer_end_tpl or cls.ConfigFFLayer(base_ff, **ff)
    if trans_atten_tpl is not None:
      p.trans_atten_tpl = trans_atten_tpl
    elif layer_order != 'conv':
      atten_tpl = cls._ConfigSelfAttenContext(
          atten_left_context, atten_right_context,
          use_relative_atten=True if use_relative_atten is None else use_relative_atten,
          atten_chunk_size=atten_chunk_size, query_stride=query_stride,
          relative_pos_emb_dim=input_dim)
      atten_tpl.atten_logit_cap = atten_logit_cap
      p.trans_atten_tpl = attention_lib.TransformerAttentionLayer.Params().Set(
          atten_tpl=atten_tpl, num_heads=atten_num_heads)
    if lconv_tpl is not None:
      p.lconv_tpl = lconv_tpl
    if kernel_size:
      p.lconv_tpl.kernel_size = kernel_size
    if conv_norm_layer_tpl is not None:
      p.lconv_tpl.conv_norm_layer_tpl = conv_norm_layer_tpl
    if fprop_dtype is not None:
      cls.SetFPropDtype(p, fprop_dtype)
    if layer_order == 'mhsa':
      p.lconv_tpl = None
    return p

  @classmethod
  def SetFPropDtype(cls, p, dtype):
    p.fprop_dtype = dtype
    for sub in (p.fflayer_start_tpl, p.fflayer_end_tpl, p.trans_atten_tpl, p.lconv_tpl):
      if sub is not None:
        sub.fprop_dtype = dtype
    return p

  @classmethod
  def NumOutputNodes(cls, p):
    return p.input_dim

  @classmethod
  def Stride(cls, params):
    """Time reduction of the block: the funnel attention's stride, else 1 (ref :730)."""
    if 'funnel_tpl' in params.trans_atten_tpl:
      return params.trans_atten_tpl.funnel_tpl.stride
    return 1

  @classmethod
  def RightContext(cls, params):
    if 'atten_tpl' in params:
      return params.atten_tpl.right_context
    raise ValueError(
        f'Failed to resolve right context for {params.cls}: "atten_tpl" should have been '
        'declared in the ConformerLayer params')

  @classmethod
  def ConfigMoEParams(cls, *, tpl, input_dim, hidden_dim, activation, residual_weight,
                      dropout_prob):
    """A gshard MoE builder configured as this block's FFN (ref :823)."""
    from lingvo_b200.core import gshard_builder  # pylint: disable=g-import-not-at-top
    moe_p = tpl.Copy().Set(model_dim=input_dim, dropout_rate=dropout_prob,
                           moe_hidden_dim=hidden_dim, moe_activation=activation)
    if moe_p.cls is gshard_builder.MoEBuilder and moe_p.num_devices is None:
      raise ValueError('num_devices must be specified for MoEBuilder.')
    if residual_weight != 0.5:
      raise ValueError('residual_weight must be 0.5')
    return moe_p

  @staticmethod
  def _IsMoE(tpl):
    from lingvo_b200.core import gshard_builder  # pylint: disable=g-import-not-at-top
    return tpl is not None and isinstance(tpl.cls, type) and issubclass(
        tpl.cls, gshard_builder.MoEBuilder)

  @staticmethod
  def _IsHashMoE(tpl):
    from lingvo_b200.core import gshard_builder  # pylint: disable=g-import-not-at-top
    return tpl is not None and isinstance(tpl.cls, type) and issubclass(
        tpl.cls, gshard_builder.MoEHashBuilder)

  def _ConfigFFLayerOrMoEParams(self, fflayer_tpl, name_prefix):
    """A dense FFN template bound to `input_dim`, or — for a MoE builder template — the
    builder's `EncoderLayer(MoE)` block named `<prefix>_moe` (ref :932)."""
    p = self.params
    fflayer_tpl = fflayer_tpl.Copy()
    if not self._IsMoE(fflayer_tpl):
      if 'input_dim' in fflayer_tpl:
        fflayer_tpl.Set(input_dim=p.input_dim)
      if _PGet(fflayer_tpl, 'num_tasks', 0):
        assert p.fflayer_task_ids, 'fflayer_task_ids must be provided for multitask FFNs.'
      if p.dropout_prob is not None:
        for n in ('residual_dropout_prob', 'relu_dropout_prob'):
          if n in fflayer_tpl:
            fflayer_tpl.Set(**{n: p.dropout_prob})
      return fflayer_tpl
    fflayer_tpl.model_dim = p.input_dim
    moe_builder = fflayer_tpl.Instantiate()
    name = name_prefix + '_moe'
    return moe_builder.EncoderLayer(name, moe_builder.MoE(name), residual_weight=0.5)

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.layer_order in ('mhsa', 'conv', 'mhsa_before_conv', 'conv_before_mhsa')
    if p.layer_order == 'mhsa':
      assert not self.has_lconv, 'mhsa must not have a lconv block.'
    d = p.input_dim

    def _Drop(tpl, *names):
      if p.dropout_prob is not None:
        for n in names:
          if n in tpl:
            tpl.Set(**{n: p.dropout_prob})
      return tpl

    start_p = None
    if self.has_fflayer_start:
      start_p = self._ConfigFFLayerOrMoEParams(p.fflayer_start_tpl, 'fflayer_start')
      if start_p.name:
        assert start_p.name == 'fflayer_start_moe'
      else:
        start_p.name = 'fflayer_start'
      self.CreateChild(start_p.name, start_p)
    end_p = self._ConfigFFLayerOrMoEParams(p.fflayer_end_tpl, 'fflayer_end')
    if end_p.name:
      assert end_p.name == 'fflayer_end_moe'
    else:
      end_p.name = 'fflayer_end'
    if not p.fflayer_weight_sharing:
      self.CreateChild(end_p.name, end_p)
    else:
      assert start_p is not None, 'fflayer_weight_sharing needs a start FFN.'
      # Same module under both names; only the start FFN owns the variables.
      self.__dict__['_shared_ff_end'] = (end_p.name, start_p.name)
    if self.has_mhsa:
      self.CreateChild('trans_atten', _Drop(
          p.trans_atten_tpl.Copy().Set(input_dim=d),
          'residual_dropout_prob', 'atten_dropout_prob'))
    if self.has_lconv:
      self.CreateChild('lconv', _Drop(
          p.lconv_tpl.Copy().Set(input_dim=d, is_causal=p.is_causal), 'dropout_prob'))
    self.CreateChild('final_ln', p.final_ln_tpl.Copy().Set(input_dim=d))
    if p.adapter_tpl is not None:
      tpl = p.adapter_tpl
      if hasattr(tpl.cls, 'SetNumInputNodes'):
        tpl.cls.SetNumInputNodes(tpl, d)
      elif 'input_dim' in tpl and not tpl.input_dim:
        tpl = tpl.Copy().Set(input_dim=d)
      if p.adapter_pos in ('block_sequential', 'block_parallel'):
        self.CreateChild('adapter', tpl.Copy())
      elif p.adapter_pos in ('ff_sequential', 'ff_parallel'):
        if start_p is not None:
          self.CreateChild('fflayer_start_adapter', tpl.Copy().Set(name='fflayer_start_adapter'))
        self.CreateChild('fflayer_end_adapter', tpl.Copy().Set(name='fflayer_end_adapter'))
      else:
        raise ValueError(
            f'Wrong adapter_pos: {p.adapter_pos}. Valid options are '
            '[block_sequential, block_parallel, ff_sequential, ff_parallel].')

  @property
  def has_lconv(self):
    return bool(self.params.lconv_tpl) and 'conv' in self.params.layer_order

  @property
  def has_mhsa(self):
    return 'mhsa' in self.params.layer_order

  @property
  def has_fflayer_start(self):
    return bool(self.params.fflayer_start_tpl)

  def _FF(self, theta, name):
    """(layer, theta) of the FFN child `name` or its `_moe` twin; None when absent."""
    shared = self.__dict__.get('_shared_ff_end')
    if shared is not None and name in ('fflayer_end', shared[0]):
      name = shared[1] if name == shared[0] else 'fflayer_start'
    for n in (name, name + '_moe'):
      if n in self.children:
        return n, self.children[n], theta.GetItem(n)
    raise AssertionError('{} child layer not present.'.format(name + '_moe'))

  def _RunAdapter(self, adapter, adapter_theta, nmap):
    """Adapters come in two call conventions: NestedMap → NestedMap[, extra] wrappers and
    per-task residual adapters `FProp(theta, inputs, tasks)`; returns the adapter features."""
    p = self.params
    tasks = nmap.Get(p.fflayer_task_ids) if p.fflayer_task_ids else nmap.Get('task_ids')
    if hasattr(adapter.params, 'num_tasks') and tasks is not None:
      t = tasks.reshape(tasks.shape[0], -1)[:, :1].expand(-1, nmap.features.shape[1])
      return adapter.FProp(adapter_theta, nmap.features, t)
    out = adapter.FProp(adapter_theta, nmap)
    out = out[0] if isinstance(out, tuple) else out
    return out.features if isinstance(out, NestedMap) else out

  def _MaybeFFLayerAdapter(self, theta, fflayer_name, in_nmap, features):
    """Adds the `<ffn>_adapter` output inside the FFN's residual branch (ref :979)."""
    p = self.params
    if p.adapter_tpl is None or p.adapter_pos not in ('ff_sequential', 'ff_parallel'):
      return features
    _, fflayer, _ = self._FF(theta, fflayer_name)
    fp = fflayer.params
    assert _PGet(fp, 'residual_droppath_prob', 0.0) == 0.0, (
        'residual droppath prob is not supported by adapter.')
    adapter = self.children[fflayer_name + '_adapter']
    adapter_theta = theta.GetItem(fflayer_name + '_adapter')
    skip = _PGet(fp, 'add_skip_connection', True)
    rw = _PGet(fp, 'residual_weight', 1.0)
    if skip:
      features = (features - in_nmap.features) / rw
    if p.adapter_pos == 'ff_sequential':
      in_nmap = in_nmap.copy()
      residual_in = in_nmap.features
      in_nmap.features = features
    else:
      residual_in = in_nmap.features
    features = features + self._RunAdapter(adapter, adapter_theta, in_nmap)
    if skip:
      features = residual_in + features * rw
    return features

  def _MoeOrFFLayer(self, theta, fflayer_name, features, paddings, aux_loss, expert_ids=None,
                    task_ids=None):
    """Dense FFN or MoE block (ref :1006) → (features, paddings, aux_loss). The MoE auxiliary
    (load-balancing) loss is added to `aux_loss` (broadcast over a per-example vector)."""
    name, fflayer, ff_theta = self._FF(theta, fflayer_name)
    if not name.endswith('_moe'):
      if _PGet(fflayer.params, 'num_tasks', 0):
        assert task_ids is not None, 'task_ids should not be None for multitask FFN layers.'
        out = fflayer.FProp(ff_theta, features, paddings, task_ids.reshape(features.shape[0]))
      else:
        out = fflayer.FProp(ff_theta, features, paddings)
      return out, paddings, aux_loss
    assert task_ids is None, 'MoE layer does not support multitask yet.'
    seg = (1.0 - paddings.float()).to(torch.int32)
    moe_in = NestedMap(vec=features, segment_id=seg, segment_pos=torch.zeros_like(seg),
                       aux_loss=torch.zeros((), dtype=torch.float32, device=features.device))
    if expert_ids is not None:
      moe_in.expert_id = expert_ids
    moe_out = fflayer.FProp(ff_theta, moe_in)
    moe_aux = moe_out.aux_loss
    if aux_loss is not None:
      assert moe_aux.dim() == 0, 'MoE aux-loss should be a scalar.'
      aux_loss = aux_loss + (moe_aux.expand(aux_loss.shape[0]) if aux_loss.dim() == 1
                             else moe_aux)
    else:
      aux_loss = moe_aux
    return moe_out.vec, paddings, aux_loss

  def _SelfAtten(self, theta, x, paddings):
    """→ (features, paddings, atten_probs); a funnel attention also pools the paddings."""
    out = self.trans_atten.FProp(theta.trans_atten, x, None, paddings)
    if len(out) == 3:
      return out
    return out[0], paddings, out[1]

  def _LConv(self, theta, x, paddings):
    return self.lconv.FProp(theta.lconv, x, paddings)

  def _AddAttentionSummaries(self, name, atten_probs):
    p = self.params
    if not p.allow_attention_summaries or atten_probs is None:
      return
    from lingvo_b200.core import summary_utils  # pylint: disable=g-import-not-at-top
    probs = atten_probs.detach().float()
    summary_utils.histogram(f'{name}/atten_probs', probs)
    if probs.dim() == 4:                     # [B, N, T, S]: one image per head of example 0
      for h in range(min(probs.shape[1], 4)):
        summary_utils.image(f'{name}/atten_probs_head{h}', probs[0, h].unsqueeze(0))

  def _Body(self, theta, in_nmap, x, paddings):
    p = self.params
    hash_moe = (self.has_fflayer_start and self._IsHashMoE(p.fflayer_start_tpl)) or \
        self._IsHashMoE(p.fflayer_end_tpl)
    expert_ids = None
    if hash_moe:
      expert_ids = in_nmap.Get(p.moe_expert_id_field_name)
      expert_ids = expert_ids.reshape(x.shape[0], -1)[:, :1].expand(-1, x.shape[1])
    aux_loss = in_nmap.Get('aux_loss')
    task_ids = in_nmap.Get(p.fflayer_task_ids) if p.fflayer_task_ids else None
    if self.has_fflayer_start:
      ad_in = in_nmap.copy()
      ad_in.features = x
      x, paddings, aux_loss = self._MoeOrFFLayer(theta, 'fflayer_start', x, paddings, aux_loss,
                                                 expert_ids, task_ids)
      x = self._MaybeFFLayerAdapter(theta, 'fflayer_start', ad_in, x)
    atten_probs = None
    if p.layer_order == 'mhsa':
      x, paddings, atten_probs = self._SelfAtten(theta, x, paddings)
    elif p.layer_order == 'conv':
      x, paddings = self._LConv(theta, x, paddings)
    elif p.layer_order == 'mhsa_before_conv':
      x, paddings, atten_probs = self._SelfAtten(theta, x, paddings)
      x, paddings = self._LConv(theta, x, paddings)
    else:
      x, paddings = self._LConv(theta, x, paddings)
      x, paddings, atten_probs = self._SelfAtten(theta, x, paddings)
    ad_in = in_nmap.copy()
    ad_in.features, ad_in.paddings = x, paddings
    if expert_ids is not None and expert_ids.shape[1] != x.shape[1]:
      expert_ids = expert_ids[:, :1].expand(-1, x.shape[1])
    x, paddings, aux_loss = self._MoeOrFFLayer(theta, 'fflayer_end', x, paddings, aux_loss,
                                               expert_ids, task_ids)
    x = self._MaybeFFLayerAdapter(theta, 'fflayer_end', ad_in, x)
    x = self.final_ln.FProp(theta.final_ln, x)
    if p.adapter_tpl is not None and p.adapter_pos in ('block_sequential', 'block_parallel'):
      ad_in = in_nmap.copy()
      if p.adapter_pos == 'block_sequential':
        ad_in.features, ad_in.paddings = x, paddings
      x = x + self._RunAdapter(self.adapter, theta.adapter, ad_in)
    return x, paddings, aux_loss, atten_probs

  def _FProp(self, theta, in_nmap):
    x, paddings = in_nmap.features, in_nmap.paddings
    x = self._CastToFPropDtype(x)
    x, paddings, aux_loss, atten_probs = self._Body(theta, in_nmap, x, paddings)
    x = py_utils.ApplyPadding(paddings.unsqueeze(-1), x)
    out = NestedMap(in_nmap.copy() if hasattr(in_nmap, 'copy') else in_nmap)
    out.features = self._CastToFPropDtype(x)
    out.paddings = paddings
    if aux_loss is not None:
      out.aux_loss = aux_loss
    self._AddAttentionSummaries(self.params.name, atten_probs)
    return out

  def FProp(self, theta, in_nmap):
    """in_nmap: NestedMap(features [B,T,D], paddings [B,T][, aux_loss, task / expert ids]) →
    same keys (time pooled by `Stride` under a funnel attention)."""
    p = self.params
    if not (p.remat and torch.is_grad_enabled()):
      return self._FProp(theta, in_nmap)
    from torch.utils import checkpoint as ckpt  # pylint: disable=g-import-not-at-top
    keys = [k for k, v in in_nmap.FlattenItems() if isinstance(v, torch.Tensor)]
    side = {}

    def _Fn(*tensors):
      nm = in_nmap.copy()
      for k, t in zip(keys, tensors):
        nm.Set(k, t)
      out = self._FProp(theta, nm)
      side['keys'] = [k for k, v in out.FlattenItems() if isinstance(v, torch.Tensor)]
      return tuple(out.GetItem(k) for k in side['keys'])

    outs = ckpt.checkpoint(_Fn, *[in_nmap.GetItem(k) for k in keys], use_reentrant=False)
    res = in_nmap.copy()
    for k, t in zip(side['keys'], outs):
      res.Set(k, t)
    return res

  def zero_state(self, batch_size):
    st = NestedMap()
    if self.has_mhsa:
      st.atten_state = self.trans_atten.atten.zero_state(batch_size)
    if self.has_lconv:
      st.lconv_state = self.lconv.zero_state(batch_size)
    return st

  def StreamStep(self, theta, in_nmap, state0):
    """Streaming FProp of a `[B, Q, D]` chunk for causal configs (ref :1190)."""
    p = self.params
    assert p.is_causal
    x, paddings = in_nmap.features, in_nmap.paddings
    st = NestedMap()
    if self.has_fflayer_start:
      x, _, _ = self._MoeOrFFLayer(theta, 'fflayer_start', x, paddings, None)

    def _Atten(x):
      ta, tt = self.trans_atten, theta.trans_atten
      normed = ta.layer_norm.FProp(tt.layer_norm, x) if ta.params.pre_layer_norm else x
      out, _, st.atten_state = ta.atten.StreamStep(tt.atten, normed, paddings,
                                                   state0.atten_state)
      out = x + out
      if not ta.params.pre_layer_norm:
        out = ta.layer_norm.FProp(tt.layer_norm, out)
      return out

    def _Conv(x):
      out, _, st.lconv_state = self.lconv.StreamStep(theta.lconv, x, paddings,
                                                     state0.lconv_state)
      return out

    if p.layer_order == 'mhsa':
      x = _Atten(x)
    elif p.layer_order == 'conv':
      x = _Conv(x)
    elif p.layer_order == 'mhsa_before_conv':
      x = _Conv(_Atten(x))
    else:
      x = _Atten(_Conv(x))
    x, _, _ = self._MoeOrFFLayer(theta, 'fflayer_end', x, paddings, None)
    x = self.final_ln.FProp(theta.final_ln, x)
    x = py_utils.ApplyPadding(paddings.unsqueeze(-1), x)
    return NestedMap(features=x, paddings=paddings), st


def ApplyGshard(conformer_tpl, device_mesh=None, proj_w_split_list=None,
                proj_activation_split_list=None, atten_dnh_w_split=None,
                atten_blnh_activation_split=None, atten_bld_activation_split=None,
                lconv_df_w_split=None, lconv_hwim_w_split=None, lconv_fd_w_split=None,
                lconv_blf_activation_split=None, lconv_bld_activation_split=None):
  """Annotates a conformer template with GShard sharding specs (ref :1344).
  The specs are recorded on the params; the tensor-parallel engine consumes them."""
  conformer_tpl.device_mesh = device_mesh
  for tpl in (conformer_tpl.fflayer_start_tpl, conformer_tpl.fflayer_end_tpl):
    if tpl is not None:
      tpl.device_mesh = device_mesh
      tpl.weight_split_dims_mapping = proj_w_split_list
      tpl.activation_split_dims_mapping = proj_activation_split_list
  if conformer_tpl.trans_atten_tpl is not None:
    a = conformer_tpl.trans_atten_tpl.atten_tpl
    a.device_mesh = device_mesh
    a.weight_split_dims_mapping = atten_dnh_w_split
    a.activation_split_dims_mapping = NestedMap(
        blnh=atten_blnh_activation_split, bld=atten_bld_activation_split)
  if conformer_tpl.lconv_tpl is not None:
    l = conformer_tpl.lconv_tpl
    l.device_mesh = device_mesh
    l.weight_split_dims_mapping = NestedMap(df=lconv_df_w_split, hwim=lconv_hwim_w_split,
                                            fd=lconv_fd_w_split)
    l.activation_split_dims_mapping = NestedMap(blf=lconv_blf_activation_split,
                                                bld=lconv_bld_activation_split)
  return conformer_tpl
