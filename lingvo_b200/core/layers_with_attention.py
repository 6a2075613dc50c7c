"""Time-major Transformer building blocks (ref `lingvo/core/layers_with_attention.py`).

`TransformerAttentionLayer` (:85), `TransformerFeedForwardLayer` (:529),
`MoEFeedforwardLayer` (:740), `HybridFeedforwardLayer` (:788),
`TransformerLayer` (:1334), `TransformerLayerWithMultitaskAdapters` (:2192),
`SelfAttentiveLayer` (:2984), `StochasticResidualLayer` (:32).

Inputs are `[time, batch, dim]`. The self-attention of a whole sequence is
computed batch-major through the fused kernel (`ops.attention`) using the same
projection variables (`source_proj`, `query_proj`, `ctx_post_proj`) the
step-wise `attention.MultiHeadedAttention` owns, so FProp is O(1) kernel
launches in T while ExtendStep stays incremental.
"""

from __future__ import annotations

import torch
import torch.nn.functional as F

from lingvo_b200.core import attention
from lingvo_b200.core import base_layer
from lingvo_b200.core import layers
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.core.py_utils import WeightInit
from lingvo_b200.core.py_utils import WeightParams
from lingvo_b200.ops import attention as attention_ops

_NEG = -0.7 * torch.finfo(torch.float32).max


class StochasticResidualLayer(base_layer.BaseLayer):
  """x + drop_path(f(x)); in eval f(x) is scaled by the survival prob (:32)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('residual_weight', 1.0, 'Residual weight.')
    p.Define('survival_prob', 1.0, 'Probability of keeping the residual branch.')
    return p

  def FProp(self, theta, x, y):
    p = self.params
    if self.do_eval:
      return x + p.residual_weight * p.survival_prob * y
    keep = (torch.rand((), device=y.device) < p.survival_prob).to(y.dtype)
    return x + p.residual_weight * keep * y


class TransformerAttentionLayer(base_layer.BaseLayer):
  """LN → multi-headed attention → dropout → residual, time-major (:85)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('source_dim', 0, 'Query/source dim.')
    p.Define('context_dim', 0, 'Aux (cross-attention) source dim.')
    p.Define('atten_hidden_dim', 0, 'Attention hidden dim.')
    p.Define('num_attention_heads', 8, 'Heads.')
    p.Define('is_masked', False, 'Masked self-attention.')
    p.Define('mask_ngram_order', 0, 'For mask_type=ngram.')
    p.Define('mask_type', 'future', 'future | eye | ngram.')
    p.Define('ln_tpl', layers.LayerNorm.Params(), 'LN template.')
    p.Define('atten_tpl', attention.MultiHeadedAttention.Params().Set(
        use_source_vec_as_attention_value=False, enable_ctx_post_proj=True,
        enable_ctx_pre_proj=True), 'Attention template.')
    p.Define('atten_dropout_prob', 0.0, 'Attention dropout.')
    p.Define('residual_dropout_prob', 0.0, 'Residual dropout.')
    p.Define('residual_dropout_tpl', layers.DropoutLayer.Params(), 'Dropout tpl.')
    p.Define('packed_input', False, 'Packed input.')
    p.Define('add_unnormalized_input', False, 'Residual on the raw input.')
    p.Define('residual_function', None, 'Gated residual layer params.')
    p.Define('pre_layer_norm', True, 'Pre-LN.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.source_dim
    hid = p.atten_hidden_dim or p.source_dim
    ctx = p.context_dim or p.source_dim
    self.CreateChild('atten', p.atten_tpl.Copy().Set(
        source_dim=ctx, query_dim=p.source_dim, context_dim=ctx, hidden_dim=hid,
        ctx_post_proj_dim=p.source_dim, num_attention_heads=p.num_attention_heads,
        atten_dropout_prob=p.atten_dropout_prob, packed_input=p.packed_input))
    self.CreateChild('layer_norm', p.ln_tpl.Copy().Set(input_dim=p.source_dim))
    self.CreateChild('residual_dropout', p.residual_dropout_tpl.Copy().Set(
        keep_prob=1.0 - p.residual_dropout_prob))
    if p.residual_function is not None:
      self.CreateChild('residual_function', p.residual_function.Copy().Set(
          input_dim=p.source_dim))

  def _StepMask(self, t, device):
    """[T, T] True where query i may NOT see key j."""
    p = self.params
    i = torch.arange(t, device=device).unsqueeze(1)
    j = torch.arange(t, device=device).unsqueeze(0)
    if p.mask_type == 'future':
      return j > i
    if p.mask_type == 'eye':
      return j == i
    if p.mask_type == 'ngram':
      return (j > i) | (j <= i - p.mask_ngram_order)
    raise ValueError(p.mask_type)

  def _Residual(self, theta, base, ctx):
    p = self.params
    ctx = self.residual_dropout.FProp(theta.residual_dropout, ctx)
    if p.residual_function is None:
      return base + ctx
    return self.residual_function.FProp(theta.residual_function, base, ctx)

  def FProp(self, theta, query_vec, source_paddings, source_vecs=None,
            query_segment_id=None, source_segment_id=None, context_vecs=None,
            **kwargs):
    """query_vec [T, B, D]; source_vecs [S, B, D] (None ⇒ self-attention).
    Returns (output [T, B, D], probs [T, B, S])."""
    p = self.params
    a, th = self.atten, theta.atten
    unnormalized = query_vec
    q_in = self.layer_norm.FProp(theta.layer_norm, query_vec) if p.pre_layer_norm \
        else query_vec
    if source_vecs is None:
      source_vecs, source_segment_id = q_in, query_segment_id
    if context_vecs is None:
      context_vecs = source_vecs
    t, b = q_in.shape[:2]
    s = source_vecs.shape[0]
    n = p.num_attention_heads
    packed = a.PackSource(th, source_vecs, context_vecs, source_paddings,
                          source_segment_id)
    qp = a._Apply(th, 'query_proj', q_in.transpose(0, 1)) if a.params.enable_query_proj \
        else q_in.transpose(0, 1)                    # pylint: disable=protected-access
    qh = qp.reshape(b, t, n, -1)
    if isinstance(a.atten, attention.DotProductAttention):
      qh = a.atten._ScaleQuery(th.atten, qh)        # pylint: disable=protected-access
    mask = (packed.source_padding > 0).view(b, 1, 1, s)
    if p.is_masked:
      mask = mask | self._StepMask(t, q_in.device).view(1, 1, t, s)
    if p.packed_input and query_segment_id is not None:
      mask = mask | (query_segment_id.t().view(b, 1, t, 1) !=
                     packed.source_segment_id.view(b, 1, 1, s))
    bias = mask.float() * _NEG
    drop = 0.0 if self.do_eval else p.atten_dropout_prob
    ctx, probs = attention_ops.dot_product_attention(
        qh, packed.source_vecs, packed.source_contexts, bias, 1.0,
        dropout_prob=drop, return_probs=True)
    ctx = ctx.reshape(b, t, -1)
    if a.params.enable_ctx_post_proj:
      ctx = a._Apply(th, 'ctx_post_proj', ctx)       # pylint: disable=protected-access
    ctx = ctx.transpose(0, 1)
    base = unnormalized if p.add_unnormalized_input else q_in
    out = self._Residual(theta, base, ctx)
    if not p.pre_layer_norm:
      out = self.layer_norm.FProp(theta.layer_norm, out)
    return out, probs.mean(1).transpose(0, 1)       # [T, B, S]

  def ExtendStep(self, theta, query_vec, prefix_state, t=None):
    """query_vec [B, D]; prefix_state {key,value: [t, B, D]} grows by one."""
    p = self.params
    assert p.is_masked
    a, th = self.atten, theta.atten
    unnormalized = query_vec
    q_in = self.layer_norm.FProp(theta.layer_norm, query_vec) if p.pre_layer_norm \
        else query_vec
    if t is None:
      key = torch.cat([prefix_state.key, q_in.unsqueeze(0)], 0)
      value = torch.cat([prefix_state.value, q_in.unsqueeze(0)], 0)
      pad = torch.zeros(key.shape[0], key.shape[1], device=q_in.device)
    else:
      key = prefix_state.key.clone()
      value = prefix_state.value.clone()
      key[t] = q_in
      value[t] = q_in
      pad = (torch.arange(key.shape[0], device=q_in.device) > t).float().unsqueeze(1) \
          .expand(key.shape[0], key.shape[1])
    packed = a.PackSource(th, key, value, pad)
    ctx, probs, _ = a.ComputeContextVectorWithSource(th, packed, q_in)
    base = unnormalized if p.add_unnormalized_input else q_in
    out = self._Residual(theta, base, ctx)
    if not p.pre_layer_norm:
      out = self.layer_norm.FProp(theta.layer_norm, out)
    return out, probs, NestedMap(key=key, value=value)


class TransformerMultiSourceAttentionLayer(TransformerAttentionLayer):
  """Cross-attention over several named sources (:480)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_source', 0, 'Number of sources.')
    p.Define('primary_source_index', 0, 'Which source returns probs.')
    p.Define('multi_source_atten', attention.MultiSourceAttention.Params(), 'Wrapper.')
    return p

  def FProp(self, theta, query_vec, source_paddings, source_vecs=None, **kwargs):
    outs, probs = [], None
    for i in range(self.params.num_source):
      k = 'source_%d' % i
      o, pr = super().FProp(theta, query_vec, source_paddings[k], source_vecs[k])
      outs.append(o)
      if i == self.params.primary_source_index:
        probs = pr
    return sum(outs) / len(outs), probs


class TransformerFeedForwardLayer(base_layer.BaseLayer):
  """LN → FFN(hidden) → dropout → residual (:529). Works on [..., D] inputs."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('output_dim', 0, 'Output dim (0 ⇒ input_dim).')
    p.Define('hidden_dim', 0, 'Hidden dim.')
    p.Define('num_tasks', 0, 'Kept for parity.')
    p.Define('ln_tpl', layers.LayerNorm.Params(), 'LN template.')
    p.Define('activation', 'RELU', 'Activation (GATED_* use a gated unit).')
    p.Define('residual_weight', 1.0, 'Weight of f(x) in the residual add.')
    p.Define('fflayer_tpl', layers.FeedForwardNet.Params().Set(
        activation=['RELU', 'NONE']), 'FFN template.')
    p.Define('res_proj_tpl', layers.ProjectionLayer.Params().Set(batch_norm=True),
             'Residual re-projection when dims differ.')
    p.Define('residual_dropout_prob', 0.0, 'Residual dropout.')
    p.Define('residual_dropout_tpl', layers.DropoutLayer.Params(), 'Dropout tpl.')
    p.Define('relu_dropout_prob', 0.0, 'Hidden dropout.')
    p.Define('add_skip_connection', True, 'Residual add.')
    p.Define('pre_layer_norm', True, 'Pre-LN.')
    p.Define('primer_hybrid_norm', False, 'Pre- and post-LN.')
    p.Define('residual_droppath_prob', 0.0, 'Stochastic depth.')
    p.Define('use_block_diagonal_matmul_pl', False, 'Kept for parity.')
    p.Define('num_blocks_pl', 1, 'Kept for parity.')
    p.Define('memory_augmentation', False, 'Kept for parity.')
    p.Define('memory', None, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.input_dim and p.hidden_dim
    odim = p.output_dim or p.input_dim
    self._odim = odim
    act = p.activation
    self._gated = isinstance(act, str) and act.startswith('GATED_')
    # `fflayer_tpl.dropout` (a single Params) chooses the dropout flavour of the hidden
    # layer — GPipe swaps in DeterministicDropoutLayer there (ref layers_with_gpipe.py:207)
    drop_tpl = p.fflayer_tpl.dropout if hasattr(p.fflayer_tpl.dropout, 'Copy') \
        else layers.DropoutLayer.Params()
    ff = p.fflayer_tpl.Copy().Set(
        input_dim=p.input_dim, hidden_layer_dims=[p.hidden_dim, odim],
        dropout=[drop_tpl.Copy().Set(keep_prob=1.0 - p.relu_dropout_prob),
                 drop_tpl.Copy().Set(keep_prob=1.0)])
    if self._gated:
      ff.activation = [act[len('GATED_'):], 'NONE']
      self.CreateChild('gate', layers.ProjectionLayer.Params().Set(
          input_dim=p.input_dim, output_dim=p.hidden_dim, activation='NONE',
          batch_norm=False, has_bias=True))
    else:
      ff.activation = [act, 'NONE']
    self.CreateChild('fflayer', ff)
    ln_name = 'pre_layer_norm' if p.primer_hybrid_norm else 'layer_norm'
    self.CreateChild(ln_name, p.ln_tpl.Copy().Set(
        input_dim=p.input_dim if p.pre_layer_norm else odim))
    if p.primer_hybrid_norm:
      self.CreateChild('post_layer_norm', p.ln_tpl.Copy().Set(input_dim=odim))
    self.CreateChild('residual_dropout', p.residual_dropout_tpl.Copy().Set(
        keep_prob=1.0 - p.residual_dropout_prob))
    if p.add_skip_connection and odim != p.input_dim:
      self.CreateChild('res_proj_layer', p.res_proj_tpl.Copy().Set(
          input_dim=p.input_dim, output_dim=odim, activation='NONE'))
    if p.residual_droppath_prob:
      self.CreateChild('residual_droppath', StochasticResidualLayer.Params().Set(
          residual_weight=p.residual_weight,
          survival_prob=1.0 - p.residual_droppath_prob))

  @property
  def output_dim(self):
    return self._odim

  @classmethod
  def NumOutputNodes(cls, p):
    return p.output_dim or p.input_dim

  def FProp(self, theta, inputs, paddings=None, tasks=None):
    p = self.params
    del tasks
    inputs = self._CastToFPropDtype(inputs)
    if p.pre_layer_norm:
      ln = self.pre_layer_norm if p.primer_hybrid_norm else self.layer_norm
      lt = theta.pre_layer_norm if p.primer_hybrid_norm else theta.layer_norm
      normed = ln.FProp(lt, inputs)
    else:
      normed = inputs
    pad = paddings.unsqueeze(-1) if paddings is not None else None
    if self._gated:
      ff, ft = self.fflayer, theta.fflayer
      h = ff.fc[0].FProp(ft.fc[0], normed) * self.gate.FProp(theta.gate, normed)
      h = ff.dropout[0].FProp(ft.dropout[0], h)
      h = ff.fc[1].FProp(ft.fc[1], h)
      if pad is not None:
        h = py_utils.ApplyPadding(pad, h)
    else:
      h = self.fflayer.FProp(theta.fflayer, normed, pad)
    if p.primer_hybrid_norm:
      h = self.post_layer_norm.FProp(theta.post_layer_norm, h)
    h = self.residual_dropout.FProp(theta.residual_dropout, h)
    if p.add_skip_connection:
      res = inputs
      if hasattr(self, 'res_proj_layer'):
        res = self.res_proj_layer.FProp(theta.res_proj_layer, inputs)
      if p.residual_droppath_prob:
        h = self.residual_droppath.FProp(theta.residual_droppath, res, h)
      else:
        h = res + h * p.residual_weight
    if not p.pre_layer_norm:
      h = self.layer_norm.FProp(theta.layer_norm, h)
    return h


class ReshapedTransformerFeedForwardLayer(TransformerFeedForwardLayer):
  """Inputs arrive `[..., N, D/N]`; flattened, processed, reshaped back (:1246)."""

  def FProp(self, theta, inputs, paddings=None, tasks=None):
    shp = inputs.shape
    out = super().FProp(theta, inputs.reshape(*shp[:-2], -1), paddings, tasks)
    return out.reshape(*shp[:-2], shp[-2], -1)


class TransformerFeedForwardLayerWithTaskId(TransformerFeedForwardLayer):
  """FFN whose projections are selected per task id (:bma 7720)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('use_task_ids', False, 'Select per-task weights.')
    return p


class MoEFeedforwardLayer(base_layer.BaseLayer):
  """GShard MoE layer behind the time-major FFN interface (:740)."""

  @classmethod
  def Params(cls):
    from lingvo_b200.core import gshard_builder  # pylint: disable=g-import-not-at-top
    p = super().Params()
    p.Define('moe_builder_p', gshard_builder.MoEBuilder.Params(), 'MoE builder.')
    p.Define('fflayer_residual_weight', 0.5, 'Residual weight.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    b = p.moe_builder_p.Instantiate()
    self.CreateChild('moe_fflayer', b.EncoderLayer(
        p.name, b.MoE(p.name), residual_weight=p.fflayer_residual_weight))

  def FProp(self, theta, inputs, paddings):
    seg = (1.0 - paddings).to(torch.int32)
    moe_in = NestedMap(vec=inputs, segment_id=seg, segment_pos=torch.zeros_like(seg))
    out = self.moe_fflayer.FProp(theta.moe_fflayer, moe_in)
    ctx = py_utils.AuxLossContext.Current()
    if ctx is None:
      raise ValueError('MoEFeedforwardLayer needs an AuxLossContext.')
    ctx.AddLoss(out.aux_loss)
    return out.vec


class HybridFeedforwardLayer(base_layer.BaseLayer):
  """Named sub-FFNs, chosen by `sub_key` at FProp time (:788)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('sub', None, 'Dict name → FFN layer params.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self._keys = sorted(p.sub.keys())
    for k in self._keys:
      self.CreateChild(k, p.sub[k])

  def FProp(self, theta, inputs, paddings, sub_key=None):
    k = sub_key or self._keys[0]
    return getattr(self, k).FProp(theta[k], inputs, paddings)


class TransformerLayer(base_layer.BaseLayer):
  """Time-major Transformer block: self-atten [→ aux-atten] → FFN (:1334)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('source_dim', 0, 'Input dim.')
    p.Define('output_dim', 0, 'Output dim.')
    p.Define('tr_atten_tpl', TransformerAttentionLayer.Params().Set(
        num_attention_heads=8), 'Self-attention tpl.')
    p.Define('tr_post_ln_tpl', None, 'Optional output LN.')
    p.Define('tr_fflayer_tpl', TransformerFeedForwardLayer.Params().Set(hidden_dim=2048),
             'FFN tpl.')
    p.Define('has_aux_atten', False, 'Cross attention.')
    p.Define('tr_aux_atten_tpl', None, 'Cross-attention tpl (defaults to tr_atten_tpl).')
    p.Define('mask_self_atten', False, 'Masked self-attention.')
    p.Define('packed_input', False, 'Packed input.')
    p.Define('is_decoder', False, 'Kept for parity.')
    p.Define('num_aux_atten_post_proj', 1, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.source_dim
    self.CreateChild('self_atten', p.tr_atten_tpl.Copy().Set(
        source_dim=p.source_dim, is_masked=p.mask_self_atten,
        packed_input=p.packed_input))
    if p.has_aux_atten:
      aux = (p.tr_aux_atten_tpl or p.tr_atten_tpl).Copy().Set(
          source_dim=p.source_dim, is_masked=False, packed_input=p.packed_input)
      self.CreateChild('atten', aux)
    self.CreateChild('fflayer', p.tr_fflayer_tpl.Copy().Set(
        input_dim=p.source_dim, output_dim=p.output_dim or p.source_dim))
    if p.tr_post_ln_tpl is not None:
      self.CreateChild('layer_norm', p.tr_post_ln_tpl.Copy().Set(
          input_dim=p.output_dim or p.source_dim))

  @property
  def output_dim(self):
    return self.fflayer.output_dim

  @classmethod
  def NumOutputNodes(cls, p):
    return p.output_dim or p.source_dim

  def FProp(self, theta, source_vecs, source_paddings, aux_vecs=None,
            aux_paddings=None, source_segment_id=None, aux_segment_id=None,
            **kwargs):
    p = self.params
    out, probs = self.self_atten.FProp(
        theta.self_atten, source_vecs, source_paddings,
        query_segment_id=source_segment_id)
    if p.has_aux_atten:
      assert aux_vecs is not None
      out, probs = self.atten.FProp(
          theta.atten, out, aux_paddings, aux_vecs,
          query_segment_id=source_segment_id, source_segment_id=aux_segment_id)
    out = self.fflayer.FProp(theta.fflayer, out, source_paddings)
    if p.tr_post_ln_tpl is not None:
      out = self.layer_norm.FProp(theta.layer_norm, out)
    return out, probs

  def ExtendStep(self, theta, source_vecs, prefix_states, aux_vecs=None,
                 aux_paddings=None, t=None, **kwargs):
    """source_vecs [B, D] → (out [B, D], probs [B, S], new prefix state)."""
    p = self.params
    out, probs, state = self.self_atten.ExtendStep(
        theta.self_atten, source_vecs, prefix_states, t)
    if p.has_aux_atten:
      o, pr = self.atten.FProp(theta.atten, out.unsqueeze(0), aux_paddings, aux_vecs)
      out, probs = o.squeeze(0), pr.squeeze(0)
    out = self.fflayer.FProp(theta.fflayer, out.unsqueeze(0),
                             torch.zeros(1, out.shape[0], device=out.device)).squeeze(0)
    if p.tr_post_ln_tpl is not None:
      out = self.layer_norm.FProp(theta.layer_norm, out)
    return out, probs, state


class TransformerLayerWithMultitaskAdapters(TransformerLayer):
  """TransformerLayer followed by per-task residual adapters (:2192)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('adapter_tpl', layers.MultitaskAdapterLayer.Params(), 'Adapter tpl.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('adapters', p.adapter_tpl.Copy().Set(
        input_dim=p.output_dim or p.source_dim))

  def FProp(self, theta, source_vecs, source_paddings, aux_vecs=None,
            aux_paddings=None, source_segment_id=None, aux_segment_id=None,
            source_task_id=None, **kwargs):
    out, probs = super().FProp(theta, source_vecs, source_paddings, aux_vecs,
                               aux_paddings, source_segment_id, aux_segment_id)
    out = self.adapters.FProp(theta.adapters, out, source_task_id)
    return out, probs


class SelfAttentiveLayer(base_layer.BaseLayer):
  """Structured self-attentive sentence embedding (Lin et al. 2017) (:2984):
  A = softmax(W2·tanh(W1·Hᵀ)); M = A·H, plus the ‖AAᵀ − I‖² penalty."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_heads', 5, 'Attention hops.')
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('hidden_dim', 0, 'Hidden dim.')
    p.Define('penalty_coef', 1.0, 'Coefficient of the orthogonality penalty.')
    p.Define('penalty_terms', [1.0, 1.0], 'Kept for parity.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('w1', WeightParams([p.input_dim, p.hidden_dim], p.params_init, p.dtype))
    self.CreateVariable('w2', WeightParams([p.hidden_dim, p.num_heads], p.params_init, p.dtype))

  def FProp(self, theta, inputs, paddings=None):
    """inputs [B, T, D] → ([B, N, D], penalty scalar)."""
    p = self.params
    hid = torch.tanh(torch.matmul(inputs, theta.w1.to(inputs.dtype)))
    logits = torch.matmul(hid, theta.w2.to(hid.dtype)).transpose(1, 2).float()
    if paddings is not None:
      logits = logits.masked_fill(paddings.unsqueeze(1) > 0, _NEG)
    a = torch.softmax(logits, -1)
    out = torch.bmm(a.to(inputs.dtype), inputs)
    eye = torch.eye(p.num_heads, device=a.device)
    pen = ((torch.bmm(a, a.transpose(1, 2)) - eye) ** 2).sum((1, 2)).mean()
    return out, p.penalty_coef * pen


# =================================================================================
# GShard MoE as a layer (reference :832-1242)
# =================================================================================
class TransformerShardedMoeLayer(base_layer.BaseLayer):
  """LN → group tokens → top-2 (or expert-choice) gating → expert FFNs → combine →
  dropout → residual; the layer-style twin of `gshard_builder.MoEBuilder.MoE`.

  inputs `[B, T, D]` (or `[B, T, G, D/G]`), paddings `[B, T]`. Tokens are reshaped to
  `[num_groups, group_size, D]`; `min_group_size` shrinks `num_groups` until every group
  holds at least that many tokens. The load-balancing aux loss goes to the enclosing
  `py_utils.AuxLossContext`. Expert weights `wi_<k> [E, D, H/shards]`, `wo_<k>`.

  On a GPU, with bf16 activations, ReLU experts and top-2 gating, the expert path is the
  fused peer-memory exchange of `parallel/symm.py` (gate+dispatch kernel, grouped wgmma
  GEMMs, row-pointer combine); otherwise the index-dispatch reference path.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Dimension of the layer input.')
    p.Define('output_dim', 0, 'Dimension of the layer output (0 ⇒ input_dim).')
    p.Define('hidden_dim', 0, 'Dimension of the expert hidden layer.')
    p.Define('ln_tpl', layers.LayerNorm.Params(), 'Layer norm params.')
    p.Define('activation', 'RELU', 'Non-linearity.')
    p.Define('use_glu', False, 'Gated experts: act(x·wi) ⊙ (x·wi_gate).')
    p.Define('dropout_tpl', layers.DropoutLayer.Params(), 'Dropout template.')
    p.Define('add_skip_connection', True, 'Residual connection input → output.')
    p.Define('residual_weight', 1.0, 'Output = residual_weight · f(x) + x.')
    p.Define('residual_dropout_prob', 0.0, 'Dropout on f(x).')
    p.Define('relu_dropout_prob', 0.0, 'Dropout on the expert hidden layer.')
    p.Define('pre_layer_norm', True, 'Pre or post layer norm.')
    p.Define('residual_droppath_prob', 0.0, 'Probability of dropping the residual path.')
    p.Define('gating_func', 'top_2', 'top_2 or expert_choice.')
    p.Define('num_experts', 0, 'Total number of experts.')
    p.Define('num_groups', 0, 'Groups for dispatching (≈ number of devices).')
    p.Define('disable_grouping', False, 'One group per batch element / whole batch.')
    p.Define('min_group_size', None, 'Lower bound on tokens per group.')
    p.Define('expert_capacity_dim', 0, 'Tokens per group per expert.')
    p.Define('expert_capacity_factor', 1.5, 'Capacity factor (≥ 1).')
    p.Define('expert_weight_shards', 1, 'Split each expert weight into this many vars.')
    p.Define('second_expert_policy', 'all', 'all | sampling | random.')
    from lingvo_b200.core import hyperparams  # pylint: disable=g-import-not-at-top
    if p.weight_split_dims_mapping is None:
      p.weight_split_dims_mapping = hyperparams.Params()
    if p.activation_split_dims_mapping is None:
      p.activation_split_dims_mapping = hyperparams.Params()
    wp = p.weight_split_dims_mapping
    wp.Define('me', None, 'Sharding of the gating weight [input_dim, num_experts].')
    wp.Define('emh', None, 'Sharding of wi [E, M, H].')
    wp.Define('ehm', None, 'Sharding of wo [E, H, M].')
    ap = p.activation_split_dims_mapping
    for k in ('gsm', 'gs', 'gsec', 'egcm', 'egch', 'gecm'):
      ap.Define(k, None, 'Sharding of the %s tensors.' % k)
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.num_experts > 0 and p.input_dim and p.hidden_dim
    assert p.expert_capacity_factor >= 1.0
    assert p.hidden_dim % p.expert_weight_shards == 0
    self._odim = p.output_dim or p.input_dim
    self.CreateChild('layer_norm', p.ln_tpl.Copy().Set(input_dim=p.input_dim))
    self.CreateChild('residual_dropout', p.dropout_tpl.Copy().Set(
        keep_prob=1.0 - p.residual_dropout_prob))
    self.CreateChild('relu_dropout', p.dropout_tpl.Copy().Set(
        keep_prob=1.0 - p.relu_dropout_prob))
    if p.residual_droppath_prob > 0:
      assert p.add_skip_connection
      self.CreateChild('residual_droppath', StochasticResidualLayer.Params().Set(
          residual_weight=p.residual_weight,
          survival_prob=1.0 - p.residual_droppath_prob))

  def _CreateLayerVariables(self):
    p = self.params
    m, e = p.input_dim, p.num_experts
    hs = p.hidden_dim // p.expert_weight_shards
    odim = p.output_dim or p.input_dim
    self.CreateVariable('gate', WeightParams([m, e], WeightInit.Xavier(1.0), p.dtype))
    for ii in range(p.expert_weight_shards):
      self.CreateVariable('wi_%d' % ii, WeightParams(
          [e, m, hs], WeightInit.Xavier(1.0), p.dtype))
      if p.use_glu:
        self.CreateVariable('wi_gate_%d' % ii, WeightParams(
            [e, m, hs], WeightInit.Xavier(1.0), p.dtype))
      self.CreateVariable('wo_%d' % ii, WeightParams(
          [e, hs, odim], WeightInit.Xavier(1.0), p.dtype))

  @property
  def output_dim(self):
    return self._odim

  def _NumGroups(self, tokens: int, batch: int) -> int:
    p = self.params
    if p.disable_grouping:
      return 1
    g = p.num_groups or batch
    if p.min_group_size is not None:
      g = max(1, min(g, tokens // max(1, p.min_group_size)))
    while tokens % g:
      g -= 1
    return g

  def FProp(self, theta, inputs, paddings):
    from lingvo_b200.core import activations  # pylint: disable=g-import-not-at-top
    from lingvo_b200.core import gshard_layers  # pylint: disable=g-import-not-at-top
    p = self.params
    orig_shape = inputs.shape
    if inputs.dim() == 4:
      inputs = inputs.reshape(orig_shape[0], orig_shape[1], -1)
    b, t, m = inputs.shape
    fd = inputs.dtype
    x = self.layer_norm.FProp(theta.layer_norm, inputs) if p.pre_layer_norm else inputs
    tokens = b * t
    g = self._NumGroups(tokens, b)
    s = tokens // g
    xg = x.reshape(g, s, m)
    pad_g = paddings.reshape(g, s).float()
    e = p.num_experts
    # fp32 gating logits; expert capacity scaled ×2 for top-2 like the reference (:1090)
    logits = torch.matmul(xg.float(), theta.gate.float())
    cap_factor = p.expert_capacity_factor * (2.0 if p.gating_func == 'top_2' else 1.0)
    wi = torch.cat([theta['wi_%d' % i] for i in range(p.expert_weight_shards)], -1)
    wo = torch.cat([theta['wo_%d' % i] for i in range(p.expert_weight_shards)], 1)
    act = p.activation.upper()
    if p.gating_func in ('top_2', 'top2'):
      seeds = None
      if p.second_expert_policy != 'all':
        seeds = py_utils.GenerateStepSeedPair(p)
      gating = gshard_layers.Top2GatingIndices(
          logits, pad_g, e, p.expert_capacity_dim, torch.float32, p.second_expert_policy,
          0.0, False, cap_factor, seeds)
      if p.use_glu:
        wg = torch.cat([theta['wi_gate_%d' % i] for i in range(p.expert_weight_shards)], -1)
        wi_arg = torch.stack([wi, wg])
      else:
        wi_arg = wi
      if p.relu_dropout_prob and not self.do_eval:
        # dropout on the hidden layer: explicit expert path
        xin = gshard_layers.MoEDispatchIndexed(xg.reshape(g * s, m), gating, g, s, e)
        h = activations.GetFn(act)(torch.einsum('EAM,EMH->EAH', xin, wi.to(fd)))
        if p.use_glu:
          h = h * torch.einsum('EAM,EMH->EAH', xin, wg.to(fd))
        h = self.relu_dropout.FProp(theta.relu_dropout, h)
        out = torch.einsum('EAH,EHM->EAM', h, wo.to(fd))
        y = gshard_layers.MoECombineIndexed(out, gating, g, s).reshape(g, s, -1)
      else:
        y = gshard_layers.MoEApplyIndexed(xg, gating, wi_arg.to(fd), wo.to(fd), act,
                                          use_glu=p.use_glu)
      aux_loss = gating.aux_loss
    elif p.gating_func == 'expert_choice':
      # every expert picks its top-C tokens of the group (no token is dropped by overflow,
      # some may be picked by no expert) — GECS dispatch of the reference (:2496)
      cap = gshard_layers.ExpertCapacity(s, e, p.expert_capacity_dim, cap_factor)
      cap = min(cap, s)
      probs = torch.softmax(logits, -1) * (1.0 - pad_g).unsqueeze(-1)
      top = torch.topk(probs.transpose(1, 2), cap, dim=-1)            # [G, E, C]
      idx = top.indices
      xin = torch.gather(xg.unsqueeze(1).expand(g, e, s, m), 2,
                         idx.unsqueeze(-1).expand(g, e, cap, m))      # [G, E, C, M]
      h = activations.GetFn(act)(torch.einsum('GECM,EMH->GECH', xin, wi.to(fd)))
      if p.use_glu:
        wg = torch.cat([theta['wi_gate_%d' % i] for i in range(p.expert_weight_shards)], -1)
        h = h * torch.einsum('GECM,EMH->GECH', xin, wg.to(fd))
      h = self.relu_dropout.FProp(theta.relu_dropout, h)
      out = torch.einsum('GECH,EHM->GECM', h, wo.to(fd)) * top.values.unsqueeze(-1).to(fd)
      y = torch.zeros(g, s, out.shape[-1], dtype=out.dtype, device=out.device)
      y.scatter_add_(1, idx.reshape(g, e * cap, 1).expand(g, e * cap, out.shape[-1]),
                     out.reshape(g, e * cap, -1))
      aux_loss = torch.zeros((), device=inputs.device)
    else:
      raise ValueError('Unsupported gating function %s' % p.gating_func)
    ctx = py_utils.AuxLossContext.Current()
    if ctx is not None:
      ctx.AddLoss(aux_loss)
    self.last_aux_loss = aux_loss
    y = y.reshape(b, t, -1).to(fd)
    y = y * (1.0 - paddings.to(fd)).unsqueeze(-1)
    y = self.residual_dropout.FProp(theta.residual_dropout, y)
    if p.add_skip_connection:
      if p.residual_droppath_prob:
        y = self.residual_droppath.FProp(theta.residual_droppath, inputs, y)
      else:
        y = inputs + y * p.residual_weight
    if not p.pre_layer_norm:
      y = self.layer_norm.FProp(theta.layer_norm, y)
    return y.reshape(orig_shape) if len(orig_shape) == 4 else y


# =================================================================================
# Evolved Transformer (So et al. 2019; reference :1807-2290)
# =================================================================================
def _SepConv1D(name, in_dim, out_dim, kernel, causal=False):
  """Depthwise-separable conv over time as (depthwise, pointwise) layer params."""
  from lingvo_b200.core import conv_layers_with_time_padding as ctp  # pylint: disable=g-import-not-at-top
  cls = ctp.CausalDepthwiseConv2DLayer if causal else ctp.DepthwiseConv2DLayer
  dw = cls.Params().Set(name=name + '_dw', filter_shape=(kernel, 1, in_dim, 1),
                        filter_stride=(1, 1))
  pw = layers.FCLayer.Params().Set(name=name + '_pw', input_dim=in_dim, output_dim=out_dim,
                                   activation='NONE')
  return dw, pw


class _ConvBranchMixin:
  """Runs time-major [T, B, D] tensors through [B, T, 1, D] conv layers."""

  @staticmethod
  def _Conv(layer, theta, x, paddings):
    xb = x.transpose(0, 1).unsqueeze(2)                # [B, T, 1, D]
    yb, _ = layer.FProp(theta, xb, paddings.transpose(0, 1))
    return yb.squeeze(2).transpose(0, 1)


class EvolvedTransformerEncoderBranchedConvsLayer(base_layer.BaseLayer, _ConvBranchMixin):
  """ET encoder conv block: LN → {dense(4D)+relu → dropout ‖ conv3×1(D/2)+relu} summed
  (right branch zero-padded) → LN → sep-conv 9×1 → residual (reference :1807)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('ln_tpl', layers.LayerNorm.Params(), 'LN template.')
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('activation', 'RELU', 'Branch activation.')
    p.Define('dropout_tpl', layers.DropoutLayer.Params(), 'Dropout template.')
    p.Define('dense_tpl', layers.FCLayer.Params(), 'Left branch dense.')
    p.Define('conv_tpl', None, 'Kept for parity.')
    p.Define('separable_conv_tpl', None, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    from lingvo_b200.core import conv_layers_with_time_padding as ctp  # pylint: disable=g-import-not-at-top
    p = self.params
    d = p.input_dim
    self.CreateChild('first_layer_norm', p.ln_tpl.Copy().Set(input_dim=d))
    self.CreateChild('dense_layer', p.dense_tpl.Copy().Set(
        input_dim=d, output_dim=4 * d, activation=p.activation))
    self.CreateChild('conv_layer', ctp.Conv2DLayerWithPadding.Params().Set(
        filter_shape=(3, 1, d, d // 2), filter_stride=(1, 1)))
    self.CreateChild('second_layer_norm', p.ln_tpl.Copy().Set(input_dim=4 * d))
    dw, pw = _SepConv1D('separable_conv', 4 * d, d // 2, 9)
    self.CreateChild('separable_conv_dw', dw)
    self.CreateChild('separable_conv_pw', pw)
    self.CreateChild('dropout', p.dropout_tpl.Copy())

  def FProp(self, theta, inputs, paddings):
    p = self.params
    d = p.input_dim
    mask = (1.0 - paddings).unsqueeze(-1).to(inputs.dtype)
    x = self.first_layer_norm.FProp(theta.first_layer_norm, inputs) * mask
    left = self.dropout.FProp(theta.dropout, self.dense_layer.FProp(theta.dense_layer, x))
    right = F.relu(self._Conv(self.conv_layer, theta.conv_layer, x, paddings))
    right = self.dropout.FProp(theta.dropout, right)
    h = left + F.pad(right, (0, 4 * d - right.shape[-1]))
    h = self.second_layer_norm.FProp(theta.second_layer_norm, h) * mask
    h = self._Conv(self.separable_conv_dw, theta.separable_conv_dw, h, paddings)
    h = self.separable_conv_pw.FProp(theta.separable_conv_pw, h)
    h = self.dropout.FProp(theta.dropout, h)
    return inputs + F.pad(h, (0, d - h.shape[-1]))


class EvolvedTransformerDecoderBranchedConvsLayer(base_layer.BaseLayer, _ConvBranchMixin):
  """ET decoder conv block: LN → {causal sep-conv 11×1 (2D)+relu ‖ causal sep-conv 7×1
  (D/2)} → LN → causal sep-conv 7×1 (D) → residual (reference :1935)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('ln_tpl', layers.LayerNorm.Params(), 'LN template.')
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('activation', 'RELU', 'Branch activation.')
    p.Define('dropout_tpl', layers.DropoutLayer.Params(), 'Dropout template.')
    p.Define('separable_conv_tpl', None, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    d = p.input_dim
    self.CreateChild('first_layer_norm', p.ln_tpl.Copy().Set(input_dim=d))
    for nm, k, od in (('left', 11, 2 * d), ('right', 7, d // 2)):
      dw, pw = _SepConv1D(nm, d, od, k, causal=True)
      self.CreateChild('separable_conv_%s_dw' % nm, dw)
      self.CreateChild('separable_conv_%s_pw' % nm, pw)
    self.CreateChild('second_layer_norm', p.ln_tpl.Copy().Set(input_dim=2 * d))
    dw, pw = _SepConv1D('final', 2 * d, d, 7, causal=True)
    self.CreateChild('separable_conv_final_dw', dw)
    self.CreateChild('separable_conv_final_pw', pw)
    self.CreateChild('dropout', p.dropout_tpl.Copy())

  def FProp(self, theta, inputs, paddings):
    p = self.params
    d = p.input_dim
    mask = (1.0 - paddings).unsqueeze(-1).to(inputs.dtype)
    x = self.first_layer_norm.FProp(theta.first_layer_norm, inputs) * mask

    def sep(nm, t):
      h = self._Conv(getattr(self, 'separable_conv_%s_dw' % nm),
                     theta['separable_conv_%s_dw' % nm], t, paddings)
      return getattr(self, 'separable_conv_%s_pw' % nm).FProp(
          theta['separable_conv_%s_pw' % nm], h)
    left = self.dropout.FProp(theta.dropout, F.relu(sep('left', x)))
    right = self.dropout.FProp(theta.dropout, sep('right', x))
    h = left + F.pad(right, (0, 2 * d - right.shape[-1]))
    h = self.second_layer_norm.FProp(theta.second_layer_norm, h) * mask
    h = self.dropout.FProp(theta.dropout, sep('final', h))
    return inputs + h


class EvolvedTransformerBaseLayer(base_layer.BaseLayer):
  """Shared plumbing of the ET encoder/decoder layers."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('source_dim', 0, 'Model dim.')
    p.Define('has_aux_atten', False, 'Kept for parity.')
    p.Define('packed_input', False, 'Packed input.')
    return p


class EvolvedTransformerEncoderLayer(EvolvedTransformerBaseLayer):
  """GLU → branched convs → self-attention → FFN (reference :2085)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('glu_tpl', layers.GluLayer.Params(), 'Gated linear unit.')
    p.Define('branched_convs_tpl', EvolvedTransformerEncoderBranchedConvsLayer.Params(),
             'Branched convs.')
    p.Define('transformer_tpl', TransformerLayer.Params(), 'Attention + FFN.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('glu_layer', p.glu_tpl.Copy().Set(input_dim=p.source_dim))
    self.CreateChild('branched_convs_layer', p.branched_convs_tpl.Copy().Set(
        input_dim=p.source_dim))
    self.CreateChild('transformer_layer', p.transformer_tpl.Copy().Set(
        source_dim=p.source_dim, packed_input=p.packed_input))

  def FProp(self, theta, source_vecs, source_paddings, aux_vecs=None, aux_paddings=None,
            source_segment_id=None, aux_segment_id=None):
    h = self.glu_layer.FProp(theta.glu_layer, source_vecs, source_paddings)
    h = self.branched_convs_layer.FProp(theta.branched_convs_layer, h, source_paddings)
    return self.transformer_layer.FProp(
        theta.transformer_layer, h, source_paddings, aux_vecs, aux_paddings,
        source_segment_id, aux_segment_id)


class EvolvedTransformerDecoderLayer(EvolvedTransformerBaseLayer):
  """{16-head self-attention ‖ encoder attention} → branched causal convs →
  self-attention → encoder attention → swish FFN (reference :2170)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('tr_atten_tpl', TransformerAttentionLayer.Params().Set(num_attention_heads=8),
             'Attention template.')
    p.Define('tr_double_heads_atten_tpl',
             TransformerAttentionLayer.Params().Set(num_attention_heads=16),
             'Double-heads self-attention.')
    p.Define('branched_convs_tpl', EvolvedTransformerDecoderBranchedConvsLayer.Params(),
             'Branched convs.')
    p.Define('transformer_tpl', TransformerLayer.Params().Set(
        tr_fflayer_tpl=TransformerFeedForwardLayer.Params().Set(
            hidden_dim=2048, activation='SWISH')), 'Final attention + FFN.')
    p.has_aux_atten = True
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    d = p.source_dim
    self.CreateChild('self_atten_double_heads', p.tr_double_heads_atten_tpl.Copy().Set(
        source_dim=d, is_masked=True, packed_input=p.packed_input))
    self.CreateChild('attend_to_encoder', p.tr_atten_tpl.Copy().Set(
        source_dim=d, is_masked=False, packed_input=p.packed_input))
    self.CreateChild('branched_convs', p.branched_convs_tpl.Copy().Set(input_dim=d))
    self.CreateChild('transformer_layer', p.transformer_tpl.Copy().Set(
        source_dim=d, has_aux_atten=True, mask_self_atten=True,
        packed_input=p.packed_input))

  def FProp(self, theta, source_vecs, source_paddings, aux_vecs=None, aux_paddings=None,
            source_segment_id=None, aux_segment_id=None):
    left, _ = self.self_atten_double_heads.FProp(
        theta.self_atten_double_heads, source_vecs, source_paddings,
        query_segment_id=source_segment_id)
    right, _ = self.attend_to_encoder.FProp(
        theta.attend_to_encoder, source_vecs, aux_paddings, aux_vecs,
        query_segment_id=source_segment_id, source_segment_id=aux_segment_id)
    h = left + right - source_vecs            # each branch already carries one residual
    h = self.branched_convs.FProp(theta.branched_convs, h, source_paddings)
    return self.transformer_layer.FProp(
        theta.transformer_layer, h, source_paddings, aux_vecs, aux_paddings,
        source_segment_id, aux_segment_id)


# =================================================================================
# Style / context / conditional-computation variants
# =================================================================================
class StyleLayer(base_layer.BaseLayer):
  """Global style tokens: a query attends over a bank of learned style embeddings and the
  result is broadcast over time (reference `StyleLayer` :2290)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Query (reference encoder) dim.')
    p.Define('output_dim', 0, 'Style embedding dim.')
    p.Define('num_styles', 0, 'Number of style tokens.')
    p.Define('num_heads', 4, 'Attention heads.')
    p.Define('enable_ctx_post_proj', True, 'Project the mixed style.')
    p.Define('use_bias', True, 'Bias in projections.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.num_styles > 0 and p.input_dim and p.output_dim
    self.CreateChild('atten', attention.MultiHeadedAttention.Params().Set(
        source_dim=p.output_dim, context_dim=p.output_dim, hidden_dim=p.output_dim,
        query_dim=p.input_dim, ctx_post_proj_dim=p.output_dim,
        num_attention_heads=p.num_heads, use_source_vec_as_attention_value=False,
        enable_ctx_pre_proj=True, enable_ctx_post_proj=p.enable_ctx_post_proj))

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('styles_w', WeightParams(
        [p.num_styles, 1, p.output_dim], WeightInit.Gaussian(0.5), p.dtype))

  def EmbLookup(self, theta, ids):
    """Style vectors of explicit ids `[B]` → `[B, output_dim]` (inference control)."""
    return torch.tanh(theta.styles_w)[ids.long(), 0]

  def StyleEmbFromProbs(self, theta, probs):
    """Mixture `[B, num_styles]` → `[B, output_dim]`."""
    return torch.matmul(probs.to(theta.styles_w.dtype), torch.tanh(theta.styles_w[:, 0]))

  def FProp(self, theta, inputs):
    """inputs `[B, input_dim]` → style embedding `[B, output_dim]`."""
    p = self.params
    b = inputs.shape[0]
    src = torch.tanh(theta.styles_w).expand(p.num_styles, b, p.output_dim).to(inputs.dtype)
    pad = torch.zeros(p.num_styles, b, device=inputs.device)
    packed = self.atten.InitForSourcePacked(theta.atten, src, src, pad)
    ctx, _, _ = self.atten.ComputeContextVectorWithSource(theta.atten, packed, inputs)
    return ctx


class TransformerWithContextLayer(TransformerLayer):
  """Decoder block with a third attention over an extra *context* sequence besides the
  encoder output (reference :2775): self-atten → source-atten → context-atten → FFN."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('tr_context_atten_tpl', None, 'Context attention (defaults to tr_atten_tpl).')
    p.has_aux_atten = True
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    ctx_tpl = (p.tr_context_atten_tpl or p.tr_aux_atten_tpl or p.tr_atten_tpl).Copy().Set(
        source_dim=p.source_dim, is_masked=False, packed_input=p.packed_input)
    self.CreateChild('context_atten', ctx_tpl)

  def FProp(self, theta, source_vecs, source_paddings, aux_vecs, aux_paddings,
            tertiary_vecs, tertiary_paddings, source_segment_id=None, aux_segment_id=None,
            tertiary_segment_id=None, **kwargs):
    p = self.params
    out, _ = self.self_atten.FProp(theta.self_atten, source_vecs, source_paddings,
                                   query_segment_id=source_segment_id)
    out, probs = self.atten.FProp(theta.atten, out, aux_paddings, aux_vecs,
                                  query_segment_id=source_segment_id,
                                  source_segment_id=aux_segment_id)
    out, _ = self.context_atten.FProp(theta.context_atten, out, tertiary_paddings,
                                      tertiary_vecs, query_segment_id=source_segment_id,
                                      source_segment_id=tertiary_segment_id)
    out = self.fflayer.FProp(theta.fflayer, out, source_paddings)
    if p.tr_post_ln_tpl is not None:
      out = self.layer_norm.FProp(theta.layer_norm, out)
    return out, probs


class CCTAttentionLayer(base_layer.BaseLayer):
  """Conditional-computation attention block (reference `CCTAttentionLayer` :2484): a
  gating network decides per position how much of the query / key-value transformation
  to apply; the continuous gates (train) are thresholded at inference."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('source_dim', 0, 'Model dim.')
    p.Define('num_attention_heads', 8, 'Heads.')
    p.Define('is_masked', False, 'Masked self-attention.')
    p.Define('ln_tpl', layers.LayerNorm.Params(), 'LN template.')
    p.Define('atten_tpl', TransformerAttentionLayer.Params(), 'Attention block.')
    p.Define('gating_tpl', layers.CCTGatingNetwork.Params(), 'Gating network.')
    p.Define('residual_dropout_prob', 0.0, 'Residual dropout.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('atten', p.atten_tpl.Copy().Set(
        source_dim=p.source_dim, num_attention_heads=p.num_attention_heads,
        is_masked=p.is_masked, residual_dropout_prob=p.residual_dropout_prob))
    self.CreateChild('gating', p.gating_tpl.Copy().Set(
        input_dim=p.source_dim, hidden_layer_dim=p.source_dim, num_outputs=1))

  def FProp(self, theta, query_vec, source_paddings, source_vecs=None, **kwargs):
    out, probs = self.atten.FProp(theta.atten, query_vec, source_paddings, source_vecs,
                                  **kwargs)
    gate = self.gating.FProp(theta.gating, query_vec)            # [T, B, 1]
    self.last_gate_mean = gate.mean()
    return query_vec + gate * (out - query_vec), probs


class CCTFeedForwardLayer(base_layer.BaseLayer):
  """Conditional-computation FFN (reference :2620): the hidden layer is split into
  `num_blocks` blocks, each switched by its own gate."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Model dim.')
    p.Define('hidden_dim', 0, 'Hidden dim.')
    p.Define('num_blocks', 1, 'Gated blocks of the hidden layer.')
    p.Define('ln_tpl', layers.LayerNorm.Params(), 'LN template.')
    p.Define('gating_tpl', layers.CCTGatingNetwork.Params(), 'Gating network.')
    p.Define('activation', 'RELU', 'Activation.')
    p.Define('residual_dropout_prob', 0.0, 'Residual dropout.')
    p.Define('relu_dropout_prob', 0.0, 'Hidden dropout.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.hidden_dim % p.num_blocks == 0
    self.CreateChild('layer_norm', p.ln_tpl.Copy().Set(input_dim=p.input_dim))
    self.CreateChild('fc_in', layers.FCLayer.Params().Set(
        input_dim=p.input_dim, output_dim=p.hidden_dim, activation=p.activation))
    self.CreateChild('fc_out', layers.FCLayer.Params().Set(
        input_dim=p.hidden_dim, output_dim=p.input_dim, activation='NONE'))
    self.CreateChild('gating', p.gating_tpl.Copy().Set(
        input_dim=p.input_dim, hidden_layer_dim=p.input_dim, num_outputs=p.num_blocks))
    self.CreateChild('relu_dropout', layers.DropoutLayer.Params().Set(
        keep_prob=1.0 - p.relu_dropout_prob))
    self.CreateChild('residual_dropout', layers.DropoutLayer.Params().Set(
        keep_prob=1.0 - p.residual_dropout_prob))

  def FProp(self, theta, inputs, paddings=None):
    p = self.params
    x = self.layer_norm.FProp(theta.layer_norm, inputs)
    gate = self.gating.FProp(theta.gating, x)                    # [..., num_blocks]
    h = self.fc_in.FProp(theta.fc_in, x)
    h = self.relu_dropout.FProp(theta.relu_dropout, h)
    blk = p.hidden_dim // p.num_blocks
    h = (h.reshape(*h.shape[:-1], p.num_blocks, blk) * gate.unsqueeze(-1)).reshape(h.shape)
    y = self.fc_out.FProp(theta.fc_out, h)
    if paddings is not None:
      y = y * (1.0 - paddings).unsqueeze(-1).to(y.dtype)
    self.last_gate_mean = gate.mean()
    return inputs + self.residual_dropout.FProp(theta.residual_dropout, y)
