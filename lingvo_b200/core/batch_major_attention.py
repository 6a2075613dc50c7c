"""Batch-major multi-headed attention and Transformer layers.

API-parity re-implementation of `lingvo/core/batch_major_attention.py`
(ref :52-190 mask helpers, :192 PerDimScaleLayer, :253
MultiHeadedProjectionLayer, :481 MultiHeadedAttention, :2233 …XL, :2413 …RPE,
:2656 LocalSelfAttention, :4008 ChunkwiseSelfAttention, :5226
TransformerAttentionLayer, :6265 TransformerLayer, :7116
StackedTransformerLayers, :8591 Builder).

H100-first design choices (not a translation):
  * Every mask (padding, causal, per-step, segment, local band, chunk) and every
    relative-position term (XL, RPE) is folded into ONE additive bias and the
    core runs through `ops.attention.dot_product_attention`, whose CUDA path is
    a fused online-softmax kernel — the `[B,N,T,S]` logits are only
    materialised when the caller asks for probabilities.
  * Projections `[D, N, H]` are stored exactly like the reference (checkpoint
    parity) and run as flat `[D, N·H]` wgmma GEMMs with fused bias.
  * Decode caches are `[T, B, N, H]` like the reference's `InitStates`.
"""

from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F

from lingvo_b200.core import activations
from lingvo_b200.core import base_layer
from lingvo_b200.core import builder
from lingvo_b200.core import builder_layers
from lingvo_b200.core import layers
from lingvo_b200.core import py_utils
from lingvo_b200.core import quant_utils
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.core.py_utils import WeightInit
from lingvo_b200.core.py_utils import WeightParams
from lingvo_b200.ops import attention as attention_ops
from lingvo_b200.ops import gemm

_FP32_MAX = torch.finfo(torch.float32).max


def GetDtypeMin(dtype=torch.float32):
  """The reference's "very negative" logit: -0.7 · dtype.max (:156)."""
  return -0.7 * torch.finfo(dtype).max


def CausalPadding(slen, dtype=torch.float32, device=None):
  """[slen, slen] 0/1 matrix, 1 where key position > query position (:82)."""
  return torch.triu(torch.ones(slen, slen, dtype=dtype, device=device), 1)


def SegmentMask(segment_id, source_segment_id, dtype=torch.float32,
                apply_dtype_min=True):
  """[B, 1, T, S] additive (or 0/1) mask separating packed segments (:160)."""
  if segment_id is None or source_segment_id is None:
    return None
  ret = (segment_id.unsqueeze(2) != source_segment_id.unsqueeze(1)).to(dtype)
  if apply_dtype_min:
    ret = ret * GetDtypeMin(dtype)
  return ret.unsqueeze(1)


def CausalSegmentMask(segment_ids, dtype=torch.float32):
  """[B, 1, T, T] additive mask = causal ∪ cross-segment (:52)."""
  slen = segment_ids.shape[1]
  seg = segment_ids.unsqueeze(2) != segment_ids.unsqueeze(1)
  causal = torch.triu(torch.ones(slen, slen, dtype=torch.bool,
                                 device=segment_ids.device), 1)
  return ((seg | causal).to(dtype) * GetDtypeMin(dtype)).unsqueeze(1)


def CrossAttentionPaddingWithTimestamp(timestamp, source_paddings, left_context,
                                       right_context):
  """[B, T, S] 0/1 padding restricting each query to a window around its
  aligned source timestamp (:86)."""
  s = source_paddings.shape[1]
  pos = torch.arange(s, device=timestamp.device).view(1, 1, s)
  ts = timestamp.unsqueeze(-1)
  out_of_window = (pos <= ts - left_context) | (pos > ts + right_context)
  pad = out_of_window | (source_paddings.unsqueeze(1) > 0)
  return pad.to(source_paddings.dtype if source_paddings.is_floating_point()
                else torch.float32)


def _CombineBias(*terms):
  """Sums additive masks, clamped so two 'very negative' terms never reach -inf."""
  out = None
  for t in terms:
    if t is None:
      continue
    out = t if out is None else out + t
  if out is None:
    return None
  return torch.clamp(out.float(), min=GetDtypeMin(torch.float32))


def _PaddingBias(paddings):
  """[B, S] 0/1 (or bool) → [B, 1, 1, S] additive."""
  if paddings is None:
    return None
  pad = paddings if paddings.dtype == torch.bool else paddings > 0
  return pad.view(pad.shape[0], 1, 1, pad.shape[1]).float() * GetDtypeMin()


class PerDimScaleLayer(base_layer.BaseLayer):
  """x · softplus(w)·1.4427/√dim, w init 0 ⇒ plain 1/√dim at start (:192)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('dim', 0, 'Number of individual dims.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('per_dim_scale', WeightParams(
        [p.dim], WeightInit.Constant(0.0), p.dtype,
        [self.__class__.__name__ + '_vars']))

  def Scale(self, theta):
    p = self.params
    return (1.442695041 / math.sqrt(p.dim)) * F.softplus(theta.per_dim_scale.float())

  def FProp(self, theta, inputs):
    return (inputs.float() * self.Scale(theta)).to(inputs.dtype)

  @classmethod
  def FPropMeta(cls, p, inputs):
    return NestedMap(flops=inputs.num_elements() * 5, out_shapes=(inputs,))


class MultiHeadedProjectionLayer(quant_utils.QuantizableLayer):
  """`BTD,DNH->BTNH` (input) or `BTNH,DNH->BTD` (output) projection (:253)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Input dimension D.')
    p.Define('num_heads', 0, 'Number of heads N.')
    p.Define('dim_per_head', 0, 'Size of each head H.')
    p.Define('is_output_projection', False, 'Project [B,T,N,H] back to [B,T,D].')
    p.Define('make_output_proj_no_op', False, 'Output projection is a reshape.')
    p.Define('use_bias', True, 'Add bias.')
    p.Define('input_proj_bias_rank_3', False, 'Bias shaped [N, 1, H].')
    p.Define('xla_num_partitions', None, 'Kept for parity.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    if p.make_output_proj_no_op:
      assert p.is_output_projection
      return
    coll = [self.__class__.__name__ + '_vars']
    self.CreateVariable('w', WeightParams(
        [p.input_dim, p.num_heads, p.dim_per_head], p.params_init, p.dtype, coll))
    if p.use_bias:
      if p.is_output_projection:
        shape = [p.input_dim]
      elif p.input_proj_bias_rank_3:
        shape = [p.num_heads, 1, p.dim_per_head]
      else:
        shape = [p.num_heads, p.dim_per_head]
      self.CreateVariable('b', WeightParams(shape, WeightInit.Constant(0.0),
                                            p.dtype, coll))

  def FProp(self, theta, inputs, eqn=None):
    p = self.params
    n, h, d = p.num_heads, p.dim_per_head, p.input_dim
    inputs = self._CastToFPropDtype(inputs)
    if p.make_output_proj_no_op:
      return inputs.reshape(*inputs.shape[:-2], n * h)
    w = theta.w.to(inputs.dtype)
    b = theta.b if p.use_bias else None
    if p.is_output_projection:
      x = inputs.reshape(*inputs.shape[:-2], n * h)
      # y = x · w[D, N·H]ᵀ : the weight is the K-major B operand, no transpose copy.
      return gemm.linear_t(x, w.reshape(d, n * h), b)
    y = gemm.linear(inputs, w.reshape(d, n * h),
                    b.reshape(n * h) if b is not None else None)
    return y.reshape(*inputs.shape[:-1], n, h)


class ReshapedMultiHeadedProjectionLayer(MultiHeadedProjectionLayer):
  """MultiHeadedProjectionLayer whose model dim D is presented as `[M, d]` with
  `M = device_mesh.shape[1]` (the layout 2-D sharded models keep activations in): inputs /
  outputs are `[B, T, M, d]` on the model side, `[B, T, N, H]` on the head side (:438)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    if 'device_mesh' not in p:
      p.Define('device_mesh', None, 'numpy mesh; its second axis splits the model dim.')
    return p

  def FProp(self, theta, inputs, eqn=None):
    p = self.params
    assert p.device_mesh is not None and p.device_mesh.ndim >= 2
    inputs = self._CastToFPropDtype(inputs)
    if p.make_output_proj_no_op:
      return inputs
    m = int(p.device_mesh.shape[1])
    w = theta.w.to(inputs.dtype)
    w = w.reshape(m, w.shape[0] // m, p.num_heads, p.dim_per_head)
    if p.is_output_projection:
      ret = torch.einsum(eqn or 'BTNH,MdNH->BTMd', inputs, w)
      if p.use_bias:
        ret = ret + theta.b.to(ret.dtype).reshape(m, -1)
      return ret
    ret = torch.einsum(eqn or 'BTMd,MdNH->BTNH', inputs, w)
    if p.use_bias:
      ret = ret + theta.b.to(ret.dtype)
    return ret


class MultiHeadedAttention(quant_utils.QuantizableLayer):
  """Dot-product attention over N heads; GQA / MQA / RoPE / packed inputs (:481).

  q:[B,T,D] k,v:[B,S,D] → encoded [B,T,D], probs [B,N,T,S] (probs only when
  `p.return_atten_probs`, default True for parity with callers that plot them;
  set False to stay on the fused kernel).
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'int, or dict with keys key/value/query.')
    p.Define('hidden_dim', 0, 'Number of hidden nodes (N·H).')
    p.Define('output_dim', None, 'Output dim; defaults to the query input dim.')
    p.Define('num_heads', 1, 'Number of attention heads.')
    p.Define('num_kv_heads', None, 'GQA: number of kv heads (divides num_heads).')
    p.Define('dim_per_head', None, 'H; defaults to hidden_dim // num_heads.')
    p.Define('dropout_tpl', layers.DropoutLayer.Params(), 'Dropout template.')
    p.Define('enable_value_proj', True, 'Project values.')
    p.Define('enable_query_scale', True, 'Scale the query.')
    p.Define('enable_per_dim_scale', True, 'Learned per-dim query scale.')
    p.Define('enable_qkv_proj_in_onestep', False, 'Kept for parity.')
    p.Define('enable_qk_proj_in_onestep', False, 'Kept for parity.')
    p.Define('use_mqa', False, 'Multi-query attention (one kv head).')
    p.Define('enable_shaped_attention', False, 'Shaped attention (arXiv 2311.01906).')
    p.Define('query_stride', 1, 'Strided queries: S == stride · T.')
    p.Define('query_first_n', None, 'Only the first N query positions.')
    p.Define('rope_tpl', None, 'RotaryPositionalEmbeddingLayer params.')
    p.Define('atten_dropout_prob', 0.0, 'Dropout on attention weights.')
    p.Define('proj_tpl', MultiHeadedProjectionLayer.Params(), 'Projection tpl.')
    p.Define('packed_input', False, 'Inputs are packed (segment_mask given).')
    p.Define('use_bias', True, 'Bias in the projections.')
    p.Define('enable_scaling_code_motion', False, 'Kept for parity.')
    p.Define('atten_extra_logit', None, 'Extra softmax logit (None ≠ 0).')
    p.Define('atten_logit_cap', 0.0, 'tanh soft cap on logits if > 0.')
    p.Define('use_scale_invariant_atten', False, 'relu + L1 norm instead of softmax.')
    p.Define('enable_ctx_pre_proj_ln', False, 'LN on the context before post-proj.')
    p.Define('enable_ctx_post_proj_ln', False, 'LN after post-proj.')
    p.Define('pre_softmax_probs_fn', None, 'Optional fn applied to probs.')
    p.Define('return_atten_probs', True,
             'Materialise [B,N,T,S] probabilities. False keeps the fused path.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.hidden_dim, p.name
    if isinstance(p.input_dim, dict):
      kd, vd, qd = p.input_dim['key'], p.input_dim['value'], p.input_dim['query']
    else:
      kd = vd = qd = p.input_dim
    assert qd > 0
    self._query_dim = qd
    n = p.num_heads
    h = self.dim_per_head
    nkv = 1 if p.use_mqa else (p.num_kv_heads or n)
    assert n % nkv == 0
    self._num_kv_heads = nkv

    def _Proj(dim, heads, out=False):
      return p.proj_tpl.Copy().Set(
          input_dim=dim, num_heads=heads, dim_per_head=h,
          is_output_projection=out, use_bias=p.use_bias)

    self.CreateChild('key', _Proj(kd, nkv))
    self.CreateChild('query', _Proj(qd, n))
    if p.enable_value_proj:
      self.CreateChild('value', _Proj(vd, nkv))
    if p.enable_query_scale and p.enable_per_dim_scale:
      self.CreateChild('per_dim_scale', PerDimScaleLayer.Params().Set(dim=h))
    if p.rope_tpl is not None:
      self.CreateChild('rope', p.rope_tpl.Copy().Set(embedding_dim=h))
    self.CreateChild('atten_dropout', p.dropout_tpl.Copy().Set(
        keep_prob=1.0 - p.atten_dropout_prob))
    if p.enable_ctx_pre_proj_ln:
      self.CreateChild('ctx_pre_proj_ln', layers.LayerNorm.Params().Set(
          input_dim=n * h))
    self.CreateChild('post', _Proj(p.output_dim or qd, n, out=True))
    if p.enable_ctx_post_proj_ln:
      self.CreateChild('ctx_post_proj_ln', layers.LayerNorm.Params().Set(
          input_dim=p.output_dim or qd))

  @property
  def dim_per_head(self):
    p = self.params
    return p.dim_per_head or p.hidden_dim // p.num_heads

  # -- pieces -------------------------------------------------------------------
  def _MaybeScaleQuery(self, theta, query):
    p = self.params
    if not p.enable_query_scale:
      return query
    if p.enable_per_dim_scale:
      return self.per_dim_scale.FProp(theta.per_dim_scale, query)
    return query * (self.dim_per_head ** -0.5)

  def _RoPE(self, theta, proj, stride=1, time_step=None):
    if self.params.rope_tpl is None:
      return proj
    b, t = proj.shape[0], proj.shape[1]
    if time_step is not None:
      pos = torch.as_tensor(time_step, device=proj.device).reshape(-1, 1).expand(b, 1)
    else:
      pos = (torch.arange(t, device=proj.device) * stride).unsqueeze(0).expand(b, t)
    return self.rope.FProp(theta.rope, proj, pos)

  def _HeadsProj(self, theta, query_vec, key_vec, value_vec):
    p = self.params
    q = self.query.FProp(theta.query, query_vec)
    k = self.key.FProp(theta.key, key_vec)
    if p.enable_value_proj:
      v = self.value.FProp(theta.value, value_vec)
    else:
      v = value_vec.reshape(*value_vec.shape[:2], self._num_kv_heads, -1)
    return q, k, v

  def _RelativeBias(self, theta, query, key, time_step=None):
    """Extra additive [B or 1, N, T, S] logit term (XL / RPE subclasses)."""
    del theta, query, key, time_step
    return None

  def _StructuralBias(self, t, s, device):
    """Static band/chunk mask of local-attention subclasses, [1,1,T,S] or None."""
    del t, s, device
    return None

  def _Core(self, theta, q, k, v, bias, want_probs):
    """q scaled & rotated. Returns (context [B,T,N,H], probs or None)."""
    p = self.params
    rel = self._RelativeBias(theta, q, k)
    bias = _CombineBias(bias, rel, self._StructuralBias(q.shape[1], k.shape[1],
                                                        q.device))
    drop = 0.0 if self.do_eval else p.atten_dropout_prob
    special = (p.use_scale_invariant_atten or p.enable_shaped_attention or
               p.pre_softmax_probs_fn is not None)
    if special:
      return self._CoreExplicit(theta, q, k, v, bias, drop)
    out = attention_ops.dot_product_attention(
        q, k, v, bias, 1.0, p.atten_logit_cap, p.atten_extra_logit, drop,
        return_probs=want_probs)
    return out if want_probs else (out, None)

  def _CoreExplicit(self, theta, q, k, v, bias, drop):
    p = self.params
    n = q.shape[2]
    kx, vx = attention_ops._ExpandKv(k, n), attention_ops._ExpandKv(v, n)  # pylint: disable=protected-access
    logits = torch.einsum('BTNH,BSNH->BNTS', q.float(), kx.float())
    if p.atten_logit_cap:
      logits = p.atten_logit_cap * torch.tanh(logits / p.atten_logit_cap)
    if bias is not None:
      logits = logits + bias
    if p.use_scale_invariant_atten:
      probs = F.relu(logits)
      probs = probs / probs.sum(-1, keepdim=True).clamp_min(1e-30)
    else:
      probs = py_utils.Softmax(logits, extra_logit=p.atten_extra_logit)
    if p.enable_shaped_attention:
      t, s = probs.shape[-2:]
      eye = torch.eye(t, s, device=probs.device)
      valid = (bias > GetDtypeMin() * 0.5).float() if bias is not None else (
          torch.ones_like(probs))
      center = valid / valid.sum(-1, keepdim=True).clamp_min(1.0)
      probs = probs + eye - center
    if p.pre_softmax_probs_fn is not None:
      probs = p.pre_softmax_probs_fn(probs)
    pd = probs.to(v.dtype)
    if drop:
      pd = F.dropout(pd, drop, training=True)
    return torch.einsum('BNTS,BSNH->BTNH', pd, vx), probs

  def _PostProj(self, theta, encoded):
    p = self.params
    if p.enable_ctx_pre_proj_ln:
      shp = encoded.shape
      encoded = self.ctx_pre_proj_ln.FProp(
          theta.ctx_pre_proj_ln, encoded.reshape(*shp[:-2], -1)).reshape(shp)
    out = self.post.FProp(theta.post, encoded)
    if p.enable_ctx_post_proj_ln:
      out = self.ctx_post_proj_ln.FProp(theta.ctx_post_proj_ln, out)
    return out

  def _Bias(self, paddings, segment_mask, per_step_padding):
    p = self.params
    if p.packed_input and segment_mask is not None:
      base = segment_mask.float()          # paddings already folded in
    else:
      base = _PaddingBias(paddings)
    if per_step_padding is not None:
      psp = per_step_padding if per_step_padding.dtype == torch.bool else (
          per_step_padding > 0)
      base = _CombineBias(base, psp.unsqueeze(1).float() * GetDtypeMin())
    return base

  # -- public -------------------------------------------------------------------
  def FProp(self, theta, query_vec, key_vec, value_vec, paddings,
            segment_mask=None, per_step_padding=None):
    p = self.params
    if p.query_first_n is not None:
      query_vec = query_vec[:, :p.query_first_n]
      if per_step_padding is not None:
        per_step_padding = per_step_padding[:, :p.query_first_n]
      if segment_mask is not None:
        segment_mask = segment_mask[:, :, :p.query_first_n]
    elif p.query_stride > 1:
      query_vec = query_vec[:, ::p.query_stride]
      if per_step_padding is not None:
        per_step_padding = per_step_padding[:, ::p.query_stride]
      if segment_mask is not None:
        segment_mask = segment_mask[:, :, ::p.query_stride]
    q, k, v = self._HeadsProj(theta, query_vec, key_vec, value_vec)
    q = self._RoPE(theta, q, stride=p.query_stride)
    k = self._RoPE(theta, k)
    q = self._MaybeScaleQuery(theta, q)
    bias = self._Bias(paddings, segment_mask, per_step_padding)
    ctx, probs = self._Core(theta, q, k, v, bias, p.return_atten_probs)
    return self._PostProj(theta, ctx), probs

  def InitStates(self, theta, target_batch_size, target_max_length):
    """Empty decode cache: key/value `[T, B, Nkv, H]`."""
    del theta
    dev = self.Device()
    dtype = py_utils.FPropDtype(self.params)
    shape = (target_max_length, target_batch_size, self._num_kv_heads,
             self.dim_per_head)
    return NestedMap(key=torch.zeros(shape, dtype=dtype, device=dev),
                     value=torch.zeros(shape, dtype=dtype, device=dev))

  def ExtendStep(self, theta, query_vec, cached_states, paddings,
                 segment_mask=None, per_step_padding=None, time_step=0,
                 use_short_seq_opt=False):
    """One decode step. query_vec `[B, 1, D]` (or `[B, D]`); returns
    (encoded `[B, 1, D]`, updated cache)."""
    del use_short_seq_opt
    p = self.params
    squeeze = query_vec.dim() == 2
    if squeeze:
      query_vec = query_vec.unsqueeze(1)
    t = int(time_step)
    q, k_new, v_new = self._HeadsProj(theta, query_vec, query_vec, query_vec)
    q = self._RoPE(theta, q, time_step=t)
    k_new = self._RoPE(theta, k_new, time_step=t)
    q = self._MaybeScaleQuery(theta, q)
    key = cached_states.key.clone()
    value = cached_states.value.clone()
    key[t] = k_new[:, 0].to(key.dtype)
    value[t] = v_new[:, 0].to(value.dtype)
    k = key.transpose(0, 1).to(q.dtype)       # [B, T, N, H]
    v = value.transpose(0, 1).to(q.dtype)
    s = k.shape[1]
    future = (torch.arange(s, device=q.device) > t).view(1, 1, 1, s).float() * GetDtypeMin()
    if per_step_padding is not None and per_step_padding.dim() == 2:
      per_step_padding = per_step_padding.unsqueeze(1)
    bias = _CombineBias(self._Bias(paddings, segment_mask, per_step_padding), future)
    rel = self._RelativeBias(theta, q, k, time_step=t)
    bias = _CombineBias(bias, rel)
    ctx = attention_ops.dot_product_attention(
        q, k, v, bias, 1.0, p.atten_logit_cap, p.atten_extra_logit, 0.0)
    out = self._PostProj(theta, ctx)
    if squeeze:
      out = out.squeeze(1)
    return out, NestedMap(key=key, value=value)

  @classmethod
  def FPropMeta(cls, p, *args):
    q = args[0]
    b, t, d = q[0], q[1], q[2]
    s = args[1][1]
    h = p.hidden_dim
    flops = 2 * b * (t * d * h + 2 * s * d * h + 2 * t * s * h + t * h * d)
    return NestedMap(flops=flops, out_shapes=(q,))


class SingleHeadedAttention(MultiHeadedAttention):
  """N = 1 special case kept for API parity (:1765)."""

  def __init__(self, params):
    params.num_heads = 1
    super().__init__(params)


class ReshapedMultiHeadedAttention(MultiHeadedAttention):
  """Inputs arrive as `[B, T, N, D/N]`; flattened on entry (:2063)."""

  def FProp(self, theta, query_vec, key_vec, value_vec, paddings,
            segment_mask=None, per_step_padding=None):
    flat = lambda x: x.reshape(*x.shape[:2], -1) if x.dim() == 4 else x
    out, probs = super().FProp(theta, flat(query_vec), flat(key_vec),
                               flat(value_vec), paddings, segment_mask,
                               per_step_padding)
    return out.reshape(*out.shape[:2], self.params.num_heads, -1), probs


def _SinusoidTable(length_range, dim, device, min_ts=1.0, max_ts=1.0e4):
  """Sinusoid embeddings for integer positions `length_range` → [L, dim]."""
  half = dim // 2
  inc = math.log(max_ts / min_ts) / max(half - 1, 1)
  inv = min_ts * torch.exp(torch.arange(half, device=device).float() * -inc)
  ang = length_range.float().unsqueeze(1) * inv.unsqueeze(0)
  emb = torch.cat([torch.sin(ang), torch.cos(ang)], 1)
  if dim % 2:
    emb = F.pad(emb, (0, 1))
  return emb


def _ToeplitzFromRelative(term, t, s, offset):
  """term[..., t, R] indexed by relative distance r = (s_idx - t_idx) + offset →
  [..., T, S] without an index tensor (strided view over a padded copy)."""
  # out[..., i, j] = term[..., i, j - i + offset]
  r = term.shape[-1]
  idx = (torch.arange(s, device=term.device).unsqueeze(0) -
         torch.arange(t, device=term.device).unsqueeze(1) + offset)
  valid = (idx >= 0) & (idx < r)
  out = torch.gather(term, -1, idx.clamp(0, r - 1).expand(*term.shape[:-2], t, s))
  return out * valid.to(out.dtype)


class MultiHeadedAttentionXL(MultiHeadedAttention):
  """Transformer-XL relative attention: (q+u)·k + (q+v)·W_r·R(i−j) (:2233)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('rel_pos_emb_dim', None, 'Sinusoid embedding dim.')
    p.Define('skip_term_b', False, 'Drop the position term (q·R).')
    p.Define('pos_atten_logits_tpl', None, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.rel_pos_emb_dim and p.rel_pos_emb_dim > 0
    self.CreateChild('pos_proj', p.proj_tpl.Copy().Set(
        input_dim=p.rel_pos_emb_dim, num_heads=p.num_heads,
        dim_per_head=self.dim_per_head, use_bias=False))

  def _CreateLayerVariables(self):
    super()._CreateLayerVariables()
    p = self.params
    shape = [p.num_heads, self.dim_per_head]
    coll = [self.__class__.__name__ + '_vars']
    self.CreateVariable('u', WeightParams(shape, WeightInit.Constant(0.0), p.dtype, coll))
    self.CreateVariable('v', WeightParams(shape, WeightInit.Constant(0.0), p.dtype, coll))

  def _RelativeBias(self, theta, query, key, time_step=None):
    p = self.params
    b, t, n, h = query.shape
    s = key.shape[1]
    kx = attention_ops._ExpandKv(key, n).float()  # pylint: disable=protected-access
    # term (c): u·k — content bias, [B,N,1,S]
    term_c = torch.einsum('NH,BSNH->BNS', theta.u.float(), kx).unsqueeze(2)
    if p.skip_term_b:
      return term_c
    # distances d = i − j ∈ [−(S−1), T−1]; table over r = j − i + (T−1) reversed
    if time_step is not None:
      dist = time_step - torch.arange(s, device=query.device)
      sin = _SinusoidTable(dist, p.rel_pos_emb_dim, query.device)
      r = self.pos_proj.FProp(theta.pos_proj, sin.unsqueeze(0).to(query.dtype))[0]
      qv = query.float() + theta.v.float()
      term_bd = torch.einsum('BTNH,SNH->BNTS', qv, r.float())
      return term_c + term_bd
    dist = torch.arange(t - 1, -s, -1, device=query.device)       # [T+S−1]
    sin = _SinusoidTable(dist, p.rel_pos_emb_dim, query.device)
    r = self.pos_proj.FProp(theta.pos_proj, sin.unsqueeze(0).to(query.dtype))[0]
    qv = query.float() + theta.v.float()
    term = torch.einsum('BTNH,RNH->BNTR', qv, r.float())           # R = T+S−1
    # element (i, j) needs distance i−j ⇒ index (T−1) − (i−j) = j − i + T − 1
    term_bd = _ToeplitzFromRelative(term, t, s, t - 1)
    return term_c + term_bd


class MultiHeadedAttentionRPE(MultiHeadedAttention):
  """Learned relative-position embeddings on keys (and optionally values),
  distances clipped to ±radius (Shaw et al.) (:2413)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('rel_pos_emb_tpl', layers.RelativePositionalEmbeddingLayer.Params(),
             'Relative embedding template.')
    p.Define('rel_pos_radius', None, 'Clip radius.')
    p.Define('skip_value_emb', False, 'No relative embedding on values.')
    p.Define('use_global_emb', True, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.rel_pos_radius
    tpl = p.rel_pos_emb_tpl.Copy().Set(radius=p.rel_pos_radius,
                                       dim=self.dim_per_head)
    self.CreateChild('key_emb', tpl.Copy())
    if not p.skip_value_emb:
      self.CreateChild('value_emb', tpl.Copy())

  def _RelIndex(self, t, s, device, time_step=None):
    r = self.params.rel_pos_radius
    qi = (torch.arange(t, device=device) if time_step is None else
          torch.full((1,), int(time_step), device=device))
    d = torch.arange(s, device=device).unsqueeze(0) - qi.unsqueeze(1)
    return d.clamp(-r, r) + r

  def _RelativeBias(self, theta, query, key, time_step=None):
    t, s = query.shape[1], key.shape[1]
    emb = theta.key_emb.w.float()                      # [2r+1, H]
    term = torch.einsum('BTNH,RH->BNTR', query.float(), emb)
    idx = self._RelIndex(t, s, query.device, time_step)
    return torch.gather(term, -1, idx.expand(*term.shape[:2], t, s))

  def _Core(self, theta, q, k, v, bias, want_probs):
    p = self.params
    if p.skip_value_emb:
      return super()._Core(theta, q, k, v, bias, want_probs)
    bias = _CombineBias(bias, self._RelativeBias(theta, q, k))
    ctx, probs = attention_ops.attention_ref(
        q, k, v, bias, 1.0, p.atten_logit_cap, p.atten_extra_logit,
        0.0 if self.do_eval else p.atten_dropout_prob, return_probs=True)
    t, s = q.shape[1], k.shape[1]
    idx = self._RelIndex(t, s, q.device)
    r = 2 * p.rel_pos_radius + 1
    onehot = F.one_hot(idx, r).float()                 # [T, S, R]
    pr = torch.einsum('BNTS,TSR->BNTR', probs, onehot)
    ctx = ctx + torch.einsum('BNTR,RH->BTNH', pr, theta.value_emb.w.float()).to(ctx.dtype)
    return ctx, (probs if want_probs else None)


class LocalSelfAttention(MultiHeadedAttention):
  """Each query sees `left_context − 1` past and `right_context` future keys
  (:2656). Implemented as a band bias on the fused kernel; `StreamStep`
  keeps a rolling key/value cache of `left_context − 1 + right_context` frames.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('block_size', None, 'Kept for parity (blocking is internal).')
    p.Define('left_context', None, 'Past frames incl. the current one.')
    p.Define('right_context', 0, 'Future frames.')
    p.Define('force_consistent_probs_shape', False, 'Kept for parity.')
    p.Define('inference_step_max_length', None, 'Kept for parity.')
    p.Define('use_3d_recurrent_state', False, 'Kept for parity.')
    p.Define('minimize_state_size', False, 'Kept for parity.')
    return p

  def _StructuralBias(self, t, s, device):
    p = self.params
    i = torch.arange(t, device=device).unsqueeze(1)
    j = torch.arange(s, device=device).unsqueeze(0)
    bad = torch.zeros(t, s, dtype=torch.bool, device=device)
    if p.left_context is not None:
      bad |= j < i - (p.left_context - 1)
    if p.right_context is not None:
      bad |= j > i + p.right_context
    return bad.view(1, 1, t, s).float() * GetDtypeMin()

  def zero_state(self, batch_size):
    p = self.params
    ctx = (p.left_context - 1) + p.right_context
    dev, dt = self.Device(), py_utils.FPropDtype(p)
    shape = (batch_size, ctx, self._num_kv_heads, self.dim_per_head)
    return NestedMap(key=torch.zeros(shape, dtype=dt, device=dev),
                     value=torch.zeros(shape, dtype=dt, device=dev),
                     masks=torch.ones(batch_size, ctx, device=dev),
                     query=torch.zeros(batch_size, p.right_context, self._query_dim,
                                       dtype=dt, device=dev) if p.right_context else None,
                     out_masks=torch.ones(batch_size, p.right_context, device=dev)
                     if p.right_context else None)

  def StreamStep(self, theta, query_vec, paddings, state0):
    """Streaming FProp over a chunk `[B, Q, D]`; output delayed by `right_context`."""
    p = self.params
    b, qn, _ = query_vec.shape
    r = p.right_context
    q_new, k_new, v_new = self._HeadsProj(theta, query_vec, query_vec, query_vec)
    k_all = torch.cat([state0.key.to(k_new.dtype), k_new], 1)
    v_all = torch.cat([state0.value.to(v_new.dtype), v_new], 1)
    m_all = torch.cat([state0.masks, paddings.float()], 1)
    if r:
      q_in = torch.cat([state0.query.to(query_vec.dtype), query_vec], 1)[:, :qn]
      out_pad = torch.cat([state0.out_masks, paddings.float()], 1)[:, :qn]
      q = self.query.FProp(theta.query, q_in)
    else:
      q, out_pad = q_new, paddings.float()
    q = self._MaybeScaleQuery(theta, q)
    ctx_len = state0.key.shape[1]
    # query i (absolute pos ctx_len − r + i in k_all coords … ) band mask:
    qpos = torch.arange(qn, device=q.device).unsqueeze(1) + (ctx_len - r)
    kpos = torch.arange(k_all.shape[1], device=q.device).unsqueeze(0)
    bad = (kpos < qpos - (p.left_context - 1)) | (kpos > qpos + r)
    bias = _CombineBias(bad.view(1, 1, qn, -1).float() * GetDtypeMin(),
                        _PaddingBias(m_all))
    ctx = attention_ops.dot_product_attention(q, k_all, v_all, bias, 1.0,
                                              p.atten_logit_cap, p.atten_extra_logit)
    out = self._PostProj(theta, ctx)
    state1 = NestedMap(
        key=k_all[:, -ctx_len:] if ctx_len else k_all[:, :0],
        value=v_all[:, -ctx_len:] if ctx_len else v_all[:, :0],
        masks=m_all[:, -ctx_len:] if ctx_len else m_all[:, :0],
        query=torch.cat([state0.query.to(query_vec.dtype), query_vec], 1)[:, -r:] if r else None,
        out_masks=torch.cat([state0.out_masks, paddings.float()], 1)[:, -r:] if r else None)
    return out, out_pad, state1


class LocalSelfAttentionXL(LocalSelfAttention):
  """Local attention + Transformer-XL relative term (:3754)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('rel_pos_emb_dim', None, 'Sinusoid embedding dim.')
    p.Define('skip_term_b', False, 'Drop the position term.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('pos_proj', p.proj_tpl.Copy().Set(
        input_dim=p.rel_pos_emb_dim, num_heads=p.num_heads,
        dim_per_head=self.dim_per_head, use_bias=False))

  def _CreateLayerVariables(self):
    super()._CreateLayerVariables()
    p = self.params
    shape = [p.num_heads, self.dim_per_head]
    coll = [self.__class__.__name__ + '_vars']
    self.CreateVariable('u', WeightParams(shape, WeightInit.Constant(0.0), p.dtype, coll))
    self.CreateVariable('v', WeightParams(shape, WeightInit.Constant(0.0), p.dtype, coll))

  _RelativeBias = MultiHeadedAttentionXL._RelativeBias


class ChunkwiseSelfAttention(MultiHeadedAttention):
  """Queries attend within their own chunk plus `left_context`/`right_context`
  neighbouring frames of it (:4008)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('chunk_size', None, 'Chunk length.')
    p.Define('left_context', 0, 'Extra frames before the chunk.')
    p.Define('right_context', 0, 'Extra frames after the chunk.')
    return p

  def _StructuralBias(self, t, s, device):
    p = self.params
    c = p.chunk_size
    i = torch.arange(t, device=device).unsqueeze(1)
    j = torch.arange(s, device=device).unsqueeze(0)
    start = (i // c) * c
    bad = (j < start - p.left_context) | (j >= start + c + p.right_context)
    return bad.view(1, 1, t, s).float() * GetDtypeMin()


class MultiSourceAttention(base_layer.BaseLayer):
  """One attention per named source; outputs summed/merged (:5113)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('source_atten_tpls', None, 'List of (source_key, atten params).')
    p.Define('input_dim', 0, 'Default input dim.')
    p.Define('hidden_dim', 0, 'Default hidden dim.')
    p.Define('primary_source_key', 'source_0', 'Source whose probs are returned.')
    p.Define('atten_merger_tpl', None, 'Merger layer params (defaults to sum).')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self._keys = []
    for key, tpl in p.source_atten_tpls:
      tpl = tpl.Copy()
      if tpl.hidden_dim <= 0:
        tpl.hidden_dim = p.hidden_dim
      if not tpl.input_dim:
        tpl.input_dim = p.input_dim
      self.CreateChild('atten_%s' % key, tpl)
      self._keys.append(key)
    if p.atten_merger_tpl is not None:
      self.CreateChild('atten_merger', p.atten_merger_tpl)

  def FProp(self, theta, query_vec, key_vec, value_vec, paddings,
            segment_mask=None, per_step_padding=None):
    p = self.params
    outs, primary_probs = [], None
    for key in self._keys:
      child = getattr(self, 'atten_%s' % key)
      out, probs = child.FProp(theta['atten_%s' % key], query_vec, key_vec[key],
                               value_vec[key], paddings[key],
                               segment_mask[key] if segment_mask else None,
                               per_step_padding)
      outs.append(out)
      if key == p.primary_source_key:
        primary_probs = probs
    if p.atten_merger_tpl is not None:
      return self.atten_merger.FProp(theta.atten_merger, outs, query_vec), primary_probs
    return sum(outs), primary_probs


class TransformerAttentionLayer(base_layer.BaseLayer):
  """LN → (self|cross) attention → dropout → residual (:5226)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Model dim.')
    p.Define('hidden_dim', 0, 'Attention hidden dim.')
    p.Define('num_heads', 8, 'Heads.')
    p.Define('is_masked', False, 'Causal self-attention.')
    p.Define('atten_dropout_prob', 0.0, 'Attention-weights dropout.')
    p.Define('residual_dropout_prob', 0.0, 'Dropout before the residual add.')
    p.Define('pre_layer_norm', True, 'Pre- or post-LN.')
    p.Define('primer_hybrid_norm', False, 'Pre- and post-LN.')
    p.Define('add_unnormalized_input', True, 'Residual uses the raw input.')
    p.Define('add_skip_connection', True, 'Residual add.')
    p.Define('ln_tpl', layers.LayerNorm.Params(), 'LN template.')
    p.Define('atten_tpl', MultiHeadedAttention.Params().Set(
        use_bias=False, enable_per_dim_scale=False), 'Attention template.')
    p.Define('dropout_tpl', layers.DropoutLayer.Params(), 'Dropout template.')
    p.Define('residual_droppath_prob', 0.0, 'Stochastic depth.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    hid = p.hidden_dim or p.input_dim
    qdim = p.input_dim['query'] if isinstance(p.input_dim, dict) else p.input_dim
    tpl = p.atten_tpl
    if isinstance(tpl, (list, tuple)):
      srcs = [('source_%d' % i, self._Atten(t, hid)) for i, t in enumerate(tpl)]
      self.CreateChild('atten', MultiSourceAttention.Params().Set(
          source_atten_tpls=srcs, input_dim=p.input_dim, hidden_dim=hid))
    else:
      self.CreateChild('atten', self._Atten(tpl, hid))
    self.CreateChild('layer_norm', p.ln_tpl.Copy().Set(input_dim=qdim))
    if p.primer_hybrid_norm:
      self.CreateChild('post_layer_norm', p.ln_tpl.Copy().Set(input_dim=qdim))
    self.CreateChild('residual_dropout', p.dropout_tpl.Copy().Set(
        keep_prob=1.0 - p.residual_dropout_prob))

  def _Atten(self, tpl, hid):
    p = self.params
    t = tpl.Copy()
    t.input_dim = t.input_dim or p.input_dim
    t.hidden_dim = t.hidden_dim or hid
    t.num_heads = p.num_heads
    t.atten_dropout_prob = p.atten_dropout_prob
    return t

  def _Norm(self, theta, x):
    return self.layer_norm.FProp(theta.layer_norm, x)

  def _Finish(self, theta, unnormalized, normalized, ctx):
    p = self.params
    if p.primer_hybrid_norm:
      ctx = self.post_layer_norm.FProp(theta.post_layer_norm, ctx)
    ctx = self.residual_dropout.FProp(theta.residual_dropout, ctx)
    if p.add_skip_connection:
      res = unnormalized if p.add_unnormalized_input else normalized
      if p.residual_droppath_prob and not self.do_eval:
        keep = 1.0 - p.residual_droppath_prob
        mask = (torch.rand(ctx.shape[0], *([1] * (ctx.dim() - 1)),
                           device=ctx.device) < keep).to(ctx.dtype) / keep
        ctx = ctx * mask
      ctx = res + ctx
    if not p.pre_layer_norm:
      ctx = self._Norm(theta, ctx)
    return ctx

  def FProp(self, theta, query_vec, source_vecs, paddings,
            per_step_padding_override=None, segment_mask=None):
    """query_vec [B,T,D]; source_vecs None ⇒ self-attention."""
    p = self.params
    b, t, _ = query_vec.shape
    unnormalized = query_vec
    q = self._Norm(theta, query_vec) if p.pre_layer_norm else query_vec
    src = q if source_vecs is None else source_vecs
    psp = per_step_padding_override
    if p.is_masked and psp is None and segment_mask is None:
      psp = CausalPadding(t, device=q.device).unsqueeze(0).expand(b, t, t)
    elif p.is_masked and psp is None:
      # packed: fold the causal mask into the segment mask
      segment_mask = _CombineBias(
          segment_mask, CausalPadding(t, device=q.device).view(1, 1, t, t) * GetDtypeMin())
    ctx, probs = self.atten.FProp(theta.atten, q, src, src, paddings,
                                  segment_mask=segment_mask, per_step_padding=psp)
    return self._Finish(theta, unnormalized, q, ctx), probs

  def InitStates(self, theta, target_batch_size, target_max_length):
    return self.atten.InitStates(theta.atten, target_batch_size, target_max_length)

  def ExtendStep(self, theta, query_vec, cached_states, time_step,
                 use_short_seq_opt=False, *, segment_mask=None,
                 per_step_padding=None, paddings=None):
    p = self.params
    assert p.is_masked
    unnormalized = query_vec
    q = self._Norm(theta, query_vec) if p.pre_layer_norm else query_vec
    ctx, states = self.atten.ExtendStep(
        theta.atten, q, cached_states, paddings, segment_mask, per_step_padding,
        time_step, use_short_seq_opt)
    return self._Finish(theta, unnormalized, q, ctx), states


class TransformerMultiSourceAttentionLayer(TransformerAttentionLayer):
  """Cross attention over several named sources (:6206)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_source', 0, 'Number of sources.')
    p.Define('primary_source_index', 0, 'Which source returns probs.')
    p.Define('multi_source_atten', MultiSourceAttention.Params(), 'Wrapper tpl.')
    return p

  def __init__(self, params):
    p = params
    tpl = p.atten_tpl
    if not isinstance(tpl, (list, tuple)):
      p.atten_tpl = [tpl.Copy() for _ in range(p.num_source)]
    super().__init__(p)


class ReZeroAddLayer(base_layer.BaseLayer):
  """x + α·f(x), α learnable, init 0 (:7958)."""

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('alpha', WeightParams([1], WeightInit.Constant(0.0), p.dtype))

  def FProp(self, theta, x, y):
    return x + theta.alpha.to(y.dtype) * y


class ResidualAddLayer(base_layer.BaseLayer):
  """x + w·y (optionally y = f(y)) (:8017)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('residual_weight', 1.0, 'Weight of the residual branch.')
    p.Define('apply_residual', True, 'If False return y only.')
    return p

  def FProp(self, theta, x, y):
    p = self.params
    return x + p.residual_weight * y if p.apply_residual else y


class PaddingLayer(base_layer.BaseLayer):
  """Zeroes padded positions (:8056)."""

  def FProp(self, theta, inputs, paddings):
    return py_utils.ApplyPadding(paddings.unsqueeze(-1), inputs)


class StrideLayer(base_layer.BaseLayer):
  """Keeps every `stride`-th frame (or the first `first_n`) (:8085)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('stride', 0, '0 ⇒ keep only frame 0; 1 ⇒ identity.')
    p.Define('first_n', None, 'Keep only the first n (strided) frames.')
    p.Define('axis', 1, 'Time axis.')
    return p

  def FProp(self, theta, x):
    p = self.params
    if p.stride == 1 and not p.first_n:
      return x
    idx = [slice(None)] * x.dim()
    if p.stride == 0:
      idx[p.axis] = slice(0, 1)
    else:
      end = p.first_n * p.stride if p.first_n else None
      idx[p.axis] = slice(0, end, p.stride)
    return x[tuple(idx)]


class FunnelPoolingLayer(StrideLayer):
  """Funnel-Transformer pooling over time with padding-aware mean/max (:8162)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('pooling_type', 'AVG', 'AVG or MAX.')
    p.Define('padding_algorithm', 'SAME', 'SAME or VALID.')
    p.Define('begin_intact', 0, 'Leading frames (e.g. CLS) left unpooled.')
    p.Define('trunc_seq', True, 'Truncate so intact+pooled has length T/stride.')
    p.Define('exclude_pad_effect', True, 'Mask pads out of the pooling.')
    return p

  def FProp(self, theta, x, paddings=None):
    p = self.params
    if p.stride in (0, 1):
      y = super().FProp(theta, x)
      if paddings is None:
        return y
      return y, StrideLayer.FProp(self, theta, paddings)
    intact, rest = x[:, :p.begin_intact], x[:, p.begin_intact:]
    pad_rest = paddings[:, p.begin_intact:] if paddings is not None else None
    t = rest.shape[1]
    t_out = -(-t // p.stride) if p.padding_algorithm == 'SAME' else t // p.stride
    pad_t = t_out * p.stride - t
    xr = F.pad(rest, (0, 0, 0, max(pad_t, 0)))[:, :t_out * p.stride]
    w = torch.ones(x.shape[0], t, device=x.device) if pad_rest is None else (
        1.0 - pad_rest.float())
    w = F.pad(w, (0, max(pad_t, 0)))[:, :t_out * p.stride]
    xr = xr.reshape(x.shape[0], t_out, p.stride, -1)
    w = w.reshape(x.shape[0], t_out, p.stride, 1)
    if not p.exclude_pad_effect:
      w = torch.ones_like(w)
    if p.pooling_type == 'AVG':
      y = (xr * w.to(xr.dtype)).sum(2) / w.sum(2).clamp_min(1.0).to(xr.dtype)
    else:
      y = xr.masked_fill(w == 0, torch.finfo(xr.dtype).min).max(2).values
      y = y * (w.sum(2) > 0).to(y.dtype)
    y = torch.cat([intact, y], 1)
    if paddings is None:
      return y
    new_pad = (w.sum(2).squeeze(-1) == 0).to(paddings.dtype)
    return y, torch.cat([paddings[:, :p.begin_intact], new_pad], 1)


class FunnelUpsampleLayer(base_layer.BaseLayer):
  """Repeat (or deconv) frames `upsample_rate`× (:8423)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('begin_intact', 0, 'Leading frames left untouched.')
    p.Define('upsample_rate', 1, 'Repeat factor.')
    p.Define('upsample_type', 'REPEAT', 'REPEAT or DECONV.')
    p.Define('hidden_dim', 0, 'For DECONV.')
    p.Define('trunc_seq', True, 'Kept for parity.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    if p.upsample_type == 'DECONV':
      self.CreateVariable('weight', WeightParams(
          [p.hidden_dim, p.upsample_rate, p.hidden_dim], p.params_init, p.dtype))
      self.CreateVariable('bias', WeightParams(
          [p.upsample_rate, p.hidden_dim], WeightInit.Constant(0.0), p.dtype))

  def FProp(self, theta, x):
    p = self.params
    intact, rest = x[:, :p.begin_intact], x[:, p.begin_intact:]
    if p.upsample_type == 'REPEAT':
      up = rest.repeat_interleave(p.upsample_rate, dim=1)
    else:
      up = torch.einsum('BTD,DRE->BTRE', rest, theta.weight.to(rest.dtype))
      up = (up + theta.bias.to(up.dtype)).reshape(x.shape[0], -1, p.hidden_dim)
    return torch.cat([intact, up], 1)


class MeshSplitLayer(base_layer.BaseLayer):
  """Sharding annotation; identity on one device (:8556)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('split_dims_mapping', None, 'Mapping.')
    return p

  def FProp(self, theta, x):
    return x


class TransformerLayer(base_layer.BaseLayer):
  """self-attention [→ cross-attention] → feed-forward (:6265).

  FProp(query_vec [B,T,D], paddings [B,T], aux_vec, aux_paddings, …) →
  (output, cross-attention probs or self-attention probs).
  """

  @classmethod
  def Params(cls):
    from lingvo_b200.core import layers_with_attention  # pylint: disable=g-import-not-at-top
    p = super().Params()
    p.Define('has_aux_atten', False, 'Add a cross-attention sub-layer.')
    p.Define('mask_self_atten', False, 'Causal self-attention.')
    p.Define('input_dim', 0, 'Input dim.')
    p.Define('output_dim', 0, 'Output dim (defaults to input_dim).')
    p.Define('num_heads', None, 'Override heads of both attentions.')
    p.Define('aux_atten_input_dim', None, 'Dim of the aux source.')
    p.Define('tr_atten_tpl', TransformerAttentionLayer.Params(), 'Self-atten tpl.')
    p.Define('tr_self_atten_tpl', None, 'Separate self-atten tpl (decoder).')
    p.Define('tr_fflayer_tpl',
             layers_with_attention.TransformerFeedForwardLayer.Params().Set(
                 hidden_dim=2048), 'Feed-forward tpl.')
    p.Define('packed_input', False, 'Packed inputs.')
    p.Define('compute_flops', False, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self_tpl = (p.tr_self_atten_tpl or p.tr_atten_tpl).Copy()
    self_tpl.input_dim = p.input_dim
    self_tpl.is_masked = p.mask_self_atten
    if p.num_heads:
      self_tpl.num_heads = p.num_heads
    self._SetPacked(self_tpl)
    self.CreateChild('self_atten', self_tpl)
    if p.has_aux_atten:
      cross = p.tr_atten_tpl.Copy()
      cross.is_masked = False
      if p.num_heads:
        cross.num_heads = p.num_heads
      if p.aux_atten_input_dim and p.aux_atten_input_dim != p.input_dim:
        cross.input_dim = {'query': p.input_dim, 'key': p.aux_atten_input_dim,
                           'value': p.aux_atten_input_dim}
      else:
        cross.input_dim = p.input_dim
      self._SetPacked(cross)
      self.CreateChild('cross_atten', cross)
    ff = p.tr_fflayer_tpl.Copy()
    ff.input_dim = p.input_dim
    ff.output_dim = p.output_dim or p.input_dim
    self.CreateChild('fflayer', ff)

  def _SetPacked(self, tpl):
    if not self.params.packed_input:
      return
    a = tpl.atten_tpl
    for t in (a if isinstance(a, (list, tuple)) else [a]):
      t.packed_input = True

  @classmethod
  def SetFPropDtype(cls, p, fprop_dtype):
    p.fprop_dtype = fprop_dtype
    for sub in (p.tr_atten_tpl, p.tr_self_atten_tpl, p.tr_fflayer_tpl):
      if sub is not None:
        sub.fprop_dtype = fprop_dtype
    return p

  @classmethod
  def CommonParams(cls, input_dim, atten_num_heads, atten_is_relative_position=False,
                   atten_local_context=None, atten_left_context=None,
                   atten_right_context=None, has_aux_atten=False,
                   mask_self_atten=False, fflayer_hidden_dim=None,
                   fflayer_output_dim=None, dropout_prob=0.):
    p = cls.Params().Set(input_dim=input_dim, has_aux_atten=has_aux_atten,
                         mask_self_atten=mask_self_atten, num_heads=atten_num_heads,
                         output_dim=fflayer_output_dim or input_dim)
    p.tr_atten_tpl.Set(num_heads=atten_num_heads, residual_dropout_prob=dropout_prob,
                       atten_dropout_prob=dropout_prob)
    if atten_local_context or atten_left_context or atten_right_context:
      left = atten_left_context or (atten_local_context + 1 if atten_local_context else None)
      right = atten_right_context if atten_right_context is not None else (
          atten_local_context or 0)
      base = LocalSelfAttentionXL if atten_is_relative_position else LocalSelfAttention
      p.tr_atten_tpl.atten_tpl = base.Params().Set(
          left_context=left, right_context=right, use_bias=False,
          enable_per_dim_scale=False)
      if atten_is_relative_position:
        p.tr_atten_tpl.atten_tpl.rel_pos_emb_dim = input_dim
    elif atten_is_relative_position:
      p.tr_atten_tpl.atten_tpl = MultiHeadedAttentionXL.Params().Set(
          rel_pos_emb_dim=input_dim, use_bias=False, enable_per_dim_scale=False)
    p.tr_fflayer_tpl.Set(hidden_dim=fflayer_hidden_dim or 4 * input_dim,
                         residual_dropout_prob=dropout_prob,
                         relu_dropout_prob=dropout_prob)
    return p

  def FProp(self, theta, query_vec, paddings, aux_vec=None, aux_paddings=None,
            per_step_padding_override=None, segment_mask=None,
            aux_segment_mask=None):
    p = self.params
    out, probs = self.self_atten.FProp(
        theta.self_atten, query_vec, None, paddings,
        per_step_padding_override=per_step_padding_override,
        segment_mask=segment_mask)
    if p.has_aux_atten:
      assert aux_vec is not None
      out, probs = self.cross_atten.FProp(
          theta.cross_atten, out, aux_vec, aux_paddings,
          segment_mask=aux_segment_mask)
    out = self.fflayer.FProp(theta.fflayer, out, paddings)
    return out, probs

  def InitStates(self, theta, target_batch_size, target_max_length):
    return self.self_atten.InitStates(theta.self_atten, target_batch_size,
                                      target_max_length)

  def ExtendStep(self, theta, query_vec, aux_vec, aux_paddings, cached_states,
                 time_step, use_short_seq_opt=False, *, segment_mask=None,
                 aux_segment_mask=None, per_step_padding=None):
    """query_vec [B, 1, D] → (output [B, 1, D], cross-atten probs, new cache)."""
    p = self.params
    out, states = self.self_atten.ExtendStep(
        theta.self_atten, query_vec, cached_states, time_step, use_short_seq_opt,
        segment_mask=segment_mask, per_step_padding=per_step_padding)
    probs = None
    if p.has_aux_atten:
      out, probs = self.cross_atten.FProp(theta.cross_atten, out, aux_vec,
                                          aux_paddings, segment_mask=aux_segment_mask)
    pad = torch.zeros(out.shape[0], out.shape[1], device=out.device)
    out = self.fflayer.FProp(theta.fflayer, out, pad)
    return out, probs, states


class TransformerDecoderLayer(TransformerLayer):
  """TransformerLayer with masked self-attention + cross-attention (:6954)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.has_aux_atten = True
    p.mask_self_atten = True
    return p


class MultiSourceTransformerLayer(TransformerLayer):
  """Cross attention over multiple sources (:6820)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_source', 0, 'Number of sources.')
    p.Define('primary_source_index', 0, 'Source whose probs are returned.')
    return p

  def __init__(self, params):
    p = params
    assert p.has_aux_atten
    cross = TransformerMultiSourceAttentionLayer.Params().Set(
        num_source=p.num_source, primary_source_index=p.primary_source_index)
    for k, v in p.tr_atten_tpl.IterParams():
      if k in cross and k not in ('cls', 'name'):
        cross.Set(**{k: v})
    p.tr_self_atten_tpl = p.tr_self_atten_tpl or p.tr_atten_tpl.Copy()
    p.tr_atten_tpl = cross
    super().__init__(p)


class MultiSourceTransformerDecoderLayer(MultiSourceTransformerLayer):

  @classmethod
  def Params(cls):
    p = super().Params()
    p.has_aux_atten = True
    p.mask_self_atten = True
    return p


def UseRelativeAttentionInTransformerLayer(transformer_params, rel_pos_emb_dim,
                                           atten_type=None):
  """Swaps the self-attention template for an XL variant (:6866)."""
  tpl = transformer_params.tr_self_atten_tpl or transformer_params.tr_atten_tpl
  old = tpl.atten_tpl
  cls = {None: MultiHeadedAttentionXL, 'multihead': MultiHeadedAttentionXL,
         'local': LocalSelfAttentionXL}[atten_type]
  new = cls.Params()
  for k, v in old.IterParams():
    if k in new and k not in ('cls',):
      new.Set(**{k: v})
  new.rel_pos_emb_dim = rel_pos_emb_dim
  tpl.atten_tpl = new
  return transformer_params


def ClearRelativeAttentionInTransformerLayer(transformer_params):
  """Reverts to plain (local) attention (:6921)."""
  tpl = transformer_params.tr_self_atten_tpl or transformer_params.tr_atten_tpl
  old = tpl.atten_tpl
  base = LocalSelfAttention if issubclass(old.cls, LocalSelfAttention) else (
      MultiHeadedAttention)
  new = base.Params()
  for k, v in old.IterParams():
    if k in new and k not in ('cls',):
      new.Set(**{k: v})
  tpl.atten_tpl = new
  return transformer_params


class StackedTransformerLayers(base_layer.BaseLayer):
  """N TransformerLayers + optional final LN (:7116)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('has_aux_atten', False, 'Cross attention in every layer.')
    p.Define('mask_self_atten', False, 'Causal self attention.')
    p.Define('num_layers', 0, 'Number of layers.')
    p.Define('mdl_dim', 0, 'Model dim.')
    p.Define('hidden_dim', 0, 'FFN hidden dim.')
    p.Define('num_atten_heads', 0, 'Heads.')
    p.Define('dropout_prob', 0.0, 'Dropout everywhere.')
    p.Define('stochastic_depth_droppath_prob', 0.0, 'Max droppath (linear ramp).')
    p.Define('add_unnormalized_input', True, 'Residual uses raw input.')
    p.Define('transformer_layer_params_tpl', TransformerLayer.Params(),
             'Layer template or list of templates.')
    p.Define('funnel_pool_strides', None, 'Kept for parity.')
    p.Define('funnel_pool_begin_intacts', None, 'Kept for parity.')
    p.Define('final_layer_norm', False, 'Apply LN on the output.')
    p.Define('packed_input', False, 'Packed inputs.')
    p.Define('use_fused_layernorm', False, 'Kept for parity.')
    p.Define('layernorm_tpl', layers.LayerNorm.Params(), 'Final LN template.')
    p.Define('splits', None, 'Kept for parity (GPipe split points).')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.num_layers > 0 and p.mdl_dim > 0
    tpls = p.transformer_layer_params_tpl
    if not isinstance(tpls, (list, tuple)):
      tpls = [tpls] * p.num_layers
    layer_ps = []
    for i in range(p.num_layers):
      lp = tpls[i % len(tpls)].Copy()
      lp.name = 'layer_%d' % i
      lp.has_aux_atten = p.has_aux_atten
      lp.mask_self_atten = p.mask_self_atten
      lp.input_dim = p.mdl_dim
      lp.output_dim = p.mdl_dim
      lp.packed_input = p.packed_input
      if p.num_atten_heads:
        lp.num_heads = p.num_atten_heads
      for at in (lp.tr_atten_tpl, lp.tr_self_atten_tpl):
        if at is None:
          continue
        at.atten_dropout_prob = p.dropout_prob
        at.residual_dropout_prob = p.dropout_prob
        at.add_unnormalized_input = p.add_unnormalized_input
        if p.num_atten_heads:
          at.num_heads = p.num_atten_heads
        if p.stochastic_depth_droppath_prob:
          at.residual_droppath_prob = (
              p.stochastic_depth_droppath_prob * i / max(p.num_layers - 1, 1))
      if p.hidden_dim:
        lp.tr_fflayer_tpl.hidden_dim = p.hidden_dim
      lp.tr_fflayer_tpl.residual_dropout_prob = p.dropout_prob
      lp.tr_fflayer_tpl.relu_dropout_prob = p.dropout_prob
      layer_ps.append(lp)
    self.CreateChildren('x_layers', layer_ps)
    if p.final_layer_norm:
      self.CreateChild('final_ln', p.layernorm_tpl.Copy().Set(input_dim=p.mdl_dim))

  @classmethod
  def GetSplitForLayer(cls, buckets, layer_index):
    for i, b in enumerate(buckets):
      if layer_index <= b:
        return i
    return -1

  def FProp(self, theta, query_vec, paddings, aux_vec=None, aux_paddings=None,
            segment_mask=None, aux_segment_mask=None):
    """`aux_vec` may be a list with one source encoding per layer (transparent encoders)."""
    p = self.params
    x = query_vec
    for i, layer in enumerate(self.x_layers):
      aux_i = aux_vec[i] if isinstance(aux_vec, (list, tuple)) else aux_vec
      x, _ = layer.FProp(theta.x_layers[i], x, paddings, aux_i, aux_paddings,
                         segment_mask=segment_mask,
                         aux_segment_mask=aux_segment_mask)
    if p.final_layer_norm:
      x = self.final_ln.FProp(theta.final_ln, x)
    return x, paddings

  def InitStates(self, theta, *args, **kwargs):
    return NestedMap(x_layers=[
        layer.InitStates(theta.x_layers[i], *args, **kwargs)
        for i, layer in enumerate(self.x_layers)])

  def ExtendStep(self, theta, query_vec, aux_vec, aux_paddings, cached_states,
                 time_step, use_short_seq_opt=False, **kwargs):
    p = self.params
    x = query_vec
    new_states = NestedMap(x_layers=[])
    for i, layer in enumerate(self.x_layers):
      aux_i = aux_vec[i] if isinstance(aux_vec, (list, tuple)) else aux_vec
      x, _, st = layer.ExtendStep(theta.x_layers[i], x, aux_i, aux_paddings,
                                  cached_states.x_layers[i], time_step,
                                  use_short_seq_opt, **kwargs)
      new_states.x_layers.append(st)
    if p.final_layer_norm:
      x = self.final_ln.FProp(theta.final_ln, x)
    return x, new_states


class RepeatedTransformerLayer(builder_layers.RepeatLayer):
  """`repeat` copies of one TransformerLayer body with stacked weights (:6976)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    if 'atten_prob_aggregation' not in p:
      p.Define('atten_prob_aggregation', None, 'None | "mean".')
    return p

  def FProp(self, theta, query_vec, paddings, aux_vec=None, aux_paddings=None,
            segment_mask=None, aux_segment_mask=None):
    p = self.params
    x = query_vec
    probs_acc = []
    for i in range(p.repeat):
      th = self._SliceTheta(theta, i) if hasattr(self, '_SliceTheta') else theta.body
      x, probs = self.body.FProp(th, x, paddings, aux_vec, aux_paddings,
                                 segment_mask=segment_mask,
                                 aux_segment_mask=aux_segment_mask)
      probs_acc.append(probs)
    agg = None
    if p.atten_prob_aggregation == 'mean' and probs_acc[0] is not None:
      agg = torch.stack(probs_acc).mean(0)
    return x, agg


class TransformerFeedForwardLayerWithTaskId(base_layer.BaseLayer):
  """Placeholder factory: see layers_with_attention (:7720)."""

  @classmethod
  def Params(cls):
    from lingvo_b200.core import layers_with_attention  # pylint: disable=g-import-not-at-top
    return layers_with_attention.TransformerFeedForwardLayerWithTaskId.Params()


class GPipeBatchMajorTransformerLayer(TransformerLayer):
  """TransformerLayer with the GPipe calling convention: all tensors in, all
  tensors out, so stages can be chained by `gpipe.PipeliningLayer` (:7762)."""

  def FProp(self, theta, source_vecs, source_paddings, target_vecs=None,
            target_paddings=None, encoder_self_atten_segment_mask=None,
            decoder_self_atten_segment_mask=None,
            decoder_cross_atten_segment_mask=None):
    p = self.params
    if p.has_aux_atten:
      out, _ = super().FProp(theta, target_vecs, target_paddings, source_vecs,
                             source_paddings,
                             segment_mask=decoder_self_atten_segment_mask,
                             aux_segment_mask=decoder_cross_atten_segment_mask)
      target_vecs = out
    else:
      out, _ = super().FProp(theta, source_vecs, source_paddings,
                             segment_mask=encoder_self_atten_segment_mask)
      source_vecs = out
    return (source_vecs, source_paddings, target_vecs, target_paddings,
            encoder_self_atten_segment_mask, decoder_self_atten_segment_mask,
            decoder_cross_atten_segment_mask)

  @classmethod
  def FPropMeta(cls, p, inputs, *args):
    b, t, d = inputs[0], inputs[1], inputs[2]
    ff = p.tr_fflayer_tpl.hidden_dim
    flops = b * t * (8 * d * d + 4 * t * d + 4 * d * ff)
    return NestedMap(flops=flops, out_shapes=(inputs,) + args)


class Builder(builder.Base):
  """Composition DSL for Transformer stacks (:8591). Produces the same child
  naming as the reference for the commonly used blocks."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('model_dim', 4, 'Model dim.')
    p.Define('num_heads', 1, 'Heads.')
    p.Define('ff_hidden_dim', 4, 'FFN hidden.')
    p.Define('attention_hidden_dim', None, 'Attention hidden; default model_dim.')
    p.Define('residual_dropout_prob', 0.0, 'Residual dropout.')
    p.Define('ff_activation_fn', 'RELU', 'FFN activation.')
    p.Define('ff_residual_weight', 1.0, 'FFN residual weight.')
    p.Define('relu_dropout_prob', 0.0, 'FFN hidden dropout.')
    p.Define('atten_dropout_prob', 0.0, 'Attention dropout.')
    p.Define('selfatten_add_unnormalized_input', True, 'Residual on raw input.')
    p.Define('selfatten_enable_value_proj', True, 'Value projection.')
    p.Define('conv_activation', 'RELU', 'LConv activation.')
    p.Define('num_splits', 1, 'GPipe splits.')
    p.Define('num_micro_batches', 1, 'GPipe micro-batches.')
    p.Define('glu_with_tanh', False, 'GLU variant.')
    p.Define('packed_input', False, 'Packed input.')
    p.Define('enable_per_dim_scale', True, 'Per-dim query scale.')
    p.Define('use_fused_layernorm', False, 'Kept for parity.')
    p.Define('layernorm_tpl', layers.LayerNorm.Params(), 'LN template.')
    p.Define('use_bias', True, 'Bias in projections.')
    p.Define('norm_layer_tpl', None, 'Overrides layernorm_tpl.')
    p.Define('funnel_pool_tpl', FunnelPoolingLayer.Params(), 'Funnel pooling tpl.')
    p.Define('survival_prob', 1.0, 'Stochastic depth survival.')
    p.Define('atten_tpl', MultiHeadedAttention.Params(), 'Attention template.')
    p.Define('ff_use_paddings', True, 'Zero the padded positions after the FFN.')
    p.Define('ff_apply_residual', True, 'x + f(x) (else f(x) only).')
    p.Define('num_experts', 0, 'MoE: number of experts.')
    p.Define('num_groups', 1, 'MoE: token groups.')
    p.Define('expert_capacity_dim', 0, 'MoE: fixed expert capacity (0: from the factor).')
    p.Define('expert_capacity_factor', 1.5, 'MoE: capacity = factor · S / E.')
    p.Define('moe_activation', 'RELU', 'MoE expert activation.')
    return p

  # -- leaves -------------------------------------------------------------------
  def _ExpandDims(self, name):
    return self._Fn(name, lambda x: x.unsqueeze(2))

  def _Squeeze(self, name):
    return self._Fn(name, lambda x: x.squeeze(2))

  def _Glu(self, name):
    """[gate ‖ act] halves → act · σ(gate) (tanh(act) with `glu_with_tanh`) (ref :8760)."""
    with_tanh = self.params.glu_with_tanh

    def Fn(x):
      gate, act = x.chunk(2, -1)
      return (torch.tanh(act) if with_tanh else act) * torch.sigmoid(gate)
    return self._Fn(name, Fn)

  def Seq(self, name, *subs):
    return self._Seq(name, *subs)

  def _Stride(self, name, stride, first_n=None, axis=1):
    return StrideLayer.Params().Set(name=name, stride=stride, first_n=first_n, axis=axis)

  def _Pool(self, name, stride, first_n=None):
    return self.params.funnel_pool_tpl.Copy().Set(name=name, stride=stride, first_n=first_n)

  def _DefaultLN(self, name):
    p = self.params
    return (p.norm_layer_tpl or p.layernorm_tpl).Copy().Set(
        name=name, input_dim=p.model_dim)

  def _Dropout(self, name, drop_prob):
    return layers.DropoutLayer.Params().Set(name=name, keep_prob=1.0 - drop_prob)

  def _Linear(self, name, idims, odims):
    return builder_layers.LinearLayer.Params().Set(
        name=name, input_dims=idims, output_dims=odims)

  def _Bias(self, name, dims):
    return builder_layers.BiasLayer.Params().Set(name=name, dims=dims)

  def _Activation(self, name, fn='RELU'):
    return activations.ActivationLayer.Params().Set(name=name, activation=fn)

  def _Add(self, name, residual_weight=1.0):
    return ResidualAddLayer.Params().Set(name=name, residual_weight=residual_weight)

  def _Pad(self, name):
    return PaddingLayer.Params().Set(name=name)

  def _MultiHeadedAtten(self, name, num_heads=None):
    p = self.params
    return p.atten_tpl.Copy().Set(
        name=name, input_dim=p.model_dim,
        hidden_dim=p.attention_hidden_dim or p.model_dim,
        num_heads=num_heads or p.num_heads, atten_dropout_prob=p.atten_dropout_prob,
        enable_value_proj=p.selfatten_enable_value_proj,
        enable_per_dim_scale=p.enable_per_dim_scale, packed_input=p.packed_input,
        use_bias=p.use_bias)

  # -- blocks -------------------------------------------------------------------
  def Feedforward(self, name, is_causal=False, ff_hidden_dim=None):
    del is_causal
    p = self.params
    h = ff_hidden_dim or p.ff_hidden_dim
    body = self._Seq(
        'ff',
        self._DefaultLN('ln'),
        self._Linear('linear01', p.model_dim, h),
        self._Bias('bias01', h),
        self._Activation('act', p.ff_activation_fn),
        self._Dropout('relu_dropout', p.relu_dropout_prob),
        self._Linear('linear02', h, p.model_dim),
        self._Bias('bias02', p.model_dim),
        self._Dropout('dropout', p.residual_dropout_prob))
    return self._Graph(
        name, ['i'], ['o'],
        ('i.vec->after_ff', body),
        ('i.vec,after_ff->added', self._Add('add', p.ff_residual_weight)),
        ('added,i.paddings->o.vec', self._Pad('pad')),
        ('i.paddings->o.paddings', self._Id('id')))

  def _Id(self, name):
    return layers.IdentityLayer.Params().Set(name=name)

  def GatedFeedforward(self, name, is_causal=False, ff_hidden_dim=None, activation_fn='RELU',
                       use_paddings=None):
    """LN → act(x·wi0) ⊙ (x·wi1) → wo, bias-free (T5 v1.1 / GLU-variants FFN) (ref :8880)."""
    del is_causal
    p = self.params
    use_paddings = p.ff_use_paddings if use_paddings is None else use_paddings
    h = ff_hidden_dim or p.ff_hidden_dim
    act = activations.GetFn(activation_fn) if isinstance(activation_fn, str) else activation_fn
    sub_list = [
        ('i.vec->after_gelu', self._Graph(
            'feedforward', ['x'], ['y'],
            ('x->x1', self._DefaultLN('ln')),
            ('x1->h0', self._Linear('wi0', p.model_dim, h)),
            ('x1->h1', self._Linear('wi1', p.model_dim, h)),
            ('h0,h1->h', self._Fn('gelu', lambda a, b: act(a) * b)),
            ('h->h_dropout', self._Dropout('dropout', p.relu_dropout_prob)),
            ('h_dropout->y', self._Linear('wo', h, p.model_dim)))),
        ('after_gelu->y', self._Dropout('dropout', p.residual_dropout_prob)),
        ('i.vec,y->added', ResidualAddLayer.Params().Set(
            name='add', residual_weight=p.ff_residual_weight,
            apply_residual=p.ff_apply_residual)),
    ]
    if use_paddings:
      sub_list += [('added,i.paddings->o.vec', self._Pad('pad')),
                   ('i.paddings->o.paddings', self._Id('id'))]
    else:
      sub_list += [('added->o.vec', self._Id('id_vec')),
                   ('i.paddings->o.paddings', self._Id('id'))]
    if p.packed_input:
      sub_list.append(('i.segment_mask->o.segment_mask', self._Id('segment_mask')))
    return self._Graph(name, ['i'], ['o'], *sub_list)

  def GatedGeluFeedforward(self, name, is_causal=False, ff_hidden_dim=None):
    return self.GatedFeedforward(name, is_causal, ff_hidden_dim,
                                 activation_fn='GELU_APPROXIMATE')

  def MoE(self, name, is_causal=False, ff_hidden_dim=None):
    """Sharded mixture-of-experts FFN in place of the dense one (ref :8836)."""
    del is_causal
    from lingvo_b200.core import layers_with_attention   # pylint: disable=g-import-not-at-top
    p = self.params
    assert not p.packed_input and p.num_experts > 0 and p.expert_capacity_factor >= 1.0
    moe_p = layers_with_attention.TransformerShardedMoeLayer.Params().Set(
        name=name, input_dim=p.model_dim, output_dim=p.model_dim,
        hidden_dim=ff_hidden_dim or p.ff_hidden_dim, activation=p.moe_activation,
        residual_weight=p.ff_residual_weight, residual_dropout_prob=p.residual_dropout_prob,
        relu_dropout_prob=p.relu_dropout_prob, num_groups=p.num_groups,
        expert_capacity_dim=p.expert_capacity_dim, min_group_size=None,
        num_experts=p.num_experts, expert_capacity_factor=p.expert_capacity_factor)
    if p.deterministic_dropout:
      moe_p.dropout_tpl = layers.DeterministicDropoutLayer.Params()
    return self._Graph(name, ['i'], ['o'],
                       ('i.vec,i.paddings->o.vec', moe_p),
                       ('i.paddings->o.paddings', self._Id('id')))

  # -- lightweight convolutions (https://arxiv.org/abs/1901.10430) -----------------------------
  def _NormalizedDepthwiseConv2D(self, name, kernel_size, is_causal=False, qdomain=None):
    del qdomain
    from lingvo_b200.core import conv_layers_builder   # pylint: disable=g-import-not-at-top
    p = self.params
    return conv_layers_builder.Builder.Params().Instantiate().NormalizedDepthwiseConv2D(
        name=name, kernel_size=kernel_size, num_heads=p.num_heads, in_dim=p.model_dim,
        dropconnect_prob=p.atten_dropout_prob, deterministic_dropout=p.deterministic_dropout,
        is_causal=is_causal)

  def LConv(self, name, kernel_size, is_causal=False, convolution_fn=None,
            linear_qdomain=None, conv_qdomain=None):
    """LN → linear(2D) → GLU → softmax-normalised depthwise conv over time → linear →
    dropout → residual: the self-attention replacement of "Pay Less Attention" (ref :8985)."""
    del linear_qdomain, conv_qdomain
    p = self.params
    convolution_fn = convolution_fn or self._NormalizedDepthwiseConv2D
    sub_list = [
        ('i.vec->pre_conv', self._Seq(
            'pre_conv', self._DefaultLN('ln'),
            self._Linear('linear', p.model_dim, p.model_dim * 2),
            self._Bias('bias', p.model_dim * 2), self._Glu('glu'),
            self._ExpandDims('expand'))),
        ('pre_conv,i.paddings->post_conv,o.paddings',
         convolution_fn('conv', kernel_size, is_causal)),
        ('post_conv->after_dropout', self._Seq(
            'post_conv', self._Squeeze('squeeze'),
            self._Linear('linear', p.model_dim, p.model_dim), self._Bias('bias', p.model_dim),
            self._Dropout('dropout', p.residual_dropout_prob))),
        ('i.vec,after_dropout->o.vec', self._Add('add')),
    ]
    if p.packed_input:
      sub_list.append(('i.segment_mask->o.segment_mask', self._Id('segment_mask')))
    return self._Graph(name, ['i'], ['o'], *sub_list)

  def LconvBlock(self, name, kernel_size, is_causal, convolution_fn):
    return self._Seq(name,
                     self.LConv('lconv', kernel_size, is_causal, convolution_fn),
                     self.Feedforward('ff', is_causal))

  def LConvStack(self, name, kernel_sizes, is_causal=False):
    blocks = [self.LconvBlock('block_{}'.format(i), k, is_causal, None)
              for i, k in enumerate(kernel_sizes)]
    return self._MaybeSplit(name, blocks) or self._Seq(name, *blocks)

  def _MaybeSplit(self, name, blocks):
    """With `num_splits` / `num_micro_batches` > 1 the blocks become GPipe cells."""
    p = self.params
    if p.num_splits == 1 and p.num_micro_batches == 1:
      return None
    from lingvo_b200.core import gpipe   # pylint: disable=g-import-not-at-top
    assert len(blocks) >= p.num_splits
    per = (len(blocks) - 1) // p.num_splits + 1
    cells = [self._Seq('cell_{}'.format(i // per), *blocks[i:i + per])
             for i in range(0, len(blocks), per)]
    assert len(cells) == p.num_splits
    return gpipe.PipeliningLayer.Params().Set(
        name=name, cell_tpl=cells, nested_map_fprop=True,
        num_micro_batches=p.num_micro_batches)

  def FunnelEncoderLayer(self, name, stride=1, first_n=None, ff_hidden_dim=None,
                         num_heads=None):
    """Funnel-Transformer block (ref :9290): the query (and the shortcut) is pooled by
    `stride`, keys / values stay at full resolution; then a feed-forward block."""
    p = self.params
    tr = FunnelTransformerAttentionAdapter.Params().Set(
        name='self_atten', stride=stride, first_n=first_n,
        pool=self._Pool('pool', stride, first_n), ln=self._DefaultLN('LN'),
        atten=self._MultiHeadedAtten('atten', num_heads),
        dropout=self._Dropout('dropout', p.residual_dropout_prob),
        add_unnormalized_input=p.selfatten_add_unnormalized_input)
    return self._Seq(name, tr, self.Feedforward('ff', False, ff_hidden_dim))

  def SelfAttention(self, name, is_causal=False, num_heads=None):
    p = self.params
    tr = TransformerAttentionLayer.Params().Set(
        name=name, input_dim=p.model_dim,
        hidden_dim=p.attention_hidden_dim or p.model_dim,
        num_heads=num_heads or p.num_heads, is_masked=is_causal,
        atten_dropout_prob=p.atten_dropout_prob,
        residual_dropout_prob=p.residual_dropout_prob,
        add_unnormalized_input=p.selfatten_add_unnormalized_input,
        ln_tpl=(p.norm_layer_tpl or p.layernorm_tpl).Copy(),
        atten_tpl=self._MultiHeadedAtten('atten', num_heads))
    return _SelfAttenAdapter.Params().Set(name=name, body=tr)

  def TransformerEncoderLayer(self, name, is_causal=False, ff_hidden_dim=None,
                              num_heads=None):
    return self._Seq(name,
                     self.SelfAttention('self_atten', is_causal, num_heads),
                     self.Feedforward('ff', is_causal, ff_hidden_dim))

  def TransformerEncoderStack(self, name, num_layers, is_causal=False):
    return self._Seq(name, *[
        self.TransformerEncoderLayer('iter_%03d' % i, is_causal)
        for i in range(num_layers)])

  Stack = TransformerEncoderStack


class FunnelTransformerAttentionAdapter(base_layer.BaseLayer):
  """NestedMap(vec, paddings) → NestedMap at 1/stride of the time resolution: pooled
  queries attend to the full-resolution normalised input; residual on the pooled input."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('stride', 1, 'Pooling stride of the query.')
    p.Define('first_n', None, 'Only the first n positions are pooled / output.')
    p.Define('pool', None, 'FunnelPoolingLayer params.')
    p.Define('ln', None, 'LayerNorm params.')
    p.Define('atten', None, 'MultiHeadedAttention params.')
    p.Define('dropout', None, 'Dropout params.')
    p.Define('add_unnormalized_input', True, 'Residual on the raw (pooled) input.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    for n in ('pool', 'ln', 'atten', 'dropout'):
      self.CreateChild(n, p.Get(n))

  def FProp(self, theta, i):
    p = self.params
    after_ln = self.ln.FProp(theta.ln, i.vec)
    query, out_pad = self.pool.FProp(theta.pool, after_ln, i.paddings)
    ctx, _ = self.atten.FProp(theta.atten, query, after_ln, after_ln, i.paddings)
    ctx = self.dropout.FProp(theta.dropout, ctx)
    if p.add_unnormalized_input:
      shortcut, _ = self.pool.FProp(theta.pool, i.vec, i.paddings)
    else:
      shortcut = query
    return NestedMap(vec=shortcut + ctx, paddings=out_pad)


class _SelfAttenAdapter(base_layer.BaseLayer):
  """NestedMap(vec, paddings[, segment_mask]) in/out wrapper used by Builder."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('body', None, 'TransformerAttentionLayer params.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self.CreateChild('atten', self.params.body)

  def FProp(self, theta, i):
    out, _ = self.atten.FProp(theta.atten, i.vec, None, i.paddings,
                              segment_mask=i.get('segment_mask'))
    ret = NestedMap(vec=out, paddings=i.paddings)
    if 'segment_mask' in i:
      ret.segment_mask = i.segment_mask
    return ret


class LmBuilder(Builder):
  """Decoder-only stack: every layer causal (:9883)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('xla_num_partitions', None, 'Kept for parity.')
    p.Define('dtype', torch.float32, 'Weights dtype.')
    return p

  def TransformerEncoderLayer(self, name, is_causal=True, ff_hidden_dim=None,
                              num_heads=None):
    return super().TransformerEncoderLayer(name, True, ff_hidden_dim, num_heads)

  def TransformerEncoderStack(self, name, num_layers, is_causal=True):
    return super().TransformerEncoderStack(name, num_layers, True)


def TransformerFlops(inputs_shape, num_heads, ff_dim, atten_dim, model_dim):
  """FLOPs of one TransformerLayer FProp on `[B, T, D]` (:6778)."""
  del num_heads
  b, t = inputs_shape[0], inputs_shape[1]
  proj = 2 * 4 * b * t * model_dim * atten_dim
  attn = 2 * 2 * b * t * t * atten_dim
  ff = 2 * 2 * b * t * model_dim * ff_dim
  return proj + attn + ff


# ==================================================================================
# Sub-quadratic / structured attention variants (long-context toolbox, SURVEY §5.7)
# ==================================================================================
class ChunkwiseSelfAttentionXL(ChunkwiseSelfAttention):
  """Chunk-wise attention + Transformer-XL relative term (reference :4318)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('rel_pos_emb_dim', None, 'Sinusoid embedding dim.')
    p.Define('skip_term_b', False, 'Drop the position term.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.rel_pos_emb_dim and p.rel_pos_emb_dim > 0
    self.CreateChild('pos_proj', p.proj_tpl.Copy().Set(
        input_dim=p.rel_pos_emb_dim, num_heads=p.num_heads,
        dim_per_head=self.dim_per_head, use_bias=False))

  def _CreateLayerVariables(self):
    super()._CreateLayerVariables()
    p = self.params
    shape = [p.num_heads, self.dim_per_head]
    coll = [self.__class__.__name__ + '_vars']
    self.CreateVariable('u', WeightParams(shape, WeightInit.Constant(0.0), p.dtype, coll))
    self.CreateVariable('v', WeightParams(shape, WeightInit.Constant(0.0), p.dtype, coll))

  _RelativeBias = MultiHeadedAttentionXL._RelativeBias


class MultiHeadedFavorAttention(MultiHeadedAttention):
  """Performer (FAVOR+) attention: O(L) softmax-kernel approximation (reference :2125).

  `attention_type`: 'softmax' (positive random features), 'relu' (deterministic) or
  'cossim'. Probabilities are never formed, so `probs` is None. `causal` selects the
  prefix-sum form (the reference only exposes the bidirectional one).
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_random_features', 384, 'Random projection features.')
    p.Define('attention_type', 'softmax', 'relu|softmax|cossim.')
    p.Define('redraw', False, 'Redraw the random features at every call.')
    p.Define('causal', False, 'Causal (prefix-sum) FAVOR.')
    return p

  def __init__(self, params):
    super().__init__(params)
    assert not self.params.packed_input, 'Packed input not supported.'
    self._proj = None
    self._draws = 0

  def _Projection(self, dim, device):
    from lingvo_b200.core import favor_attention as favor  # pylint: disable=g-import-not-at-top
    p = self.params
    if p.redraw or self._proj is None or self._proj.device != device:
      seed = self._draws if p.redraw else 0
      self._draws += 1
      self._proj = favor.create_projection_matrix(p.num_random_features, dim, seed=seed).to(device)
    return self._proj

  def FProp(self, theta, query_vec, key_vec, value_vec, paddings,
            segment_mask=None, per_step_padding=None):
    from lingvo_b200.core import favor_attention as favor  # pylint: disable=g-import-not-at-top
    p = self.params
    q, k, v = self._HeadsProj(theta, query_vec, key_vec, value_vec)
    q = self._RoPE(theta, q)
    k = self._RoPE(theta, k)
    if p.enable_query_scale and p.enable_per_dim_scale:
      q = self.per_dim_scale.FProp(theta.per_dim_scale, q)
    n = q.shape[2]
    k, v = attention_ops._ExpandKv(k, n), attention_ops._ExpandKv(v, n)  # pylint: disable=protected-access
    qf, kf, vf = q.float(), k.float(), v.float()
    if p.attention_type == 'relu':
      ctx = favor.favor_attention(qf, kf, vf, paddings, favor.relu_kernel_transformation,
                                  p.causal)
    elif p.attention_type == 'softmax':
      ctx = favor.favor_attention(qf, kf, vf, paddings, favor.softmax_kernel_transformation,
                                  p.causal, self._Projection(q.shape[-1], q.device))
    elif p.attention_type == 'cossim':
      proj = self._Projection(q.shape[-1], q.device)
      kp = favor.cossim_kernel_transformation(kf, False, proj)
      qp = favor.cossim_kernel_transformation(qf, True, proj)
      scores = torch.einsum('BXHD,BYHD->BXYH', qp, kp)
      if paddings is not None:
        scores = scores + (paddings.float() * GetDtypeMin()).view(
            paddings.shape[0], 1, -1, 1)
      ctx = torch.einsum('BXYH,BYHD->BXHD', torch.softmax(scores, dim=2), vf)
    else:
      raise ValueError('FAVOR attention type %s is not supported' % p.attention_type)
    return self._PostProj(theta, ctx.to(v.dtype)), None


class RoutingAttention(MultiHeadedAttention):
  """Sparse attention by online k-means routing (Routing Transformer; reference :4458).

  Queries and keys are layer-normalised and assigned to `num_clusters` centroids per head
  (`attention_util.KMeansClusteringForAtten`, EMA-updated while training). A query only
  attends to the `attention_window` keys closest to *its* centroid: O(T·W) instead of
  O(T·S). `causal_masking` additionally hides keys at later positions.
  """

  @classmethod
  def Params(cls):
    from lingvo_b200.core import attention_util  # pylint: disable=g-import-not-at-top
    p = super().Params()
    p.Define('num_clusters', 0, 'Clusters per head (≈ sqrt(sequence length)).')
    p.Define('attention_window', 0, 'Keys each query attends to.')
    p.Define('clustering', attention_util.KMeansClusteringForAtten.Params(), 'k-means tpl.')
    p.Define('causal_masking', False, 'Position idx only sees positions <= idx.')
    p.Define('fast_path', True, 'Kept for parity (one gather-based implementation).')
    p.Define('query_group_size_factor', 1.2, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.num_clusters and p.attention_window
    assert not p.packed_input
    self.CreateChild('clustering', p.clustering.Copy().Set(
        num_clusters=p.num_clusters, num_heads=p.num_heads,
        dim_per_head=self.dim_per_head, apply_layer_norm=False))
    self._clustering_loss = None

  @property
  def clustering_loss(self):
    return self._clustering_loss

  def FProp(self, theta, query_vec, key_vec, value_vec, paddings,
            segment_mask=None, per_step_padding=None, query_paddings=None):
    from lingvo_b200.core import attention_util  # pylint: disable=g-import-not-at-top
    p = self.params
    q, k, v = self._HeadsProj(theta, query_vec, key_vec, value_vec)
    n = q.shape[2]
    k, v = attention_ops._ExpandKv(k, n), attention_ops._ExpandKv(v, n)  # pylint: disable=protected-access
    h = q.shape[-1]
    # Euclidean closeness must imply a large dot product: normalise both sides.
    qn = F.layer_norm(q.float(), (h,))
    kn = F.layer_norm(k.float(), (h,))
    b, t = q.shape[0], q.shape[1]
    s = k.shape[1]
    q_dists, q_loss = self.clustering.FProp(theta.clustering, qn, query_paddings,
                                            update=not self.do_eval)
    k_dists, k_loss = self.clustering.FProp(theta.clustering, kn, paddings,
                                            update=not self.do_eval)
    self._clustering_loss = q_loss + k_loss
    # keys never selectable when padded
    if paddings is not None:
      k_dists = k_dists + paddings.float().view(b, s, 1, 1) * 1e6
    w = min(p.attention_window, s)
    # closest W keys of every (head, cluster): [B, N, K, W]
    top = torch.topk(-k_dists.permute(0, 2, 3, 1), w, dim=-1).indices
    q_cluster = q_dists.argmin(-1)                               # [B, T, N]
    idx = torch.gather(top, 2, q_cluster.permute(0, 2, 1).unsqueeze(-1).expand(b, n, t, w))
    if p.causal_masking:
      pos = torch.arange(t, device=q.device).view(1, 1, t, 1)
      idx = torch.where(idx <= pos, idx, torch.full_like(idx, -1))
    qs = qn.permute(0, 2, 1, 3)
    ctx, probs = attention_util.ComputeSparseAttention(
        qs, kn.permute(0, 2, 1, 3), v.float().permute(0, 2, 1, 3), idx, paddings)
    ctx = ctx.permute(0, 2, 1, 3).to(v.dtype)
    return self._PostProj(theta, ctx), probs


class FunnelTransformerAttentionLayer(TransformerAttentionLayer):
  """Self-attention whose *queries* are pooled first (Funnel-Transformer; reference :5943):
  `[B, T, D]` in, `[B, T/stride, D]` out, keys/values at full resolution."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('query_pooling_tpl', FunnelPoolingLayer.Params(), 'Pooling of the queries.')
    p.Define('begin_intact', 0, 'Leading positions (e.g. [CLS]) kept un-pooled.')
    p.Define('trunc_seq', True, 'Truncate so that the length divides the stride.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('query_pooling', p.query_pooling_tpl.Copy().Set(
        begin_intact=p.begin_intact, trunc_seq=p.trunc_seq))

  def FProp(self, theta, query_vec, source_vecs, paddings,
            per_step_padding_override=None, segment_mask=None):
    p = self.params
    assert source_vecs is None, 'funnel attention is self-attention'
    normed = self._Norm(theta, query_vec) if p.pre_layer_norm else query_vec
    pooled, pooled_paddings = self.query_pooling.FProp(theta.query_pooling, normed, paddings)
    res_in, _ = self.query_pooling.FProp(theta.query_pooling, query_vec, paddings)
    ctx, probs = self.atten.FProp(theta.atten, pooled, normed, normed, paddings,
                                  segment_mask=segment_mask,
                                  per_step_padding=per_step_padding_override)
    return self._Finish(theta, res_in, pooled, ctx), probs, pooled_paddings


class MemoryAddLayer(base_layer.BaseLayer):
  """Adds a learned (or supplied) memory bank in front of a sequence (reference
  `MemoryAddLayer`, used by the sketch-memory builder): `[B, T, D]` → `[B, M + T, D]`."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_dim', 0, 'Model dim.')
    p.Define('num_memory_slots', 0, 'M.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('memory', WeightParams(
        [p.num_memory_slots, p.input_dim], WeightInit.Gaussian(p.input_dim**-0.5), p.dtype))

  def FProp(self, theta, inputs, paddings=None):
    b = inputs.shape[0]
    mem = theta.memory.to(inputs.dtype).unsqueeze(0).expand(b, -1, -1)
    out = torch.cat([mem, inputs], 1)
    if paddings is None:
      return out
    pad = torch.cat([torch.zeros(b, mem.shape[1], dtype=paddings.dtype,
                                 device=paddings.device), paddings], 1)
    return out, pad


class PerformerBuilder(Builder):
  """`Builder` whose self-attention is FAVOR+ (reference `PerformerBuilder`)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_random_features', 384, 'Random features.')
    p.Define('attention_type', 'softmax', 'relu|softmax|cossim.')
    return p

  def _MultiHeadedAtten(self, name, num_heads=None):
    p = self.params
    return MultiHeadedFavorAttention.Params().Set(
        name=name, input_dim=p.model_dim, hidden_dim=p.attention_hidden_dim or p.model_dim,
        num_heads=num_heads or p.num_heads, num_random_features=p.num_random_features,
        attention_type=p.attention_type, use_bias=p.use_bias,
        enable_per_dim_scale=p.enable_per_dim_scale, return_atten_probs=False)

  def SelfAttention(self, name, is_causal=False, num_heads=None):
    """FAVOR has no [T, S] mask: causality is the prefix-sum form of the kernel."""
    adapter = super().SelfAttention(name, False, num_heads)
    adapter.body.atten_tpl.causal = is_causal
    return adapter


class SketchMemTransformerBuilder(Builder):
  """Transformer whose layers read a small learned sketch memory in addition to the
  sequence (reference `SketchMemTransformerBuilder`): memory slots are prepended once and
  every layer attends over [memory; tokens]."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_memory_slots', 16, 'Sketch memory size M.')
    return p

  def MemoryAdd(self, name):
    return MemoryAddLayer.Params().Set(name=name, input_dim=self.params.model_dim,
                                       num_memory_slots=self.params.num_memory_slots)

  def TransformerEncoderStack(self, name, num_layers, is_causal=False):
    """[memory; tokens] → layers → tokens (memory slots are dropped at the end)."""
    body = super().TransformerEncoderStack('body', num_layers, is_causal)
    return _SketchMemStack.Params().Set(name=name, memory=self.MemoryAdd('memory'), body=body,
                                        num_memory_slots=self.params.num_memory_slots)

  Stack = TransformerEncoderStack


class _SketchMemStack(base_layer.BaseLayer):
  """NestedMap(vec, paddings) → same, running `body` over [memory; tokens]."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('memory', None, 'MemoryAddLayer params.')
    p.Define('body', None, 'Stack params.')
    p.Define('num_memory_slots', 0, 'M.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self.CreateChild('memory', self.params.memory)
    self.CreateChild('body', self.params.body)

  def FProp(self, theta, i):
    vec, pad = self.memory.FProp(theta.memory, i.vec, i.paddings)
    o = self.body.FProp(theta.body, NestedMap(vec=vec, paddings=pad))
    m = self.params.num_memory_slots
    return NestedMap(vec=o.vec[:, m:], paddings=o.paddings[:, m:])


class _PipelineStageAdapter(base_layer.BaseLayer):
  """NestedMap(vec, paddings[, segment_mask]) in/out around a `StackedTransformerLayers`
  stage, so the shifting-buffer pipeline can carry the side inputs with the activations."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('stage', None, 'StackedTransformerLayers params.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self.CreateChild('stage', self.params.stage)

  def FProp(self, theta, i):
    vec, pad = self.stage.FProp(theta.stage, i.vec, i.paddings,
                                segment_mask=i.get('segment_mask'))
    o = NestedMap(vec=vec, paddings=pad)
    if 'segment_mask' in i:
      o.segment_mask = i.segment_mask
    return o


class PipelinedTransformerLayers(base_layer.BaseLayer):
  """`num_pipeline_stages` (× `circular_repeat`) `StackedTransformerLayers` stages run
  through `gshard_layers.LayerwiseShardablePipelinedLayer` (reference :7512): micro-batches
  flow through a shifting buffer; with `AttachStageGroup` each rank holds one stage."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('pipeline_stage', StackedTransformerLayers.Params(), 'Params of each stage.')
    p.Define('num_pipeline_stages', None, 'Number of pipeline stages.')
    p.Define('num_pipeline_microbatches', None, 'Number of micro-batches.')
    p.Define('pipeline_microbatch_size', None, 'Size of each micro-batch.')
    p.Define('shard_stages_1d', False, 'One stage per rank (see `stage_group`).')
    p.Define('final_layer_norm', False, 'LN after all stages.')
    p.Define('final_ln_at_each_stage', False, 'LN at the end of each stage instead.')
    p.Define('circular_repeat', 1, 'Circular pipeline repeats.')
    p.Define('pipeline_stage_mesh_dim', None, 'Kept for parity.')
    p.Define('unroll', 'never', 'Kept for parity.')
    return p

  def __init__(self, params, stage_group=None):
    super().__init__(params)
    from lingvo_b200.core import gshard_layers  # pylint: disable=g-import-not-at-top
    p = self.params
    assert p.num_pipeline_stages and p.num_pipeline_stages > 0
    stage = p.pipeline_stage.Copy().Set(name='stage')
    stage.final_layer_norm = bool(p.final_ln_at_each_stage)
    pp = gshard_layers.LayerwiseShardablePipelinedLayer.Params().Set(
        name='pipeline', num_stages=p.num_pipeline_stages,
        single_stage_body=_PipelineStageAdapter.Params().Set(name='body', stage=stage),
        num_microbatches=p.num_pipeline_microbatches,
        microbatch_size=p.pipeline_microbatch_size, circular_repeat=p.circular_repeat)
    if p.shard_stages_1d and stage_group is not False:
      import torch.distributed as dist  # pylint: disable=g-import-not-at-top
      if dist.is_available() and dist.is_initialized() and (
          dist.get_world_size(stage_group) == p.num_pipeline_stages):
        self.AddChild('pipeline', gshard_layers.LayerwiseShardablePipelinedLayer.ForStageGroup(
            pp, stage_group))
    if 'pipeline' not in self.children:
      self.CreateChild('pipeline', pp)
    if p.final_layer_norm:
      self.CreateChild('final_ln', p.pipeline_stage.layernorm_tpl.Copy().Set(
          input_dim=p.pipeline_stage.mdl_dim))

  def FProp(self, theta, query_vec, paddings, aux_vec=None, aux_paddings=None,
            segment_mask=None, aux_segment_mask=None):
    p = self.params
    assert aux_vec is None, 'pipelined cross attention is not supported'
    inp = NestedMap(vec=query_vec, paddings=paddings)
    if segment_mask is not None:
      inp.segment_mask = segment_mask
    out = self.pipeline.FProp(theta.pipeline, inp)
    x = out.vec
    if p.final_layer_norm:
      x = self.final_ln.FProp(theta.final_ln, x)
    return x, out.paddings
