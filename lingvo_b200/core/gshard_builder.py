"""GShard builders (`MoEBuilder`, `DenseBuilder`) and the `UniTransformer` LM.

Reference `lingvo/core/gshard_builder.py` (5375 LoC): builder params
(:55-330, :2269-2330), `DecoderLayer` (:558-666), `DecoderLayerStack`
(:675-906), attention (`_AttentionWeights :1973`, `Attention :2697`,
`_ComputeQKVCombine :2819`, `_ComputeAttenOutputs :2908`, T5 relative bias
:1431-1514, RoPE :409-426), norms (`_LN` RMS :1833, `_TrueLN :1856`, `_PN`),
FFN (`DenseReluDense :2939`, gated :3054), MoE (`MoE :2465`,
`_ShardedFeedForwardNetworksWeights :2484`, gating weights), embedding
(:457-466, :2550), and `UniTransformer` (:3939-4483).

Re-design: the reference composes every block from a string-signature graph
DSL and relies on XLA to fuse/shard it. Here each block is an explicit layer
class whose `FProp` calls the fused sm_90a kernels directly (RMS-norm,
wgmma GEMM w/ fused epilogues, index-based MoE dispatch/combine, fused
xent), and whose collectives are explicit (`lingvo_b200.parallel`). The
builder API (method names, params, sub-layer type lists) is kept so
experiment configs port 1:1.
"""

from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from lingvo_b200 import ops
from lingvo_b200.core import activations
from lingvo_b200.core import base_layer
from lingvo_b200.core import base_model
from lingvo_b200.core import builder
from lingvo_b200.core import gshard_layers
from lingvo_b200.core import gshard_utils
from lingvo_b200.core import layers
from lingvo_b200.core import py_utils
from lingvo_b200.core import summary_utils
from lingvo_b200.core.nested_map import NestedMap

WeightParams = py_utils.WeightParams
WeightInit = py_utils.WeightInit


def ShardedWeightParams(shape, init=None, dtype=None, collections=None,
                        tensor_split_dims_mapping=None, device_mesh=None):
  return WeightParams(shape, init, dtype, collections, device_mesh,
                      tensor_split_dims_mapping)


def _Act(name: str):
  n = name.upper()
  if n in ('GELU',):
    return lambda x: F.gelu(x, approximate='tanh')
  if n in ('SQR_RELU',):
    return lambda x: torch.square(F.relu(x))
  return activations.GetFn(n)


def _ContextParallel(b) -> bool:
  """Context parallelism requested by the builder and a process group to run it on."""
  if not ('context_parallel' in b and b.context_parallel):
    return False
  import torch.distributed as dist   # pylint: disable=g-import-not-at-top
  return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


# =========================================================================
# Layer classes
# =========================================================================
def KLDiv(f_old, f_new):
  """KL(f_old ‖ f_new) of two probability tensors `[B, L, D]`, summed and divided by the
  batch size (ref :32; distillation between an old and a new gating / feature
  distribution)."""
  eps = 1e-7
  p = f_old.float().clamp(eps, 1.0)
  q = f_new.float().clamp(eps, 1.0)
  return (p * torch.log(p / q)).sum() / f_old.shape[0]


class _BuilderLayer(base_layer.BaseLayer):
  """Base of builder-produced layers; carries the builder params."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('b', None, 'Builder params (shared hyper-parameters).')
    return p

  @property
  def bp(self):
    return self.params.b

  def _TensorParallel(self, split, dim):
    """The tensor-parallel context if `split[dim]` puts that weight dim on the model axis
    (mesh axis 1) of a [dp, tp] device mesh and the job runs with tp_size > 1; else None."""
    from lingvo_b200.parallel import mesh as mesh_lib   # pylint: disable=g-import-not-at-top
    b = self.bp
    if 'device_mesh_shape' in b:
      mesh_lib.ConfigureFromMeshShape(b.device_mesh_shape)
    ctx = mesh_lib.TensorParallel()
    if ctx is None or split is None or len(split) <= dim or split[dim] != 1:
      return None
    return ctx

  def _TagTpVars(self, names_dims):
    """Tags `{var name: (sharded dim, logical size)}` after instantiation."""
    from lingvo_b200.parallel import tp_layers   # pylint: disable=g-import-not-at-top
    for n, (dim, logical) in names_dims.items():
      if n in self._private_vars:
        tp_layers.MarkSharded(self._private_vars[n], self._tp, dim, logical)


def _CommonFrom(parent_params, p, name):
  """Child params inheriting the builder handle and dtypes of `parent_params`."""
  p.name = name
  p.b = parent_params.b
  p.dtype = parent_params.dtype
  p.fprop_dtype = parent_params.fprop_dtype
  return p


class RmsNormLayer(_BuilderLayer):
  """Bias-less RMS "layer norm" `x·rsqrt(mean(x²)+eps)·scale` (:1833-1854)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('dim', 0, 'Model dim.')
    p.Define('epsilon', 1e-6, 'Epsilon.')
    p.Define('no_scale', False, 'No learned scale (`_LNNoScale`).')
    p.Define('kind', 'rms', 'rms|true_ln|pn|none.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    if p.kind == 'none' or (p.no_scale and p.kind == 'rms'):
      return
    self.CreateVariable('scale', WeightParams([p.dim], WeightInit.Constant(1.0),
                                              p.dtype))
    if p.kind == 'true_ln':
      self.CreateVariable('shift', WeightParams(
          [p.dim], WeightInit.Constant(0.0), p.dtype))

  def FPropPass(self, theta, x):
    """→ (norm(x), x_pass). `x_pass` is x routed through the same autograd node as the norm,
    so `x_pass + f(norm(x))` back-propagates with the residual-gradient add fused into the
    norm backward kernel (ops/norm.py `_NormPassFn`). Falls back to (FProp(x), x)."""
    p = self.params
    if (p.kind == 'rms' and ops.use_cuda_kernels(x) and x.dtype == torch.bfloat16 and
        x.requires_grad):
      from lingvo_b200.ops import norm
      return norm.rms_norm_pass(x, None if p.no_scale else theta.scale, p.epsilon)
    return self.FProp(theta, x), x

  def FProp(self, theta, x):
    p = self.params
    if p.kind == 'none':
      return x
    if p.kind == 'rms':
      scale = None if p.no_scale else theta.scale
      if ops.use_cuda_kernels(x) and x.dtype == torch.bfloat16:
        from lingvo_b200.ops import norm
        return norm.rms_norm(x, scale, p.epsilon)
      xf = x.float()
      y = xf * torch.rsqrt(xf.square().mean(-1, keepdim=True) + p.epsilon)
      if scale is not None:
        y = y * scale.float()
      return y.to(x.dtype)
    xf = x.float()
    if p.kind == 'true_ln':
      c = xf - xf.mean(-1, keepdim=True)
      y = c * torch.rsqrt(c.square().mean(-1, keepdim=True) + p.epsilon)
      return (y * theta.scale.float() + theta.shift.float()).to(x.dtype)
    if p.kind == 'pn':   # power norm: mean |x| based
      y = xf / (xf.abs().mean(-1, keepdim=True) + p.epsilon)
      return (y * theta.scale.float()).to(x.dtype)
    raise ValueError(p.kind)


class _EmbedRows(torch.autograd.Function):
  """out[i] = w[ids[i]]; d_w = sum of d_out rows per id, accumulated in fp32 in a fixed
  (sorted-index) order, so duplicate tokens give the same gradient on every run."""

  @staticmethod
  def forward(ctx, w, ids):
    flat = ids.reshape(-1)
    ctx.save_for_backward(flat)
    ctx.w_shape, ctx.w_dtype = w.shape, w.dtype
    return w.index_select(0, flat).reshape(*ids.shape, w.shape[1])

  @staticmethod
  def backward(ctx, dy):
    (flat,) = ctx.saved_tensors
    dw = torch.zeros(ctx.w_shape, dtype=torch.float32, device=dy.device)
    # index_put_(accumulate=True) sorts the indices on CUDA: duplicate ids are summed in a
    # fixed order, so the gradient is the same on every run (index_add_ uses atomics).
    dw.index_put_((flat,), dy.reshape(-1, dy.shape[-1]).float(), accumulate=True)
    return dw.to(ctx.w_dtype), None


class EmbeddingLayer(_BuilderLayer):
  """`w.embedding [V, M]`; gather lookup (reference one-hot einsum :457)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_dim', 0, 'Vocabulary size.')
    p.Define('model_dim', 0, 'Model dim.')
    p.Define('scale_by_dim', False, 'Multiply by sqrt(model_dim).')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('embedding', ShardedWeightParams(
        [p.vocab_dim, p.model_dim], WeightInit.Gaussian(), p.dtype,
        tensor_split_dims_mapping=p.b.emb_w_split if p.b else None))

  def FProp(self, theta, ids):
    p = self.params
    if theta.embedding.is_cuda:
      out = _EmbedRows.apply(theta.embedding, ids.long())
    else:
      out = F.embedding(ids.long(), theta.embedding)
    if p.scale_by_dim:
      out = out * (p.model_dim**0.5)
    return out


def RelativePositionBucket(relative_position, num_buckets, max_distance,
                           bidirectional=False):
  """T5 bucketing of `key_pos - query_pos` (reference :1431-1456)."""
  ret = 0
  n = -relative_position
  if bidirectional:
    num_buckets //= 2
    ret = (n < 0).to(torch.int32) * num_buckets
    n = n.abs()
  else:
    n = n.clamp(min=0)
  max_exact = num_buckets // 2
  is_small = n < max_exact
  large = max_exact + (torch.log(n.float().clamp(min=1) / max_exact) /
                       math.log(max_distance / max_exact) *
                       (num_buckets - max_exact)).to(torch.int32)
  large = large.clamp(max=num_buckets - 1)
  return ret + torch.where(is_small, n.to(torch.int32), large)


class _BucketGather(torch.autograd.Function):
  """table[h, i] = w[h, bucket[i]]; d_w[h, k] = Σ_{i: bucket[i]=k} d_table[h, i]."""

  @staticmethod
  def forward(ctx, w, bucket):
    ctx.save_for_backward(bucket)
    ctx.nb = w.shape[1]
    return w.index_select(1, bucket)

  @staticmethod
  def backward(ctx, dt):
    (bucket,) = ctx.saved_tensors
    # Summed in a fixed order (sorted indices), unlike index_add_'s atomics.
    dw = torch.zeros(ctx.nb, dt.shape[0], dtype=dt.dtype, device=dt.device)
    dw.index_put_((bucket,), dt.t(), accumulate=True)
    return dw.t(), None


class SelfAttentionLayer(_BuilderLayer):
  """Decoder/encoder self-attention in `BLHD` layout (:1249-1700, :2697).

  Weights `w.{wq,wk,wv,wo}` are `[M, H·D]`/`[H·D, M]` (combine_dims) and
  `wrb [H, buckets]` for the T5 relative bias. Logits are fp32; masking uses
  packed `segment_id`/`segment_pos` (+ causal for decoders); MQA via
  `attention_num_memory_heads == 1`.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('decoder', True, 'Causal (decoder) masking.')
    p.Define('relative_bias', False, 'Use T5 relative attention bias.')
    p.Define('multi_dconv_head', False,
             'Primer multi-dconv-head attention (ref :1349): a 3-tap causal depthwise '
             'convolution over time on each of q, k, v after the projections.')
    return p

  def __init__(self, params):
    super().__init__(params)
    b = self.bp
    # Heads on the model axis (`mhd_w_split = [0, 1, -1]`, ref :2806-2851): every TP rank owns
    # H/tp heads — wq/wk/wv column-parallel, wo row-parallel, one all-reduce per direction.
    self._tp = self._TensorParallel(b.mhd_w_split if 'mhd_w_split' in b else None, 1)
    if self._tp is not None:
      h = b.attention_num_heads
      hk = b.attention_num_memory_heads or h
      assert h % self._tp.tp_size == 0 and hk % self._tp.tp_size == 0, (
          'tensor parallelism needs heads (%d, kv %d) divisible by tp_size %d' %
          (h, hk, self._tp.tp_size))

    if self.params.multi_dconv_head:
      assert self._tp is None, 'multi-dconv-head attention is not tensor-parallel yet'
      hh, hk2, dd = b.attention_num_heads, (b.attention_num_memory_heads or
                                            b.attention_num_heads), b.attention_key_value_dim
      for nm, heads in (('q_dconv', hh), ('k_dconv', hk2), ('v_dconv', hk2)):
        self.CreateChild(nm, _CommonFrom(
            self.params, DepthwiseConvAutoregressiveLayer.Params().Set(
                kernel_size=3, model_dims=[heads, dd]), nm))

  def _LocalHeads(self):
    b = self.bp
    h = b.attention_num_heads
    hk = b.attention_num_memory_heads or h
    if self._tp is None:
      return h, hk
    return h // self._tp.tp_size, hk // self._tp.tp_size

  def _CreateLayerVariables(self):
    b = self.bp
    h, d, m = b.attention_num_heads, b.attention_key_value_dim, b.model_dim
    hk = b.attention_num_memory_heads or h
    hl, hkl = self._LocalHeads()
    q_std = (m * d)**-0.5
    tp = self._tp

    def Shard(wp, dim):
      if tp is not None:
        wp.init_shard = (dim, tp.tp_rank, tp.tp_size)
      return wp

    self.CreateVariable('wq', Shard(ShardedWeightParams(
        [m, hl * d], WeightInit.Gaussian(q_std), self.params.dtype), 1))
    self.CreateVariable('wk', Shard(ShardedWeightParams(
        [m, hkl * d], WeightInit.Gaussian(m**-0.5), self.params.dtype), 1))
    self.CreateVariable('wv', Shard(ShardedWeightParams(
        [m, hkl * d], WeightInit.Gaussian(m**-0.5), self.params.dtype), 1))
    self.CreateVariable('wo', Shard(ShardedWeightParams(
        [hl * d, m], WeightInit.Gaussian((h * d)**-0.5), self.params.dtype), 0))
    if self.params.relative_bias:
      self.CreateVariable('wrb', Shard(WeightParams(
          [hl, b.relative_attention_num_buckets], WeightInit.Gaussian(1.0),
          self.params.dtype), 0))

  def _InstantiateSelfAndChildren(self):
    super()._InstantiateSelfAndChildren()
    if self._tp is not None:
      b = self.bp
      h, d = b.attention_num_heads, b.attention_key_value_dim
      hk = b.attention_num_memory_heads or h
      self._TagTpVars({'wq': (1, h * d), 'wk': (1, hk * d), 'wv': (1, hk * d),
                       'wo': (0, h * d), 'wrb': (0, h)})

  _MASK_CACHE = {}

  def _Mask(self, segment_id, segment_pos, dtype):
    """Additive visibility mask `[B, 1, L, L]`, shared by all layers of a step."""
    b = self.bp
    key = (segment_id.data_ptr(), segment_pos.data_ptr(), tuple(segment_id.shape),
           dtype, self.params.decoder, segment_id._version)
    hit = SelfAttentionLayer._MASK_CACHE.get('k')
    if hit is not None and hit[0] == key:
      return hit[1]
    a, c = segment_id.unsqueeze(-1), segment_id.unsqueeze(-2)
    not_vis = ((a == 0) & (c == 0)) | (a != c)
    if self.params.decoder and not b.decoder_skip_causal_mask:
      not_vis = not_vis | (segment_pos.unsqueeze(-1) < segment_pos.unsqueeze(-2))
    mask = (not_vis.to(dtype) * -1e9).unsqueeze(1)
    SelfAttentionLayer._MASK_CACHE['k'] = (key, mask)
    return mask

  def _RelTable(self, theta, l, device):
    """fp32 `[H, 2L-1]` table indexed by (query_pos - key_pos + L - 1)."""
    b = self.bp
    bidi = (not self.params.decoder) or b.decoder_bidirectional_relative_attention
    rel = torch.arange(l - 1, -l, -1, device=device)           # key - query
    bucket = RelativePositionBucket(
        rel, b.relative_attention_num_buckets,
        b.relative_attention_max_distance, bidirectional=bidi)
    if theta.wrb.is_cuda:
      # gather forward, sorted index_put_ backward: replaces a one-hot fp32 matmul per layer
      # and direction.
      return _BucketGather.apply(theta.wrb.float(), bucket.long())
    onehot = F.one_hot(bucket.long(), b.relative_attention_num_buckets).float()
    return torch.matmul(theta.wrb.float(), onehot.t())

  def _Bias(self, theta, segment_id, segment_pos, dtype=torch.float32):
    """Additive bias `[B or 1, H or 1, L, L]` in `dtype`."""
    b = self.bp
    bias = self._Mask(segment_id, segment_pos, dtype)
    if self.params.relative_bias:
      bidi = (not self.params.decoder) or (
          b.decoder_bidirectional_relative_attention)
      if b.relative_attention_use_universal_1d_position:
        # Toeplitz structure: bias[h, i, j] = T[h, j - i + L - 1] with a
        # (2L-1)-entry table per head. Building T costs a 2L-1 gather and the
        # [H, L, L] expansion is a strided window view (no 16M-element
        # scatter-add in the backward pass, unlike the one-hot einsum
        # `HX,...LJX->...LHJ` of the reference :1487).
        l = segment_pos.shape[-1]
        rel = torch.arange(-(l - 1), l, device=segment_pos.device)
        bucket = RelativePositionBucket(
            rel, b.relative_attention_num_buckets,
            b.relative_attention_max_distance, bidirectional=bidi)
        table = theta.wrb.float()[:, bucket.long()].to(dtype)  # [H, 2L-1]
        rb = table.unfold(-1, l, 1).flip(1).unsqueeze(0)       # [1, H, L, L]
      else:
        rel = segment_pos.unsqueeze(-2) - segment_pos.unsqueeze(-1)
        bucket = RelativePositionBucket(
            rel, b.relative_attention_num_buckets,
            b.relative_attention_max_distance, bidirectional=bidi)
        oh = F.one_hot(bucket.long(), b.relative_attention_num_buckets).float()
        rb = torch.einsum('HX,BLJX->BHLJ', theta.wrb.float(), oh).to(dtype)
      bias = bias + rb
    return bias

  def _ContextParallelCore(self, theta, q, k, v, segment_id):
    """Sequence-sharded attention: local queries against the all-gathered keys / values.
    Causality and the relative bias use *global* token indices (inside a packed segment the
    index difference equals the position difference; across segments the mask removes the
    pair), so the result equals the unsharded layer's rows of this rank."""
    from lingvo_b200.parallel import cp   # pylint: disable=g-import-not-at-top
    import torch.distributed as dist   # pylint: disable=g-import-not-at-top
    b = self.bp
    w, r = dist.get_world_size(), dist.get_rank()
    lq = q.shape[1]
    lg = lq * w
    bias = None
    if self.params.relative_bias:
      table = self._RelTable(theta, lg, q.device)                 # [H, 2L−1], idx q−k+L−1
      qpos = torch.arange(lq, device=q.device) + r * lq
      kpos = torch.arange(lg, device=q.device)
      idx = qpos.unsqueeze(1) - kpos.unsqueeze(0) + lg - 1
      bias = table[:, idx]                                        # [H, L/W, L]
    causal = self.params.decoder and not b.decoder_skip_causal_mask
    return cp.Attention(q, k, v, causal=causal, segment_ids=segment_id, bias=bias, scale=1.0)

  supports_fused_residual = True

  def FProp(self, theta, x, segment_id, segment_pos, residual=None):
    if self._tp is not None:
      # f: identity / all-reduce(dx); the partial outputs of the head shards are summed by
      # g before the residual is added (once, on the replicated result).
      from lingvo_b200.parallel import tp_layers   # pylint: disable=g-import-not-at-top
      out, aux = self._FPropLocal(theta, tp_layers.CopyToTensorParallel(x, self._tp),
                                  segment_id, segment_pos, None)
      out = tp_layers.ReduceFromTensorParallel(out, self._tp)
      return (out + residual if residual is not None else out), aux
    return self._FPropLocal(theta, x, segment_id, segment_pos, residual)

  def _ProjectQkv(self, theta, x, segment_id, segment_pos):
    """x `[B,L,M]` → q `[B,L,H,D]`, k / v `[B,L,Hk,D]` of this rank's heads, after the
    multi-dconv-head convolutions and RoPE."""
    b = self.bp
    bsz, l, _ = x.shape
    d = b.attention_key_value_dim
    h, hk = self._LocalHeads()
    from lingvo_b200.ops import gemm
    wq, wk, wv = theta.wq, theta.wk, theta.wv
    if b.attention_combine_qkv and hk == h:
      wqkv = torch.cat([wq, wk, wv], dim=1)
      qkv = gemm.linear(x, wqkv.to(x.dtype))
      q, k, v = qkv.split([h * d, hk * d, hk * d], dim=-1)
    else:
      q = gemm.linear(x, wq.to(x.dtype))
      k = gemm.linear(x, wk.to(x.dtype))
      v = gemm.linear(x, wv.to(x.dtype))
    q = q.reshape(bsz, l, h, d)
    k = k.reshape(bsz, l, hk, d)
    v = v.reshape(bsz, l, hk, d)
    if self.params.multi_dconv_head:
      live = (segment_id != 0).to(q.dtype).reshape(bsz, l, 1, 1)
      q = self.q_dconv.FProp(theta.q_dconv, q * live, segment_pos)
      k = self.k_dconv.FProp(theta.k_dconv, k * live, segment_pos)
      v = self.v_dconv.FProp(theta.v_dconv, v * live, segment_pos)
    if b.use_rotary_position_emb or (self.params.multi_dconv_head and b.mdha_rope):
      q = _Rope(q, segment_pos, b.rope_emb_max_timescale)
      k = _Rope(k, segment_pos, b.rope_emb_max_timescale)
    return q, k, v

  def _FPropLocal(self, theta, x, segment_id, segment_pos, residual=None):
    b = self.bp
    bsz, l, _ = x.shape
    d = b.attention_key_value_dim
    h, _ = self._LocalHeads()
    from lingvo_b200.ops import gemm
    wo = theta.wo
    q, k, v = self._ProjectQkv(theta, x, segment_id, segment_pos)
    if _ContextParallel(b):
      o = self._ContextParallelCore(theta, q, k, v, segment_id)
      out = gemm.linear(o.reshape(bsz, l, h * d), wo.to(x.dtype), residual=residual)
      return out, torch.zeros((), device=x.device, dtype=torch.float32)
    simple = (not b.atten_logit_cap) and b.attention_extra_logit is None
    drop = b.attention_dropout_prob if not self.do_eval else 0.0
    toeplitz = (not self.params.relative_bias) or b.relative_attention_use_universal_1d_position
    if toeplitz:
      from lingvo_b200.ops import attention as attention_ops
      if attention_ops.flash_attention_supported(q, k, drop):
        # Our wgmma flash attention: bias table + packed-input mask applied in registers (after
        # the logit cap), dRel folded into the backward; grouped / multi-query KV heads are
        # read in place; output already `[B, L, H, D]`.
        rel = self._RelTable(theta, l, x.device) if self.params.relative_bias else None
        causal = self.params.decoder and not b.decoder_skip_causal_mask
        o = attention_ops.flash_attention(q, k, v, rel, segment_id, segment_pos, 1.0, causal,
                                          **_LogitOptions(b))
        out = gemm.linear(o.reshape(bsz, l, h * d), wo.to(x.dtype), residual=residual)
        return out, torch.zeros((), device=x.device, dtype=torch.float32)
    bias = self._Bias(theta, segment_id, segment_pos,
                      x.dtype if (simple and x.is_cuda) else torch.float32)
    o = _AttentionCore(q, k, v, bias, b.atten_logit_cap,
                       b.attention_extra_logit, b.attention_dropout_prob
                       if not self.do_eval else 0.0)
    out = gemm.linear(o.reshape(bsz, l, h * d), wo.to(x.dtype), residual=residual)
    return out, torch.zeros((), device=x.device, dtype=torch.float32)


def _SelfAttentionInitCache(layer, batch, max_len, device, dtype):
  b = layer.bp
  _, hk = layer._LocalHeads()   # pylint: disable=protected-access
  d = b.attention_key_value_dim
  cache = NestedMap(k=torch.zeros(batch, max_len, hk, d, device=device, dtype=dtype),
                    v=torch.zeros(batch, max_len, hk, d, device=device, dtype=dtype))
  if layer.params.multi_dconv_head:
    cache.q_conv = layer.q_dconv.InitState(batch, device, dtype)
    cache.k_conv = layer.k_dconv.InitState(batch, device, dtype)
    cache.v_conv = layer.v_dconv.InitState(batch, device, dtype)
  return cache


def _SelfAttentionExtendStep(layer, theta, x, cache, t):
  """One decode step: x `[B,1,M]` at position `t` (python int or 0-dim tensor) attends to
  the cached keys/values of positions ≤ t. The cache is updated in place (static
  buffers → the whole step is CUDA-graph capturable with `t` as a device scalar)."""
  b = layer.bp
  bsz, _, m = x.shape
  d = b.attention_key_value_dim
  h, hk = layer._LocalHeads()   # pylint: disable=protected-access  (this rank's heads under TP)
  xd = x.dtype
  q = torch.matmul(x, theta.wq.to(xd)).reshape(bsz, 1, h, d)
  k = torch.matmul(x, theta.wk.to(xd)).reshape(bsz, 1, hk, d)
  v = torch.matmul(x, theta.wv.to(xd)).reshape(bsz, 1, hk, d)
  if layer.params.multi_dconv_head:
    q, cache.q_conv = layer.q_dconv.ExtendStep(theta.q_dconv, q, cache.q_conv)
    k, cache.k_conv = layer.k_dconv.ExtendStep(theta.k_dconv, k, cache.k_conv)
    v, cache.v_conv = layer.v_dconv.ExtendStep(theta.v_dconv, v, cache.v_conv)
  tmax = cache.k.shape[1]
  dev = x.device
  tt = torch.as_tensor(t, device=dev).reshape(())
  if b.use_rotary_position_emb or (layer.params.multi_dconv_head and b.mdha_rope):
    pos = tt.reshape(1, 1).expand(bsz, 1)
    q, k = _Rope(q, pos, b.rope_emb_max_timescale), _Rope(k, pos, b.rope_emb_max_timescale)
  # Fused cache append + attention over the live keys (our split-KV kernel on the GPU; the
  # fp32 step of `decode_attention_ref`, in the forward's order, with a cap or extra logit).
  from lingvo_b200.ops import attention as attention_ops
  rel = _DecodeRelTable(layer, theta, tmax, dev)
  o = attention_ops.decode_attention(q, k, v, cache.k, cache.v, tt, rel, **_LogitOptions(b))
  o = o.reshape(bsz, 1, h * d)
  out = torch.matmul(o, theta.wo.to(xd))
  if layer._tp is not None:   # pylint: disable=protected-access
    from lingvo_b200.parallel import tp_layers   # pylint: disable=g-import-not-at-top
    out = tp_layers.ReduceFromTensorParallel(out, layer._tp)   # pylint: disable=protected-access
  return out


def _LogitOptions(b):
  """The builder's `atten_logit_cap` / `attention_extra_logit` as the keyword arguments of the
  attention ops, only those that are set: a layer without them calls the ops exactly as
  before they existed, so wrappers written against the plain signatures keep working."""
  opts = {}
  if b.atten_logit_cap:
    opts['logit_cap'] = float(b.atten_logit_cap)
  if b.attention_extra_logit is not None:
    opts['extra_logit'] = float(b.attention_extra_logit)
  return opts


def _DecodeRelTable(layer, theta, tmax, dev):
  """fp32 `[H, 2T-1]` relative-bias table of a decode step over a `T`-row cache, indexed by
  query − key + T − 1; None for a layer without relative bias."""
  if not layer.params.relative_bias:
    return None
  b = layer.bp
  bucket = RelativePositionBucket(     # table[:, i] for key − query = T − 1 − i
      torch.arange(tmax - 1, -tmax, -1, device=dev), b.relative_attention_num_buckets,
      b.relative_attention_max_distance,
      bidirectional=b.decoder_bidirectional_relative_attention)
  return theta.wrb.float()[:, bucket.long()]


def _SelfAttentionOut(layer, theta, o, xd):
  """Output projection of the attended heads `[B, L, H·D]` of a decode call."""
  out = torch.matmul(o, theta.wo.to(xd))
  if layer._tp is not None:   # pylint: disable=protected-access
    from lingvo_b200.parallel import tp_layers   # pylint: disable=g-import-not-at-top
    out = tp_layers.ReduceFromTensorParallel(out, layer._tp)   # pylint: disable=protected-access
  return out


def _SelfAttentionPrefill(layer, theta, x, segment_id, segment_pos, cache):
  """The whole prompt x `[B,P,M]` in one call: writes the post-RoPE keys / values into cache
  rows [0, P) and the positions into `cache.pos`, and returns the block output `[B,P,M]`.
  Pads carry segment id 0: they see nothing and nothing sees them. Where the layer's forward
  takes our flash kernel, so does this call (P padded to a multiple of 128); elsewhere it
  takes the layer's fp32 path."""
  b = layer.bp
  bsz, plen, _ = x.shape
  d = b.attention_key_value_dim
  h, _ = layer._LocalHeads()   # pylint: disable=protected-access
  q, k, v = layer._ProjectQkv(theta, x, segment_id, segment_pos)   # pylint: disable=protected-access
  cache.k[:, :plen] = k.to(cache.k.dtype)
  cache.v[:, :plen] = v.to(cache.v.dtype)
  cache.pos[:, :plen] = segment_pos.to(cache.pos.dtype)
  from lingvo_b200.ops import attention as attention_ops
  toeplitz = (not layer.params.relative_bias) or b.relative_attention_use_universal_1d_position
  causal = layer.params.decoder and not b.decoder_skip_causal_mask
  pad = -plen % 128
  padded = [F.pad(t, (0, 0, 0, 0, 0, pad)) for t in (q, k, v)]
  if toeplitz and attention_ops.flash_attention_supported(padded[0], padded[1]):
    rel = layer._RelTable(theta, plen + pad, x.device) if layer.params.relative_bias else None   # pylint: disable=protected-access
    o = attention_ops.flash_attention(*padded, rel, F.pad(segment_id, (0, pad)),
                                      F.pad(segment_pos, (0, pad)), 1.0, causal,
                                      **_LogitOptions(b))[:, :plen]
  else:
    bias = layer._Bias(theta, segment_id, segment_pos, torch.float32)   # pylint: disable=protected-access
    o = _AttentionCore(q, k, v, bias, b.atten_logit_cap, b.attention_extra_logit)
  return _SelfAttentionOut(layer, theta, o.reshape(bsz, plen, h * d), x.dtype)


def _SelfAttentionBeamStep(layer, theta, x, cache, slot0, vis, qpos):
  """One flat-beam-search step: x `[B,K,M]` holds one token per hypothesis at positions
  `qpos [B,K]`. Appends their keys / values at cache rows slot0 … slot0+K-1 and lets
  hypothesis k attend over the rows set in its bit mask `vis [B,K,⌈N/32⌉]`."""
  b = layer.bp
  bsz, kk, _ = x.shape
  d = b.attention_key_value_dim
  h, hk = layer._LocalHeads()   # pylint: disable=protected-access
  xd = x.dtype
  q = torch.matmul(x, theta.wq.to(xd)).reshape(bsz, kk, h, d)
  k = torch.matmul(x, theta.wk.to(xd)).reshape(bsz, kk, hk, d)
  v = torch.matmul(x, theta.wv.to(xd)).reshape(bsz, kk, hk, d)
  if b.use_rotary_position_emb:
    q, k = _Rope(q, qpos, b.rope_emb_max_timescale), _Rope(k, qpos, b.rope_emb_max_timescale)
  tmax = cache.k.shape[1]
  rows = torch.as_tensor(slot0, device=x.device).reshape(()) + torch.arange(kk, device=x.device)
  cache.pos.scatter_(1, rows.unsqueeze(0).expand(bsz, kk), qpos.to(cache.pos.dtype))
  from lingvo_b200.ops import attention as attention_ops
  o = attention_ops.flat_beam_attention(
      q, k, v, cache.k, cache.v, slot0, vis, qpos, cache.pos,
      _DecodeRelTable(layer, theta, tmax, x.device), 1.0, b.atten_logit_cap,
      b.attention_extra_logit)
  return _SelfAttentionOut(layer, theta, o.reshape(bsz, kk, h * d), xd)


def _Rope(x, pos, max_timescale):
  """Half-split rotary embedding on `[B, L, H, D]` (reference :409-426)."""
  d = x.shape[-1]
  half = d // 2
  frac = torch.arange(half, dtype=torch.float32, device=x.device) * 2.0 / d
  ts = max_timescale**frac
  ang = pos.float().unsqueeze(-1) / ts
  sin, cos = torch.sin(ang).unsqueeze(-2), torch.cos(ang).unsqueeze(-2)
  xf = x.float()
  a, b = xf[..., :half], xf[..., half:]
  return torch.cat([a * cos - b * sin, b * cos + a * sin], -1).to(x.dtype)


def _AttentionCore(q, k, v, bias, logit_cap=0.0, extra_logit=None,
                   dropout_prob=0.0):
  """softmax(q·kᵀ + bias)·v with fp32 logits; `BLHD` in/out."""
  bsz, l, h, d = q.shape
  hk = k.shape[2]
  if hk != h:
    k = k.expand(bsz, k.shape[1], h, d) if hk == 1 else (
        k.repeat_interleave(h // hk, dim=2))
    v = v.expand(bsz, v.shape[1], h, d) if hk == 1 else (
        v.repeat_interleave(h // hk, dim=2))
  simple = (not logit_cap) and extra_logit is None
  if simple and q.is_cuda:
    # NOTE: no 1/sqrt(D) scaling in GShard attention (folded into wq init).
    o = F.scaled_dot_product_attention(
        q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
        attn_mask=bias.expand(bsz, h, l, k.shape[1]),
        dropout_p=dropout_prob, scale=1.0)
    return o.transpose(1, 2)
  logits = torch.einsum('BLHD,BMHD->BHLM', q.float(), k.float())
  if logit_cap and logit_cap > 0:
    logits = logit_cap * torch.tanh(logits / logit_cap)
  logits = logits + bias
  if extra_logit is not None:
    extra = torch.full_like(logits[..., :1], float(extra_logit))
    probs = torch.softmax(torch.cat([logits, extra], -1), -1)[..., :-1]
  else:
    probs = torch.softmax(logits, -1)
  probs = probs.to(q.dtype)
  if dropout_prob:
    probs = F.dropout(probs, dropout_prob, training=True)
  return torch.einsum('BHLM,BMHD->BLHD', probs, v)


class DepthwiseConvAutoregressiveLayer(_BuilderLayer):
  """Causal depthwise convolution over time (ref :1749; Primer / MTF
  `sublayer_depthwise_conv_autoregressive`): `Y[:, t] = Σ_k W[k] ⊙ X[:, t − k]` with one
  weight vector per tap (`w_k/scale`, init 0.5 for k = 0 and 0.5/K otherwise). The input may
  carry several model dims (`[B, L, H, D]` for per-head convolutions). Positions do not
  look across packed-segment boundaries when `segment_pos` is given (a tap that would reach
  before position 0 of the segment reads zero)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('kernel_size', 3, 'Number of taps K.')
    p.Define('model_dims', None, 'Trailing dims of the input (default [model_dim]).')
    return p

  def _Dims(self):
    return list(self.params.model_dims or [self.bp.model_dim])

  def _CreateLayerVariables(self):
    p = self.params
    for k in range(p.kernel_size):
      self.CreateVariable('w_%d' % k, WeightParams(
          self._Dims(), WeightInit.Constant(0.5 if k == 0 else 0.5 / p.kernel_size),
          p.dtype))

  def FProp(self, theta, x, segment_pos=None):
    p = self.params
    out = x * theta.w_0.to(x.dtype)
    shifted = x
    for k in range(1, p.kernel_size):
      shifted = torch.cat([torch.zeros_like(shifted[:, :1]), shifted[:, :-1]], 1)
      term = shifted * theta['w_%d' % k].to(x.dtype)
      if segment_pos is not None:
        ok = (segment_pos >= k).to(x.dtype)
        term = term * ok.reshape(list(ok.shape) + [1] * (x.dim() - 2))
      out = out + term
    return out

  def InitState(self, batch, device, dtype):
    """The K−1 previous inputs, newest last (incremental decoding)."""
    return torch.zeros([batch, self.params.kernel_size - 1] + self._Dims(), device=device,
                       dtype=dtype)

  def ExtendStep(self, theta, x, state):
    """x `[B, 1, …]` → (y `[B, 1, …]`, new state)."""
    p = self.params
    out = x * theta.w_0.to(x.dtype)
    for k in range(1, p.kernel_size):
      out = out + state[:, -k:state.shape[1] - k + 1 or None][:, :1] * theta['w_%d' % k].to(
          x.dtype)
    new_state = torch.cat([state[:, 1:], x.to(state.dtype)], 1) if p.kernel_size > 1 else state
    return out, new_state


class AttentionCoreLayer(_BuilderLayer):
  """`softmax(q·kᵀ + bias)·v` for already projected `BLHD` / `BMHD` tensors (ref :1081
  `Attention`): fp32 logits, optional tanh cap, extra logit and attention dropout."""

  def FProp(self, theta, q, k, v, bias):
    b = self.bp
    while bias.dim() < 4:
      bias = bias.unsqueeze(1)                       # BLM → B1LM
    return _AttentionCore(q, k, v, bias.float(), b.atten_logit_cap, b.attention_extra_logit,
                          b.attention_dropout_prob if not self.do_eval else 0.0)


class CrossAttentionLayer(_BuilderLayer):
  """Decoder → encoder attention (ref :1206 `DecEncAttention`): queries from the decoder
  stream, keys / values from `encoder_output`; a query sees the encoder positions of its own
  packed segment only (`_EncNotVisible`, ref :1171)."""

  needs_encoder = True

  def _CreateLayerVariables(self):
    b = self.bp
    h, d, m = b.attention_num_heads, b.attention_key_value_dim, b.model_dim
    hk = b.attention_num_memory_heads or h
    dt = self.params.dtype
    self.CreateVariable('wq', WeightParams([m, h * d], WeightInit.Gaussian((m * d)**-0.5), dt))
    self.CreateVariable('wk', WeightParams([m, hk * d], WeightInit.Gaussian(m**-0.5), dt))
    self.CreateVariable('wv', WeightParams([m, hk * d], WeightInit.Gaussian(m**-0.5), dt))
    self.CreateVariable('wo', WeightParams([h * d, m], WeightInit.Gaussian((h * d)**-0.5), dt))

  def ProjectEncoder(self, theta, encoder_output):
    """K / V of the encoder output — computed once per sequence when decoding."""
    b = self.bp
    bsz, s, _ = encoder_output.shape
    hk = b.attention_num_memory_heads or b.attention_num_heads
    d = b.attention_key_value_dim
    xd = encoder_output.dtype
    k = torch.matmul(encoder_output, theta.wk.to(xd)).reshape(bsz, s, hk, d)
    v = torch.matmul(encoder_output, theta.wv.to(xd)).reshape(bsz, s, hk, d)
    return k, v

  def FProp(self, theta, x, segment_id, segment_pos, encoder_output=None,
            encoder_segment_id=None, kv=None):
    del segment_pos
    b = self.bp
    bsz, l, _ = x.shape
    h, d = b.attention_num_heads, b.attention_key_value_dim
    q = torch.matmul(x, theta.wq.to(x.dtype)).reshape(bsz, l, h, d)
    k, v = kv if kv is not None else self.ProjectEncoder(theta, encoder_output)
    a, c = segment_id.unsqueeze(-1), encoder_segment_id.unsqueeze(-2)
    not_visible = ((a == 0) & (c == 0)) | (a != c)
    bias = (not_visible.float() * -1e9).unsqueeze(1)                     # [B, 1, L, S]
    o = _AttentionCore(q, k, v, bias, b.atten_logit_cap, b.attention_extra_logit,
                       b.attention_dropout_prob if not self.do_eval else 0.0)
    out = torch.matmul(o.reshape(bsz, l, h * d), theta.wo.to(x.dtype))
    return out, torch.zeros((), device=x.device, dtype=torch.float32)


class ParallelAttentionFFNLayer(_BuilderLayer):
  """Attention and feed-forward applied to the SAME normalised input and summed (ref :2619
  `ParallelDecSelfAttentionRelativeBiasFFN`; the PaLM / GPT-J block): one norm, two
  branches, one residual add — the two branches' GEMMs are independent."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('atten', None, 'Self-attention layer params.')
    p.Define('ffn', None, 'Feed-forward layer params.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self.CreateChild('atten', self.params.atten)
    self.CreateChild('ffn', self.params.ffn)

  def FProp(self, theta, x, segment_id, segment_pos):
    a, aux_a = self.atten.FProp(theta.atten, x, segment_id, segment_pos)
    f, aux_f = self.ffn.FProp(theta.ffn, x, segment_id, segment_pos)
    return a + f, aux_a + aux_f


class SmoothedSoftmaxLayer(_BuilderLayer):
  """Output softmax with its own `[M, V]` weight and label-smoothed cross entropy
  (ref :2258 `SmoothedSoftmax`): FProp(vec `[B, L, M]`, label ids, weights) →
  NestedMap(logits, per_token_loss, loss); z-loss is added by the task."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_dim', 0, 'Vocabulary size V.')
    p.Define('label_smoothing', None, 'Overrides the builder value.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    m = self.bp.model_dim
    self.CreateVariable('w', WeightParams([m, p.vocab_dim], WeightInit.Gaussian(m**-0.5),
                                          p.dtype))

  def Logits(self, theta, vec):
    return torch.matmul(vec, theta.w.to(vec.dtype))

  def FProp(self, theta, vec, label_ids, label_weights=None):
    p = self.params
    ls = self.bp.label_smoothing if p.label_smoothing is None else p.label_smoothing
    logits = self.Logits(theta, vec).float()
    logp = torch.log_softmax(logits, -1)
    nll = -logp.gather(-1, label_ids.long().unsqueeze(-1)).squeeze(-1)
    if ls:
      # off value ls/(V−1), on value 1−ls (the reference's smoothing)
      off = ls / (p.vocab_dim - 1)
      per_token = (1.0 - ls - off) * nll + off * (-logp.sum(-1))
    else:
      per_token = nll
    if label_weights is None:
      label_weights = torch.ones_like(per_token)
    w = label_weights.float()
    return NestedMap(logits=logits, per_token_loss=per_token,
                     loss=(per_token * w).sum() / w.sum().clamp_min(1e-8))


class DenseReluDenseLayer(_BuilderLayer):
  """`wi [M, H]` → act → dropout → `wo [H, M]` (:2939-2998); gated variant
  with `wi_0, wi_1` (:3054-)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('activation', 'relu', 'relu|gelu|sqr_relu|silu.')
    p.Define('gated', False, 'GLU variant: act(x·wi_0) ⊙ (x·wi_1).')
    return p

  def __init__(self, params):
    super().__init__(params)
    b = self.bp
    # Hidden dim on the model axis (`mh_wi_split = [0, 1]`, `hm_wo_split = [1, 0]`, ref
    # :2939-2998): wi column-parallel, wo row-parallel — Megatron's MLP.
    self._tp = self._TensorParallel(b.mh_wi_split if 'mh_wi_split' in b else None, 1)
    if self._tp is not None:
      assert b.ff_dim % self._tp.tp_size == 0, (b.ff_dim, self._tp.tp_size)

  def _CreateLayerVariables(self):
    b = self.bp
    m, h = b.model_dim, b.ff_dim
    tp = self._tp
    hl = h // tp.tp_size if tp is not None else h
    dt = self.params.dtype
    wi_init = WeightInit.Uniform(((1. / m)**0.5) * 3.**0.5)
    wo_init = WeightInit.Uniform(((1. / h)**0.5) * 3.**0.5)

    def Shard(wp, dim):
      if tp is not None:
        wp.init_shard = (dim, tp.tp_rank, tp.tp_size)
      return wp

    if self.params.gated:
      self.CreateVariable('wi_0', Shard(ShardedWeightParams(
          [m, hl], wi_init, dt, tensor_split_dims_mapping=b.mh_wi_split), 1))
      self.CreateVariable('wi_1', Shard(ShardedWeightParams(
          [m, hl], wi_init, dt, tensor_split_dims_mapping=b.mh_wi_split), 1))
    else:
      self.CreateVariable('wi', Shard(ShardedWeightParams(
          [m, hl], wi_init, dt, tensor_split_dims_mapping=b.mh_wi_split), 1))
    self.CreateVariable('wo', Shard(ShardedWeightParams(
        [hl, m], wo_init, dt, tensor_split_dims_mapping=b.hm_wo_split), 0))
    if b.ff_use_bias:
      self.CreateVariable('bi', Shard(WeightParams([hl], WeightInit.Constant(0.), dt), 0))
      self.CreateVariable('bo', WeightParams([m], WeightInit.Constant(0.), dt))

  def _InstantiateSelfAndChildren(self):
    super()._InstantiateSelfAndChildren()
    if self._tp is not None:
      h = self.bp.ff_dim
      self._TagTpVars({'wi': (1, h), 'wi_0': (1, h), 'wi_1': (1, h), 'wo': (0, h),
                       'bi': (0, h)})

  supports_fused_residual = True

  def FProp(self, theta, x, segment_id=None, segment_pos=None, residual=None):
    if self._tp is not None:
      from lingvo_b200.parallel import tp_layers   # pylint: disable=g-import-not-at-top
      th = theta
      bo = None
      if self.bp.ff_use_bias:          # the output bias is added once, after the reduction
        th = NestedMap(theta)
        bo = theta.bo
        th.bo = torch.zeros_like(theta.bo)
      out, aux = self._FPropLocal(th, tp_layers.CopyToTensorParallel(x, self._tp), None)
      out = tp_layers.ReduceFromTensorParallel(out, self._tp)
      if bo is not None:
        out = out + bo.to(out.dtype)
      return (out + residual if residual is not None else out), aux
    return self._FPropLocal(theta, x, residual)

  def _FPropLocal(self, theta, x, residual=None):
    from lingvo_b200.ops import gemm
    b = self.bp
    p = self.params
    bi = theta.bi if b.ff_use_bias else None
    bo = theta.bo if b.ff_use_bias else None
    act = p.activation.upper()
    if p.gated:
      h = _Act(p.activation)(gemm.linear(x, theta.wi_0.to(x.dtype), bi)) * (
          gemm.linear(x, theta.wi_1.to(x.dtype)))
    elif act == 'RELU' and bi is None and bo is None and not (
        b.dropout_rate and not self.do_eval):
      out = gemm.ffn_relu(x, theta.wi.to(x.dtype), theta.wo.to(x.dtype), residual=residual)
      return out, torch.zeros((), device=x.device, dtype=torch.float32)
    elif act == 'RELU':
      h = gemm.linear(x, theta.wi.to(x.dtype), bi, act='RELU')
    else:
      h = _Act(p.activation)(gemm.linear(x, theta.wi.to(x.dtype), bi))
    if b.dropout_rate and not self.do_eval:
      h = F.dropout(h, b.dropout_rate, training=True)
    out = gemm.linear(h, theta.wo.to(x.dtype), bo, residual=residual)
    return out, torch.zeros((), device=x.device, dtype=torch.float32)


class MoELayer(_BuilderLayer):
  """Sharded MoE position-wise FFN (reference :2465-2548).

  Variables: `top_2_gating.w [M, E]`, `wi [E(_local), M, H]`,
  `wo [E(_local), H, M]` (GLU: `wi_0/wi_1`). Tokens `[B, L, M]` are grouped
  to `[G, S, M]`, gated (fp32 logits), dispatched to experts, and combined.
  `mode`: 'indexed' (H100 path) or 'dense' (reference einsum oracle).
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('gated', False, 'GLU experts (`MoEGated`).')
    p.Define('mode', 'indexed', 'indexed|dense.')
    return p

  def __init__(self, params):
    super().__init__(params)
    from lingvo_b200.parallel import mesh as mesh_lib
    self._ep = mesh_lib.ExpertParallelFor(self.bp.e_dim)

  @property
  def ep_engine(self):
    return self._ep

  def _CreateLayerVariables(self):
    b = self.bp
    m, h, e = b.model_dim, b.moe_hidden_dim, b.e_dim
    dt = self.params.dtype
    e_local = e if self._ep is None else self._ep.num_local_experts
    wi_init = WeightInit.Uniform(((1. / m)**0.5) * 3.**0.5)
    wo_init = WeightInit.Uniform(((1. / h)**0.5) * 3.**0.5)
    self.CreateVariable('gw', WeightParams(
        [m, e], WeightInit.Gaussian(m**-0.5), dt))
    names = ['wi_0', 'wi_1'] if self.params.gated else ['wi']
    shard = None
    if self._ep is not None:
      shard = (0, self._ep.ep_rank, self._ep.ep_size)
    for n in names:
      wp = ShardedWeightParams(
          [e_local, m, h], wi_init, dt, tensor_split_dims_mapping=b.emh_split)
      wp.init_shard = shard
      self.CreateVariable(n, wp)
    wp = ShardedWeightParams(
        [e_local, h, m], wo_init, dt, tensor_split_dims_mapping=b.ehm_split)
    wp.init_shard = shard
    self.CreateVariable('wo', wp)
    # Expert weights are *not* replicated across the EP group: mark them so
    # the data-parallel engine skips / narrows their gradient reduction.
    self._expert_var_names = names + ['wo']

  def _InstantiateSelfAndChildren(self):
    super()._InstantiateSelfAndChildren()
    for n in self._expert_var_names:
      self._private_vars[n].expert_parallel = self._ep is not None
      if self._ep is not None:
        # (ep_rank, ep_size, num_experts): dim-0 slice of the logical `[E, …]` tensor.
        self._private_vars[n].ep_shard = (self._ep.ep_rank, self._ep.ep_size, self.bp.e_dim)

  def _FusedExchange(self, x, act):
    """The fused gate+dispatch/expert-GEMM/combine engine when applicable."""
    b = self.bp
    p = self.params
    if not (ops.use_cuda_kernels(x) and x.dtype == torch.bfloat16 and
            act == 'RELU' and not p.gated and b.gating_func == 'top_2' and
            b.second_expert_policy == 'all' and x.shape[-1] % 8 == 0 and
            b.moe_hidden_dim % 8 == 0 and not (b.moe_dropout_rate and
                                              not self.do_eval)):
      return None
    from lingvo_b200.parallel import mesh as mesh_lib
    if mesh_lib.Get().mode != 'fused':
      return None
    if self._ep is not None:
      return self._ep.GetExchange(x.device)
    from lingvo_b200.parallel import symm
    return symm.LocalExchange(b.e_dim, x.device)

  def FProp(self, theta, x, segment_id, segment_pos=None, expert_id=None):
    b = self.bp
    p = self.params
    bsz, l, m = x.shape
    groups = b.num_groups or bsz
    tokens = bsz * l
    assert tokens % groups == 0
    s = tokens // groups
    xg = x.reshape(groups, s, m)
    paddings = (segment_id == 0).float().reshape(groups, s)
    ldt = b.gating_logits_dtype or torch.float32
    act = b.moe_activation.upper()
    pad_idx = b.Get('expert_padding_idx') if 'expert_padding_idx' in b else None
    if p.mode == 'dense' or b.gating_func == 'hashing' or pad_idx is not None:
      eid = expert_id.reshape(groups, s) if expert_id is not None else None
      gating = gshard_layers.ComputeGating(
          theta.gw, xg, paddings, b.num_devices, b.e_dim, b.c_dim or 0, True,
          x.dtype, b.gating_func, False, b.second_expert_policy,
          b.second_expert_threshold, b.legacy_mtf_behavior, b.capacity_factor,
          None, b.mask_dtype or torch.float32, ldt, expert_id=eid,
          expert_padding_idx=pad_idx)
      wi = torch.stack([theta.wi_0, theta.wi_1]) if p.gated else theta.wi
      out, aux = gshard_layers.FeedForwardNetworksApplyGating(
          gating, x, xg, wi, theta.wo, b.num_devices, groups,
          dropout_rate=b.moe_dropout_rate if not self.do_eval else 0.0,
          use_glu=p.gated, activation_name=act)
      return out.reshape(bsz, l, m), aux.float()
    # Gating logits in fp32: [G,S,M]·[M,E] is tiny (E = 8); keep it exact. On the GPU one
    # streaming kernel reads the bf16 activations directly (no fp32 upcast, no N=8 SGEMM).
    from lingvo_b200.ops import gate as gate_ops
    if ldt == torch.float32 and gate_ops.supported(xg, theta.gw):
      if xg.requires_grad:
        # x also feeds the expert exchange: take it from the router's autograd node so the
        # two input gradients are summed inside the router's dx kernel.
        logits, xg = gate_ops.gate_logits_pass(xg, theta.gw)
      else:
        logits = gate_ops.gate_logits(xg, theta.gw)
    else:
      logits = torch.matmul(xg.to(ldt), theta.gw.to(ldt))
    ex = self._FusedExchange(x, act)
    if ex is not None:
      cap = gshard_layers.ExpertCapacity(s, b.e_dim, b.c_dim or 0,
                                         b.capacity_factor)
      out, aux = ex.Apply(id(self), xg.reshape(groups * s, m).contiguous(),
                          logits, paddings, cap, bool(b.legacy_mtf_behavior),
                          theta.wi.to(x.dtype), theta.wo.to(x.dtype))
      return out.reshape(bsz, l, m), aux.float()
    seeds = None
    if b.second_expert_policy != 'all':
      seeds = py_utils.GenerateStepSeedPair(p)
    gating = gshard_layers.Top2GatingIndices(
        logits, paddings, b.e_dim, b.c_dim or 0, torch.float32,
        b.second_expert_policy, b.second_expert_threshold,
        b.legacy_mtf_behavior, b.capacity_factor, seeds)
    wi = torch.stack([theta.wi_0, theta.wi_1]) if p.gated else theta.wi
    out = gshard_layers.MoEApplyIndexed(
        xg, gating, wi, theta.wo, act, use_glu=p.gated, ep_engine=self._ep)
    return out.reshape(bsz, l, m), gating.aux_loss.float()


class DecoderBlock(_BuilderLayer):
  """mask → norm → sub-layer → dropout → residual add (reference :558-666)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('layer', None, 'Sub-layer params.')
    p.Define('norm', None, 'Norm layer params.')
    p.Define('norm_policy', 'pre', 'pre|primer|primer_hybrid.')
    p.Define('post_norm', None, 'Post-norm params for primer_hybrid.')
    p.Define('residual_weight', 1.0, 'x + residual_weight · f(norm(x)) (ref :488).')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('ln', p.norm)
    self.CreateChild('layer', p.layer)
    if p.post_norm is not None:
      self.CreateChild('post_ln', p.post_norm)

  def FProp(self, theta, i: NestedMap) -> NestedMap:
    p = self.params
    b = self.bp
    if i.get('all_valid', False):
      # The input generator vouched (from host data) that this batch has no padding:
      # the mask is all ones, skip the elementwise pass (and its backward).
      x_in = i.vec
    else:
      mask = (i.segment_id != 0).unsqueeze(-1).to(i.vec.dtype)
      x_in = i.vec * mask
    x_res = x_in
    if p.norm_policy != 'primer_post':
      x, x_res = self.ln.FPropPass(theta.ln, x_in)
    else:
      x = x_in
    fuse_res = (getattr(self.layer, 'supports_fused_residual', False) and
                p.residual_weight == 1.0 and
                i.get('expert_id') is None and p.post_norm is None and not (b.dropout_rate and not self.do_eval))
    if fuse_res:
      # x_in + f(x) comes out of the sub-layer's last GEMM epilogue.
      y, aux = self.layer.FProp(theta.layer, x, i.segment_id, i.segment_pos, residual=x_res)
      o = i.copy()
      o.vec = y
      o.aux_loss = i.aux_loss + aux
      return o
    if getattr(self.layer, 'needs_encoder', False):
      y, aux = self.layer.FProp(theta.layer, x, i.segment_id, i.segment_pos,
                                encoder_output=i.encoder_output,
                                encoder_segment_id=i.encoder_segment_id)
    elif i.get('expert_id') is not None and isinstance(self.layer, MoELayer):
      y, aux = self.layer.FProp(theta.layer, x, i.segment_id, i.segment_pos,
                                expert_id=i.expert_id)
    else:
      y, aux = self.layer.FProp(theta.layer, x, i.segment_id, i.segment_pos)
    if p.post_norm is not None:
      y = self.post_ln.FProp(theta.post_ln, y)
    if b.dropout_rate and not self.do_eval:
      y = F.dropout(y, b.dropout_rate, training=True)
    o = i.copy()
    o.vec = x_res + (y if p.residual_weight == 1.0 else y * p.residual_weight)
    o.aux_loss = i.aux_loss + aux
    return o


class LayerStack(_BuilderLayer):
  """`num` repetitions of the sub-layer list + final norm (:675-906)."""

  # -- incremental decoding ----------------------------------------------------------
  def InitDecodeState(self, batch, max_len, device, dtype):
    """KV caches for every self-attention block (None for the other blocks)."""
    return [(_SelfAttentionInitCache(blk.layer, batch, max_len, device, dtype)
             if isinstance(blk.layer, SelfAttentionLayer) else None) for blk in self.layers]

  def InitEncoderState(self, theta, encoder_output, encoder_segment_id=None):
    """Per cross-attention block the encoder keys / values (computed once per sequence);
    pass the result as `ExtendStep(..., encoder_state=…)`."""
    if encoder_segment_id is None:
      encoder_segment_id = torch.ones(encoder_output.shape[:2], dtype=torch.long,
                                      device=encoder_output.device)
    kvs = {}
    for idx, blk in enumerate(self.layers):
      if getattr(blk.layer, 'needs_encoder', False):
        kvs[idx] = blk.layer.ProjectEncoder(theta.layers[idx].layer, encoder_output)
    return NestedMap(kv=kvs, segment_id=encoder_segment_id)

  def _CheckBeamSupported(self):
    """Prefill / BeamExtendStep handle self-attention (without multi-dconv heads) and
    position-wise blocks only; anything else would decode wrongly, so it is refused."""
    for blk in self.layers:
      lyr = blk.layer
      if isinstance(lyr, SelfAttentionLayer):
        if lyr.params.multi_dconv_head:
          raise NotImplementedError(
              '%s: multi-dconv-head attention cannot be prefilled or beam-stepped' %
              blk.params.name)
      elif not isinstance(lyr, (DenseReluDenseLayer, MoELayer)):
        raise NotImplementedError(
            '%s: %s cannot be prefilled or beam-stepped; only self-attention and '
            'feed-forward / MoE blocks can' % (blk.params.name, type(lyr).__name__))

  def _RunBlocks(self, theta, x, attend, seg, pos):
    """The ExtendStep block loop over x `[R, L, M]`: self-attention blocks call
    `attend(layer, theta, y, cache)`, the others run on `seg` / `pos` `[R, L]`."""
    for idx, blk in enumerate(self.layers):
      th = theta.layers[idx]
      y = blk.ln.FProp(th.ln, x)
      if isinstance(blk.layer, SelfAttentionLayer):
        y = attend(blk.layer, th.layer, y, idx)
      else:
        y, _ = blk.layer.FProp(th.layer, y, seg, pos)
      if blk.params.residual_weight != 1.0:
        y = y * blk.params.residual_weight
      if blk.params.post_norm is not None:
        y = blk.post_ln.FProp(th.post_ln, y)
      x = x + y
    if 'final_layer_norm' in self.children:
      x = self.final_layer_norm.FProp(theta.final_layer_norm, x)
    return x

  def Prefill(self, theta, vec, segment_id, segment_pos, state):
    """Runs a prompt `vec [B,P,M]` through the stack in one call and writes every
    self-attention block's keys / values into cache rows [0, P) of `state` (from
    `InitDecodeState`). Tokens with `segment_id` 0 are padding. Returns `[B,P,M]`."""
    self._CheckBeamSupported()
    bsz, plen, _ = vec.shape
    for cache in state:
      if cache is not None:
        assert plen <= cache.k.shape[1], (plen, cache.k.shape)
        cache.pos = torch.zeros(bsz, cache.k.shape[1], dtype=torch.int32, device=vec.device)

    def Attend(layer, th, y, idx):
      return _SelfAttentionPrefill(layer, th, y, segment_id, segment_pos, state[idx])
    return self._RunBlocks(theta, vec, Attend, segment_id, segment_pos)

  def BeamExtendStep(self, theta, vec, state, slot0, vis, qpos):
    """One flat-beam-search step after `Prefill`: `vec [B,K,M]` holds the token of each of
    the K hypotheses at positions `qpos [B,K]`; they are appended at cache rows
    slot0 … slot0+K-1 (slot0 a Python int or 0-dim device tensor), and hypothesis k attends
    over the rows set in its int32 bit mask `vis [B,K,⌈N/32⌉]` (`ops.attention.
    pack_visibility`). Every other block sees B·K rows of one token, as in `ExtendStep`, so
    no hypothesis depends on its siblings. Returns `[B,K,M]`."""
    self._CheckBeamSupported()
    bsz, kk, m = vec.shape
    for cache in state:
      if cache is not None and 'pos' not in cache:
        raise ValueError('BeamExtendStep needs a state filled by Prefill')
    seg = torch.ones(bsz * kk, 1, dtype=torch.long, device=vec.device)
    pos = qpos.reshape(bsz * kk, 1).long()

    def Attend(layer, th, y, idx):
      return _SelfAttentionBeamStep(layer, th, y.reshape(bsz, kk, m), state[idx], slot0, vis,
                                    qpos).reshape(bsz * kk, 1, m)
    return self._RunBlocks(theta, vec.reshape(bsz * kk, 1, m), Attend, seg, pos).reshape(
        bsz, kk, m)

  def ExtendStep(self, theta, vec, state, t, encoder_state=None):
    """vec `[B,1,M]` at position t → `[B,1,M]`; `state` from `InitDecodeState`."""
    bsz = vec.shape[0]
    seg = torch.ones(bsz, 1, dtype=torch.long, device=vec.device)
    pos = torch.as_tensor(t, device=vec.device).reshape(1, 1).expand(bsz, 1)
    x = vec
    for idx, blk in enumerate(self.layers):
      th = theta.layers[idx]
      y = blk.ln.FProp(th.ln, x)
      if state[idx] is not None:
        y = _SelfAttentionExtendStep(blk.layer, th.layer, y, state[idx], t)
      elif getattr(blk.layer, 'needs_encoder', False):
        assert encoder_state is not None, 'cross-attention needs InitEncoderState()'
        y, _ = blk.layer.FProp(th.layer, y, seg, pos, kv=encoder_state.kv[idx],
                               encoder_segment_id=encoder_state.segment_id)
      else:
        y, _ = blk.layer.FProp(th.layer, y, seg, pos)
      if blk.params.residual_weight != 1.0:
        y = y * blk.params.residual_weight
      if blk.params.post_norm is not None:
        y = blk.post_ln.FProp(th.post_ln, y)
      x = x + y
    if 'final_layer_norm' in self.children:
      x = self.final_layer_norm.FProp(theta.final_layer_norm, x)
    return x

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('blocks', [], 'Flat list of DecoderBlock params.')
    p.Define('final_norm', None, 'Final norm layer params (or None).')
    p.Define('remat', False, 'Rematerialise each block in the backward pass.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChildren('layers', list(p.blocks))
    if p.final_norm is not None:
      self.CreateChild('final_layer_norm', p.final_norm)

  def FProp(self, theta, i: NestedMap) -> NestedMap:
    p = self.params
    x = i
    for idx, blk in enumerate(self.layers):
      if p.remat and not self.do_eval:
        keys = sorted(x.keys())

        def run(*vals, blk=blk, th=theta.layers[idx], keys=keys):
          o = blk.FProp(th, NestedMap(dict(zip(keys, vals))))
          return tuple(o[k] for k in keys)
        outs = py_utils.RematerializeFn(run, *[x[k] for k in keys])
        x = NestedMap(dict(zip(keys, outs)))
      else:
        x = blk.FProp(theta.layers[idx], x)
    if 'final_layer_norm' in self.children:
      x.vec = self.final_layer_norm.FProp(theta.final_layer_norm, x.vec)
      if not x.get('all_valid', False):
        mask = (x.segment_id != 0).unsqueeze(-1).to(x.vec.dtype)
        x.vec = x.vec * mask
      if self.bp.dropout_rate and not self.do_eval and (
          not self.bp.skip_output_dropout):
        x.vec = F.dropout(x.vec, self.bp.dropout_rate, training=True)
    return x


class MeshSplitLayer(base_layer.BaseLayer):
  """Sharding annotation layer (`MeshSplit`)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('tensor_split_dims_mapping', None, 'Mesh axis per tensor dim.')
    return p

  def FProp(self, theta, x):
    p = self.params
    return gshard_utils.MeshSplit(x, p.device_mesh, p.tensor_split_dims_mapping)


# =========================================================================
# Builders
# =========================================================================
class MoEBuilder(builder.Base):
  """Mixture-of-Experts Transformer builder (reference :55-2268)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_devices', 1, 'Obsolete: number of devices for Split().')
    p.Define('num_groups', None, 'MoE token groups G (default: batch dim).')
    p.Define('layer_norm_epsilon', 1e-6, 'Epsilon for norms.')
    p.Define('model_dim', 1024, 'Model dimension M.')
    p.Define('dropout_rate', 0.0, 'Residual/FFN dropout.')
    p.Define('noise_shape_broadcast_dims', None, 'Dropout broadcast dims.')
    p.Define('attention_num_heads', 1, 'Attention heads H.')
    p.Define('attention_num_memory_heads', None, '1 ⇒ multi-query attention.')
    p.Define('attention_key_value_dim', None, 'Per-head dim D.')
    p.Define('attention_dropout_prob', 0.0, 'Attention dropout.')
    p.Define('moe_dropout_rate', 0.0, 'Dropout inside experts.')
    p.Define('attention_combine_dims', False, 'Store weights as [M, H·D].')
    p.Define('attention_combine_qkv', True, 'One GEMM for q, k, v.')
    p.Define('mdha_rope', False, 'Primer multi-dconv-head attention w/ RoPE.')
    p.Define('use_rotary_position_emb', False, 'Apply RoPE to q/k.')
    p.Define('rope_emb_max_timescale', 10000.0, 'RoPE max timescale.')
    p.Define('ff_dim', None, 'Dense FFN hidden dim.')
    p.Define('e_dim', None, 'Number of experts E.')
    p.Define('c_dim', None, 'Expert capacity C (0/None ⇒ from factor).')
    p.Define('moe_hidden_dim', None, 'Expert hidden dim H.')
    p.Define('moe_activation', 'RELU', 'Expert activation.')
    p.Define('second_expert_policy', 'all', 'all|sampling|random.')
    p.Define('second_expert_threshold', 0., 'Threshold for `random`.')
    p.Define('legacy_mtf_behavior', True, 'Renormalise before capacity.')
    p.Define('label_smoothing', 0.1, 'Label smoothing.')
    p.Define('capacity_factor', None, 'C ≥ S·factor/E.')
    p.Define('gating_func', 'top_2', 'top_2|token_shuffle|hashing.')
    p.Define('relative_attention_type', None, 'None|bias|bias_shared.')
    p.Define('relative_attention_num_buckets', 32, 'T5 buckets.')
    p.Define('relative_attention_max_distance', 128, 'T5 max distance.')
    p.Define('relative_attention_use_universal_1d_position', False,
             'Positions 0..L-1 regardless of packing.')
    p.Define('inflate_universal_relative_bias_to_match_batch_dimension', False,
             'Kept for parity.')
    p.Define('attention_extra_logit', None, 'Extra softmax logit.')
    p.Define('attention_logits_dtype', None, 'Logits dtype (fp32 here).')
    p.Define('mask_dtype', None, 'Mask dtype.')
    p.Define('gating_logits_dtype', None, 'Gating logits dtype.')
    p.Define('conv_vars_reshape', False, 'Kept for parity.')
    p.Define('use_fused_depthwise_conv_autoregressive', False, 'Kept.')
    p.Define('ln_no_scale', False, 'RMS norm without scale.')
    p.Define('model_dim_reshape_segments', None, 'Reshape M → [segments, M/s].')
    p.Define('use_xla_dynamic_update_slice', True, 'Kept for parity.')
    p.Define('decoder_skip_causal_mask', False, 'Skip the causal mask.')
    p.Define('decoder_bidirectional_relative_attention', False, 'Bidi buckets.')
    p.Define('final_norm_type', 'ln', 'ln|true_ln|pn|none.')
    p.Define('skip_output_dropout', False, 'No dropout after the final norm.')
    p.Define('device_mesh_shape', None, 'Device mesh shape.')
    p.Define('emb_w_split', None, 'Mesh split for embedding weight.')
    p.Define('mhd_w_split', [0, 1, -1], 'Mesh split for attention MHD weight.')
    p.Define('kv_mhd_w_split', None, 'Mesh split for K/V MHD weight.')
    p.Define('mh_wi_split', [0, 1], 'Mesh split for dense MH weight.')
    p.Define('hm_wo_split', [1, 0], 'Mesh split for dense HM weight.')
    p.Define('one_hot_ids_split', None, 'Split for one-hot ids.')
    p.Define('emb_out_split', [0, -1, -1], 'Split for embedding outputs.')
    p.Define('qkv_split', [0, -1, 1, -1], 'Split for QKV BLHD activation.')
    p.Define('blm_split', [0, -1, -1], 'Split for BLM activation.')
    p.Define('blh_split', [0, -1, 1], 'Split for BLH activation.')
    p.Define('egcm_split', [0, -1, -1, -1], 'Split for EGCM.')
    p.Define('gecm_split', [0, -1, -1, -1], 'Split for GECM.')
    p.Define('gsec_split', [0, -1, -1, -1], 'Split for GSEC.')
    p.Define('gecs_split', [0, -1, -1, -1], 'Split for GECS.')
    p.Define('gec_split', [0, -1, -1], 'Split for GEC.')
    p.Define('eah_split', [0, -1, 1], 'Split for EAH.')
    p.Define('eam_split', [0, -1, -1], 'Split for EAM.')
    p.Define('emh_split', [0, -1, 1], 'Split for expert EMH weight.')
    p.Define('ehm_split', [0, 1, -1], 'Split for expert EHM weight.')
    p.Define('logits_split', [0, -1, -1], 'Split for logits.')
    p.Define('experimental_fix_split_dims_mapping', False, 'Kept for parity.')
    p.Define('atten_logit_cap', 0.0, 'tanh cap on attention logits.')
    p.Define('scale_input_embedding_by_dim', False, 'Scale embeddings.')
    p.Define('softplus_scale_q', False, 'Kept for parity.')
    p.Define('ff_use_bias', False, 'Bias in dense FFN.')
    p.Define('moe_mode', 'indexed', 'indexed (fused H100 path) | dense oracle.')
    p.Define('remat', False, 'Rematerialise blocks in backward.')
    p.Define('context_parallel', False,
             'Shard the *sequence* dimension over the ranks (context parallelism, '
             '`parallel/cp.py`): every rank holds L/W tokens of each sequence, attention '
             'all-gathers K/V (dK/dV are reduce-scattered in backward), everything else is '
             'token-local. For sequences too long for one GPU.')
    return p

  @property
  def _device_mesh(self):
    return self.params.device_mesh

  def _Common(self, p, name):
    p.name = name
    p.b = self.params
    p.dtype = self.params.dtype
    p.fprop_dtype = self.params.fprop_dtype
    return p

  # ---- sharding -----------------------------------------------------------
  def MeshSplit(self, name, tensor_split_dims_mapping):
    return MeshSplitLayer.Params().Set(
        name=name, device_mesh=self.params.device_mesh,
        tensor_split_dims_mapping=tensor_split_dims_mapping)

  def _AdjustMSplit(self, split, m_dim):
    """Adjusts split dims for `model_dim_reshape_segments` (reference)."""
    if split is None or self.params.model_dim_reshape_segments is None:
      return split
    seg = self.params.model_dim_reshape_segments
    n = len(seg) if isinstance(seg, (list, tuple)) else 1
    if m_dim < 0:
      m_dim += len(split)
    return list(split[:m_dim]) + [split[m_dim]] + [-1] * n + list(
        split[m_dim + 1:])

  # ---- norms --------------------------------------------------------------
  def _Norm(self, name, kind):
    p = self.params
    return self._Common(RmsNormLayer.Params().Set(
        dim=p.model_dim, epsilon=p.layer_norm_epsilon, kind=kind,
        no_scale=p.ln_no_scale and kind == 'rms'), name)

  def _LN(self, name):
    return self._Norm(name, 'rms')

  def _LNNoScale(self, name):
    q = self._Norm(name, 'rms')
    q.no_scale = True
    return q

  def _TrueLN(self, name):
    return self._Norm(name, 'true_ln')

  def _PN(self, name):
    return self._Norm(name, 'pn')

  def _NormByType(self, name, norm_type):
    if norm_type == 'ln':
      return self._LN(name)
    if norm_type in ('true_ln', 'jax_replica_ln'):
      return self._TrueLN(name)
    if norm_type == 'pn':
      return self._PN(name)
    if norm_type in ('none', 'no_ln'):
      return self._Norm(name, 'none')
    raise ValueError('Norm type %s not supported.' % norm_type)

  # ---- embedding ----------------------------------------------------------
  def Embedding(self, name, vocab_dim):
    p = self.params
    return self._Common(EmbeddingLayer.Params().Set(
        vocab_dim=vocab_dim, model_dim=p.model_dim,
        scale_by_dim=p.scale_input_embedding_by_dim), name)

  SharedEmbSoftmax = Embedding

  def SoftmaxWeight(self, name, vocab_dim):
    """A stand-alone `[M, V]` softmax weight (ref :468) as a logits layer."""
    return self._Common(SmoothedSoftmaxLayer.Params().Set(vocab_dim=vocab_dim,
                                                          label_smoothing=0.0), name)

  def SmoothedSoftmax(self, name, vocab_dim, label_smoothing=None):
    """Untied output softmax + label-smoothed cross entropy (ref :2258)."""
    return self._Common(SmoothedSoftmaxLayer.Params().Set(
        vocab_dim=vocab_dim, label_smoothing=label_smoothing), name)

  def Mask(self):
    """(vec, segment_id) → vec with padded positions (segment_id == 0) zeroed (ref :478)."""
    return self._Fn('mask', lambda x, segment_id: x * (segment_id != 0).unsqueeze(-1).to(
        x.dtype))

  def Split(self, name):
    """Batch-dim sharding annotation of the data-parallel axis (ref :1956): one process per
    GPU already holds its own batch shard, so this is the identity layer."""
    return self._Identity(name)

  def LN(self, name):
    return self._LN(name)

  def PN(self, name):
    return self._PN(name)

  def Repeat(self, name, body, repeat=1, per_layer_vars=True, start_layer_id=0):
    """`body` applied `repeat` times (ref :710): stacked variables + loop, or — with
    `per_layer_vars` — `repeat` independently named copies (checkpoint compatible with an
    unrolled stack)."""
    del start_layer_id
    from lingvo_b200.core import builder_layers   # pylint: disable=g-import-not-at-top
    return builder_layers.RepeatLayer.Params().Set(name=name, body=body, repeat=repeat,
                                                   per_layer_vars=per_layer_vars)

  def ShardablePipeline(self, name, body, stages, num_micro_batches=1):
    """`stages` copies of `body` run as a layer-wise shardable (shifting-buffer) pipeline
    over micro-batches (ref :720)."""
    from lingvo_b200.core import gshard_layers   # pylint: disable=g-import-not-at-top
    return gshard_layers.LayerwiseShardablePipelinedLayer.Params().Set(
        name=name, num_stages=stages, single_stage_body=body,
        num_microbatches=num_micro_batches)

  @classmethod
  def SetFPropDtype(cls, p, fprop_dtype):
    """Sets the activation dtype on builder params (ref :274); bf16 keeps fp32 attention
    logits and gating."""
    p.fprop_dtype = fprop_dtype
    if fprop_dtype == torch.bfloat16 and not p.attention_logits_dtype:
      p.attention_logits_dtype = torch.float32
    return p

  # ---- attention ----------------------------------------------------------
  def _Atten(self, name, decoder, relative_bias):
    return self._Common(SelfAttentionLayer.Params().Set(
        decoder=decoder, relative_bias=relative_bias), name)

  def DecSelfAttention(self, name, *unused):
    return self._Atten(name, True, False)

  def DecSelfAttentionRelativeBias(self, name, *unused):
    assert self.params.relative_attention_type in ('bias', 'bias_shared')
    return self._Atten(name, True, True)

  def SelfAttention(self, name, *unused):
    return self._Atten(name, False, False)

  def SelfAttentionRelativeBias(self, name, *unused):
    return self._Atten(name, False, True)

  EncSelfAttention = SelfAttention

  def Attention(self, name):
    """(q, k, v, bias) → context for already projected `BLHD` tensors (ref :1081)."""
    return self._Common(AttentionCoreLayer.Params(), name)

  def DecEncAttention(self, name, *unused):
    """Decoder → encoder cross attention (ref :1206); the enclosing `DecoderLayer` feeds it
    `encoder_output` / `encoder_segment_id` from the layer-stack input map."""
    return self._Common(CrossAttentionLayer.Params(), name)

  def DecMultiDconvHeadAttention(self, name, *unused):
    """Primer's multi-dconv-head decoder self-attention (ref :1349)."""
    return self._Common(SelfAttentionLayer.Params().Set(
        decoder=True, relative_bias=False, multi_dconv_head=True), name)

  def DecMultiDconvHeadAttentionRelativeBias(self, name, *unused):
    assert self.params.relative_attention_type in ('bias', 'bias_shared')
    return self._Common(SelfAttentionLayer.Params().Set(
        decoder=True, relative_bias=True, multi_dconv_head=True), name)

  def DepthwiseConvAutoregressive(self, name, kernel_size, model_dims=None):
    """Causal depthwise conv over time with one weight vector per tap (ref :1749)."""
    return self._Common(DepthwiseConvAutoregressiveLayer.Params().Set(
        kernel_size=kernel_size, model_dims=list(model_dims) if model_dims else None), name)

  CausalDepthwiseConv = DepthwiseConvAutoregressive        # same math, one fused layer here

  def ParallelDecSelfAttentionRelativeBiasFFN(self, name, activation_fn='relu',
                                              gated=False, relative_bias=True, **unused):
    """Attention ‖ FFN on one normalised input (ref :2619)."""
    if isinstance(activation_fn, str):
      act = activation_fn
    else:
      act = getattr(activation_fn, '_lingvo_name', 'relu')
    atten = self._Atten('atten', True, relative_bias)
    ffn = (self.DenseReluDenseGated('ffn', act) if gated else
           self.DenseReluDense('ffn', activation=act))
    return self._Common(ParallelAttentionFFNLayer.Params().Set(atten=atten, ffn=ffn), name)

  # ---- FFN / MoE ----------------------------------------------------------
  def DenseReluDense(self, name, decoder=False, activation='relu'):
    return self._Common(DenseReluDenseLayer.Params().Set(
        activation=activation, gated=False), name)

  def DenseReluDenseGated(self, name, activation_fn, decoder=False):
    act = activation_fn if isinstance(activation_fn, str) else getattr(
        activation_fn, '_lingvo_name', 'gelu')
    return self._Common(DenseReluDenseLayer.Params().Set(
        activation=act, gated=True), name)

  def DenseReluDenseGatedGELU(self, name, decoder=False):
    return self.DenseReluDenseGated(name, 'gelu', decoder=decoder)

  def DenseReluDenseGatedSILU(self, name, decoder=False):
    return self.DenseReluDenseGated(name, 'silu', decoder=decoder)

  def MoE(self, name, decoder=False):
    return self._Common(MoELayer.Params().Set(
        gated=False, mode=self.params.moe_mode), name)

  def MoEGated(self, name, decoder=False):
    return self._Common(MoELayer.Params().Set(
        gated=True, mode=self.params.moe_mode), name)

  # ---- blocks & stacks ----------------------------------------------------
  def DecoderLayer(self, name, layer, conv_kernel_size=None, norm_type='ln',
                   norm_policy='pre'):
    post = None
    if norm_policy == 'primer_hybrid':
      post = self._NormByType('post_' + norm_type, norm_type)
    return self._Common(DecoderBlock.Params().Set(
        layer=layer.Copy(), norm=self._NormByType(norm_type, norm_type),
        norm_policy=norm_policy, post_norm=post), name)

  def EncoderLayer(self, name, layer, residual_weight=1.0, norm_type='ln',
                   norm_policy='pre'):
    """Encoder block: x + residual_weight · layer(norm(x)) (ref :488)."""
    blk = self.DecoderLayer(name, layer, None, norm_type, norm_policy)
    blk.residual_weight = residual_weight
    return blk

  def _LayerStack(self, name, sub_layers, num, conv_kernel_size=None,
                  norm_type='ln', norm_policy='pre', start_layer_id=0,
                  has_final_layer=True, decoder=True, **unused):
    blocks = []
    for i in range(num):
      for j, sub in enumerate(sub_layers):
        idx = start_layer_id + i * len(sub_layers) + j
        blocks.append(self.DecoderLayer('layer_%03d' % idx, sub,
                                        conv_kernel_size, norm_type,
                                        norm_policy))
    final = None
    if has_final_layer:
      final = self._NormByType('final_layer_norm', self.params.final_norm_type)
    return self._Common(LayerStack.Params().Set(
        blocks=blocks, final_norm=final, remat=self.params.remat), name)

  def DecoderLayerStack(self, name, sub_layers, num=1, **kwargs):
    return self._LayerStack(name, sub_layers, num, decoder=True, **kwargs)

  def EncoderLayerStack(self, name, sub_layers, num=1, **kwargs):
    return self._LayerStack(name, sub_layers, num, decoder=False, **kwargs)


class DenseBuilder(MoEBuilder):
  """Builder for dense / hybrid models with 2-D sharding (reference :2269)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.emb_w_split = None
    return p


RecurrentDenseBuilder = DenseBuilder


class RecurrentDenseBuilderParallelDecode(DenseBuilder):
  """`DenseBuilder` whose projection weights are split into *micro variables* of shape
  `[model_dim, proj_weight_hdim, d_kv]` (reference :3478) so that no single variable of a
  very deep repeated stack exceeds one host's memory. On H100 the 80 GB of HBM hold the
  fused `[M, H·D]` weights directly and the kernels want them contiguous, so the weights
  stay fused; the class keeps the knob (checkpoint converters use it to split / merge the
  micro variables) and forces deterministic dropout like the reference."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('proj_weight_hdim', 64,
             'Micro-variable width (None disables); used by checkpoint conversion.')
    p.deterministic_dropout = True
    return p

  def MicroVariableShapes(self, out_dim):
    """Shapes the reference would create for a `[model_dim, out_dim]` projection."""
    p = self.params
    d_kv = p.attention_key_value_dim
    if not p.proj_weight_hdim or not d_kv:
      return [[p.model_dim, out_dim]]
    per = p.proj_weight_hdim * d_kv
    assert out_dim % per == 0, (out_dim, per)
    return [[p.model_dim, p.proj_weight_hdim, d_kv]] * (out_dim // per)


class MoEHashBuilder(DenseBuilder):
  """MoE with hash routing (reference :3829): a token goes to expert `id mod E`; there is
  no learned gate and no auxiliary loss. The task passes `expert_id` alongside the
  activations (see `BertTransformer._ComputeEncInput`)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.gating_func = 'hashing'
    return p


class DenseLifelongBuilder(DenseBuilder):
  """Builder for lifelong learning with growing expert sets (reference :3198): the gate
  can be widened from `e_dim_old` to `e_dim` experts, ranges of experts can be masked out
  of the routing (`expert_padding_idx = [lo, hi)`), and a learning-without-forgetting
  penalty (`lwf_scale`) ties the new model's outputs to the frozen old model's."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('e_dim_old', None, 'Number of experts of the previous stage.')
    p.Define('expert_padding_idx', None, '[lo, hi): experts excluded from routing.')
    p.Define('expert_padding_idx_old', None, 'Same, for the old model in LwF.')
    p.Define('lwf_scale', 0, 'Weight of the LwF distillation loss.')
    return p

  @staticmethod
  def ExpandGate(old_gw, e_dim, init_scale=None):
    """Widens a trained gate `[M, E_old]` to `[M, E]`, new columns ~ U(±init_scale)."""
    m, e_old = old_gw.shape
    scale = init_scale if init_scale is not None else (1.0 / m) ** 0.5 * 3.0 ** 0.5
    extra = (torch.rand(m, e_dim - e_old, dtype=old_gw.dtype, device=old_gw.device) * 2 - 1)
    return torch.cat([old_gw, extra * scale], 1)

  @staticmethod
  def ExpandExperts(old_w, e_dim):
    """Grows expert weights `[E_old, …]` to `[E, …]` by cloning experts round-robin."""
    e_old = old_w.shape[0]
    idx = torch.arange(e_dim, device=old_w.device) % e_old
    return old_w.index_select(0, idx).clone()


# =========================================================================
# UniTransformer LM task
# =========================================================================
class UniTransformer(base_model.BaseTask):
  """Decoder-only LM with z-loss, label smoothing and MoE aux loss."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('debug', False, 'Emit per-example tensors.')
    p.Define('builder', None, 'GShard builder params.')
    p.Define('vocab_size', None, 'Vocabulary size.')
    p.Define('sequence_length', None, 'Sequence length.')
    p.Define('max_length', 512, 'Max sequence length (positional table).')
    p.Define('batch_size', None, 'Batch size (unused).')
    p.Define('num_transformer_layers', None, 'Number of blocks.')
    p.Define('loss_denominator', 0, 'Fixed loss denominator if > 0.')
    p.Define('use_tgt_labels_size_as_loss_denominator', True,
             'Denominator = labels size instead of #non-pad tokens.')
    p.Define('aux_loss_coef', 0.01, 'Multiplier for the MoE aux loss.')
    p.Define('enable_tpu_summary', True, 'Kept for parity.')
    p.Define('label_smoothing', 0.1, 'Label smoothing.')
    p.Define('logits_abs_max', None, 'Logits clipping.')
    p.Define('z_loss', 1e-4, 'z_loss · logsumexp(logits)² added to the loss.')
    p.Define('positional_embedding', True, 'Learned positional embedding.')
    p.Define('sub_layer_types', None, "e.g. ['attn','moe','attn','ffw'].")
    p.Define('sinusoid_positional_embedding', False, 'Sinusoid positions.')
    p.Define('gated_gelu', False, 'Deprecated: gated_ffn_activation=gelu.')
    p.Define('moe_gated_gelu', False, 'GLU experts.')
    p.Define('gated_ffn_activation', None, 'silu|gelu|None.')
    p.Define('softmax_bias', False, 'Bias in the softmax.')
    p.Define('parallel_ffn', False, 'Kept for parity.')
    p.Define('hidden_dim_reshape_segments', 4, 'Kept for parity.')
    p.Define('conv_kernel_size', None, 'Optional depthwise conv in the norm.')
    p.Define('scale_decoder_outputs', True, 'Scale outputs by M^-0.5.')
    p.Define('use_per_layer_vars_for_recurrent', False, 'Kept for parity.')
    p.Define('use_repeat_layer', False, 'Kept for parity.')
    p.Define('num_spmd_pipeline_stages', 1, 'SPMD pipeline stages.')
    p.Define('num_spmd_pipeline_microbatches', None, 'SPMD micro-batches.')
    p.Define('moe', False, 'Mixture-of-Experts model.')
    p.Define('activation', 'relu', 'Non-gated FFN activation.')
    p.Define('norm_type', 'ln', 'ln|pn|true_ln|jax_replica_ln|no_ln.')
    p.Define('norm_policy', 'pre', 'pre|primer|primer_hybrid.')
    p.Define('multi_dconv_head_att', False, "Primer's multi-dconv-head attention.")
    p.Define('decoder_max_steps', 64, 'Max decode steps.')
    p.Define('decoder_beam_size', 4, 'Beam size.')
    p.Define('decoder_eos_id', 1, '</s> id.')
    p.Define('decoder_bos_id', 0, '<s> id.')
    p.Define('start_layer_id', 0, 'Start layer id.')
    p.Define('pos_emb_max_timescale', 10000.0, 'Sinusoid max timescale.')
    p.Define('has_embedding_layer', True, 'Model has the embedding layer.')
    p.Define('has_final_layer', True, 'Model has the final layer.')
    p.Define('softmax_logit_cap', 0.0, 'Softmax logit cap.')
    p.Define('is_quantize', False, 'Kept for parity.')
    p.Define('use_log_softmax_normalization', True, 'Kept for parity.')
    p.Define('fused_xent', True, 'Use the fused logits+xent kernel path.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    b = p.builder.Instantiate()
    bp = b.params
    gated = p.gated_ffn_activation or ('gelu' if p.gated_gelu else None)
    if p.has_embedding_layer:
      self.CreateChild('dec_emb', b.Embedding('dec_emb', p.vocab_size))
      if p.positional_embedding:
        if p.sinusoid_positional_embedding:
          self.CreateChild('dec_pos_emb',
                           layers.PositionalEmbeddingLayer.Params().Set(
                               name='dec_pos_emb', embedding_dim=bp.model_dim,
                               max_timescale=p.pos_emb_max_timescale))
        else:
          self.CreateChild('dec_pos_emb', b.Embedding('dec_pos_emb',
                                                      p.max_length))
    if p.multi_dconv_head_att:
      atten = (b.DecMultiDconvHeadAttention('multi_dconv_head_att') if p.positional_embedding
               else b.DecMultiDconvHeadAttentionRelativeBias('multi_dconv_head_att'))
    elif p.positional_embedding:
      atten = b.DecSelfAttention('dec_self_attention')
    else:
      atten = b.DecSelfAttentionRelativeBias('dec_self_attention')
    if gated is None:
      ffw = b.DenseReluDense('dense_relu_dense', decoder=True,
                             activation=p.activation)
    else:
      ffw = b.DenseReluDenseGated('dense_relu_dense', gated, decoder=True)
    if p.moe:
      moe = (b.MoEGated('moe', decoder=True) if p.moe_gated_gelu
             else b.MoE('moe', decoder=True))
      table = {'attn': atten, 'moe': moe, 'ffw': ffw}
      if p.sub_layer_types:
        n_types = len(p.sub_layer_types)
        if p.num_transformer_layers * 2 % n_types != 0:
          raise ValueError('Unsupported Sub-layer types length!')
        subs = [table[t] for t in p.sub_layer_types]
        num = p.num_transformer_layers * 2 // n_types
      else:
        subs = [atten, moe, atten, ffw]
        num = p.num_transformer_layers // 2
    else:
      subs = [atten, ffw]
      num = p.num_transformer_layers
    dec = b.DecoderLayerStack(
        'decoder', subs, num, conv_kernel_size=p.conv_kernel_size,
        norm_type=p.norm_type, norm_policy=p.norm_policy,
        start_layer_id=p.start_layer_id, has_final_layer=p.has_final_layer)
    dec.params_init = WeightInit.Xavier(scale=1.0, seed=0)
    self.CreateChild('dec', dec)
    self.CreateChild('emb_w_split', b.MeshSplit('w_split', bp.emb_w_split))
    self.CreateChild('dec_out_split', b.MeshSplit('dec_out_split', bp.blm_split))
    self.CreateChild('logits_split', b.MeshSplit('logits_split',
                                                 bp.logits_split))
    if p.has_final_layer and p.softmax_bias:
      self.CreateVariable('softmax_bias', WeightParams(
          [p.vocab_size], WeightInit.Constant(0.0), p.dtype))

  # ---------------------------------------------------------------- input --
  def _ComputeInputBatch(self, input_batch):
    if 'tgt' not in input_batch:
      input_batch.tgt = NestedMap(
          ids=input_batch.ids, paddings=input_batch.paddings,
          labels=input_batch.labels, segment_ids=input_batch.segment_ids,
          segment_pos=input_batch.segment_pos)
    if _ContextParallel(self.params.builder) and not input_batch.tgt.get('_cp_sharded', False):
      # context parallelism: this rank keeps its L/W slice of every [B, L, …] input
      from lingvo_b200.parallel import cp   # pylint: disable=g-import-not-at-top
      tgt = input_batch.tgt
      full_len = tgt.ids.shape[1]
      for k, v in list(tgt.items()):
        if isinstance(v, torch.Tensor) and v.dim() >= 2 and v.shape[1] == full_len:
          tgt[k] = cp.ShardSequence(v, 1)
      tgt._cp_sharded = True   # pylint: disable=protected-access
    return input_batch

  def _ComputeDecoderInput(self, theta, input_batch):
    p = self.params
    input_batch = self._ComputeInputBatch(input_batch)
    tgt = input_batch.tgt
    fd = self.fprop_dtype
    y = self.dec_emb.FProp(theta.dec_emb, tgt.ids).to(fd)
    if p.positional_embedding:
      if p.sinusoid_positional_embedding:
        y = y + self.dec_pos_emb.FPropWithPosition(theta.dec_pos_emb,
                                                   tgt.segment_pos).to(fd)
      else:
        y = y + self.dec_pos_emb.FProp(theta.dec_pos_emb,
                                       tgt.segment_pos).to(fd)
    return NestedMap(vec=y, segment_id=tgt.segment_ids,
                     segment_pos=tgt.segment_pos,
                     aux_loss=torch.zeros((), device=y.device),
                     all_valid=bool(tgt.get('all_valid', False)))

  # --------------------------------------------------------- predictions --
  def ComputePredictions(self, theta, input_batch):
    p = self.params
    dec_in = self._ComputeDecoderInput(theta, input_batch)
    out = self.dec.FProp(theta.dec, dec_in)
    dec_outputs, aux_loss = out.vec, out.aux_loss
    if not p.has_final_layer:
      return dec_outputs, aux_loss
    if p.scale_decoder_outputs:
      dec_outputs = dec_outputs * (p.builder.model_dim**-0.5)
    return NestedMap(dec_outputs=dec_outputs, aux_loss=aux_loss)

  def _ComputeLogits(self, theta, dec_outputs):
    p = self.params
    w = theta.dec_emb.embedding.to(dec_outputs.dtype)    # [V, M]
    from lingvo_b200.ops import gemm
    logits = gemm.gemm(dec_outputs.reshape(-1, dec_outputs.shape[-1]), w,
                       True, True) if (ops.use_cuda_kernels(dec_outputs) and
                                       dec_outputs.dtype == torch.bfloat16 and
                                       not torch.is_grad_enabled()) else (
                                           torch.matmul(dec_outputs, w.t()))
    logits = logits.reshape(list(dec_outputs.shape[:-1]) + [w.shape[0]])
    if p.has_final_layer and p.softmax_bias:
      logits = logits + theta.softmax_bias.to(logits.dtype)
    if p.softmax_logit_cap and p.softmax_logit_cap > 0:
      logits = p.softmax_logit_cap * torch.tanh(logits / p.softmax_logit_cap)
    if p.logits_abs_max is not None:
      logits = logits.clamp(-p.logits_abs_max, p.logits_abs_max)
    return logits

  def _ComputeNonPadding(self, input_batch):
    tgt = input_batch.tgt
    if 'paddings' in tgt:
      return (1.0 - tgt.paddings.float())
    non_padding = (tgt.segment_ids != 0).float()
    return non_padding * (tgt.labels > 0).float()

  # ----------------------------------------------------------------- loss --
  def ComputeLoss(self, theta, predictions, input_batch):
    p = self.params
    input_batch = self._ComputeInputBatch(input_batch)
    tgt = input_batch.tgt
    v = p.vocab_size
    aux_loss = predictions.aux_loss
    x = predictions.dec_outputs
    labels = tgt.labels.long().clamp(min=0)
    non_padding = self._ComputeNonPadding(input_batch)
    stats = None
    if (p.fused_xent and ops.use_cuda_kernels(x) and x.dtype == torch.bfloat16
        and p.logits_abs_max is None and not p.softmax_logit_cap and
        not p.softmax_bias):
      from lingvo_b200.ops import xent as xent_ops
      stats = xent_ops.lm_head_xent(
          x.reshape(-1, x.shape[-1]), theta.dec_emb.embedding.to(x.dtype),
          labels.reshape(-1), p.label_smoothing, p.z_loss)
    if stats is None:
      logits = self._ComputeLogits(theta, x).float()
      lse = torch.logsumexp(logits, -1)
      true_logit = torch.gather(logits, -1, labels.unsqueeze(-1)).squeeze(-1)
      entropy = lse - true_logit
      off = p.label_smoothing / v
      on = 1.0 - p.label_smoothing + off
      # xent with soft labels: lse − Σ soft·logit
      soft_dot = (on - off) * true_logit + off * logits.sum(-1)
      loss = lse - soft_dot
      zinc = p.z_loss * lse.square() if p.z_loss else torch.zeros_like(lse)
      top1 = logits.argmax(-1)
    else:
      shape = labels.shape
      entropy = stats.entropy.reshape(shape)
      loss = stats.soft_xent.reshape(shape)
      zinc = stats.z_inc.reshape(shape)
      top1 = stats.argmax.reshape(shape)
    soft_labels_entropy = loss
    loss = loss + zinc
    acc1 = (tgt.labels.long() == top1).float()
    per_token_loss = loss * non_padding
    if p.loss_denominator:
      denom = float(p.loss_denominator)
    elif p.use_tgt_labels_size_as_loss_denominator:
      denom = float(non_padding.numel())
    else:
      denom = non_padding.sum()
    avg_loss = per_token_loss.sum() / denom
    avg_z = (zinc * non_padding).sum() / denom if p.z_loss else torch.zeros(
        (), device=loss.device)
    np_sum = non_padding.sum()
    safe = torch.clamp(np_sum, min=1.0)
    avg_loss = avg_loss + p.aux_loss_coef * aux_loss
    num_items = tgt.segment_ids.amax(dim=1).sum().float()
    num_nonpad = (tgt.segment_ids != 0).float().sum()
    whole = ((acc1 * non_padding).sum(1) == non_padding.sum(1)).float()
    one = torch.ones((), device=loss.device)
    metrics = {
        'num_packed_examples': (num_items, one),
        'batch_utilized_ratio': (num_nonpad / float(tgt.labels.numel()), one),
        'acc1': ((acc1 * non_padding).sum() / safe, np_sum),
        'whole_tgt_accuracy': (whole.mean(), one),
        'mean_xent': ((entropy * non_padding).sum() / safe, np_sum),
        'soft_labels_xent': ((soft_labels_entropy * non_padding).sum() / safe,
                             np_sum),
        'weight': (np_sum, one),
        'loss': (avg_loss, one),
        'aux_loss': (p.aux_loss_coef * aux_loss, one),
        'avg_z_loss_increment': (avg_z, one),
    }
    per_step = {'loss': avg_loss.reshape(1)}
    return metrics, per_step

  def FilterPerExampleTensors(self, per_step):
    return per_step if self.params.debug else {}

  # --------------------------------------------------------------- decode --
  def InitDecodeState(self, batch, max_len, device):
    return self.dec.InitDecodeState(batch, max_len, device, self.fprop_dtype)

  def _EmbedDecodeIds(self, theta, ids, pos):
    """Token + positional embedding of ids `[B, L]` at positions `[B, L]`."""
    p = self.params
    fd = self.fprop_dtype
    y = self.dec_emb.FProp(theta.dec_emb, ids).to(fd)
    if p.positional_embedding:
      if p.sinusoid_positional_embedding:
        y = y + self.dec_pos_emb.FPropWithPosition(theta.dec_pos_emb, pos).to(fd)
      else:
        y = y + self.dec_pos_emb.FProp(theta.dec_pos_emb, pos).to(fd)
    return y

  def _DecodeLogits(self, theta, out):
    p = self.params
    if p.scale_decoder_outputs:
      out = out * (p.builder.model_dim ** -0.5)
    return self._ComputeLogits(theta, out).float()

  def DecodeStep(self, theta, ids, state, t):
    """ids `[B]` at position t → logits `[B, V]` (fp32); updates `state` in place."""
    ids = ids.reshape(-1, 1)
    pos = torch.as_tensor(t, device=ids.device).reshape(1, 1).expand(ids.shape[0], 1)
    y = self._EmbedDecodeIds(theta, ids, pos)
    out = self.dec.ExtendStep(theta.dec, y, state, t)
    return self._DecodeLogits(theta, out).squeeze(1)

  def Prefill(self, theta, ids, segment_id, segment_pos, state):
    """Writes a prompt `ids [B, P]` (padding: segment id 0) into the caches of `state` (from
    `InitDecodeState`) in one pass through the stack. No LM head runs on the prompt."""
    y = self._EmbedDecodeIds(theta, ids, segment_pos)
    self.dec.Prefill(theta.dec, y, segment_id, segment_pos, state)

  def BeamDecodeStep(self, theta, ids, pos, state, slot0, vis):
    """One flat-beam-search step after `Prefill`: ids `[B, K]` at positions `pos [B, K]`,
    appended at cache rows slot0 … slot0+K-1; hypothesis k sees the rows of its bit mask
    `vis [B, K, ⌈N/32⌉]`. Returns logits `[B, K, V]` (fp32)."""
    y = self._EmbedDecodeIds(theta, ids, pos)
    out = self.dec.BeamExtendStep(theta.dec, y, state, slot0, vis, pos)
    return self._DecodeLogits(theta, out)

  def Decode(self, input_batch):
    """Greedy / sampled decode of continuations (see gshard_decode)."""
    from lingvo_b200.core import gshard_decode
    return gshard_decode.DecodeIds(self, self.theta, input_batch)

  def BeamDecode(self, input_batch):
    """Flat beam search of continuations with `decoder_beam_size` hypotheses."""
    from lingvo_b200.core import gshard_decode
    return gshard_decode.BeamDecodeIds(self, self.theta, input_batch)


class TunableUniTransformer(UniTransformer):
  """UniTransformer whose stack is `top_layer_types` + repeated `sub_layer_types` +
  `bottom_layer_types` (reference :5001), e.g. dense layers at both ends and MoE in the
  middle."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('top_layer_types', None, 'Layer types of the first layers.')
    p.Define('bottom_layer_types', None, 'Layer types of the last layers.')
    return p

  def __init__(self, params):
    p = params
    if p.top_layer_types and p.bottom_layer_types:
      n_mid = (p.num_transformer_layers * 2 - len(p.top_layer_types) -
               len(p.bottom_layer_types))
      if not p.sub_layer_types or n_mid % len(p.sub_layer_types) != 0:
        raise ValueError('Undivided Sub-layer types length!')
      params = p.Copy()
      params.sub_layer_types = (list(p.top_layer_types) +
                                list(p.sub_layer_types) * (n_mid // len(p.sub_layer_types)) +
                                list(p.bottom_layer_types))
      params.moe = True
    super().__init__(params)


class LifelongUniTransformer(UniTransformer):
  """UniTransformer for continual training with `DenseLifelongBuilder` (reference :4643).

  With `builder.lwf_scale > 0` and `builder.e_dim_old` set, a frozen copy of the previous
  stage's model (`old`, `e_dim_old` experts, restored from its checkpoint by the caller
  via `LoadOldModel`) is run on the same batch and the KL between the two output
  distributions is added to the loss (learning without forgetting)."""

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    bp = p.builder
    self._has_old = bool('lwf_scale' in bp and bp.lwf_scale and bp.e_dim_old)
    if self._has_old:
      old = p.Copy()
      old.name = 'old'
      old.cls = UniTransformer
      old_dict = {k: v for k, v in old.IterParams()}
      op = UniTransformer.Params()
      for k, v in old_dict.items():
        if k in op and k != 'cls':
          op.Set(**{k: v})
      ob = DenseBuilder.Params()
      for k, v in bp.IterParams():
        if k in ob and k != 'cls':
          ob.Set(**{k: v})
      ob.e_dim = bp.e_dim_old
      op.builder = ob
      op.name = 'old'
      self.CreateChild('old', op)

  def _InstantiateSelfAndChildren(self):
    super()._InstantiateSelfAndChildren()
    if self._has_old:
      for v in self.old.vars.Flatten():
        v.requires_grad_(False)

  def LoadOldModel(self, state):
    """Copies a NestedMap of tensors (same structure as `self.old.vars`) into the frozen
    old model."""
    with torch.no_grad():
      for dst, src in zip(self.old.vars.Flatten(), state.Flatten()):
        dst.copy_(src)

  def ComputeLoss(self, theta, predictions, input_batch):
    metrics, per_step = super().ComputeLoss(theta, predictions, input_batch)
    if not self._has_old or self.do_eval:
      return metrics, per_step
    p = self.params
    with torch.no_grad():
      old_pred = self.old.ComputePredictions(self.old.theta, input_batch)
      old_logits = self.old._ComputeLogits(self.old.theta, old_pred.dec_outputs).float()
    new_logits = self._ComputeLogits(theta, predictions.dec_outputs).float()
    non_padding = self._ComputeNonPadding(self._ComputeInputBatch(input_batch))
    kl = (torch.softmax(old_logits, -1) *
          (torch.log_softmax(old_logits, -1) - torch.log_softmax(new_logits, -1))).sum(-1)
    lwf = (kl * non_padding).sum() / non_padding.sum().clamp_min(1.0)
    one = torch.ones((), device=lwf.device)
    total = metrics['loss'][0] + p.builder.lwf_scale * lwf
    metrics['lwf_loss'] = (lwf, one)
    metrics['loss'] = (total, one)
    per_step['loss'] = total.reshape(1)
    return metrics, per_step


class BertTransformer(base_model.BaseTask):
  """Encoder-only masked-LM Transformer on the GShard builder (reference :5054).

  Input batch: `ids, segment_ids, segment_pos` (+ `paddings`); either pre-masked
  (`masked_ids`, `masked_pos`) or masked on the fly by `masked_lm`. The loss is the
  (label-smoothed, z-regularised) cross entropy at the masked positions; the softmax
  shares the embedding matrix."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('builder', None, 'GShard builder params.')
    p.Define('vocab_size', None, 'Vocabulary size.')
    p.Define('sequence_length', None, 'Sequence length.')
    p.Define('max_length', 512, 'Positional table size.')
    p.Define('batch_size', None, 'Unused.')
    p.Define('num_transformer_layers', None, 'Number of blocks.')
    p.Define('loss_denominator', 0, 'Fixed loss denominator if > 0.')
    p.Define('aux_loss_coef', 0.01, 'Multiplier of the MoE aux loss.')
    p.Define('label_smoothing', 0.1, 'Label smoothing.')
    p.Define('logits_abs_max', None, 'Logits clipping.')
    p.Define('z_loss', 1e-4, 'z_loss · logsumexp(logits)².')
    p.Define('positional_embedding', True, 'Learned positions (else relative bias).')
    p.Define('gated_ffn_activation', None, 'silu|gelu|None.')
    p.Define('use_repeat_layer', False, 'Kept for parity.')
    p.Define('num_spmd_pipeline_stages', 1, 'SPMD pipeline stages.')
    p.Define('num_spmd_pipeline_microbatches', None, 'SPMD micro-batches.')
    p.Define('moe', False, 'Mixture-of-Experts model.')
    p.Define('moe_gated_gelu', False, 'GLU experts.')
    p.Define('activation', 'relu', 'Non-gated FFN activation.')
    p.Define('mlm_loss_weight', 1.0, 'Weight of the masked-LM loss.')
    p.Define('masked_lm', layers.MaskedLmDataAugmenter.Params(), 'On-the-fly masking.')
    p.Define('mask_token_id', 0, 'Id of the [MASK] token.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    if p.mlm_loss_weight > 0:
      self.CreateChild('masked_lm', p.masked_lm.Copy().Set(
          vocab_size=p.vocab_size, mask_token_id=p.mask_token_id))
    assert p.num_transformer_layers % p.num_spmd_pipeline_stages == 0
    b = p.builder.Instantiate()
    self.CreateChild('enc_emb', b.Embedding('enc_emb', p.vocab_size))
    if p.positional_embedding:
      self.CreateChild('enc_pos_emb', b.Embedding('enc_pos_emb', p.max_length))
      atten = b.SelfAttention('self_attention')
    else:
      atten = b.SelfAttentionRelativeBias('dec_self_attention')
    if p.gated_ffn_activation:
      ffw = b.DenseReluDenseGated('dense_relu_dense', p.gated_ffn_activation)
    else:
      ffw = b.DenseReluDense('dense_relu_dense', activation=p.activation)
    if p.moe:
      moe = b.MoEGated('moe') if p.moe_gated_gelu else b.MoE('moe')
      subs, num = [atten, moe, atten, ffw], p.num_transformer_layers // 2
    else:
      subs, num = [atten, ffw], p.num_transformer_layers
    enc = b.EncoderLayerStack('encoder', subs, num)
    enc.params_init = WeightInit.Xavier(scale=1.0, seed=0)
    self.CreateChild('enc', enc)
    bp = b.params
    self.CreateChild('emb_w_split', b.MeshSplit('w_split', bp.emb_w_split))
    self.CreateChild('enc_out_split', b.MeshSplit('enc_out_split', bp.blm_split))
    self.CreateChild('logits_split', b.MeshSplit('logits_split', bp.logits_split))

  def _ComputeNonPadding(self, input_batch):
    if 'paddings' in input_batch:
      return 1.0 - input_batch.paddings.float()
    return (input_batch.segment_ids != 0).float() * (input_batch.ids > 0).float()

  def _ComputeEncInput(self, theta, input_batch):
    p = self.params
    maskables = self._ComputeNonPadding(input_batch)
    if 'masked_pos' in input_batch:
      emb_ids, masked_pos = input_batch.masked_ids, input_batch.masked_pos.float()
    elif p.mlm_loss_weight > 0:
      emb_ids, masked_pos = self.masked_lm.FProp(theta.masked_lm, input_batch.ids,
                                                 1.0 - maskables)
    else:
      emb_ids, masked_pos = input_batch.ids, 1.0 - maskables
    fd = self.fprop_dtype
    y = self.enc_emb.FProp(theta.enc_emb, emb_ids.long()).to(fd)
    if p.positional_embedding:
      y = y + self.enc_pos_emb.FProp(theta.enc_pos_emb, input_batch.segment_pos.long()).to(fd)
    out = NestedMap(vec=y, segment_id=input_batch.segment_ids.long(),
                    segment_pos=input_batch.segment_pos.long(), masked_pos=masked_pos,
                    aux_loss=torch.zeros((), device=y.device))
    if p.moe and p.builder.gating_func == 'hashing':
      out.expert_id = emb_ids.long() % p.builder.e_dim
    return out

  def ComputePredictions(self, theta, input_batch):
    p = self.params
    enc_in = self._ComputeEncInput(theta, input_batch)
    out = self.enc.FProp(theta.enc, enc_in)
    x = out.vec * (p.builder.model_dim ** -0.5)
    w = theta.enc_emb.embedding.to(x.dtype)
    logits = torch.matmul(x, w.t())
    if p.logits_abs_max is not None:
      logits = logits.clamp(-p.logits_abs_max, p.logits_abs_max)
    return NestedMap(mlm_logits=logits, mlm_masked_pos=enc_in.masked_pos,
                     aux_loss=out.aux_loss)

  def ComputePerTokenLoss(self, logits, input_batch):
    """Smoothed xent (+ z-loss) at every non-padded position."""
    p = self.params
    logits = logits.float()
    lse = torch.logsumexp(logits, -1)
    labels = input_batch.ids.long().clamp_min(0)
    true_logit = logits.gather(-1, labels.unsqueeze(-1)).squeeze(-1)
    off = p.label_smoothing / p.vocab_size
    on = 1.0 - p.label_smoothing + off
    loss = lse - ((on - off) * true_logit + off * logits.sum(-1))
    if p.z_loss > 0:
      loss = loss + p.z_loss * lse.square()
    return loss * self._ComputeNonPadding(input_batch)

  def ComputeLoss(self, theta, predictions, input_batch):
    p = self.params
    logits = predictions.mlm_logits.float()
    ids = input_batch.ids.long()
    lse = torch.logsumexp(logits, -1)
    true_logit = logits.gather(-1, ids.clamp_min(0).unsqueeze(-1)).squeeze(-1)
    entropy = lse - true_logit
    off = p.label_smoothing / p.vocab_size
    on = 1.0 - p.label_smoothing + off
    soft_xent = lse - ((on - off) * true_logit + off * logits.sum(-1))
    zinc = p.z_loss * lse.square() if p.z_loss > 0 else torch.zeros_like(lse)
    loss = soft_xent + zinc
    acc1 = (logits.argmax(-1) == ids).float()
    non_padding = self._ComputeNonPadding(input_batch)
    masked = non_padding * predictions.mlm_masked_pos.to(non_padding.dtype)
    n_masked = masked.sum()
    safe = n_masked.clamp_min(1.0)
    denom = float(p.loss_denominator) if p.loss_denominator else safe
    avg = (loss * masked).sum() / denom
    total = p.mlm_loss_weight * avg + p.aux_loss_coef * predictions.aux_loss
    one = torch.ones((), device=logits.device)
    n_items = input_batch.segment_ids.amax(dim=1).sum().float()
    metrics = {
        'num_packed_examples': (n_items, one),
        'batch_utilized_ratio': ((input_batch.segment_ids != 0).float().mean(), one),
        'acc1': ((acc1 * masked).sum() / safe, n_masked),
        'mean_xent': ((entropy * masked).sum() / safe, n_masked),
        'soft_labels_xent': ((soft_xent * masked).sum() / safe, n_masked),
        'num_masked': (n_masked, one),
        'loss': (total, one),
        'mlm_loss': (avg, one),
        'aux_loss': (p.aux_loss_coef * predictions.aux_loss, one),
        'avg_z_loss_increment': ((zinc * masked).sum() / safe, one),
    }
    return metrics, {'loss': total.reshape(1)}

  def Decode(self, input_batch):
    """Eval-as-decode: returns per-example masked accuracy."""
    with torch.no_grad():
      pred = self.ComputePredictions(self.theta, input_batch)
      masked = self._ComputeNonPadding(input_batch) * pred.mlm_masked_pos
      hit = (pred.mlm_logits.argmax(-1) == input_batch.ids.long()).float() * masked
    return NestedMap(acc1=hit.sum(1) / masked.sum(1).clamp_min(1.0), num_masked=masked.sum(1))

  def CreateDecoderMetrics(self):
    from lingvo_b200.core import metrics as metrics_lib
    return {'acc1': metrics_lib.AverageMetric()}

  def PostProcessDecodeOut(self, dec_out, dec_metrics):
    for a, n in zip(dec_out.acc1.tolist(), dec_out.num_masked.tolist()):
      if n > 0:
        dec_metrics['acc1'].Update(a, n)
    return []
