"""Self-attention layers and stacks (ref `lingvo/core/self_attention_layer.py`):
`BlockSparseAttention` (:30), the `Builder` (:294) / `SimplifiedTransformerBuilder` (:428)
DSL for encoder stacks, and `StackedTransformerEncoderLayers` (:696)."""

from __future__ import annotations

import torch

from lingvo_b200.core import base_layer
from lingvo_b200.core import batch_major_attention as bma
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap

MultiHeadedSelfAttention = bma.MultiHeadedAttention


class BlockSparseAttention(MultiHeadedSelfAttention):
  """Block-sparse attention with the diagonal band only (ref :30; BigBird, arXiv 2007.14062,
  without global / random blocks): query block l attends to key block l and nothing else.

  H100 mapping: a block-diagonal attention *is* a batched dense attention — the `L = T / w`
  blocks are folded into the batch dimension (`[B, T, N, H] → [B·L, w, N, H]`, a free view),
  and the regular attention core (flash kernel on the device) runs on B·L short sequences.
  Cost O(T·w) instead of O(T²), and no `[B, N, L, w, w]` mask tensor is materialised: key
  padding enters as the usual additive bias of the folded batch.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('src_block_size', None, 'Query block size.')
    p.Define('tgt_block_size', None, 'Key/value block size (defaults to src_block_size).')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.src_block_size is not None, 'src_block_size is not set'
    assert p.src_block_size > 0, 'src_block_size should be greater than 0'
    assert not p.packed_input, 'packed_input is not supported'
    assert not p.use_scale_invariant_atten, 'use_scale_invariant_atten is not supported.'
    assert not p.enable_scaling_code_motion, 'enable_scaling_code_motion is not supported.'

  def FProp(self, theta, query_vec, key_vec, value_vec, paddings, segment_mask=None,
            per_step_padding=None):
    """query_vec `[B, T, D]`, key/value_vec `[B, S, D]`, paddings `[B, S]` →
    (encoded `[B, T, D]`, None)."""
    p = self.params
    assert per_step_padding is None, 'per_step_padding is not supported.'
    assert segment_mask is None, 'segment_mask is not supported.'
    wt = p.src_block_size
    ws = p.tgt_block_size or p.src_block_size
    b, t = query_vec.shape[:2]
    s = key_vec.shape[1]
    assert tuple(paddings.shape) == (b, s), (paddings.shape, b, s)
    assert t % wt == 0, 'seq_length % src_block_size != 0'
    assert s % ws == 0, 'seq_length % tgt_block_size != 0'
    nblk = t // wt
    assert s // ws == nblk, 'tgt_num_blocks != src_num_blocks'
    q, k, v = self._HeadsProj(theta, query_vec, key_vec, value_vec)
    q = self._RoPE(theta, q)
    k = self._RoPE(theta, k)
    q = self._MaybeScaleQuery(theta, q)
    fold = lambda x, w: x.reshape(b * nblk, w, *x.shape[2:])
    bias = self._Bias(paddings.reshape(b * nblk, ws), None, None)
    ctx, _ = self._Core(theta, fold(q, wt), fold(k, ws), fold(v, ws), bias, False)
    ctx = ctx.reshape(b, t, *ctx.shape[2:])
    return self._PostProj(theta, ctx), None


class Builder(bma.Builder):
  """Encoder-stack builder: pre-LN self-attention + FFN blocks (ref :294).

  `p.atten_tpl` may be a list with one attention template per layer (e.g. dense attention in
  the lower layers, `BlockSparseAttention` above). `TransformerStackV2` lets the final layer
  compute strided queries or only the first n positions (`final_layer_stride`,
  `final_layer_first_n`): the output sequence — vec and paddings — shrinks accordingly, which
  is how sequence-summary encoders avoid computing positions nobody reads.
  """

  def _AttenTplFor(self, layer_idx):
    tpl = self.params.atten_tpl
    if isinstance(tpl, (list, tuple)):
      assert layer_idx is not None, 'layer_idx must be specified.'
      return tpl[layer_idx]
    return tpl

  def _LayerBuilder(self, layer_idx):
    """A builder identical to this one but with the layer's own attention template."""
    tpl = self._AttenTplFor(layer_idx)
    if tpl is self.params.atten_tpl:
      return self
    return self.params.Copy().Set(atten_tpl=tpl.Copy()).Instantiate()

  def SelfAttention(self, name, is_causal=False, num_heads=None, layer_idx=None):
    return bma.Builder.SelfAttention(self._LayerBuilder(layer_idx), name, is_causal, num_heads)

  def _StridedAttention(self, name, stride=1, first_n=None, num_heads=None, layer_idx=None):
    """Self-attention whose queries are strided / truncated; paddings follow (ref
    batch_major_attention.Builder._StridedAttention)."""
    inner = bma.Builder.SelfAttention(self._LayerBuilder(layer_idx), name, False, num_heads)
    if stride == 1 and first_n is None:
      return inner
    return _StridedSelfAtten.Params().Set(name=name, body=inner, stride=stride, first_n=first_n)

  def _TransformerLayerBlock(self, name, feed_forward_qdomain=None, layer_idx=None):
    del feed_forward_qdomain
    return self._Seq(name, self.SelfAttention('self_atten', layer_idx=layer_idx),
                     self.Feedforward('ff'))

  def _CheckTplList(self, num_layers):
    tpl = self.params.atten_tpl
    if isinstance(tpl, (list, tuple)):
      assert len(tpl) == num_layers, 'atten_tpl list must have the same length as num_layers.'

  def TransformerStack(self, name, num_layers=1, feed_forward_qdomain=None):
    self._CheckTplList(num_layers)
    return self._Seq(name, *[
        self._Seq('iter_%03d' % i, self._TransformerLayerBlock(
            'block', feed_forward_qdomain=feed_forward_qdomain, layer_idx=i))
        for i in range(num_layers)])

  def TransformerStackV2(self, name, num_layers=1, *, final_layer_first_n=None,
                         final_layer_stride=1, feed_forward_qdomain=None):
    del feed_forward_qdomain
    self._CheckTplList(num_layers)
    blocks = []
    for i in range(num_layers):
      last = i == num_layers - 1
      stride, first_n = (final_layer_stride, final_layer_first_n) if last else (1, None)
      blocks.append(self._Seq('iter_%03d' % i, self._Seq(
          'block', self._StridedAttention('self_atten', stride=stride, first_n=first_n,
                                          layer_idx=i),
          self.Feedforward('ff'))))
    return self._Seq(name, *blocks)


class _StridedSelfAtten(base_layer.BaseLayer):
  """Runs a `Builder.SelfAttention` block and keeps every `stride`-th (or the first n)
  position of its output: residual, vec, paddings and segment mask shrink together."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('body', None, 'Self-attention block params (NestedMap in/out).')
    p.Define('stride', 1, 'Keep every stride-th position.')
    p.Define('first_n', None, 'Keep only the first n positions.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self.CreateChild('body', self.params.body)

  def FProp(self, theta, i):
    p = self.params
    o = self.body.FProp(theta.body, i)
    sel = (lambda x: x[:, :p.first_n]) if p.first_n is not None else (
        lambda x: x[:, ::p.stride])
    out = NestedMap(vec=sel(o.vec), paddings=sel(o.paddings))
    if 'segment_mask' in o and o.segment_mask is not None:
      m = o.segment_mask
      out.segment_mask = (m[:, :, :p.first_n, :p.first_n] if p.first_n is not None
                          else m[:, :, ::p.stride, ::p.stride])
    return out


class _SimplifiedBlock(base_layer.BaseLayer):
  """One simplified transformer block (arXiv 2311.01906, ref `TransformerLayerBlock` :442).

  There is **no skip connection around attention**: `a = dropout(atten(LN(x)))` replaces x
  (shaped attention keeps signal propagation healthy instead). Then either
    * sequential: `o = a + FF(LN(a))` — the regular feed-forward block with its residual, or
    * parallel (`parallel_attention_mlp`, Fig. 10): `o = a + w·MLP(LN(x))` — attention and MLP
      read the same normalised input, so on the device their GEMMs are independent work
      that can overlap, and one LN is saved.
  Strided / first-n queries shrink vec, paddings and segment mask together.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('ln', None, 'LayerNorm params.')
    p.Define('atten', None, 'Attention params.')
    p.Define('dropout', None, 'Residual dropout params.')
    p.Define('ff', None, 'Sequential mode: Feedforward block params (NestedMap in/out).')
    p.Define('mlp', None, 'Parallel mode: MLP body params (vec → vec).')
    p.Define('mlp_residual_weight', 1.0, 'Weight of the MLP branch in parallel mode.')
    p.Define('stride', 1, 'Query stride.')
    p.Define('first_n', None, 'Only the first n queries.')
    p.Define('packed_input', False, 'Inputs carry a segment mask.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert (p.ff is None) != (p.mlp is None)
    self.CreateChild('LN', p.ln)
    self.CreateChild('atten', p.atten)
    self.CreateChild('dropout', p.dropout)
    if p.ff is not None:
      self.CreateChild('ff', p.ff)
    else:
      self.CreateChild('feedforward', p.mlp)

  def FProp(self, theta, i):
    p = self.params
    sel = (lambda x, ax=1: x.narrow(ax, 0, p.first_n)) if p.first_n is not None else (
        lambda x, ax=1: x.index_select(ax, torch.arange(0, x.shape[ax], p.stride,
                                                         device=x.device))
        if p.stride > 1 else x)
    after_ln = self.LN.FProp(theta.LN, i.vec)
    query = sel(after_ln)
    seg = i.get('segment_mask') if p.packed_input else None
    if seg is not None:
      seg = sel(seg, 2)
    att, _ = self.atten.FProp(theta.atten, query, after_ln, after_ln, i.paddings,
                              segment_mask=seg)
    att = self.dropout.FProp(theta.dropout, att)
    out = NestedMap(vec=att, paddings=sel(i.paddings))
    if seg is not None:
      out.segment_mask = sel(seg, 3)
    if p.mlp is not None:
      mlp = self.feedforward.FProp(theta.feedforward, query)
      out.vec = py_utils.ApplyPadding(out.paddings.unsqueeze(-1),
                                      att + p.mlp_residual_weight * mlp)
      return out
    return self.ff.FProp(theta.ff, out)


class SimplifiedTransformerBuilder(Builder):
  """Simplified transformer blocks (ref :428; arXiv 2311.01906): shaped attention, no skip
  connection around attention, optionally attention ∥ MLP."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('parallel_attention_mlp', False,
             'Attention and MLP are computed in parallel (Fig. 10 of the paper).')
    p.atten_tpl = bma.MultiHeadedAttention.Params().Set(enable_shaped_attention=True)
    return p

  def TransformerLayerBlock(self, name, stride=1, first_n=None, num_heads=None,
                            feed_forward_qdomain=None, layer_idx=None):
    """NestedMap(vec, paddings[, segment_mask]) → same, possibly shorter."""
    del feed_forward_qdomain
    p = self.params
    lb = self._LayerBuilder(layer_idx)
    atten = bma.Builder._MultiHeadedAtten(lb, 'atten', num_heads).Set(   # pylint: disable=protected-access
        query_stride=1, query_first_n=None)
    blk = _SimplifiedBlock.Params().Set(
        name=name, ln=self._DefaultLN('LN'), atten=atten,
        dropout=self._Dropout('dropout', p.residual_dropout_prob), stride=stride,
        first_n=first_n, packed_input=p.packed_input,
        mlp_residual_weight=p.ff_residual_weight)
    if p.parallel_attention_mlp:
      h = p.ff_hidden_dim
      blk.mlp = self._Seq(
          'feedforward', self._Linear('linear01', p.model_dim, h), self._Bias('bias01', h),
          self._Activation('act', p.ff_activation_fn),
          self._Dropout('relu_dropout', p.relu_dropout_prob),
          self._Linear('linear02', h, p.model_dim), self._Bias('bias02', p.model_dim),
          self._Dropout('dropout', p.residual_dropout_prob))
    else:
      blk.ff = self.Feedforward('ff')
    return blk

  def TransformerStack(self, name, num_layers=1, feed_forward_qdomain=None):
    self._CheckTplList(num_layers)
    return self._Seq(name, *[
        self._Seq('iter_%03d' % i, self.TransformerLayerBlock('block', layer_idx=i))
        for i in range(num_layers)])

  def TransformerStackV2(self, name, num_layers=1, *, final_layer_first_n=None,
                         final_layer_stride=1, feed_forward_qdomain=None):
    self._CheckTplList(num_layers)
    blocks = []
    for i in range(num_layers):
      last = i == num_layers - 1
      stride, first_n = (final_layer_stride, final_layer_first_n) if last else (1, None)
      blocks.append(self._Seq('iter_%03d' % i, self.TransformerLayerBlock(
          'block', stride=stride, first_n=first_n, layer_idx=i)))
    return self._Seq(name, *blocks)


class StackedTransformerEncoderLayers(base_layer.BaseLayer):
  """`Builder.TransformerStack` behind the `(vec, paddings) → (vec, paddings)` interface."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('builder', Builder.Params(), 'Builder params.')
    p.Define('num_layers', 1, 'Layers.')
    p.Define('mdl_dim', 0, 'Model dim.')
    p.Define('hidden_dim', 0, 'FFN hidden dim.')
    p.Define('num_atten_heads', 0, 'Heads.')
    p.Define('dropout_prob', 0.0, 'Dropout.')
    return p

  @classmethod
  def Cast(cls, params):
    """Converts `StackedTransformerLayers` params into this class's params (ref :700)."""
    p = cls.Params()
    for k in ('name', 'num_layers', 'mdl_dim', 'hidden_dim', 'num_atten_heads',
              'dropout_prob'):
      if k in params:
        p.Set(**{k: params.Get(k)})
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    b = p.builder.Copy().Set(model_dim=p.mdl_dim, ff_hidden_dim=p.hidden_dim,
                             num_heads=p.num_atten_heads,
                             residual_dropout_prob=p.dropout_prob).Instantiate()
    self.CreateChild('stack', b.TransformerStack('stack', p.num_layers))

  def FProp(self, theta, vec, paddings, segment_mask=None):
    i = NestedMap(vec=vec, paddings=paddings)
    if segment_mask is not None:
      i.segment_mask = segment_mask
    out = self.stack.FProp(theta.stack, i)
    return out.vec, out.paddings
