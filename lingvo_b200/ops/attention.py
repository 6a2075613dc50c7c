"""Attention core shared by every attention layer (SURVEY K7/K8).

`dot_product_attention` takes batch-major `[B, T, N, H]` projections plus an
additive fp32/bf16 bias broadcastable to `[B, N, T, S]` (padding, causal,
segment and relative-position terms are all folded into that one bias, the way
the reference adds them to the logits, ref
`lingvo/core/batch_major_attention.py:943-1044`).

Dispatch:
  * CUDA, no probabilities requested, no logit cap / extra logit → fused
    flash-style kernel (online softmax; logits never reach HBM).
  * otherwise → explicit fp32-softmax path (also the numerics oracle).
"""

from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn.functional as F


def _ExpandKv(k, n):
  """GQA/MQA: repeat kv heads up to `n` query heads."""
  hk = k.shape[2]
  if hk == n:
    return k
  if hk == 1:
    return k.expand(k.shape[0], k.shape[1], n, k.shape[3])
  return k.repeat_interleave(n // hk, dim=2)


def attention_ref(q, k, v, bias=None, scale=1.0, logit_cap=0.0,
                  extra_logit=None, dropout_prob=0.0, return_probs=False):
  """Explicit softmax(q·kᵀ·scale + bias)·v with fp32 logits."""
  n = q.shape[2]
  k, v = _ExpandKv(k, n), _ExpandKv(v, n)
  logits = torch.einsum('BTNH,BSNH->BNTS', q.float(), k.float())
  if scale != 1.0:
    logits = logits * scale
  if logit_cap and logit_cap > 0:
    logits = logit_cap * torch.tanh(logits / logit_cap)
  if bias is not None:
    logits = logits + bias.float()
  if extra_logit is not None:
    extra = torch.full_like(logits[..., :1], float(extra_logit))
    probs = torch.softmax(torch.cat([logits, extra], -1), -1)[..., :-1]
  else:
    probs = torch.softmax(logits, -1)
  pd = probs.to(v.dtype)
  if dropout_prob:
    pd = F.dropout(pd, dropout_prob, training=True)
  ctx = torch.einsum('BNTS,BSNH->BTNH', pd, v)
  return (ctx, probs) if return_probs else ctx


def dot_product_attention(q, k, v, bias=None, scale=1.0, logit_cap=0.0,
                          extra_logit=None, dropout_prob=0.0,
                          return_probs=False):
  """`[B,T,N,H]` × `[B,S,Nkv,H]` → context `[B,T,N,H]` (and probs if asked)."""
  fused = (q.is_cuda and not return_probs and not logit_cap and
           extra_logit is None and q.dtype in (torch.bfloat16, torch.float16))
  if not fused:
    return attention_ref(q, k, v, bias, scale, logit_cap, extra_logit,
                         dropout_prob, return_probs)
  n = q.shape[2]
  k, v = _ExpandKv(k, n), _ExpandKv(v, n)
  b, t, s = q.shape[0], q.shape[1], k.shape[1]
  mask = None
  if bias is not None:
    mask = bias.to(q.dtype)
    if mask.dim() < 4:
      mask = mask.reshape((1,) * (4 - mask.dim()) + tuple(mask.shape))
    mask = mask.expand(b, n, t, s)
  o = F.scaled_dot_product_attention(
      q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=mask,
      dropout_p=dropout_prob, scale=scale)
  return o.transpose(1, 2)


# ------------------------------------------------- relative-bias attention ----
def _RelToeplitz(rel, l):
  """rel [H, 2L-1] indexed by (i - j + L - 1) → [H, L, L] (strided view)."""
  return rel.flip(-1).unfold(-1, l, 1).flip(1)


def rel_bias_attention_ref(q, k, v, rel, mask=None, scale=1.0):
  """fp32 oracle: softmax(scale·q·kᵀ + rel[h, i-j+L-1] + mask[b,i,j])·v."""
  l = q.shape[1]
  bias = _RelToeplitz(rel.float(), l).unsqueeze(0)
  if mask is not None:
    bias = bias + mask.float().reshape(-1, 1, l, l)
  return attention_ref(q, k, v, bias, scale)


# Whether this cuDNN build accepts an additive bias together with its own causal mask
# (it then skips the fully-masked upper-triangular tiles). Probed on first use.
_CUDNN_BIAS_PLUS_CAUSAL = {'ok': None}


def _CudnnFwd(qt, kt, vt, bias, scale, causal):
  use = causal and _CUDNN_BIAS_PLUS_CAUSAL['ok'] is not False
  if use:
    try:
      res = torch.ops.aten._scaled_dot_product_cudnn_attention(
          qt, kt, vt, bias, True, 0.0, True, False, scale=scale)
      _CUDNN_BIAS_PLUS_CAUSAL['ok'] = True
      return res, True
    except RuntimeError:
      if _CUDNN_BIAS_PLUS_CAUSAL['ok'] is True:
        raise
      _CUDNN_BIAS_PLUS_CAUSAL['ok'] = False
  return torch.ops.aten._scaled_dot_product_cudnn_attention(
      qt, kt, vt, bias, True, 0.0, False, False, scale=scale), False


class _RelBiasAttnFn(torch.autograd.Function):
  """Flash attention with a learned Toeplitz bias.

  forward : `build_rel_bias` (ours) → cuDNN fused attention (library, like
            cuBLAS for plain GEMMs) producing O and the log-sum-exp.
  backward: cuDNN fused backward for dQ/dK/dV + `rel_bias_grad` (our wgmma
            kernel) for the bias-table gradient, which cuDNN cannot produce.
  """

  @staticmethod
  def forward(ctx, q, k, v, rel, mask, scale, causal):
    from lingvo_b200 import ops
    nat = ops.native()
    b, l, h, d = q.shape
    bias = nat.build_rel_bias(rel.float().contiguous(), mask, b)
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    res, cudnn_causal = _CudnnFwd(qt, kt, vt, bias, scale, causal)
    out, lse = res[0], res[1]
    ctx.save_for_backward(q, k, v, out, lse, bias, res[2], res[3], res[6], res[7])
    ctx.meta = (res[4], res[5], scale, causal, cudnn_causal)
    return out.transpose(1, 2)

  @staticmethod
  def backward(ctx, d_o):
    from lingvo_b200 import ops
    nat = ops.native()
    q, k, v, out, lse, bias, cq, ck, seed, off = ctx.saved_tensors
    max_q, max_k, scale, causal, cudnn_causal = ctx.meta
    b, l, h, d = q.shape
    d_o = d_o.contiguous()                                   # [B, L, H, D]
    dq, dk, dv = torch.ops.aten._scaled_dot_product_cudnn_attention_backward(
        d_o.transpose(1, 2), q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
        out, lse, seed, off, bias, cq, ck, max_q, max_k, 0.0, cudnn_causal, scale=scale)
    drel = None
    if ctx.needs_input_grad[3]:
      lse3 = lse.reshape(b, h, l).float().contiguous()
      drel = nat.rel_bias_grad(q, k, v, d_o, out, lse3, bias, scale, causal)
    return (dq.transpose(1, 2), dk.transpose(1, 2), dv.transpose(1, 2), drel,
            None, None, None)


def rel_bias_attention_supported(q, k, rel, dropout_prob=0.0):
  from lingvo_b200 import ops
  return (ops.use_cuda_kernels(q) and q.dtype == torch.bfloat16 and
          q.shape[-1] == 128 and q.shape[1] % 128 == 0 and
          q.shape[1] == k.shape[1] and q.shape[2] == k.shape[2] and
          not dropout_prob and rel.shape[-1] == 2 * q.shape[1] - 1)


def rel_bias_attention(q, k, v, rel, mask=None, scale=1.0, causal=False):
  """`[B,L,H,D]` self-attention with bias `rel[h, i-j+L-1] + mask[b,i,j]`.

  `causal=True` promises that `mask` hides every j > i, which lets the bias
  gradient kernel skip the upper-triangular tiles.
  """
  if not rel_bias_attention_supported(q, k, rel):
    return rel_bias_attention_ref(q, k, v, rel, mask, scale).to(q.dtype)
  if mask is not None:
    mask = mask.reshape(-1, q.shape[1], q.shape[1])
  def _View(t):   # [B,L,H,D] view with strides (*, *, D, 1), 16-byte aligned rows
    ok = (t.stride(3) == 1 and t.stride(2) == t.shape[3] and t.stride(1) % 8 == 0 and
          t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0)
    return t if ok else t.contiguous()
  return _RelBiasAttnFn.apply(_View(q), _View(k), _View(v), rel, mask,
                              float(scale), bool(causal))


# ------------------------------------------------------------ wgmma flash attention ----
def flash_attention_ref(q, k, v, rel=None, seg=None, pos=None, scale=1.0, causal=False):
  """fp32 oracle of `flash_attention`: packed-input mask built from segment ids / positions
  (visible ⇔ same non-zero segment and, if causal, pos_k <= pos_q) + Toeplitz bias."""
  b, l = q.shape[0], q.shape[1]
  dev = q.device
  if seg is None:
    seg = torch.ones(b, l, dtype=torch.int32, device=dev)
  if pos is None:
    pos = torch.arange(l, dtype=torch.int32, device=dev).unsqueeze(0).expand(b, l)
  a, c = seg.unsqueeze(-1), seg.unsqueeze(-2)
  vis = (a == c) & (a != 0)
  if causal:
    vis = vis & (pos.unsqueeze(-1) >= pos.unsqueeze(-2))
  bias = (~vis).float().unsqueeze(1) * -1e9
  if rel is not None:
    bias = bias + _RelToeplitz(rel.float(), l).unsqueeze(0)
  return attention_ref(q, k, v, bias, scale)


class _FlashAttnFn(torch.autograd.Function):
  """Our wgmma flash attention (csrc/flash_attn.cu): forward, dQ/dK/dV and the gradient
  of the relative-bias table in two kernels; no `[B,H,L,L]` tensor, no library call."""

  @staticmethod
  def forward(ctx, q, k, v, rel, seg, pos, scale, causal):
    from lingvo_b200 import ops
    out, lse = ops.native().flash_attn_fwd(q, k, v, rel, seg, pos, scale, causal)
    ctx.save_for_backward(q, k, v, out, lse, rel, seg, pos)
    ctx.meta = (scale, causal)
    return out

  @staticmethod
  def backward(ctx, d_o):
    from lingvo_b200 import ops
    q, k, v, out, lse, rel, seg, pos = ctx.saved_tensors
    scale, causal = ctx.meta
    need_drel = rel is not None and ctx.needs_input_grad[3]
    dq, dk, dv, drel = ops.native().flash_attn_bwd(
        q, k, v, out, d_o, lse, rel, seg, pos, scale, causal, need_drel)
    return dq, dk, dv, (drel if need_drel else None), None, None, None, None


def flash_attention_supported(q, k, dropout_prob=0.0):
  from lingvo_b200 import ops
  mod = ops.native(required=False) if q.is_cuda else None
  return (mod is not None and hasattr(mod, '_has_flash_attn') and
          os.environ.get('LINGVO_B200_ATTN', 'flash') == 'flash' and
          ops.use_cuda_kernels(q) and q.dtype == torch.bfloat16 and q.dim() == 4 and
          q.shape[-1] == 128 and q.shape[1] % 128 == 0 and q.shape == k.shape and
          not dropout_prob)


def flash_attention(q, k, v, rel=None, seg=None, pos=None, scale=1.0, causal=False):
  """`[B,L,H,128]` self-attention, bias `rel[h, i-j+L-1]` (fp32 `[H, 2L-1]`, optional) and
  the packed-input mask from int32 `seg` / `pos` `[B, L]` (optional). Returns `[B,L,H,128]`.

  `causal=True` additionally assumes positions grow with the index inside a segment (packed
  LM inputs), which lets both kernels skip the key blocks above the diagonal.
  """
  if not flash_attention_supported(q, k):
    return flash_attention_ref(q, k, v, rel, seg, pos, scale, causal).to(q.dtype)

  def _View(t):   # [B,L,H,D] view with strides (*, *, D, 1), 16-byte aligned rows
    ok = (t.stride(3) == 1 and t.stride(2) == t.shape[3] and t.stride(1) % 8 == 0 and
          t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0)
    return t if ok else t.contiguous()
  if rel is not None:
    rel = rel.float().contiguous()
  if seg is not None:
    seg = seg.to(torch.int32).contiguous()
  if pos is not None:
    pos = pos.to(torch.int32).contiguous()
  return _FlashAttnFn.apply(_View(q), _View(k), _View(v), rel, seg, pos, float(scale),
                            bool(causal))


# ------------------------------------------------------- incremental decoding ----
def decode_attention_ref(q, k_new, v_new, k_cache, v_cache, t, rel=None, scale=1.0):
  """fp32 oracle and CPU path of `decode_attention`: one-hot write of row t into the caches,
  fp32 logits over all T keys, −1e9 on the keys after t. Grouped / multi-query KV heads are
  expanded with `_ExpandKv`."""
  bsz, _, h, _ = q.shape
  tmax = k_cache.shape[1]
  dev = q.device
  tt = torch.as_tensor(t, device=dev).reshape(())
  onehot = (torch.arange(tmax, device=dev) == tt).to(k_cache.dtype).reshape(1, tmax, 1, 1)
  k_cache.mul_(1 - onehot).add_(k_new * onehot)
  v_cache.mul_(1 - onehot).add_(v_new * onehot)
  kk, vv = _ExpandKv(k_cache, h), _ExpandKv(v_cache, h)
  logits = torch.einsum('bqhd,bkhd->bhqk', q.float(), kk.float())      # [B,H,1,T]
  if scale != 1.0:
    logits = logits * scale
  key_pos = torch.arange(tmax, device=dev)
  if rel is not None:
    idx = (tt - key_pos + tmax - 1).clamp(0, 2 * tmax - 2)
    logits = logits + rel.float()[:, idx].reshape(1, h, 1, tmax)
  logits = logits + ((key_pos > tt).float() * -1e9).reshape(1, 1, 1, tmax)
  probs = torch.softmax(logits, -1)
  return torch.einsum('bhqk,bkhd->bqhd', probs, vv.float()).to(q.dtype)


def decode_attention_supported(q, k_cache):
  from lingvo_b200 import ops
  mod = ops.native(required=False) if q.is_cuda else None
  return (mod is not None and hasattr(mod, '_has_decode_attn') and
          ops.use_cuda_kernels(q, k_cache) and q.dtype == torch.bfloat16 and
          k_cache.dtype == torch.bfloat16 and q.dim() == 4 and k_cache.dim() == 4 and
          q.shape[-1] == 128 and k_cache.shape[-1] == 128 and
          q.shape[2] % k_cache.shape[2] == 0 and k_cache.is_contiguous())


def decode_attention(q, k_new, v_new, k_cache, v_cache, t, rel=None, scale=1.0):
  """One decode step of self-attention for a single query token per sequence.

  q `[B,1,H,D]`, k_new / v_new `[B,1,Hk,D]` (Hk divides H; query head h reads KV head
  h // (H/Hk)), caches `[B,T,Hk,D]` updated in place at row t, `t` a Python int or 0-dim
  integer tensor, `rel` an optional fp32 `[H, 2T-1]` table indexed by t − j + T − 1 (clamped
  to the table). Keys j ≤ t are visible; for t outside [0, T) no row is written and all keys
  are. Returns `[B,1,H,D]`.

  On the GPU (bf16, D = 128) this is our split-KV kernel (csrc/decode_attn.cu): it reads
  only the live rows of the cache and its launch shape does not depend on t, so a step with
  `t` as a device scalar can be captured in a CUDA graph.
  """
  if not decode_attention_supported(q, k_cache):
    return decode_attention_ref(q, k_new, v_new, k_cache, v_cache, t, rel, scale)
  from lingvo_b200 import ops
  b, _, h, d = q.shape
  hk = k_cache.shape[2]
  tt = torch.as_tensor(t, device=q.device)
  if tt.dtype not in (torch.int32, torch.int64):
    tt = tt.long()
  if rel is not None:
    rel = rel.float().contiguous()
  out = ops.native().decode_attn_fwd(
      q.reshape(b, h, d).contiguous(), k_new.reshape(b, hk, d).contiguous(),
      v_new.reshape(b, hk, d).contiguous(), k_cache, v_cache, tt.reshape(()), rel,
      float(scale))
  return out.reshape(b, 1, h, d)
