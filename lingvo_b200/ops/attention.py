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


# ------------------------------------------------------------ wgmma flash attention ----
def flash_attention_ref(q, k, v, rel=None, seg=None, pos=None, scale=1.0, causal=False,
                        logit_cap=0.0, extra_logit=None):
  """fp32 oracle of `flash_attention`: packed-input mask built from segment ids / positions
  (visible ⇔ same non-zero segment and, if causal, pos_k <= pos_q) + Toeplitz bias, both
  added after the optional cap of scale·q·k; the optional extra logit joins every softmax."""
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
  return attention_ref(q, k, v, bias, scale, logit_cap, extra_logit)


class _FlashAttnFn(torch.autograd.Function):
  """Our wgmma flash attention (csrc/flash_attn.cu): forward, dQ/dK/dV and the gradient
  of the relative-bias table in two kernels; no `[B,H,L,L]` tensor, no library call."""

  @staticmethod
  def forward(ctx, q, k, v, rel, seg, pos, scale, causal, logit_cap, extra_logit):
    from lingvo_b200 import ops
    out, lse = ops.native().flash_attn_fwd(q, k, v, rel, seg, pos, scale, causal, logit_cap,
                                           extra_logit)
    ctx.save_for_backward(q, k, v, out, lse, rel, seg, pos)
    ctx.meta = (scale, causal, logit_cap, extra_logit)
    return out

  @staticmethod
  def backward(ctx, d_o):
    from lingvo_b200 import ops
    q, k, v, out, lse, rel, seg, pos = ctx.saved_tensors
    scale, causal, logit_cap, _ = ctx.meta   # lse already counts the extra logit
    need_drel = rel is not None and ctx.needs_input_grad[3]
    dq, dk, dv, drel = ops.native().flash_attn_bwd(
        q, k, v, out, d_o, lse, rel, seg, pos, scale, causal, need_drel, logit_cap)
    return dq, dk, dv, (drel if need_drel else None), None, None, None, None, None, None


def flash_attention_supported(q, k, dropout_prob=0.0):
  from lingvo_b200 import ops
  return (ops.use_cuda_kernels(q) and q.dtype == torch.bfloat16 and q.dim() == 4 and
          q.shape[-1] == 128 and q.shape[1] % 128 == 0 and k.dim() == 4 and
          k.shape[:2] == q.shape[:2] and k.shape[3] == 128 and k.shape[2] >= 1 and
          q.shape[2] % k.shape[2] == 0 and not dropout_prob)


def flash_attention(q, k, v, rel=None, seg=None, pos=None, scale=1.0, causal=False,
                    logit_cap=0.0, extra_logit=None):
  """`[B,L,H,128]` self-attention, bias `rel[h, i-j+L-1]` (fp32 `[H, 2L-1]`, optional) and
  the packed-input mask from int32 `seg` / `pos` `[B, L]` (optional). Returns `[B,L,H,128]`.

  `logit_cap > 0` replaces scale·q·k by `logit_cap·tanh(scale·q·k / logit_cap)` before the
  bias and the mask are added. `extra_logit` (a float) adds one logit of that value, whose
  value vector is 0, to every softmax: a query that sees no key then returns exactly 0.

  k and v are `[B,L,Hk,128]` with Hk dividing H: grouped-query (Hk < H) or multi-query
  (Hk = 1) attention, where query head h reads KV head h // (H/Hk). Their gradients keep Hk
  heads, each summed over its group.

  `causal=True` additionally assumes positions grow with the index inside a segment (packed
  LM inputs), which lets both kernels skip the key blocks above the diagonal.
  """
  logit_cap = float(logit_cap or 0.0)
  if extra_logit is not None:
    extra_logit = float(extra_logit)
  if not flash_attention_supported(q, k):
    return flash_attention_ref(q, k, v, rel, seg, pos, scale, causal, logit_cap,
                               extra_logit).to(q.dtype)

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
                            bool(causal), logit_cap, extra_logit)


# ------------------------------------------------------- incremental decoding ----
def decode_attention_ref(q, k_new, v_new, k_cache, v_cache, t, rel=None, scale=1.0,
                         logit_cap=0.0, extra_logit=None):
  """fp32 oracle and CPU path of `decode_attention`: one-hot write of row t into the caches,
  fp32 logits over all T keys, −1e9 on the keys after t when t is in [0, T) (otherwise every
  key is visible, as in the kernel). Grouped / multi-query KV heads are expanded with
  `_ExpandKv`. The optional cap applies to scale·q·k before the bias and the mask, and the
  optional extra logit joins the softmax, as in `flash_attention`."""
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
  if logit_cap:
    logits = logit_cap * torch.tanh(logits / logit_cap)
  key_pos = torch.arange(tmax, device=dev)
  if rel is not None:
    idx = (tt - key_pos + tmax - 1).clamp(0, 2 * tmax - 2)
    logits = logits + rel.float()[:, idx].reshape(1, h, 1, tmax)
  masked = (key_pos > tt) & (tt >= 0) & (tt < tmax)
  logits = logits + (masked.float() * -1e9).reshape(1, 1, 1, tmax)
  if extra_logit is not None:
    extra = torch.full_like(logits[..., :1], float(extra_logit))
    probs = torch.softmax(torch.cat([logits, extra], -1), -1)[..., :-1]
  else:
    probs = torch.softmax(logits, -1)
  return torch.einsum('bhqk,bkhd->bqhd', probs, vv.float()).to(q.dtype)


def decode_attention_supported(q, k_cache):
  from lingvo_b200 import ops
  return (ops.use_cuda_kernels(q, k_cache) and q.dtype == torch.bfloat16 and
          k_cache.dtype == torch.bfloat16 and q.dim() == 4 and k_cache.dim() == 4 and
          q.shape[-1] == 128 and k_cache.shape[-1] == 128 and
          q.shape[2] % k_cache.shape[2] == 0 and k_cache.is_contiguous())


def decode_attention(q, k_new, v_new, k_cache, v_cache, t, rel=None, scale=1.0, logit_cap=0.0,
                     extra_logit=None):
  """One decode step of self-attention for a single query token per sequence.

  q `[B,1,H,D]`, k_new / v_new `[B,1,Hk,D]` (Hk divides H; query head h reads KV head
  h // (H/Hk)), caches `[B,T,Hk,D]` updated in place at row t, `t` a Python int or 0-dim
  integer tensor, `rel` an optional fp32 `[H, 2T-1]` table indexed by t − j + T − 1 (clamped
  to the table). Keys j ≤ t are visible; for t outside [0, T) no row is written and all keys
  are. `logit_cap` and `extra_logit` are those of `flash_attention`: the cap applies to
  scale·q·k before the bias and the mask. Returns `[B,1,H,D]`.

  On the GPU (bf16, D = 128, no cap, no extra logit) this is our split-KV kernel
  (csrc/decode_attn.cu): it reads only the live rows of the cache and its launch shape does
  not depend on t, so a step with `t` as a device scalar can be captured in a CUDA graph.
  With a cap or an extra logit it is `decode_attention_ref`, which is capturable too.
  """
  if logit_cap or extra_logit is not None or not decode_attention_supported(q, k_cache):
    return decode_attention_ref(q, k_new, v_new, k_cache, v_cache, t, rel, scale, logit_cap,
                                extra_logit)
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


# ------------------------------------------------------------------- flat beam search ----
def unpack_visibility(vis, n):
  """int32 `[..., ⌈n/32⌉]` bit masks (bit j%32 of word j/32 for row j) → bool `[..., n]`."""
  bits = (vis.unsqueeze(-1) >> torch.arange(32, device=vis.device, dtype=vis.dtype)) & 1
  return bits.reshape(*vis.shape[:-1], -1)[..., :n].bool()


def pack_visibility(mask):
  """bool `[..., n]` → int32 `[..., ⌈n/32⌉]` bit masks, the inverse of `unpack_visibility`."""
  n = mask.shape[-1]
  w = (n + 31) // 32
  m = F.pad(mask.to(torch.int64), (0, 32 * w - n)).reshape(*mask.shape[:-1], w, 32)
  words = (m << torch.arange(32, device=mask.device, dtype=torch.int64)).sum(-1)
  return torch.where(words >= 2**31, words - 2**32, words).to(torch.int32)


def flat_beam_attention_ref(q, k_new, v_new, k_cache, v_cache, slot0, vis, qpos, kpos, rel=None,
                            scale=1.0, logit_cap=0.0, extra_logit=None):
  """fp32 oracle and CPU path of `flat_beam_attention`: writes row slot0 + k of the caches
  from k_new / v_new[:, k], then takes fp32 logits over all N rows, applies the cap to
  scale·q·k, adds the bias (in that order, as `flash_attention` does), drops the rows that
  are not visible and adds the optional extra logit to the softmax. A query that sees no row
  returns zeros."""
  bsz, kh, h, d = q.shape
  n, hk = k_cache.shape[1], k_cache.shape[2]
  dev = q.device
  s0 = torch.as_tensor(slot0, device=dev).reshape(()).long()
  rows = torch.arange(n, device=dev)
  sel = (rows.unsqueeze(0) == s0 + torch.arange(kh, device=dev).unsqueeze(1))   # [K, N]
  written = sel.any(0).reshape(1, n, 1, 1)
  selc = sel.to(k_cache.dtype)
  k_cache.copy_(torch.where(written, torch.einsum('kn,bkhd->bnhd', selc, k_new.to(k_cache.dtype)),
                            k_cache))
  v_cache.copy_(torch.where(written, torch.einsum('kn,bkhd->bnhd', selc, v_new.to(v_cache.dtype)),
                            v_cache))
  g = h // hk
  qg = q.float().reshape(bsz, kh, hk, g, d)
  logits = torch.einsum('bkcgd,bncd->bkcgn', qg, k_cache.float()).reshape(bsz, kh, h, n)
  logits = logits * scale
  if logit_cap:
    logits = logit_cap * torch.tanh(logits / logit_cap)
  if rel is not None:
    idx = (qpos.long().unsqueeze(-1) - kpos.long().unsqueeze(1) + n - 1).clamp(0, 2 * n - 2)
    logits = logits + rel.float()[:, idx].permute(1, 2, 0, 3)                # [B,K,H,N]
  live = rows < (s0 + kh).clamp(0, n)
  visible = (unpack_visibility(vis, n) & live).unsqueeze(2)                  # [B,K,1,N]
  logits = logits.masked_fill(~visible, float('-inf'))
  if extra_logit is not None:
    extra = torch.full_like(logits[..., :1], float(extra_logit))
    probs = torch.softmax(torch.cat([logits, extra], -1), -1)[..., :-1]
  else:
    probs = torch.softmax(logits, -1).nan_to_num(0.0)
  vv = v_cache.float().unsqueeze(1).expand(bsz, kh, n, hk, d)
  out = torch.einsum('bkcgn,bkncd->bkcgd', probs.reshape(bsz, kh, hk, g, n), vv)
  return out.reshape(bsz, kh, h, d).to(q.dtype)


def flat_beam_attention_supported(q, k_cache):
  from lingvo_b200 import ops
  return (ops.use_cuda_kernels(q, k_cache) and q.dtype == torch.bfloat16 and
          k_cache.dtype == torch.bfloat16 and q.dim() == 4 and k_cache.dim() == 4 and
          1 <= q.shape[1] <= 16 and q.shape[-1] == 128 and k_cache.shape[-1] == 128 and
          q.shape[2] % k_cache.shape[2] == 0 and k_cache.is_contiguous())


def flat_beam_attention(q, k_new, v_new, k_cache, v_cache, slot0, vis, qpos, kpos, rel=None,
                        scale=1.0, logit_cap=0.0, extra_logit=None):
  """One flat-beam-search step of self-attention: K hypotheses per sequence share one token
  buffer (the caches), and each attends over its own set of rows.

  q `[B,K,H,D]`, k_new / v_new `[B,K,Hk,D]` (Hk divides H; query head h reads KV head
  h // (H/Hk)), caches `[B,N,Hk,D]` updated in place at rows slot0 + k, `slot0` a Python int
  or 0-dim integer tensor. Hypothesis k sees the rows whose bit is set in the int32 mask
  `vis[b, k]` `[B,K,⌈N/32⌉]` (see `pack_visibility`), and only rows below slot0 + K. `qpos`
  `[B,K]` and `kpos` `[B,N]` are the positions that index the optional fp32 `[H, 2N-1]` table
  `rel` at qpos − kpos + N − 1 (clamped to the table). `logit_cap` and `extra_logit` are
  those of `flash_attention`: the cap applies to scale·q·k before the bias. Returns
  `[B,K,H,D]`.

  On the GPU (bf16, D = 128, K ≤ 16, no cap, no extra logit) this is our kernel in
  csrc/decode_attn.cu: each K/V tile is read once for all hypotheses and query heads of a KV
  head, only rows below slot0 + K are read, and the launch shape does not depend on slot0,
  so a step with `slot0` as a device scalar can be captured in a CUDA graph.
  """
  if logit_cap or extra_logit is not None or not flat_beam_attention_supported(q, k_cache):
    return flat_beam_attention_ref(q, k_new, v_new, k_cache, v_cache, slot0, vis, qpos, kpos,
                                   rel, scale, logit_cap, extra_logit)
  from lingvo_b200 import ops
  s0 = torch.as_tensor(slot0, device=q.device)
  if s0.dtype not in (torch.int32, torch.int64):
    s0 = s0.long()
  if rel is not None:
    rel = rel.float().contiguous()
  return ops.native().flat_beam_attn_fwd(
      q.contiguous(), k_new.contiguous(), v_new.contiguous(), k_cache, v_cache, s0.reshape(()),
      vis.to(torch.int32).contiguous(), qpos.to(torch.int32).contiguous(),
      kpos.to(torch.int32).contiguous(), rel, float(scale))
