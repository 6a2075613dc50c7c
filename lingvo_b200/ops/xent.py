"""Fused LM-head softmax cross-entropy (csrc/xent_kernels.cu + wgmma GEMM).

`lm_head_xent(x, w, labels, label_smoothing, z_loss)` computes, per token,
the hard-label xent, the label-smoothed xent, the z-loss increment and the
argmax **without materialising any fp32 `[T, V]` tensor**: logits are one
bf16 GEMM output, statistics are one pass, and the backward pass rewrites the
logits buffer in place with `dlogits` before two more GEMMs (dx, dW).
"""

import torch

from lingvo_b200 import ops
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.ops import gemm


def available() -> bool:
  mod = ops.native(required=False)
  return mod is not None and hasattr(mod, '_has_xent')


class _LmHeadXent(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, w, labels, label_smoothing, z_loss):
    nat = ops.native()
    logits = gemm.gemm(x, w, True, True)                   # [T, V] bf16
    lse, true_logit, sum_logits, argmax = nat.xent_stats(logits, labels)
    v = w.shape[0]
    off = label_smoothing / v
    on = 1.0 - label_smoothing + off
    entropy = lse - true_logit
    soft = lse - ((on - off) * true_logit + off * sum_logits)
    zinc = z_loss * lse * lse
    ctx.save_for_backward(x, w, logits, labels, lse)
    ctx.consts = (on, off, z_loss)
    ctx.mark_non_differentiable(argmax)
    return entropy, soft, zinc, argmax

  @staticmethod
  def backward(ctx, d_ent, d_soft, d_z, _):
    x, w, logits, labels, lse = ctx.saved_tensors
    on, off, z = ctx.consts
    zeros = torch.zeros_like(lse)
    d_ent = zeros if d_ent is None else d_ent.float()
    d_soft = zeros if d_soft is None else d_soft.float()
    d_z = zeros if d_z is None else d_z.float()
    v = w.shape[0]
    # soft xent: lse − (on−off)·logit[y] − off·Σlogits  ⇒ Σ_v soft_label = 1
    a = d_soft + d_ent + d_z * (2.0 * z) * lse
    b = d_soft * off
    c = d_soft * (on - off) + d_ent
    ops.native().xent_bwd(logits, labels, lse, a.contiguous(), b.contiguous(),
                          c.contiguous())
    dlogits = logits                                       # rewritten in place
    dx = dw = None
    if ctx.needs_input_grad[0]:
      dx = gemm.gemm(dlogits, w, True, False)               # [T, M]
    if ctx.needs_input_grad[1]:
      dw = gemm.gemm(dlogits, x, False, False)              # [V, M]
    return dx, dw, None, None, None


def lm_head_xent(x, w, labels, label_smoothing=0.0, z_loss=0.0):
  """x `[T, M]` bf16, w `[V, M]` bf16, labels `[T]` → per-token stats."""
  entropy, soft, zinc, argmax = _LmHeadXent.apply(
      x.contiguous(), w.contiguous(), labels.long().contiguous(),
      float(label_smoothing), float(z_loss))
  return NestedMap(entropy=entropy, soft_xent=soft, z_inc=zinc, argmax=argmax)


def lm_head_xent_ref(x, w, labels, label_smoothing=0.0, z_loss=0.0):
  logits = torch.matmul(x.float(), w.float().t())
  lse = torch.logsumexp(logits, -1)
  tl = torch.gather(logits, -1, labels.long().unsqueeze(-1)).squeeze(-1)
  v = w.shape[0]
  off = label_smoothing / v
  on = 1.0 - label_smoothing + off
  return NestedMap(entropy=lse - tl,
                   soft_xent=lse - ((on - off) * tl + off * logits.sum(-1)),
                   z_inc=z_loss * lse * lse, argmax=logits.argmax(-1))


def linear_xent(inputs, w, b, class_ids):
  """Hook used by `SimpleFullSoftmax`; falls back (None) when a bias is used."""
  if b is not None:
    return None
  st = lm_head_xent(inputs, w.t().contiguous(), class_ids)
  return st.entropy, st.argmax, None
