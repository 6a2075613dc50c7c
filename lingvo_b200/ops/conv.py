"""Fused GLU + depthwise conv1d of the Conformer conv module (SURVEY K10)."""

from __future__ import annotations

import torch
import torch.nn.functional as F

from lingvo_b200 import ops


def glu_dwconv1d_ref(proj, w, paddings, causal=False):
  """PyTorch oracle. proj [B,T,2D] = (gated | act); w [K,D]; paddings [B,T]."""
  k, d = w.shape
  gated, act = proj.float().chunk(2, -1)
  m = (1.0 - paddings.float()).unsqueeze(-1)
  g = act * torch.sigmoid(gated) * m
  left = k - 1 if causal else (k - 1) // 2
  x = F.pad(g.transpose(1, 2), (left, k - 1 - left))            # [B, D, T+K-1]
  y = F.conv1d(x, w.float().t().unsqueeze(1), groups=d)        # [B, D, T]
  return (y.transpose(1, 2) * m).to(proj.dtype)


class _GluDwConvFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, proj, w, pad, left):
    nat = ops.native()
    ctx.save_for_backward(proj, w, pad)
    ctx.left = left
    return nat.glu_dwconv1d_fwd(proj, w, pad, left)

  @staticmethod
  def backward(ctx, dy):
    proj, w, pad = ctx.saved_tensors
    dproj, dw = ops.native().glu_dwconv1d_bwd(proj, w, pad, dy.contiguous(), ctx.left)
    return dproj, dw, None, None


def glu_dwconv1d_supported(x, conv_layer):
  """True when the fused kernel serves this depthwise conv layer. Kernel sizes above the
  backward's shared-memory limit (`glu_dwconv_max_k`) take the unfused path."""
  p = conv_layer.params
  import os  # pylint: disable=g-import-not-at-top
  if os.environ.get('LINGVO_B200_DISABLE_FUSED_CONV') == '1':   # A/B switch for benchmarks
    return False
  return (ops.use_cuda_kernels(x) and x.dtype in (torch.bfloat16, torch.float32) and
          type(conv_layer).__name__ in ('DepthwiseConv2DLayer',
                                        'CausalDepthwiseConv2DLayer') and
          p.filter_shape[1] == 1 and p.filter_shape[3] == 1 and
          tuple(p.filter_stride) == (1, 1) and tuple(p.dilation_rate) == (1, 1) and
          not p.bias and not p.partial_conv and
          p.filter_shape[0] <= ops.native().glu_dwconv_max_k)


def glu_dwconv1d(proj, w, paddings, causal=False):
  """y = (1-pad)·dwconv1d(act·σ(gated)·(1-pad)); one kernel fwd, one bwd."""
  k = w.shape[0]
  left = k - 1 if causal else (k - 1) // 2
  if not ops.use_cuda_kernels(proj):
    return glu_dwconv1d_ref(proj, w, paddings, causal)
  return _GluDwConvFn.apply(proj.contiguous(), w.float().contiguous(),
                            paddings.float().contiguous(), left)
