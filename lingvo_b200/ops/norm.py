"""Fused RMS-norm / LayerNorm (csrc/norm_kernels.cu) with autograd."""

import torch

from lingvo_b200 import ops


def available() -> bool:
  mod = ops.native(required=False)
  return mod is not None and hasattr(mod, '_has_norm')


class _NormFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, scale, bias, eps, center):
    shape = x.shape
    x2 = x.contiguous().reshape(-1, shape[-1])
    y, stats, _ = ops.native().norm_fwd(x2, None, scale, bias, eps, center, False)
    ctx.save_for_backward(x2, scale if scale is not None else torch.empty(0),
                          stats)
    ctx.center = center
    ctx.has_scale = scale is not None
    ctx.has_bias = bias is not None
    ctx.scale_dtype = scale.dtype if scale is not None else None
    ctx.bias_dtype = bias.dtype if bias is not None else None
    return y.reshape(shape)

  @staticmethod
  def backward(ctx, dy):
    x2, scale, stats = ctx.saved_tensors
    shape = dy.shape
    dy2 = dy.contiguous().reshape(-1, shape[-1])
    dx, ds, db = ops.native().norm_bwd(
        x2, dy2, None, scale if ctx.has_scale else None, stats, ctx.center,
        ctx.has_scale and ctx.needs_input_grad[1],
        ctx.has_bias and ctx.needs_input_grad[2])
    if ds is not None and ctx.scale_dtype is not None:
      ds = ds.to(ctx.scale_dtype)
    if db is not None and ctx.bias_dtype is not None:
      db = db.to(ctx.bias_dtype)
    return dx.reshape(shape), ds, db, None, None


class _NormPassFn(torch.autograd.Function):
  """(norm(x), x): the pre-norm residual pattern `x + f(norm(x))` as ONE autograd node.

  Returning x as a second output lets the residual branch take its input from this node, so
  backward receives the gradient of the normalised branch *and* the gradient flowing along
  the residual stream together and hands both to the fused kernel (`dres_in`): the
  [tokens, dim] gradient add that autograd would otherwise launch per sub-layer disappears.
  """

  @staticmethod
  def forward(ctx, x, scale, eps):
    shape = x.shape
    x2 = x.contiguous().reshape(-1, shape[-1])
    y, stats, _ = ops.native().norm_fwd(x2, None, scale, None, eps, False, False)
    ctx.save_for_backward(x2, scale if scale is not None else torch.empty(0), stats)
    ctx.has_scale = scale is not None
    ctx.scale_dtype = scale.dtype if scale is not None else None
    return y.reshape(shape), x.view_as(x)

  @staticmethod
  def backward(ctx, dy, dpass):
    x2, scale, stats = ctx.saved_tensors
    if dy is None:                      # only the residual branch was used
      return dpass, None, None
    shape = dy.shape
    dy2 = dy.contiguous().reshape(-1, shape[-1])
    dres = dpass.contiguous().reshape(-1, shape[-1]) if dpass is not None else None
    if dres is not None and dres.dtype != torch.bfloat16:
      dres = dres.to(torch.bfloat16)
    dx, ds, _ = ops.native().norm_bwd(
        x2, dy2, dres, scale if ctx.has_scale else None, stats, False,
        ctx.has_scale and ctx.needs_input_grad[1], False)
    if ds is not None and ctx.scale_dtype is not None:
      ds = ds.to(ctx.scale_dtype)
    return dx.reshape(shape), ds, None


def rms_norm(x, scale, eps):
  return _NormFn.apply(x, scale, None, float(eps), False)


def rms_norm_pass(x, scale, eps):
  """→ (rms_norm(x), x) with the residual-stream gradient add fused into the backward."""
  return _NormPassFn.apply(x, scale, float(eps))


def layer_norm(x, scale, bias, eps, center=True):
  """bf16 x → bf16 LayerNorm (center=False: no mean subtraction, as RMS norm). The bias is
  added whether or not the norm centres; without centring it is added outside the kernel."""
  if center:
    return _NormFn.apply(x, scale, bias, float(eps), True)
  y = _NormFn.apply(x, scale, None, float(eps), False)
  return y if bias is None else (y.float() + bias.float()).to(y.dtype)


def rms_norm_ref(x, scale, eps):
  xf = x.float()
  y = xf * torch.rsqrt(xf.square().mean(-1, keepdim=True) + eps)
  if scale is not None:
    y = y * scale.float()
  return y.to(x.dtype)
