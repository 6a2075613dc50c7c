"""MoE router logits `x[T,M]·gw[M,E]` with fp32 accumulation (csrc/gate_kernels.cu).

Replaces "upcast x to fp32 + SGEMM with N = E" (and its two SGEMM backward passes) by three
streaming kernels that read x once in bf16. `gate_logits_ref` is the fp32 oracle.
"""

import torch

from lingvo_b200 import ops

_SUPPORTED_E = (2, 4, 8, 16)


def supported(x, gw) -> bool:
  """The kernels read x with 16-byte loads, so a contiguous x must start 16-byte aligned (a
  strided x is copied first)."""
  return (ops.use_cuda_kernels(x, gw) and x.dtype == torch.bfloat16 and
          gw.device == x.device and (x.data_ptr() % 16 == 0 or not x.is_contiguous()) and
          gw.dtype in (torch.float32, torch.bfloat16) and gw.dim() == 2 and
          gw.shape[1] in _SUPPORTED_E and x.shape[-1] == gw.shape[0] and
          gw.shape[0] % 8 == 0 and gw.shape[0] * gw.shape[1] * 4 <= 200 * 1024)


class _GateLogitsFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, gw):
    x2 = x.reshape(-1, x.shape[-1])
    x2 = x2 if x2.is_contiguous() else x2.contiguous()
    gwc = gw if gw.is_contiguous() else gw.contiguous()
    ctx.save_for_backward(x2, gwc)
    ctx.x_shape = x.shape
    out = ops.native().gate_logits_fwd(x2, gwc)
    return out.reshape(*x.shape[:-1], gw.shape[1])

  @staticmethod
  def backward(ctx, dlogits):
    x2, gw = ctx.saved_tensors
    dl = dlogits.reshape(-1, gw.shape[1]).float()
    dl = dl if dl.is_contiguous() else dl.contiguous()
    dx, dgw = ops.native().gate_logits_bwd(x2, gw, dl, ctx.needs_input_grad[0],
                                           ctx.needs_input_grad[1], None)
    return (dx.reshape(ctx.x_shape) if dx is not None else None), dgw


class _GateLogitsPassFn(torch.autograd.Function):
  """(logits, x): the router reads x and so does the expert exchange; routing x through this
  node lets backward add the exchange's dx inside the router's dx kernel (no separate
  [tokens, dim] gradient add)."""

  @staticmethod
  def forward(ctx, x, gw):
    x2 = x.reshape(-1, x.shape[-1])
    x2 = x2 if x2.is_contiguous() else x2.contiguous()
    gwc = gw if gw.is_contiguous() else gw.contiguous()
    ctx.save_for_backward(x2, gwc)
    ctx.x_shape = x.shape
    ctx.set_materialize_grads(False)   # an unused output's gradient arrives as None
    out = ops.native().gate_logits_fwd(x2, gwc)
    return out.reshape(*x.shape[:-1], gw.shape[1]), x.view_as(x)

  @staticmethod
  def backward(ctx, dlogits, dpass):
    x2, gw = ctx.saved_tensors
    if dlogits is None:
      return dpass, None
    dl = dlogits.reshape(-1, gw.shape[1]).float()
    dl = dl if dl.is_contiguous() else dl.contiguous()
    dres = None
    if dpass is not None:
      dres = dpass.reshape(-1, x2.shape[1])
      dres = dres if dres.is_contiguous() else dres.contiguous()
      if dres.dtype != torch.bfloat16:
        dres = dres.to(torch.bfloat16)
      if dres.data_ptr() % 16:
        dres = dres.clone()            # the kernel reads dres with 16-byte loads
    dx, dgw = ops.native().gate_logits_bwd(x2, gw, dl, ctx.needs_input_grad[0],
                                           ctx.needs_input_grad[1], dres)
    return (dx.reshape(ctx.x_shape) if dx is not None else None), dgw


def gate_logits_pass(x, gw):
  """→ (logits, x_pass); use x_pass for every other consumer of x."""
  return _GateLogitsPassFn.apply(x, gw)


def gate_logits(x, gw):
  """x `[..., M]` bf16, gw `[M, E]` (fp32 or bf16) → fp32 logits `[..., E]`."""
  return _GateLogitsFn.apply(x, gw)


def gate_logits_ref(x, gw):
  return torch.matmul(x.float(), gw.float())
