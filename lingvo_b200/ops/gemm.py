"""wgmma GEMM front-end: `gemm`, and autograd-aware `linear` / `grouped_linear`.

Weights follow the reference's `[in, out]` convention (`x @ w`, SURVEY K3/K5:
`EAM,EMH->EAH`, `BLM,MH->BLH`). The three GEMMs of a linear layer map onto the
same kernel with different operand majors, so nothing is ever transposed in
HBM:
  fwd    y[M,N]  = x[M,K] @ w[K,N]        A K-major,  B MN-major
  dgrad  dx[M,K] = dy[M,N] @ w[K,N]^T     A K-major,  B K-major
  wgrad  dw[K,N] = x[M,K]^T @ dy[M,N]     A MN-major, B MN-major
"""

from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from lingvo_b200 import ops

ACT_IDS = {None: 0, 'NONE': 0, 'RELU': 1, 'GELU': 2, 'SILU': 3, 'SWISH': 3,
           'GELU_APPROXIMATE': 4, 'SQUARED_RELU': 5}
AUX_NONE, AUX_RELU_MASK, AUX_ADD = 0, 1, 2


def _act_ref(x, act):
  a = ACT_IDS[act] if not isinstance(act, int) else act
  if a == 0:
    return x
  if a == 1:
    return F.relu(x)
  if a == 2:
    return F.gelu(x)
  if a == 3:
    return F.silu(x)
  if a == 4:
    return F.gelu(x, approximate='tanh')
  if a == 5:
    return F.relu(x).square()
  raise ValueError(act)


def gemm_ref(a, b, a_kmajor=True, b_kmajor=True, bias=None, act=0, aux=None,
             aux_mode=0, row_scale=None, out_fp32=False):
  """fp32 PyTorch oracle of `gemm` (same argument meaning)."""
  a3 = a if a.dim() == 3 else a.unsqueeze(0)
  b3 = b if b.dim() == 3 else b.unsqueeze(0)
  A = a3.float() if a_kmajor else a3.float().transpose(1, 2)
  B = b3.float() if b_kmajor else b3.float().transpose(1, 2)
  y = torch.matmul(A, B.transpose(1, 2))
  if bias is not None:
    y = y + bias.float().reshape(y.shape[0], 1, -1)
  y = _act_ref(y, act)
  if aux is not None and aux_mode == AUX_RELU_MASK:
    y = y * (aux.float().reshape(y.shape) > 0)
  elif aux is not None and aux_mode == AUX_ADD:
    y = y + aux.float().reshape(y.shape)
  if row_scale is not None:
    y = y * row_scale.float().reshape(y.shape[0], -1, 1)
  if a.dim() == 2:
    y = y[0]
  return y if out_fp32 else y.to(torch.bfloat16)


def gemm(a, b, a_kmajor=True, b_kmajor=True, bias=None, act=0, aux=None,
         aux_mode=0, row_scale=None, out=None, out_fp32=False,
         accumulate=False, pre_act=None, row_ptrs=None, nblk_ptrs=None,
         a_peer_ptrs=None, nblk_ld=0):
  """C[g] = epi(A[g] · B[g]^T); see csrc/gemm_tcgen05.cu for operand layouts."""
  act = ACT_IDS[act] if not isinstance(act, int) else act
  if not ops.use_cuda_kernels(a, b):
    y = gemm_ref(a, b, a_kmajor, b_kmajor, bias, act, aux, aux_mode, row_scale,
                 out_fp32 or (out is not None and out.dtype == torch.float32))
    if out is not None:
      if accumulate:
        out.add_(y.reshape(out.shape))
      else:
        out.copy_(y.reshape(out.shape))
      return out
    return y
  res = ops.native().gemm_bf16(a, b, a_kmajor, b_kmajor, bias, act, aux,
                               aux_mode, row_scale, out, out_fp32, accumulate,
                               pre_act, row_ptrs, nblk_ptrs, a_peer_ptrs, nblk_ld)
  if out is None and a.dim() == 2:
    res = res[0]
  return res


class _LinearFn(torch.autograd.Function):
  """y = act(x @ w + b) with grouped (leading-G) or plain 2-D operands."""

  @staticmethod
  def forward(ctx, x, w, bias, act, residual=None):
    act_id = ACT_IDS[act] if not isinstance(act, int) else act
    if residual is not None:
      assert act_id == 0, 'residual epilogue needs act=None'
      y = gemm(x, w, True, False, bias=bias, aux=residual.contiguous(), aux_mode=AUX_ADD)
    else:
      y = gemm(x, w, True, False, bias=bias, act=act_id)
    ctx.has_res = residual is not None
    ctx.act_id = act_id
    ctx.has_bias = bias is not None
    if act_id not in (0, 1):
      raise NotImplementedError('fused backward supports NONE/RELU; use '
                                'linear(..., act=None) + activation for others')
    ctx.save_for_backward(x, w, y if act_id == 1 else None)
    return y

  @staticmethod
  def backward(ctx, dy):
    x, w, y = ctx.saved_tensors
    dy = dy.contiguous()
    if ctx.act_id == 1:
      # relu'(h) folded into one elementwise mask (also needed for dbias/wgrad).
      dy = torch.where(y > 0, dy, torch.zeros((), dtype=dy.dtype, device=dy.device))
    dx = dw = db = None
    if ctx.needs_input_grad[0]:
      dx = gemm(dy, w, True, True)                      # dy @ w^T
    if ctx.needs_input_grad[1]:
      dw = gemm(x, dy, False, False, out_fp32=(w.dtype == torch.float32))
      dw = dw.to(w.dtype)
    if ctx.has_bias and ctx.needs_input_grad[2]:
      db = dy.float().sum(dim=-2)
    return dx, dw, db, None, (dy if ctx.has_res else None)


def linear(x, w, bias=None, act=None, residual=None):
  """x[..., K] @ w[K, N] (+bias, act | +residual) on the wgmma path (bf16).

  `residual` (same shape as the output) is added in the GEMM epilogue — the
  sub-layer's `x + f(x)` costs no extra pass."""
  lead = x.shape[:-1]
  x2 = x.reshape(-1, x.shape[-1])
  if x2.dtype != torch.bfloat16 or w.dtype != torch.bfloat16 or not x2.is_cuda:
    y = torch.matmul(x2, w)
    if bias is not None:
      y = y + bias.to(y.dtype)
    y = _act_ref(y, act)
    if residual is not None:
      y = y + residual.reshape(y.shape).to(y.dtype)
    return y.reshape(*lead, w.shape[-1])
  r2 = residual.reshape(-1, w.shape[-1]) if residual is not None else None
  if r2 is not None and r2.dtype != torch.bfloat16:
    r2 = r2.to(torch.bfloat16)
  y = _LinearFn.apply(x2, w, bias, act, r2)
  return y.reshape(*lead, w.shape[-1])


class _LinearTFn(torch.autograd.Function):
  """y = x @ wᵀ + b for a weight stored `[N, K]` (K-major B operand)."""

  @staticmethod
  def forward(ctx, x, w, bias):
    ctx.has_bias = bias is not None
    ctx.save_for_backward(x, w)
    return gemm(x, w, True, True, bias=bias)

  @staticmethod
  def backward(ctx, dy):
    x, w = ctx.saved_tensors
    dy = dy.contiguous()
    dx = gemm(dy, w, True, False) if ctx.needs_input_grad[0] else None
    dw = gemm(dy, x, False, False) if ctx.needs_input_grad[1] else None
    db = dy.float().sum(0) if ctx.has_bias and ctx.needs_input_grad[2] else None
    return dx, dw, db


def linear_t(x, w, bias=None):
  """x[..., K] @ w[N, K]ᵀ (+bias): output projections stored `[D, N·H]`."""
  lead = x.shape[:-1]
  x2 = x.reshape(-1, x.shape[-1])
  if x2.dtype != torch.bfloat16 or w.dtype != torch.bfloat16 or not x2.is_cuda:
    y = torch.matmul(x2, w.t())
    if bias is not None:
      y = y + bias.to(y.dtype)
    return y.reshape(*lead, w.shape[0])
  return _LinearTFn.apply(x2, w, bias).reshape(*lead, w.shape[0])


def grouped_linear(x, w, bias=None, act=None):
  """x[G, M, K] @ w[G, K, N] per group (expert FFN: `EAM,EMH->EAH`)."""
  if x.dtype != torch.bfloat16 or w.dtype != torch.bfloat16 or not x.is_cuda:
    y = torch.bmm(x, w.to(x.dtype))
    if bias is not None:
      y = y + bias.to(y.dtype).unsqueeze(1)
    return _act_ref(y, act)
  return _LinearFn.apply(x, w, bias, act)


class _FfnReluFn(torch.autograd.Function):
  """y = relu(x·wi)·wo with the ReLU mask folded into the dgrad epilogue."""

  @staticmethod
  def forward(ctx, x, wi, wo, residual=None):
    h = gemm(x, wi, True, False, act=1)
    if residual is not None:
      y = gemm(h, wo, True, False, aux=residual.contiguous(), aux_mode=AUX_ADD)
    else:
      y = gemm(h, wo, True, False)
    ctx.has_res = residual is not None
    ctx.save_for_backward(x, wi, wo, h)
    return y

  @staticmethod
  def backward(ctx, dy):
    x, wi, wo, h = ctx.saved_tensors
    dy = dy.contiguous()
    dh = gemm(dy, wo, True, True, aux=h, aux_mode=AUX_RELU_MASK)
    dwo = gemm(h, dy, False, False) if ctx.needs_input_grad[2] else None
    dwi = gemm(x, dh, False, False) if ctx.needs_input_grad[1] else None
    dx = gemm(dh, wi, True, True) if ctx.needs_input_grad[0] else None
    return dx, dwi, dwo, (dy if ctx.has_res else None)


def ffn_relu(x, wi, wo, residual=None):
  """x[..., M] → relu(x·wi[M,H])·wo[H,M]; 4 wgmma GEMMs fwd+bwd, no
  elementwise passes (bias-free FFN as in the GShard dense layers)."""
  lead = x.shape[:-1]
  x2 = x.reshape(-1, x.shape[-1])
  ok = (x2.is_cuda and x2.dtype == torch.bfloat16 and wi.dtype == torch.bfloat16
        and wo.dtype == torch.bfloat16 and ops.use_cuda_kernels(x2))
  if not ok:
    y = torch.matmul(F.relu(torch.matmul(x2, wi.to(x2.dtype))), wo.to(x2.dtype))
    if residual is not None:
      y = y + residual.reshape(y.shape).to(y.dtype)
    return y.reshape(*lead, wo.shape[-1])
  r2 = residual.reshape(-1, wo.shape[-1]) if residual is not None else None
  if r2 is not None and r2.dtype != torch.bfloat16:
    r2 = r2.to(torch.bfloat16)
  return _FfnReluFn.apply(x2, wi, wo, r2).reshape(*lead, wo.shape[-1])
