"""Front-end of the fused optimizer kernels (csrc/optim_kernels.cu).

tests/test_adafactor_gpu.py checks them against float64 oracles at the MoELm8E shapes."""

import torch

from lingvo_b200 import ops

_SCRATCH = {}


def _Scratch(var, n):
  """Per-variable fp32 scratch; returns (buffer, fresh). `fresh` means the
  carried sum(w²) in it is not valid yet (first step, or after `Invalidate`)."""
  key = id(var)
  ent = _SCRATCH.get(key)
  if (ent is None or ent[0].numel() < n or ent[0].device != var.device or
      ent[1] != var.data_ptr()):
    buf = torch.zeros(n, dtype=torch.float32, device=var.device)
    # The entry holds `var` itself: id() keys are only unique while the object is alive.
    _SCRATCH[key] = (buf, var.data_ptr(), var)
    return buf, True
  return ent[0], False


def carried_sumsq(var):
  """Device scalar Σw² of `var` as left by its last fused Adafactor step (i.e. the norm²
  of the *current* weights), or None if not available."""
  ent = _SCRATCH.get(id(var))
  if ent is None or ent[1] != var.data_ptr():
    return None
  return ent[0][2:3]


def Invalidate():
  """Re-derives the carried Σw² of every variable from its current weights (call after
  weights change outside the optimizer, e.g. checkpoint restore). The scratch buffers keep
  their addresses, so a captured CUDA graph of the step stays valid."""
  with torch.no_grad():
    for key, ent in list(_SCRATCH.items()):
      buf, ptr, var = ent
      if var.data_ptr() != ptr or buf.device != var.device:
        del _SCRATCH[key]
        continue
      buf[2:3] = var.data.float().square().sum().reshape(1)


def _KernelGrad(grad, b):
  """The fused kernels take a contiguous gradient or (for a single matrix) a column slice of
  a wider row-major matrix — e.g. dwq/dwk/dwv as views of the fused qkv weight gradient —
  so those never need a `.contiguous()` copy."""
  if grad.is_contiguous():
    return grad
  if (b == 1 and grad.dim() >= 2 and grad.stride(-1) == 1 and grad.stride(-2) >= grad.shape[-1]
      and (grad.stride(-2) * grad.element_size()) % 16 == 0 and grad.data_ptr() % 16 == 0 and
      all(s == 1 for s in grad.shape[:-2])):
    return grad
  return grad.contiguous()


def _Geometry(var, d0, d1):
  nd = var.dim()
  assert sorted((d0, d1)) == [nd - 2, nd - 1]
  r, c = var.shape[-2], var.shape[-1]
  b = var.numel() // (r * c)
  return b, r, c, (d0 == nd - 1)


def adafactor_stats(var, grad, d0, d1, mult_by_param_scale, total_sumsq=None, slot=0):
  """Phase A (see csrc): row/col sums of g² (+ global Σg² into `total_sumsq`). `slot`
  names the staging buffer: 0 for the caller's stream, k for the k-th optimizer side stream."""
  b, r, c, _ = _Geometry(var, d0, d1)
  scratch, fresh = _Scratch(var, 16 + 2 * (b * r + 4) + 2 * (b * c + 4))
  g = _KernelGrad(grad, b)
  ops.native().adafactor_stats(var.data, g, scratch, b, r, c, bool(mult_by_param_scale),
                               fresh, total_sumsq, int(slot))
  return fresh


def adafactor_update(var, grad, vr, vc, d0, d1, lr, decay, eps1, eps2, clip,
                     mult_by_param_scale, grad_scale=None, fresh=False, hyper=None):
  """Phase B: factors → clip RMS → apply, using the sums left by `adafactor_stats`."""
  b, r, c, vr_is_rows = _Geometry(var, d0, d1)
  scratch, _ = _Scratch(var, 16 + 2 * (b * r + 4) + 2 * (b * c + 4))
  g = _KernelGrad(grad, b)
  compute = getattr(var, 'compute', None)
  ops.native().adafactor_update(
      var.data, g, vr, vc, scratch, compute.data if compute is not None else None,
      b, r, c, vr_is_rows, float(lr), float(decay), float(eps1), float(eps2),
      float(clip), bool(mult_by_param_scale), grad_scale, bool(fresh), hyper)


class SmallVarTable:
  """Pointer table for `adafactor_small`: rows (w, g, v, w_bf16|0, numel, g_is_bf16).

  Built on the host into a ring of pinned buffers and copied asynchronously, so neither the
  eager loop nor CUDA-graph capture ever touches pageable memory."""

  _RING = 8

  def __init__(self, device):
    self._dev = device
    self._host = []
    self._events = []
    self._i = 0
    self._last_key = None
    self._table = None

  def Build(self, rows):
    key = tuple(tuple(r) for r in rows)
    if key == self._last_key and self._table is not None:
      return self._table                       # static addresses (graph replay / fused DP)
    n = len(rows)
    if len(self._host) < self._RING:
      self._host.append(torch.empty((max(n, 1), 6), dtype=torch.int64).pin_memory())
      self._events.append(None)
    slot = self._i % len(self._host)
    self._i += 1
    if self._host[slot].shape[0] < n:
      self._host[slot] = torch.empty((n, 6), dtype=torch.int64).pin_memory()
    if self._events[slot] is not None:
      self._events[slot].synchronize()
    host = self._host[slot][:n]
    host.copy_(torch.tensor(rows, dtype=torch.int64))
    table = torch.empty((n, 6), dtype=torch.int64, device=self._dev)
    table.copy_(host, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    self._events[slot] = ev
    self._last_key, self._table = key, table
    return table


def adafactor_small(table, lr, decay, eps1, eps2, clip, mult_by_param_scale,
                    grad_scale=None, hyper=None):
  """Non-factored Adafactor for every variable in `table` with ONE kernel launch."""
  ops.native().adafactor_small(table, float(lr), float(decay), float(eps1), float(eps2),
                               float(clip), bool(mult_by_param_scale), grad_scale, hyper)


def small_sumsq(table, out):
  """out[0] += Σg², out[1] += Σw² over every variable of a `SmallVarTable` (one launch)."""
  ops.native().small_sumsq(table, out)


def adam_flat(w, g, m, v, w_bf16, lr_t, b1, b2, eps, grad_scale=1.0,
              grad_scale_t=None):
  ops.native().adam_flat(w, g, m, v, w_bf16, grad_scale_t, float(lr_t),
                         float(b1), float(b2), float(eps), float(grad_scale))


def multi_tensor_adam(variables, grads, ms, vs, lr_t, b1, b2, eps,
                      grad_scale_t=None):
  for w, g, m, v in zip(variables, grads, ms, vs):
    n = w.numel()
    if n % 8 == 0 and w.is_contiguous() and g.is_contiguous():
      compute = getattr(w, 'compute', None)
      adam_flat(w.data.view(-1), g.reshape(-1), m.view(-1), v.view(-1),
                compute.data.view(-1) if compute is not None else None,
                lr_t, b1, b2, eps, grad_scale_t=grad_scale_t)
    else:
      gg = g.to(w.dtype)
      if grad_scale_t is not None:
        gg = gg * grad_scale_t.to(gg.dtype)
      m.mul_(b1).add_(gg, alpha=1 - b1)
      v.mul_(b2).addcmul_(gg, gg, value=1 - b2)
      w.data.addcdiv_(m, v.sqrt().add_(eps), value=-lr_t)
      compute = getattr(w, 'compute', None)
      if compute is not None:
        compute.data.copy_(w.data)
