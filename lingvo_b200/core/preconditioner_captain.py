"""Asynchronous Shampoo preconditioner service (ref `ops/preconditioner_captain.{h,cc}`,
`preconditioner_op_kernels.cc`: `ComputePreconditioners` / `GetPreconditioners`).

The reference ships gradient statistics to a pool of CPU sessions that run the inverse
p-th-root graph while training continues with stale preconditioners. The H100 design keeps
the statistics on the device and runs the coupled Newton iteration on a *low-priority CUDA
stream*: training kernels on the main stream are never blocked, a finished solve is published
when its event has fired, and readers get `(preconditioner, ok)` exactly like the reference
op (ok=False until the first solve for that key lands). On CPU tensors the solves run on a
small thread pool instead.
"""

from __future__ import annotations

import concurrent.futures
import threading
from typing import Dict, Optional, Sequence

import torch

from lingvo_b200.core import matrix_functions


class PreconditionerCaptain:
  """Keyed store of statistics → inverse-p-th-root preconditioners."""

  def __init__(self, num_compute_threads: int = 4, inverse_root_fn=None, max_active: int = 0):
    self._fn = inverse_root_fn or self._DefaultRoot
    self._mu = threading.Lock()
    self._done: Dict[str, torch.Tensor] = {}
    self._steps: Dict[str, int] = {}
    self._pending: Dict[str, tuple] = {}      # key → (result tensor | future, event | None, step)
    self._pool = concurrent.futures.ThreadPoolExecutor(max(1, num_compute_threads))
    self._stream: Optional[torch.cuda.Stream] = None
    self._max_active = max_active

  @staticmethod
  def _DefaultRoot(stat, exponent):
    # exponent is the reference's "p": result = stat^(-1/p).
    p = int(round(float(exponent)))
    if stat.is_cuda:      # nothing in the solve may sync the host with the side stream
      return matrix_functions.inverse_pth_root_no_sync(stat, p)
    return matrix_functions.inlined_matrix_inverse_pth_root(stat, p)

  def _SideStream(self, device):
    if self._stream is None:
      lo, _ = torch.cuda.Stream.priority_range()
      self._stream = torch.cuda.Stream(device=device, priority=lo)
    return self._stream

  def InsertGradientStatistics(self, key: str, statistics: torch.Tensor, exponent, global_step: int,
                               sync: bool = False):
    """Schedules (or, with sync, performs) the solve for `key`. A newer request for a key whose
    solve is still in flight is dropped — the captain never queues more than one per key."""
    self._Harvest()
    with self._mu:
      if key in self._pending and not sync:
        return
      if self._max_active and len(self._pending) >= self._max_active and not sync:
        return
    stat = statistics.detach()
    if stat.is_cuda:
      side = self._SideStream(stat.device)
      side.wait_stream(torch.cuda.current_stream(stat.device))
      with torch.cuda.stream(side):
        snap = stat.clone()                 # private copy: training may keep accumulating
        out = self._fn(snap, exponent)
        ev = torch.cuda.Event()
        ev.record(side)
      snap.record_stream(side)
      with self._mu:
        self._pending[key] = (out, ev, int(global_step))
      if sync:
        ev.synchronize()
        self._Harvest()
    else:
      snap = stat.clone()
      if sync:
        with self._mu:
          self._done[key] = self._fn(snap, exponent)
          self._steps[key] = int(global_step)
          self._pending.pop(key, None)
        return
      fut = self._pool.submit(self._fn, snap, exponent)
      with self._mu:
        self._pending[key] = (fut, None, int(global_step))

  def _Harvest(self):
    with self._mu:
      for key in list(self._pending):
        res, ev, step = self._pending[key]
        if ev is not None:
          if not ev.query():
            continue
          value = res
        else:
          if not res.done():
            continue
          value = res.result()
        self._done[key] = value
        self._steps[key] = step
        del self._pending[key]

  def GetPreconditioner(self, key: str):
    """→ (tensor | None, ok)."""
    self._Harvest()
    with self._mu:
      t = self._done.get(key)
    return t, t is not None

  def StatisticsStep(self, key: str) -> int:
    with self._mu:
      return self._steps.get(key, -1)

  def WaitAll(self):
    with self._mu:
      pend = list(self._pending.values())
    for res, ev, _ in pend:
      if ev is not None:
        ev.synchronize()
      else:
        res.result()
    self._Harvest()


_CAPTAIN: Optional[PreconditionerCaptain] = None
_CAPTAIN_LOCK = threading.Lock()


def GetCaptain() -> PreconditionerCaptain:
  global _CAPTAIN
  with _CAPTAIN_LOCK:
    if _CAPTAIN is None:
      _CAPTAIN = PreconditionerCaptain()
    return _CAPTAIN


def ComputePreconditioners(inputs: Sequence[torch.Tensor], exponents: Sequence, global_step: int,
                           keys: Sequence[str], sync: bool = False):
  """Op-level entry point (ref `x_ops.cc:986`)."""
  assert len(inputs) == len(exponents) == len(keys)
  cap = GetCaptain()
  for k, s, e in zip(keys, inputs, exponents):
    cap.InsertGradientStatistics(k, s, e, int(global_step), sync)


def GetPreconditioners(shapes: Sequence[Sequence[int]], keys: Sequence[str], device=None):
  """→ (preconditioners, statuses); a missing entry is an identity-free zero tensor of the
  requested shape with status False (ref `x_ops.cc:1008`)."""
  cap = GetCaptain()
  outs, oks = [], []
  for shape, k in zip(shapes, keys):
    t, ok = cap.GetPreconditioner(k)
    if not ok:
      t = torch.zeros(tuple(int(d) for d in shape), device=device)
    outs.append(t)
    oks.append(ok)
  return outs, oks
