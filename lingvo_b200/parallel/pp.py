"""Pipeline-parallel engine: GPipe schedule over ranks with overlapped P2P links.

One rank per stage (one process per GPU). Activations move forward and gradients move
backward as `torch.distributed` point-to-point transfers — NCCL over NVLink on H100
(SURVEY K14; reference `lingvo/core/gpipe.py:421-600` + `recurrent.py:1142-1400`
Send/Recv links), gloo in the CPU tests.

Usage on every rank:
    eng = PipelineEngine(group, remat=True)   # stage id = rank in group
    pipe_layer.AttachEngine(eng)
    out = pipe_layer.FProp(theta, x)          # only the last stage gets real outputs
    loss = f(out)                             # last stage
    eng.Backward(loss)                        # all ranks call this

Design:
  * **Static shapes, no pickling.** The first transfer on a link is preceded by a fixed
    size int64 header tensor (rank, dtype code, dims per tensor); it is cached per link, so
    steady-state steps send payload only (and the step is CUDA-graph friendly).
  * **Overlap.** The receive of micro-batch m+1 is posted (`irecv`) *before* stage compute
    of micro-batch m starts and sends are asynchronous (`isend`): NCCL runs them on its own
    stream, the compute stream only waits for the tensor it is about to consume. Buffers
    stay referenced until their request completed.
  * **Rematerialisation** (`remat=True`, the reference default: `recurrent.py:780-801`
    re-runs `cell_fn` in the backward loop): the forward phase runs stages under
    `no_grad` and keeps only the micro-batch inputs; the backward phase re-runs the stage
    forward with grad enabled right before back-propagating it — O(1) activations per
    micro-batch instead of the whole stage graph.

Schedule: all micro-batch forwards, then all backwards in reverse order (GPipe).
"""

from __future__ import annotations

from typing import List, Optional

import torch
import torch.distributed as dist

_DTYPES = [torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int32,
           torch.int64, torch.int16, torch.int8, torch.uint8, torch.bool]
_MAX_TENSORS = 16
_MAX_RANK = 8
_HDR = 1 + _MAX_TENSORS * (2 + _MAX_RANK)


def _EncodeMeta(tensors) -> torch.Tensor:
  """`None` entries of the inter-stage tuple are encoded as dtype code −1."""
  assert len(tensors) <= _MAX_TENSORS
  hdr = torch.zeros(_HDR, dtype=torch.int64)
  hdr[0] = len(tensors)
  for i, t in enumerate(tensors):
    base = 1 + i * (2 + _MAX_RANK)
    if t is None:
      hdr[base] = -1
      continue
    assert t.dim() <= _MAX_RANK
    hdr[base] = _DTYPES.index(t.dtype)
    hdr[base + 1] = t.dim()
    for d, n in enumerate(t.shape):
      hdr[base + 2 + d] = n
  return hdr


def _DecodeMeta(hdr: torch.Tensor):
  hdr = hdr.tolist()
  out = []
  for i in range(int(hdr[0])):
    base = 1 + i * (2 + _MAX_RANK)
    if int(hdr[base]) < 0:
      out.append(None)
      continue
    nd = int(hdr[base + 1])
    out.append((tuple(int(x) for x in hdr[base + 2:base + 2 + nd]), _DTYPES[int(hdr[base])]))
  return out


class _Link:
  """One direction of a stage-to-stage link with cached tensor metadata."""

  def __init__(self, engine, peer: int):
    self.eng = engine
    self.peer = peer
    self.send_meta = None
    self.recv_meta = None
    self._inflight = []          # (work, tensors) kept alive until completion

  def Send(self, tensors):
    eng = self.eng
    tensors = [None if t is None else t.contiguous() for t in tensors]
    meta = [None if t is None else (tuple(t.shape), t.dtype) for t in tensors]
    if self.send_meta != meta:
      dev = next(t.device for t in tensors if t is not None)
      hdr = _EncodeMeta(tensors).to(dev if eng.device_headers else 'cpu')
      dist.send(hdr, eng.Peer(self.peer), group=eng.group)
      self.send_meta = meta
    for t in tensors:
      if t is not None:
        self._inflight.append((dist.isend(t, eng.Peer(self.peer), group=eng.group), t))
    self._Reap()

  def PostRecv(self, device):
    """Posts the receives of one tensor tuple; returns a handle for `WaitRecv`."""
    eng = self.eng
    if self.recv_meta is None:
      hdr = torch.zeros(_HDR, dtype=torch.int64,
                        device=device if eng.device_headers else 'cpu')
      dist.recv(hdr, eng.Peer(self.peer), group=eng.group)
      self.recv_meta = _DecodeMeta(hdr.cpu())
    bufs, works = [], []
    for m in self.recv_meta:
      if m is None:
        bufs.append(None)
        continue
      shape, dtype = m
      t = torch.empty(shape, dtype=dtype, device=device)
      works.append(dist.irecv(t, eng.Peer(self.peer), group=eng.group))
      bufs.append(t)
    return bufs, works

  @staticmethod
  def WaitRecv(handle):
    bufs, works = handle
    for w in works:
      w.wait()
    return bufs

  def _Reap(self, block=False):
    keep = []
    for w, t in self._inflight:
      if block:
        w.wait()
      elif not w.is_completed():
        keep.append((w, t))
    self._inflight = [] if block else keep

  def Drain(self):
    self._Reap(block=True)


class PipelineEngine:

  def __init__(self, group=None, remat: bool = False):
    self.group = group
    self.rank = dist.get_rank(group)
    self.world = dist.get_world_size(group)
    self.remat = remat
    # NCCL moves device tensors only: headers travel as device tensors there.
    self.device_headers = dist.get_backend(group) == 'nccl'
    self._saved = []        # per micro-batch: (inputs, outputs | None under remat)
    self._layer = None
    self._theta = None
    self._fwd_in = _Link(self, self.rank - 1) if self.rank > 0 else None
    self._fwd_out = _Link(self, self.rank + 1) if self.rank < self.world - 1 else None
    self._bwd_in = _Link(self, self.rank + 1) if self.rank < self.world - 1 else None
    self._bwd_out = _Link(self, self.rank - 1) if self.rank > 0 else None

  @property
  def is_first(self):
    return self.rank == 0

  @property
  def is_last(self):
    return self.rank == self.world - 1

  def Peer(self, r):
    return dist.get_global_rank(self.group, r) if self.group is not None else r

  # -- schedule -----------------------------------------------------------------
  def _RunStage(self, ins):
    return self._layer._RunCells(self._theta, tuple(ins), self.rank, self.rank + 1)  # pylint: disable=protected-access

  def Forward(self, layer, theta, micro_inputs: List[tuple]):
    """Runs this rank's stage on every micro-batch. Returns per-micro-batch
    outputs (real tensors on the last stage, detached placeholders elsewhere)."""
    assert layer.num_stages == self.world, (
        'PipelineEngine: %d cells but %d ranks' % (layer.num_stages, self.world))
    self._layer, self._theta = layer, theta
    self._saved = []
    dev = None
    for t in micro_inputs[0]:
      if isinstance(t, torch.Tensor):
        dev = t.device
        break
    n = len(micro_inputs)
    outs = []
    pending = None if self.is_first else self._fwd_in.PostRecv(dev)
    for m, mi in enumerate(micro_inputs):
      if self.is_first:
        ins = list(mi)
      else:
        ins = _Link.WaitRecv(pending)
        # next micro-batch's activations travel while this one is computed
        pending = self._fwd_in.PostRecv(dev) if m + 1 < n else None
        for t in ins:
          if t is not None and t.is_floating_point():
            t.requires_grad_(True)
      keep_graph = not self.remat or self.is_last
      if keep_graph:
        out = self._RunStage(ins)
      else:
        with torch.no_grad():
          out = self._RunStage(ins)
      if not self.is_last:
        self._fwd_out.Send([None if o is None else o.detach() for o in out])
      self._saved.append((ins, out if keep_graph else None))
      outs.append(out)
    return outs

  def Backward(self, loss=None):
    """Backward phase; the last stage passes the (already micro-batch-merged)
    loss, other stages pass nothing."""
    n = len(self._saved)

    def in_grads(ins):
      return [t.grad if t.grad is not None else torch.zeros_like(t)
              for t in ins if t is not None and t.is_floating_point()]

    if self.is_last:
      assert loss is not None
      # One backward through the merged loss populates grads of every micro-batch
      # input on this stage.
      loss.backward()
      for m in reversed(range(n)):
        if not self.is_first:
          self._bwd_out.Send(in_grads(self._saved[m][0]))
    else:
      dev = None
      for t in self._saved[0][0]:
        if isinstance(t, torch.Tensor):
          dev = t.device
          break
      # Only float outputs that take part in the graph carry a gradient back.
      pending = self._bwd_in.PostRecv(dev)
      for k, m in enumerate(reversed(range(n))):
        ins, out = self._saved[m]
        if out is None:
          # rematerialise: re-run this stage's forward for micro-batch m with grad, while
          # the gradient of its outputs is still in flight
          out = self._RunStage(ins)
        gouts = _Link.WaitRecv(pending)
        pending = self._bwd_in.PostRecv(dev) if k + 1 < n else None
        # the next stage returns one gradient per *float* tensor it received, in order
        # (also for pass-through tensors such as paddings): match them by position
        floats = [o for o in out if o is not None and o.is_floating_point()]
        pairs = [(o, g) for o, g in zip(floats, gouts) if o.requires_grad]
        torch.autograd.backward([o for o, _ in pairs], [g for _, g in pairs])
        if not self.is_first:
          self._bwd_out.Send(in_grads(ins))
        self._saved[m] = (None, None)          # free this micro-batch's graph now
    for link in (self._fwd_out, self._bwd_out):
      if link is not None:
        link.Drain()
    self._saved = []
