"""GShard LM serving loop (ref `lingvo/core/gshard_decode.py:100-538`).

The reference keeps a TPU program spinning in an infinite `while_loop`, feeding it
through infeed queues from a host thread and draining results through outfeed. The
H100 design keeps the same three-stage shape with CUDA streams instead of TPU
queues:

  infeed thread  : host batches → pinned buffers → H2D on a copy stream
  decode loop    : `task.DecodeStep`-style callable on the compute stream (optionally a
                   captured CUDA graph for static shapes)
  outfeed thread : D2H on a second copy stream → result queue / callback

`GShardDecode.decode(batches)` streams an iterable of batches through the loop and
yields outputs in order; `serve()` exposes the same loop to an RPC-ish producer via
`submit()`/`results()`.
"""

from __future__ import annotations

import queue
import threading
import time
from typing import Callable, Iterable, Optional

import numpy as np
import torch


def preload_zero(n=None, batch_size=None, max_len=None, key_size=2):  # pylint: disable=invalid-name
  """Zero batch with the decoder's input structure (ref :40)."""
  return (np.zeros([n, batch_size, key_size], np.int32),   # key
          np.zeros([n, batch_size, max_len], np.int32),    # tgt_id
          np.zeros([n, batch_size, max_len], np.float32),  # tgt_segment_id
          np.zeros([n, batch_size, max_len], np.int32),    # tgt_segment_pos
          np.zeros([n, batch_size, max_len], np.int32),    # tgt_labels
          np.zeros([n, batch_size], np.float32))           # tgt_sample_temperature


def infinite_repeat(body_fn, infeed_queue=None, stop_event=None):  # pylint: disable=invalid-name
  """Runs `body_fn(*carried)` forever, feeding its results back as the next arguments; with
  an `infeed_queue` (a `queue.Queue`) every iteration also receives the next queued tuple
  (ref :59). `stop_event` (threading.Event) or a `StopIteration` from the body / a `None`
  item in the queue ends the loop — the host-driven replacement of the device while-loop."""
  carried = ()
  while stop_event is None or not stop_event.is_set():
    args = tuple(carried)
    if infeed_queue is not None:
      item = infeed_queue.get()
      if item is None:
        break
      args += tuple(item) if isinstance(item, (list, tuple)) else (item,)
    try:
      out = body_fn(*args)
    except StopIteration:
      break
    carried = () if out is None else (tuple(out) if isinstance(out, (list, tuple)) else (out,))
  return list(carried)


def daemon(closure):  # pylint: disable=invalid-name
  t = threading.Thread(target=closure, daemon=True)
  t.start()
  return t


class GShardDecode:

  def __init__(self, decode_fn: Callable, device=None, infeed_depth=2, use_cuda_graph=False):
    """decode_fn(batch: tuple/dict of device tensors) → tuple/dict of device tensors."""
    self._fn = decode_fn
    self._device = torch.device(device) if device is not None else torch.device(
        'cuda' if torch.cuda.is_available() else 'cpu')
    self._cuda = self._device.type == 'cuda'
    self._in_q = queue.Queue(maxsize=infeed_depth)
    self._out_q = queue.Queue(maxsize=infeed_depth * 2)
    self._use_graph = use_cuda_graph and self._cuda
    self._graph = None
    self._static_in = None
    self._static_out = None
    self._threads = []
    self._stop = threading.Event()
    if self._cuda:
      self._h2d = torch.cuda.Stream(self._device)
      self._d2h = torch.cuda.Stream(self._device)

  # -- stages ---------------------------------------------------------------------
  def _ToDevice(self, batch):
    def mv(x):
      t = torch.as_tensor(x)
      if self._cuda:
        t = t.pin_memory().to(self._device, non_blocking=True)
      return t
    if isinstance(batch, dict):
      return {k: mv(v) for k, v in batch.items()}
    return tuple(mv(v) for v in batch)

  def _Infeed(self, batches: Iterable):
    for b in batches:
      if self._stop.is_set():
        break
      if self._cuda:
        with torch.cuda.stream(self._h2d):
          dev = self._ToDevice(b)
          ev = torch.cuda.Event()
          ev.record(self._h2d)
      else:
        dev, ev = self._ToDevice(b), None
      self._in_q.put((dev, ev))
    self._in_q.put(None)

  def _Run(self, dev_batch):
    if not self._use_graph:
      return self._fn(dev_batch)
    vals = list(dev_batch.values()) if isinstance(dev_batch, dict) else list(dev_batch)
    if self._graph is None:
      self._static_in = [v.clone() for v in vals]
      mk = (lambda: dict(zip(dev_batch.keys(), self._static_in))) if isinstance(
          dev_batch, dict) else (lambda: tuple(self._static_in))
      for _ in range(2):
        self._fn(mk())
      torch.cuda.synchronize()
      self._graph = torch.cuda.CUDAGraph()
      with torch.cuda.graph(self._graph):
        self._static_out = self._fn(mk())
    for s, v in zip(self._static_in, vals):
      s.copy_(v)
    self._graph.replay()
    out = self._static_out
    if isinstance(out, dict):
      return {k: v.clone() for k, v in out.items()}
    return tuple(v.clone() for v in out) if isinstance(out, (tuple, list)) else out.clone()

  def _DecodeLoop(self):
    while True:
      item = self._in_q.get()
      if item is None:
        self._out_q.put(None)
        return
      dev_batch, ev = item
      if ev is not None:
        torch.cuda.current_stream(self._device).wait_event(ev)
      with torch.no_grad():
        out = self._Run(dev_batch)
      done = None
      if self._cuda:
        done = torch.cuda.Event()
        done.record(torch.cuda.current_stream(self._device))
      self._out_q.put((out, done))

  def _ToHost(self, out, done):
    def mv(x):
      return x.to('cpu', non_blocking=self._cuda) if isinstance(x, torch.Tensor) else x
    if self._cuda:
      with torch.cuda.stream(self._d2h):
        self._d2h.wait_event(done)
        host = {k: mv(v) for k, v in out.items()} if isinstance(out, dict) else (
            tuple(mv(v) for v in out) if isinstance(out, (tuple, list)) else mv(out))
      self._d2h.synchronize()
      return host
    return out

  # -- public -----------------------------------------------------------------------
  def decode(self, batches: Iterable):  # pylint: disable=invalid-name
    """Streams `batches` through infeed → decode → outfeed; yields host outputs in order."""
    self._stop.clear()
    t_in = daemon(lambda: self._Infeed(batches))
    t_dec = daemon(self._DecodeLoop)
    while True:
      item = self._out_q.get()
      if item is None:
        break
      yield self._ToHost(*item)
    t_in.join()
    t_dec.join()

  def stop(self):  # pylint: disable=invalid-name
    self._stop.set()


def _PrefixLens(tgt):
  if 'paddings' in tgt:
    plen = (1.0 - tgt.paddings.float()).sum(1).long()
  else:
    plen = (tgt.segment_ids != 0).sum(1).long()
  return plen.clamp_min(1)


def DecodeIds(task, theta, input_batch, max_steps=None, temperature=0.0, top_k=0, seed=0):
  """Continues every row of a prefix batch with the task's incremental decoder (greedy,
  or temperature / top-k sampling) (ref :186 `_DecodeStep` + `gshard_builder` decode).

  `input_batch.tgt.ids [B, T]` with `paddings` (or `segment_ids`) marking each prefix.
  Returns NestedMap(ids [B, T+steps], prefix_lens [B], lens [B], scores [B] = Σ log p of the
  generated tokens). All control flow is on the device; the host checks `all done` every
  8 steps only."""
  from lingvo_b200.core.nested_map import NestedMap
  p = task.params
  tgt = input_batch.tgt if 'tgt' in input_batch else input_batch
  ids = tgt.ids.long()
  b, t0 = ids.shape
  dev = ids.device
  plen = _PrefixLens(tgt)
  steps = int(max_steps or p.decoder_max_steps)
  total = t0 + steps
  out = torch.full((b, total), int(p.decoder_eos_id), dtype=torch.long, device=dev)
  out[:, :t0] = ids
  gen = torch.Generator(device=dev)
  gen.manual_seed(int(seed))
  with torch.no_grad():
    state = task.InitDecodeState(b, total, dev)
    done = torch.zeros(b, dtype=torch.bool, device=dev)
    scores = torch.zeros(b, device=dev)
    lens = plen.clone()
    cur = out[:, 0]
    for t in range(total - 1):
      logits = task.DecodeStep(theta, cur, state, t)
      logp = torch.log_softmax(logits, -1)
      if temperature and temperature > 0:
        z = logits / temperature
        if top_k:
          kth = z.topk(top_k, -1).values[:, -1:]
          z = torch.where(z < kth, torch.full_like(z, -1e9), z)
        nxt = torch.multinomial(torch.softmax(z, -1), 1, generator=gen).squeeze(1)
      else:
        nxt = logits.argmax(-1)
      in_prefix = (t + 1) < plen                      # still teacher-forcing the prefix
      active = ~in_prefix & ~done
      nxt = torch.where(in_prefix, out[:, t + 1], nxt)
      out[:, t + 1] = torch.where(active | in_prefix, nxt, out[:, t + 1])
      scores = scores + torch.where(active, logp.gather(1, nxt.unsqueeze(1)).squeeze(1),
                                    torch.zeros_like(scores))
      lens = lens + active.long()
      done = done | (active & (nxt == int(p.decoder_eos_id)))
      cur = out[:, t + 1]
      if (t + 1) % 8 == 0 and t + 1 >= int(t0) and bool(done.all()):
        break
  return NestedMap(ids=out, prefix_lens=plen, lens=lens, scores=scores)


def BeamDecodeIds(task, theta, input_batch, beam_size=None, max_steps=None):
  """Flat beam search from every row's prefix (ref `gshard_builder.DecodeIds` with
  `_FlatBeamSearchCallback`): the prompts are right-aligned and written into the KV caches
  in one `task.Prefill` call, then each `task.BeamDecodeStep` extends all K hypotheses of a
  row in the shared token buffer, each attending over its own prompt and ancestors.

  `input_batch.tgt.ids [B, T]` with `paddings` (or `segment_ids`) marking each prefix, as for
  `DecodeIds`. `beam_size` / `max_steps` default to `decoder_beam_size` / `decoder_max_steps`.
  Returns NestedMap(topk_ids [B, K, S] (continuations only, EOS-terminated), topk_lens
  [B, K] (0 for an empty slot), topk_scores [B, K] (length-normalised log-probabilities,
  best first), prefix_lens [B])."""
  from lingvo_b200.core import flat_beam_search_helper as fbs
  from lingvo_b200.core.nested_map import NestedMap
  from lingvo_b200.ops import attention as attention_ops
  p = task.params
  tgt = input_batch.tgt if 'tgt' in input_batch else input_batch
  ids = tgt.ids.long()
  b, t0 = ids.shape
  dev = ids.device
  plen = _PrefixLens(tgt)
  k = int(beam_size or p.decoder_beam_size)
  steps = int(max_steps or p.decoder_max_steps)
  pmax = -(-t0 // k) * k
  src = torch.arange(pmax, device=dev) - (pmax - plen).unsqueeze(1)   # right-aligned prompts
  prefix = torch.where(src >= 0, ids.gather(1, src.clamp(0, t0 - 1)), torch.zeros_like(src))

  def Callback(tgt_id, tgt_pos, tgt_segment_id, tgt_mask, state, t):
    if tgt_mask is None:
      task.Prefill(theta, tgt_id, tgt_segment_id, tgt_pos, state)
      return None, state
    vis = attention_ops.pack_visibility(tgt_mask)
    return task.BeamDecodeStep(theta, tgt_id, tgt_pos, state, t * k, vis), state

  with torch.no_grad():
    state = task.InitDecodeState(b, pmax + k * steps, dev)
    (out, lens, scores), _ = fbs.flat_beam_search(
        b, k, steps, Callback, state, eos_id=int(p.decoder_eos_id), prefix=prefix,
        prefix_len=plen, device=dev)
  return NestedMap(topk_ids=out, topk_lens=lens, topk_scores=scores, prefix_lens=plen)
