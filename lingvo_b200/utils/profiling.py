"""Tracing / timing / roofline helpers (SURVEY §5.1).

The reference has no profiler integration beyond step-rate tracking and `py_utils.Timer`;
this framework adds what a CUDA program needs:

* `Range(name)` — NVTX range (shows up in `ncu`/nsight timelines). No-op unless
  `LINGVO_B200_NVTX=1` or `EnableNvtx()`; `InstrumentLayers(root)` wraps every layer's FProp.
* `DeviceTimer` — CUDA-event timing of a region on the launching stream, synchronised on
  both sides, max over ranks (the contract `bench.py` follows).
* `Roofline` — per-op time bound `max(flops / peak_flops, bytes / peak_bw)` against the
  measured peaks in `MEASURED_PEAKS.json` when that file exists (otherwise derated H100 SXM
  data-sheet numbers), with ready-made cost models of the fused paths.
"""

from __future__ import annotations

import contextlib
import functools
import json
import os
from typing import Dict, Optional

import torch

_NVTX = os.environ.get('LINGVO_B200_NVTX', '0') not in ('', '0')


def EnableNvtx(on: bool = True):
  global _NVTX
  _NVTX = bool(on)


@contextlib.contextmanager
def Range(name: str):
  if _NVTX and torch.cuda.is_available():
    torch.cuda.nvtx.range_push(name)
    try:
      yield
    finally:
      torch.cuda.nvtx.range_pop()
  else:
    yield


def InstrumentLayers(root_layer) -> int:
  """Wraps `FProp` of every layer under `root_layer` in an NVTX range named by its path."""
  n = 0
  for path, layer in root_layer.Walk():
    if getattr(layer, '_nvtx_wrapped', False):
      continue
    fprop = layer.FProp
    name = '%s[%s]' % (path or layer.params.name, type(layer).__name__)

    def _Wrapped(*args, _f=fprop, _n=name, **kwargs):
      with Range(_n):
        return _f(*args, **kwargs)
    layer.FProp = functools.wraps(fprop)(_Wrapped)
    layer._nvtx_wrapped = True  # pylint: disable=protected-access
    n += 1
  return n


class DeviceTimer:
  """`with DeviceTimer() as t: ...; t.ms` — device time of the region (max over ranks)."""

  def __init__(self, sync_ranks: bool = True):
    self._sync_ranks = sync_ranks
    self.ms = 0.0

  def _Barrier(self):
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    if self._sync_ranks and dist.is_available() and dist.is_initialized():
      dist.barrier()
    torch.cuda.synchronize()

  def __enter__(self):
    self._Barrier()
    self._e0 = torch.cuda.Event(enable_timing=True)
    self._e1 = torch.cuda.Event(enable_timing=True)
    self._e0.record()
    return self

  def __exit__(self, *exc):
    self._e1.record()
    self._Barrier()
    ms = torch.tensor([self._e0.elapsed_time(self._e1)], device='cuda')
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    if self._sync_ranks and dist.is_available() and dist.is_initialized():
      dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    self.ms = float(ms)
    return False


# H100 SXM data sheet (3.35 TB/s HBM3, 989 dense BF16 TFLOP/s at 700 W), derated; used when
# no measurement file exists.
_FALLBACK = {'hbm_gbs': 3350.0 * 0.92, 'bf16_tflops': 989.0 * 0.75}


def MeasuredPeaks(path: Optional[str] = None) -> Dict[str, float]:
  path = path or os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(
      os.path.abspath(__file__)))), 'MEASURED_PEAKS.json')
  try:
    with open(path) as f:
      d = json.load(f)
    return {'hbm_gbs': float(d['hbm_gbs']),
            'bf16_tflops': float(d.get('bf16_tflops_sustained') or d['bf16_tflops']),
            'source': path}
  except (OSError, KeyError, ValueError):
    return dict(_FALLBACK, source='fallback (H100 SXM data sheet × derate)')


class Roofline:
  """Time bounds of an op from its FLOPs and HBM bytes."""

  def __init__(self, peaks: Optional[Dict[str, float]] = None):
    self.peaks = peaks or MeasuredPeaks()

  def BoundUs(self, flops: float = 0.0, bytes_moved: float = 0.0) -> float:
    t_c = flops / (self.peaks['bf16_tflops'] * 1e12)
    t_m = bytes_moved / (self.peaks['hbm_gbs'] * 1e9)
    return max(t_c, t_m) * 1e6

  def Report(self, name: str, measured_us: float, flops: float = 0.0, bytes_moved: float = 0.0):
    bound = self.BoundUs(flops, bytes_moved)
    limiter = 'compute' if flops / (self.peaks['bf16_tflops'] * 1e12) * 1e6 >= bound else 'memory'
    return {'op': name, 'measured_us': measured_us, 'bound_us': bound, 'limiter': limiter,
            'fraction_of_roofline': bound / measured_us if measured_us > 0 else 0.0,
            'achieved_tflops': flops / measured_us / 1e6 if measured_us > 0 else 0.0,
            'achieved_gbs': bytes_moved / measured_us / 1e3 if measured_us > 0 else 0.0}

  # ---- cost models of the fused paths (elements are bf16 unless noted) ----
  @staticmethod
  def Gemm(m, n, k, groups=1):
    return dict(flops=2.0 * groups * m * n * k, bytes_moved=2.0 * groups * (m * k + k * n + m * n))

  @staticmethod
  def AdafactorFactored(numel):
    # stats: read g; rms: read g; apply: read g + fp32 w, write fp32 w + bf16 copy
    return dict(flops=0.0, bytes_moved=numel * (2 + 2 + 2 + 4 + 4 + 2))

  @staticmethod
  def NormFwd(rows, dim):
    return dict(flops=0.0, bytes_moved=2.0 * rows * dim * 2)

  @staticmethod
  def NormBwd(rows, dim, with_residual_grad=True):
    return dict(flops=0.0, bytes_moved=(4.0 if with_residual_grad else 3.0) * rows * dim * 2)

  @staticmethod
  def LmHeadXent(tokens, vocab, dim):
    # logits are never materialised in HBM: fwd GEMM + bwd dgrad/wgrad on recomputed chunks
    return dict(flops=3 * 2.0 * tokens * vocab * dim + 2.0 * tokens * vocab * dim,
                bytes_moved=2.0 * (3 * tokens * dim + 3 * vocab * dim))

  @staticmethod
  def GateLogits(tokens, dim, experts, backward=False):
    return dict(flops=(3 if backward else 1) * 2.0 * tokens * dim * experts,
                bytes_moved=(2 if backward else 1) * 2.0 * tokens * dim)

  @staticmethod
  def Attention(batch, heads, seq, head_dim, causal=True, with_bias=True, backward=False):
    f = 4.0 * batch * heads * seq * seq * head_dim * (0.5 if causal else 1.0)
    f = f * (2.5 if backward else 1.0)
    io = 4.0 * batch * heads * seq * head_dim * 2 * (2 if backward else 1)
    bias = batch * heads * seq * seq * 2.0 if with_bias else 0.0
    return dict(flops=f, bytes_moved=io + bias)
