"""Native (sm_90a CUDA / C++) ops of lingvo_b200.

`native()` returns the in-tree extension module `lingvo_b200/ops/_C.so`
(built by `python -m lingvo_b200.ops.build`). On a GPU box a missing
extension is a hard error: ops must never silently fall back to eager
PyTorch there. On CPU-only hosts the pure-PyTorch reference implementations
(used as numerics oracles in tests) are used instead.
"""

import importlib
import threading

import torch

_LOCK = threading.Lock()
_MOD = None
_ERR = None


def native(required: bool = True):
  """Loads (once) and returns the native extension module."""
  global _MOD, _ERR
  if _MOD is not None:
    return _MOD
  with _LOCK:
    if _MOD is None and _ERR is None:
      try:
        _MOD = importlib.import_module('lingvo_b200.ops._C')
      except Exception as e:  # pylint: disable=broad-except
        _ERR = e
  if _MOD is None and required:
    raise RuntimeError(
        'lingvo_b200 native extension is not available (%r). Build it with '
        '`python -m lingvo_b200.ops.build`.' % (_ERR,))
  return _MOD


_HOST = None


def host():
  """Loads (building on first use if needed) the torch-free host library `_H.so`:
  record yielders / batcher, tokenizers, sequence packing, MASS, best_step."""
  global _HOST
  if _HOST is not None:
    return _HOST
  with _LOCK:
    if _HOST is None:
      try:
        _HOST = importlib.import_module('lingvo_b200.ops._H')
      except ImportError:
        from lingvo_b200.ops import build as build_lib
        build_lib.BuildHost(verbose=False)
        importlib.invalidate_caches()
        _HOST = importlib.import_module('lingvo_b200.ops._H')
  return _HOST


def use_cuda_kernels(*tensors) -> bool:
  """True when the fused sm_90a path must be taken for these tensors."""
  if not tensors or not all(t.is_cuda for t in tensors if t is not None):
    return False
  native(required=True)  # fail loudly on a GPU box without the extension
  return True
