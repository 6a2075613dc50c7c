"""Sharding annotations and specs for GShard-style models.

Reference `lingvo/core/gshard_utils.py`: `Split/Replicate/MeshSplit` (:40-134)
annotate tensors and XLA's SPMD partitioner inserts the collectives — and
every annotation is a no-op off-TPU. Here an annotation *records* a
`TensorShardingSpec` on the tensor (`tensor._sharding`) which the explicit
H100 runtime (`lingvo_b200.parallel`) reads: layers that own a collective
(MoE all-to-all, TP GEMM+reduce-scatter, vocab-sharded softmax) query the
active `parallel.mesh.DeviceMesh` and run their fused kernels; everything else
stays local. `TensorShardingSpec` keeps the reference's uneven-padding
arithmetic (:262-272) for computing local shapes.
"""

from __future__ import annotations

import contextlib
import threading
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch


class _TL(threading.local):

  def __init__(self):
    super().__init__()
    self.prefix: List[int] = []
    self.manual: List[int] = []


_CTX = _TL()


def _Annotate(x, spec):
  if isinstance(x, torch.Tensor):
    try:
      x._sharding = spec  # pylint: disable=protected-access
    except Exception:  # pylint: disable=broad-except
      pass
  return x


def Split(x, split_dimension, num_devices, use_sharding_op=True,
          input_shape=None):
  """1-D split annotation along `split_dimension`."""
  if num_devices is None or not num_devices > 1:
    return x
  mapping = [-1] * x.dim()
  mapping[split_dimension] = 0
  return _Annotate(x, TensorShardingSpec(mapping,
                                         np.arange(num_devices)))


def Replicate(x, use_sharding_op=True):
  return _Annotate(x, TensorShardingSpec([-1] * x.dim(), None))


def MeshSplit(x, device_mesh, tensor_split_dims_mapping, use_sharding_op=True,
              unspecified_dims=None):
  """Mesh split annotation: dim i of x is split on mesh axis mapping[i]."""
  if tensor_split_dims_mapping is None or device_mesh is None or (
      device_mesh.size <= 1):
    return x
  mapping = list(_CTX.prefix) + list(tensor_split_dims_mapping)
  return _Annotate(x, TensorShardingSpec(mapping, device_mesh))


def GetSharding(x) -> Optional['TensorShardingSpec']:
  return getattr(x, '_sharding', None)


@contextlib.contextmanager
def MeshSplitDimPrefixContext(prefix_mesh_dim):
  if prefix_mesh_dim is not None:
    _CTX.prefix.append(prefix_mesh_dim)
  try:
    yield
  finally:
    if prefix_mesh_dim is not None:
      _CTX.prefix.pop()


def GetMeshSplitDimPrefixContext():
  return list(_CTX.prefix)


@contextlib.contextmanager
def ManualMeshDimContext(mesh_dim):
  if mesh_dim is not None:
    _CTX.manual.append(mesh_dim)
  try:
    yield
  finally:
    if mesh_dim is not None:
      _CTX.manual.pop()


def ZigzagOrderOnDeviceMesh(device_mesh, zigzag_mesh_dim):
  """Permutes a mesh so neighbours along a dim are zig-zag ordered."""
  if not isinstance(device_mesh, np.ndarray):
    device_mesh = np.array(device_mesh)
  if zigzag_mesh_dim < 0:
    zigzag_mesh_dim += len(device_mesh.shape)
  size = device_mesh.shape[zigzag_mesh_dim]
  if size % 2:
    raise ValueError('Zigzag needs an even mesh dim')
  perm = np.zeros(size, dtype=int)
  perm[:size // 2] = np.arange(0, size, 2)
  perm[size // 2:] = np.arange(size - 1, 0, -2)
  return np.take(device_mesh, perm, axis=zigzag_mesh_dim)


def GetNonPod2dMesh(device_mesh_shape, physical_mesh_shape):
  """2-D logical mesh over a 3-D physical mesh (reference :208-234)."""
  assert len(device_mesh_shape) == 2 and len(physical_mesh_shape) == 3
  assert np.prod(device_mesh_shape) == np.prod(physical_mesh_shape)
  return np.arange(np.prod(device_mesh_shape)).reshape(device_mesh_shape)


class TensorShardingSpec:
  """How a tensor is split over a device mesh (reference :237-443)."""

  def __init__(self, split_dims_mapping: Optional[List[int]] = None,
               device_mesh: Optional[np.ndarray] = None,
               uneven_padding: Optional[List[int]] = None):
    self._split_dims_mapping = (None if split_dims_mapping is None
                                else list(split_dims_mapping))
    self._device_mesh = None if device_mesh is None else np.asarray(device_mesh)
    self._uneven_padding = uneven_padding

  @classmethod
  def FromFullShape(cls, full_shape: Sequence[int], split_dims_mapping,
                    device_mesh: np.ndarray):
    """Computes the uneven padding needed so every shard has equal shape."""
    uneven = [0] * len(full_shape)
    mesh = np.asarray(device_mesh)
    for i, m in enumerate(split_dims_mapping):
      if m >= 0:
        n = mesh.shape[m]
        uneven[i] = (n - full_shape[i] % n) % n
    if all(u == 0 for u in uneven):
      uneven = None
    return cls(split_dims_mapping, mesh, uneven)

  @classmethod
  def ReplicatedSpec(cls):
    return cls(None, None, None)

  def AddLeadingDims(self, num_dims=1):
    if self.is_replicated:
      return self
    up = self._uneven_padding
    return TensorShardingSpec([-1] * num_dims + self._split_dims_mapping,
                              self._device_mesh,
                              None if up is None else [0] * num_dims + up)

  def RemoveLeadingDims(self, num_dims=1):
    if self.is_replicated:
      return self
    up = self._uneven_padding
    return TensorShardingSpec(self._split_dims_mapping[num_dims:],
                              self._device_mesh,
                              None if up is None else up[num_dims:])

  def RemoveDim(self, dim):
    if self.is_replicated:
      return self
    if dim < 0:
      dim += len(self._split_dims_mapping)
    m = self._split_dims_mapping[:dim] + self._split_dims_mapping[dim + 1:]
    up = self._uneven_padding
    if up is not None:
      up = up[:dim] + up[dim + 1:]
    return TensorShardingSpec(m, self._device_mesh, up)

  @property
  def split_dims_mapping(self):
    return self._split_dims_mapping

  @property
  def device_mesh(self):
    return self._device_mesh

  @property
  def is_replicated(self) -> bool:
    if self._device_mesh is None or self._split_dims_mapping is None:
      return True
    return all(m < 0 for m in self._split_dims_mapping)

  @property
  def uneven_padding(self):
    return self._uneven_padding

  def NumShards(self, dim: int) -> int:
    if self.is_replicated:
      return 1
    m = self._split_dims_mapping[dim]
    return 1 if m < 0 else int(self._device_mesh.shape[m])

  def ShardShape(self, full_shape: Sequence[int]) -> List[int]:
    """Shape of one shard (ceil-divided, reference `ManualToAuto…`)."""
    if self.is_replicated:
      return list(full_shape)
    out = []
    for i, s in enumerate(full_shape):
      n = self.NumShards(i)
      out.append(-(-int(s) // n))
    return out

  def ShardSlices(self, full_shape, coords: Sequence[int]):
    """Index slices of the shard at mesh coordinates `coords`."""
    shard = self.ShardShape(full_shape)
    sl = []
    for i, s in enumerate(full_shape):
      m = -1 if self.is_replicated else self._split_dims_mapping[i]
      if m < 0:
        sl.append(slice(0, s))
      else:
        c = coords[m]
        sl.append(slice(c * shard[i], min((c + 1) * shard[i], s)))
    return tuple(sl)

  def ApplyToTensor(self, tensor, use_sharding_op=True):
    if self.is_replicated:
      return Replicate(tensor, use_sharding_op)
    return MeshSplit(tensor, self._device_mesh, self._split_dims_mapping,
                     use_sharding_op)

  def ApplyToVariable(self, variable):
    return self.ApplyToTensor(variable, use_sharding_op=False)

  def ManualToAutoPartitioning(self, tensor):
    """Local shard → logical full tensor (identity in explicit-SPMD land)."""
    return tensor

  def AutoToManualPartitioning(self, tensor):
    return tensor

  def __repr__(self):
    return 'TensorShardingSpec(%s, mesh_shape=%s)' % (
        self._split_dims_mapping,
        None if self._device_mesh is None else self._device_mesh.shape)


def GetVarSharding(var) -> TensorShardingSpec:
  """Sharding spec recorded on a variable at creation."""
  mesh = getattr(var, 'device_mesh', None)
  mapping = getattr(var, 'tensor_split_dims_mapping', None)
  if mesh is None or mapping is None:
    return TensorShardingSpec.ReplicatedSpec()
  return TensorShardingSpec.FromFullShape(list(var.shape), mapping, mesh)


def GetMeshSplitSharding(device_mesh, tensor_split_dims_mapping) -> 'TensorShardingSpec':
  """The sharding spec `MeshSplit` would attach, honouring the active dim-prefix and
  manual-dim contexts (ref :89)."""
  spec = TensorShardingSpec(list(_CTX.prefix) + list(tensor_split_dims_mapping), device_mesh)
  if _CTX.manual:
    spec.manual_mesh_dims = list(_CTX.manual)
  return spec


def ReshapeDim(x, dim, dim_reshape_segments=None):
  """[..., D, ...] → [..., segments, D // segments, ...] (ref :215)."""
  if dim_reshape_segments is None:
    return x
  dim = dim % x.dim()
  assert x.shape[dim] % dim_reshape_segments == 0
  return x.reshape(list(x.shape[:dim]) + [dim_reshape_segments,
                                          x.shape[dim] // dim_reshape_segments] +
                   list(x.shape[dim + 1:]))


_SPM_CACHE = {}


def LoadSpm(model_file):
  """Cached SentencePieceProcessor for `model_file` (ref :448)."""
  if model_file not in _SPM_CACHE:
    import sentencepiece  # pylint: disable=g-import-not-at-top
    spm = sentencepiece.SentencePieceProcessor()
    spm.Load(model_file)
    _SPM_CACHE[model_file] = spm
  return _SPM_CACHE[model_file]
