"""Input placement policy (ref `lingvo/core/input_policy.py`).

`Apply(input_params)` returns params of a subclass of the input generator that is pinned to
the cluster's *input device* — the host on a H100 box: batches are assembled (and split for
towers) in host memory, ideally pinned, and only the `DevicePrefetcher` of the train engine
moves them to the GPU with an asynchronous copy that overlaps the previous step. Without the
policy an input generator written with device-agnostic factory calls could allocate on
`cuda:0` under a `torch.device` context and serialise H2D copies into the step.
`BaseTask.__init__` applies the policy to `p.input` (ref base_model.py:431).
"""

import torch

from lingvo_b200.core.nested_map import NestedMap


def _InputDevice(gen):
  dev = getattr(gen.cluster, 'input_device', None) or 'cpu'
  return torch.device(dev)


def _ToDevice(batch, dev):
  def Move(x):
    if isinstance(x, torch.Tensor) and x.device != dev:
      return x.to(dev)
    return x
  if isinstance(batch, NestedMap):
    return batch.Transform(Move)
  if isinstance(batch, (list, tuple)):
    return type(batch)(_ToDevice(b, dev) for b in batch)
  return Move(batch)


def Apply(input_params):
  """Possibly wraps `input_params` according to the input policy."""
  if getattr(input_params.cls, '_input_policy_applied', False):
    return input_params

  class _UseInputDevice(input_params.cls):
    """Places the input generator — construction, batch assembly, splitting — on the
    cluster's input device."""

    _input_policy_applied = True

    def __init__(self, params):
      with torch.device(_InputDevice(self)):
        super().__init__(params)

    def GetPreprocessedInputBatch(self):
      dev = _InputDevice(self)
      with torch.device(dev):
        return _ToDevice(super().GetPreprocessedInputBatch(), dev)

    def SplitInputBatch(self, num_splits):
      dev = _InputDevice(self)
      with torch.device(dev):
        return _ToDevice(super().SplitInputBatch(num_splits), dev)

  _UseInputDevice.__name__ = input_params.cls.__name__
  _UseInputDevice.__qualname__ = input_params.cls.__qualname__
  _UseInputDevice.__module__ = input_params.cls.__module__
  return input_params.Copy().Set(cls=_UseInputDevice)
