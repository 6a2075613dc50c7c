"""CUDA-graph capture of a whole training step.

The train step of a large model issues hundreds of kernel launches from Python, and the host
loop that enqueues them can become the critical path. `GraphedTrainStep` captures
FProp → BProp → gradient sync → optimizer of a task ONCE into a CUDA graph and replays it:
one launch per step, the host only refreshes the inputs and the two step-dependent
hyper-parameters (learning rate, Adafactor decay), which live in device memory.

Requirements (checked / arranged here):
  * static shapes (fixed batch geometry) and static input buffers (`copy_` in);
  * no host synchronisation inside the step (metrics stay on the device);
  * optimizer with `graph_capturable` (reads lr/decay from `EnableDeviceHyper` tensors);
  * cross-rank flag protocol with device-side sequence counters (`moe_sync`).
Falls back to eager execution if capture fails.
"""

from __future__ import annotations

from absl import logging
import torch

from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap


class GraphedTrainStep:

  def __init__(self, task, example_batch: NestedMap, warmup: int = 3):
    self.task = task
    self.graph = None
    self.enabled = False
    self.launches_per_step = 0
    dev = task.Device()
    assert dev.type == 'cuda'
    for lrn in task.learners:
      if not getattr(lrn.optimizer, 'graph_capturable', False):
        raise ValueError('%s cannot be graph-captured' % type(lrn.optimizer).__name__)
    self.static_in = task._MoveBatch(example_batch, dev).Transform(  # pylint: disable=protected-access
        lambda x: x.clone() if isinstance(x, torch.Tensor) else x)
    for lrn in task.learners:
      lrn.optimizer.EnableDeviceHyper(dev)
    self._SetHyper()
    # Warm-up (eager, on a side stream as the capture protocol requires): creates optimizer
    # slots, compute copies, symmetric buffers, cuDNN plans, kernel attributes.
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
      for _ in range(warmup):
        self._SetHyper()
        task.TrainStep([self.static_in])
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    from lingvo_b200 import ops  # pylint: disable=g-import-not-at-top
    nat = ops.native()
    self._SetHyper()
    before = nat.launch_count()
    # Capture records kernels without running them: host-side step counters that the
    # traced Python code advances must be rolled back afterwards.
    saved_step = task.global_step
    saved_counts = [lrn.optimizer._step_count for lrn in task.learners]  # pylint: disable=protected-access
    graph = torch.cuda.CUDAGraph()
    try:
      with torch.cuda.graph(graph, capture_error_mode='thread_local'):
        metrics, per_example = task.TrainStep([self.static_in])
    except Exception as e:  # pylint: disable=broad-except
      logging.warning('CUDA-graph capture of the train step failed (%s); running eagerly.', e)
      torch.cuda.synchronize(dev)
      raise
    self.launches_per_step = nat.launch_count() - before
    task.global_step = saved_step
    py_utils.SetGlobalStep(saved_step)
    for lrn, c in zip(task.learners, saved_counts):
      lrn.optimizer._step_count = c   # pylint: disable=protected-access
    self.graph = graph
    self.static_out = (metrics, per_example)
    self.enabled = True

  def _SetHyper(self):
    task = self.task
    with py_utils.GlobalStepContext(task.global_step):
      for lrn in task.learners:
        lrn.optimizer.SetHyper(lrn.LearningRate(), task.global_step)

  def __call__(self, batch: NestedMap):
    """Copies `batch` into the static inputs, replays the step, advances host counters."""
    task = self.task
    src = batch.Flatten()
    dst = self.static_in.Flatten()
    for s, d in zip(src, dst):
      if isinstance(d, torch.Tensor):
        d.copy_(s, non_blocking=True)
    self._SetHyper()
    self.graph.replay()
    task.global_step = task.global_step + 1
    py_utils.SetGlobalStep(task.global_step)
    for lrn in task.learners:
      lrn.optimizer._step_count += 1   # pylint: disable=protected-access
    return self.static_out
