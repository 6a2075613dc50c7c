"""Cluster topology: who am I, how many peers, which devices.

Reference: `lingvo/core/cluster.py` — `_Cluster.Params()` job specs (:72-169),
derived quantities (:377-515), variable placers (:586-654), thread-local
cluster stack (:66,254-265).

H100-first re-design: there is ONE process per GPU (torchrun). A "replica" is
a rank; `worker.replicas × worker.gpus_per_replica` therefore equals the
world size of the data-parallel group when launched distributed, and the
parameter-server job disappears: `VarPlacer` becomes the *optimizer-state
shard assigner* (ZeRO-1 style) that maps every variable to the least-loaded
rank by bytes, which is what the reference's `_LeastLoadedPlacer` does for PS
devices. Device strings are torch devices (`cuda:<local_rank>`/`cpu`).
"""

from __future__ import annotations

import collections
import contextlib
import heapq
import os
import threading
from typing import List, Optional

import numpy as np
import torch

from lingvo_b200.core import hyperparams
from lingvo_b200.core.nested_map import NestedMap


class _LocalStack(threading.local):

  def __init__(self):
    super().__init__()
    self.stack = []


_CLUSTER_STACK = _LocalStack()

_ROLES = ('controller', 'train_summaries', 'worker', 'ps', 'input', 'evaler',
          'decoder')


def _JobSpec(replicas: int, name: str = ''):
  p = hyperparams.Params()
  p.Define('name', name or '/job:localhost', 'Job name (kept for flag parity).')
  p.Define('replicas', replicas, 'Number of replicas (ranks) of this job.')
  p.Define('targets', '', 'Comma-separated host:port rendezvous targets.')
  p.Define('cpus_per_replica', 1, 'CPU devices per replica.')
  p.Define('gpus_per_replica', 0, 'GPUs per replica.')
  p.Define('tpus_per_replica', 0, 'Kept for parity; always 0 on H100.')
  p.Define('devices_per_split', 1, 'Devices one model split spans.')
  p.Define('num_tpu_hosts', 0, 'Kept for parity.')
  p.Define('additional_worker_names', [], 'Kept for parity.')
  return p


class _Cluster:
  """Describes the topology the current process runs in."""

  @classmethod
  def Params(cls):
    p = hyperparams.InstantiableParams(cls)
    p.Define('mode', 'async', 'sync|async.')
    p.Define('job', 'trainer',
             'controller|trainer|trainer_client|evaler|decoder|executor_tpu…')
    p.Define('task', 0, 'Task id (rank) within the job.')
    p.Define('logdir', '', 'Log directory.')
    p.Define('do_eval', None, 'Whether this cluster is for eval/decode.')
    p.Define('in_unit_test', None, 'True inside unit tests.')
    p.Define('split_id', 0, 'Active model-split index.')
    p.Define('require_sequential_input_order', None,
             'Input must be sequential (eval / unit tests).')
    p.Define('xla_device', None, 'Kept for parity.')
    p.Define('enable_asserts', None, 'Cluster-level override of the flag.')
    p.Define('enable_check_numerics', None, 'Cluster-level override.')
    p.Define('tf_data_service_address', '', 'Remote input workers address.')
    p.Define('add_summary', None, 'Whether summaries are emitted.')
    p.Define('immediately_instantiate_variables', True, 'Kept for parity.')
    for role in _ROLES:
      p.Define(role, _JobSpec(1 if role in ('controller', 'worker') else 0),
               'Job spec of the %s role.' % role)
    return p

  def __init__(self, params):
    self._params = params.Copy()
    p = self._params
    if p.job in ('controller', 'trainer', 'trainer_client', 'executor_tpu'):
      pass
    # Multi-process context (torchrun env) if any.
    self._rank = int(os.environ.get('RANK', '0'))
    self._world = int(os.environ.get('WORLD_SIZE', '1'))
    self._local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    self._cm = None

  # --------------------------------------------------------- context stack --
  def __enter__(self):
    _CLUSTER_STACK.stack.append(self)
    return self

  def __exit__(self, *args):
    assert _CLUSTER_STACK.stack and _CLUSTER_STACK.stack[-1] is self
    _CLUSTER_STACK.stack.pop()

  @staticmethod
  def _TopOrNone():
    return _CLUSTER_STACK.stack[-1] if _CLUSTER_STACK.stack else None

  # ------------------------------------------------------------ properties --
  @property
  def params(self):
    return self._params

  @property
  def mode(self):
    return self.params.mode

  @property
  def job(self):
    return self.params.job

  @property
  def logdir(self):
    return self.params.logdir

  @property
  def task(self):
    return self.params.task

  @property
  def rank(self):
    return self._rank

  @property
  def world_size(self):
    return self._world

  @property
  def local_rank(self):
    return self._local_rank

  @property
  def job_spec(self):
    p = self.params
    if p.job in ('controller',):
      return p.controller
    if p.job in ('trainer', 'worker', 'trainer_client', 'executor_tpu'):
      return p.worker
    if p.job == 'train_summaries':
      return p.train_summaries
    if p.job == 'evaler':
      return p.evaler
    if p.job == 'decoder':
      return p.decoder
    if p.job == 'input':
      return p.input
    if p.job == 'ps':
      return p.ps
    return p.worker

  @property
  def asynchronous(self):
    return self.params.mode == 'async'

  @property
  def synchronous(self):
    return self.params.mode == 'sync'

  @property
  def in_unit_test(self):
    return bool(self.params.in_unit_test)

  @property
  def do_eval(self):
    return bool(self.params.do_eval)

  @property
  def require_sequential_input_order(self):
    if self.params.require_sequential_input_order is not None:
      return self.params.require_sequential_input_order
    return self.do_eval

  @property
  def add_summary(self):
    p = self.params
    if p.add_summary is None:
      return p.job in ('controller', 'train_summaries', 'evaler', 'decoder',
                       'trainer', 'trainer_client', 'executor_tpu')
    return bool(p.add_summary)

  @property
  def num_replicas(self):
    return self.job_spec.replicas

  @property
  def cpus_per_replica(self):
    return self.job_spec.cpus_per_replica

  @property
  def gpus_per_replica(self):
    return self.job_spec.gpus_per_replica

  @property
  def tpus_per_replica(self):
    return 0

  @property
  def num_tpu_hosts(self):
    return 0

  @property
  def num_devices_per_replica(self):
    return self.gpus_per_replica or self.cpus_per_replica or 1

  @property
  def total_worker_devices(self):
    return self.num_devices_per_replica * self.num_replicas

  @property
  def num_devices_per_split(self):
    return self.job_spec.devices_per_split

  @property
  def num_splits_per_replica(self):
    assert self.num_devices_per_replica % self.num_devices_per_split == 0, (
        'Device count (%d) is not a multiple of device per split (%d)' %
        (self.num_devices_per_replica, self.num_devices_per_split))
    return self.num_devices_per_replica // self.num_devices_per_split

  @property
  def num_splits_per_client(self):
    """Splits handled by this process. Under torchrun every replica is its own process
    (one per GPU), so a process only ever owns its replica's splits; the reference's
    in-graph replication (one `trainer_client` driving all replicas) applies only to a
    single-process launch."""
    if self._world > 1:
      return self.num_splits_per_replica
    if self.synchronous and self.job in ('trainer_client', 'executor_tpu'):
      return self.num_splits_per_replica * self.num_replicas
    return self.num_splits_per_replica

  def RunsOnGpu(self) -> bool:
    return self.gpus_per_replica > 0 and torch.cuda.is_available()

  @property
  def available_devices(self) -> np.ndarray:
    """[replicas, devices_per_replica] array of torch device strings."""
    spec = self.job_spec
    n = self.num_devices_per_replica
    rows = []
    for r in range(max(spec.replicas, 1)):
      if spec.gpus_per_replica:
        rows.append(['cuda:%d' % ((r * n + i) if self._world == 1 else
                                  self._local_rank) for i in range(n)])
      else:
        rows.append(['cpu'] * n)
    return np.array(rows, dtype=object)

  def WorkerDeviceInModelSplit(self, device_index: int) -> str:
    """Device `device_index` of the active model split (reference :493)."""
    devices = self.available_devices.reshape([-1]).tolist()
    if not devices:
      return 'cpu'
    split = self.params.split_id * self.num_devices_per_split
    return devices[(split + device_index) % len(devices)]

  def GetPlacer(self, strategy=None):
    """Shard assigner: var → owning rank (ZeRO) (reference placers :586-654)."""
    n = max(self._world, 1)
    if strategy == 'round_robin':
      return RoundRobinPlacer(n)
    return LeastLoadedPlacer(n)

  @property
  def input_device(self) -> str:
    return 'cpu'

  @property
  def input_targets(self):
    return self.params.input.targets

  def PlaceInput(self, input_params):
    return input_params

  def ExportMetrics(self, *args, **kwargs):
    """Hook for external metric exporters (reference cluster.ExportMetrics)."""

  def InitDevices(self, sess=None):
    return None


# -- infeed context / device strings (ref cluster.py:33-63, 657) ------------------------------
InfeedContext = collections.namedtuple('InfeedContext', ['infeed_host_index',
                                                         'num_infeed_hosts'])
_INFEED_CONTEXT_STACK = _LocalStack()


@contextlib.contextmanager
def InfeedContextScope(infeed_host_index, num_infeed_hosts):
  """Names which input shard the enclosed input-generator construction serves."""
  _INFEED_CONTEXT_STACK.stack.append(InfeedContext(infeed_host_index, num_infeed_hosts))
  try:
    yield
  finally:
    _INFEED_CONTEXT_STACK.stack.pop()


def GetInfeedContext():
  """Innermost `InfeedContextScope`, else this process' rank / world size."""
  if _INFEED_CONTEXT_STACK.stack:
    return _INFEED_CONTEXT_STACK.stack[-1]
  return InfeedContext(infeed_host_index=int(os.environ.get('RANK', 0)),
                       num_infeed_hosts=int(os.environ.get('WORLD_SIZE', 1)))


def MakeDeviceString(job_name, replica_id, task_id, device_name, device_id):
  return '%s/replica:%d/task:%d/device:%s:%d' % (job_name, replica_id, task_id, device_name,
                                                 device_id)


def ParseDeviceString(device_str):
  """`/job:x/replica:r/task:t/device:GPU:i` → NestedMap(job, replica, task, device)."""
  parsed = NestedMap()
  for part in device_str.split('/'):
    if part.startswith('job:'):
      parsed.job = part[4:]
    elif part.startswith('replica:'):
      parsed.replica = int(part[8:])
    elif part.startswith('task:'):
      parsed.task = int(part[5:])
    elif part.startswith('device:'):
      parsed.device = part[7:].split(':')[0]
  return parsed


class VarPlacer:
  """Assigns each variable to an owner rank; default: everything on rank 0."""

  def __init__(self, num_owners: int):
    self._n = num_owners

  def Assign(self, name: str, nbytes: int) -> int:
    return 0


class RoundRobinPlacer(VarPlacer):

  def __init__(self, num_owners):
    super().__init__(num_owners)
    self._next = 0

  def Assign(self, name, nbytes):
    r = self._next
    self._next = (self._next + 1) % self._n
    return r


class LeastLoadedPlacer(VarPlacer):
  """Greedy bytes-balanced assignment (reference `_LeastLoadedPlacer` :624)."""

  def __init__(self, num_owners):
    super().__init__(num_owners)
    self._heap = [(0, i) for i in range(num_owners)]
    heapq.heapify(self._heap)
    self.assignment = collections.OrderedDict()

  def Assign(self, name, nbytes):
    load, idx = heapq.heappop(self._heap)
    heapq.heappush(self._heap, (load + int(nbytes), idx))
    self.assignment[name] = idx
    return idx

  def Loads(self) -> List[int]:
    return [l for l, _ in sorted(self._heap, key=lambda t: t[1])]
