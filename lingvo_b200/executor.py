"""Single-process executor time-slicing the devices between programs.

Reference `lingvo/executor.py`: `GetExecutorParams` (:67-153),
`ExecutorTpu` (:161-619: restore → compile programs → loop {save, run
schedule, export metrics, should-stop}), multi-task sampling,
`HostDrivenExecutor` (:622).

On H100 the executor is the SPMD entrypoint: every rank runs the same
schedule; the train program's model is shared (by Parameter aliasing) with
the eval/decode programs of the same rank, so no checkpoint round-trip is
needed between train and eval.
"""

from __future__ import annotations

import logging
import os
import time
from typing import Dict, Optional

from lingvo_b200 import base_runner
from lingvo_b200 import flags
from lingvo_b200.core import base_model
from lingvo_b200.core import checkpointer
from lingvo_b200.core import cluster_factory
from lingvo_b200.core import program as program_lib
from lingvo_b200.core import py_utils
from lingvo_b200.core import task_scheduler

FLAGS = flags.FLAGS
flags.DEFINE_bool('cluster_placer_in_executor', False, 'Kept for parity.')
flags.DEFINE_bool('disable_meta_optimizer_in_executor', False, 'Kept.')
flags.DEFINE_bool('use_tpu_mirrored_vars', False, 'Kept for parity.')


def GetExecutorParams(model_name, cluster_params, model_registry):
  """(program-schedule params, {dataset: task params}) (reference :67)."""
  ps_params_dict = {}
  with cluster_factory.Cluster(cluster_params):
    ps_cfg = model_registry.GetProgramSchedule(model_name)
    train_cfg = model_registry.GetParams(model_name, 'Train')
    train_cfg.cluster = cluster_params
    if issubclass(train_cfg.cls, base_model.MultiTaskModel):
      multi_task_train_cfg = train_cfg
      for k, _ in multi_task_train_cfg.task_params.IterParams():
        ps = ps_cfg[k] if isinstance(ps_cfg, dict) else ps_cfg.Copy()
        ps.task_dict = {'Train': multi_task_train_cfg}
        ps.task_name = k
        for ds in ps.dataset_names:
          cfg = model_registry.GetParams(model_name, ds)
          cfg.cluster = cluster_params
          ps.task_dict[ds] = cfg
        ps_params_dict[k] = ps
      return ps_params_dict, multi_task_train_cfg
    ps_cfg.task_dict = {'Train': train_cfg}
    for ds in ps_cfg.dataset_names:
      cfg = model_registry.GetParams(model_name, ds)
      cfg.cluster = cluster_params
      ps_cfg.task_dict[ds] = cfg
    ps_params_dict[''] = ps_cfg
    return ps_params_dict, train_cfg


class ExecutorTpu(base_runner.BaseRunner):
  """Runs program schedules until `max_steps` (name kept for parity)."""

  def __init__(self, train_cfg, ps_params_dict, *args, **kwargs):
    if args:
      model_task_name, logdir = args[0], args[1]
      args = args[2:]
    else:
      model_task_name = kwargs.pop('model_task_name', '')
      logdir = kwargs.pop('logdir')
    super().__init__(train_cfg, model_task_name, logdir, *args, **kwargs)
    self._job_name = 'executor_tpu'
    self._ps_params_dict = ps_params_dict
    tp = train_cfg.train
    self._max_steps = tp.max_steps
    if 'task' in train_cfg and train_cfg.task is not None:
      self._max_steps = min(tp.max_steps, train_cfg.task.train.max_steps)
    self._programs = []
    self._program_schedule_dict: Dict[str, program_lib.SimpleProgramSchedule] = {}
    self._is_multi_task = issubclass(train_cfg.cls, base_model.MultiTaskModel)
    for task_name, ps in ps_params_dict.items():
      ps = ps.Copy()
      ps.logdir = logdir
      sched = ps.Instantiate()
      self._program_schedule_dict[task_name] = sched
    # Build: train program first so eval/decode can alias its variables.
    shared = None
    with self._cluster:
      for task_name, sched in self._program_schedule_dict.items():
        if sched.train_program is not None:
          if shared is not None:
            sched.train_program._shared_model = shared  # pylint: disable=protected-access
          self._model = sched.train_program.BuildTpuSubgraph()
          shared = self._model
      for sched in self._program_schedule_dict.values():
        for prog in sched.eval_programs:
          prog.BuildTpuSubgraph()
          if shared is not None:
            prog.ShareVariablesFrom(shared)
      if self._model is None:
        # Eval-only executor.
        first = next(iter(self._program_schedule_dict.values()))
        self._model = first.eval_programs[0]._model  # pylint: disable=protected-access
    self._checkpointer = checkpointer.Checkpointer(
        self._train_dir, self._model, train_params=tp)
    if self._is_multi_task:
      self._task_scheduler = self._model.task_schedule
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
    if rank == 0:
      os.makedirs(os.path.join(logdir, 'control'), exist_ok=True)
      with open(os.path.join(logdir, 'control', 'params.txt'), 'w') as f:
        f.write(train_cfg.ToText())
      from lingvo_b200.core import summary_utils
      text, _ = summary_utils.ModelAnalysis(self._model)
      with open(os.path.join(logdir, 'control', 'model_analysis.txt'), 'w') as f:
        f.write(text)

  def Start(self):
    self._RunLoop('executor_tpu', self._Loop)

  def _GlobalStep(self) -> int:
    return max(t.global_step for t in self._model.tasks)

  def _Loop(self):
    with self._cluster:
      self._checkpointer.Restore()
      self._LoadProgramState()
      # Engines attach data parallelism (rank 0's variables win) after the restore.
      for sched in self._program_schedule_dict.values():
        if sched.train_program is not None:
          self._checkpointer.AttachEngine(sched.train_program.engine)
          sched.train_program.engine.PostRestore()
      while True:
        global_step = self._GlobalStep()
        py_utils.SetGlobalStep(global_step)
        self._checkpointer.MaybeSave(gsteps=global_step)
        if self._ShouldStop(step=global_step):
          break
        if self._is_multi_task:
          task_name = self._task_scheduler.Sample(global_step)
          sched = self._program_schedule_dict[task_name]
        else:
          sched = self._program_schedule_dict['']
        done, train_s, eval_s = sched.Run()
        logging.info('executor: train %.2fs eval %.2fs', train_s, eval_s)
        self._ExportMetrics(train_time=train_s, eval_time=eval_s,
                            global_step=self._GlobalStep())
        self._SaveProgramState()
        if done:
          break
      self._checkpointer.Save(gsteps=self._GlobalStep(), sync=True)
      for sched in self._program_schedule_dict.values():
        sched.Shutdown()

  def _SaveProgramState(self):
    """Trigger counters etc. next to the checkpoints (reference `RunSave` :473)."""
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    if dist.is_available() and dist.is_initialized() and dist.get_rank() != 0:
      return
    for name, sched in self._program_schedule_dict.items():
      if hasattr(sched, 'SaveProgramState'):
        sched.SaveProgramState(os.path.join(
            self._train_dir, 'program_state%s.json' % (('_' + name) if name else '')))

  def _LoadProgramState(self):
    for name, sched in self._program_schedule_dict.items():
      if hasattr(sched, 'LoadProgramState'):
        sched.LoadProgramState(os.path.join(
            self._train_dir, 'program_state%s.json' % (('_' + name) if name else '')))

  def _ExportMetrics(self, **kwargs):
    self._cluster.ExportMetrics(**kwargs)


HostDrivenExecutor = ExecutorTpu
Executor = ExecutorTpu
