"""Programs & program schedules for the executor.

Reference `lingvo/core/program.py`: `BaseProgram` (:75), `TrainProgram` (:441;
`steps_per_loop` on-device loop), `EvalProgram` (:995), `DecodeProgram`
(:1229), `MultiInputsDecodeProgram`, `ExperimentalDecodeProgram`,
`MLPerfTrainDecodeProgram`, `InputBenchmark` (:2249), `SimpleProgramSchedule`
(:2329), `MLPerfProgramSchedule`, `SimpleProgramScheduleForTask` (:2705),
`UpdateProgramSchedule` (:2835).

H100-first: a program is "run N steps of task X on this process group".
`TrainProgram.Run` executes `steps_per_loop` eager steps and syncs scalar
metrics to the host **once per loop** (the TPU-loop analogue); eval/decode
accumulate metrics on device (`DeviceEvalMetrics`).
"""

from __future__ import annotations

import abc
import logging
import os
import pickle
import time
from typing import Dict, List, Optional

import numpy as np
import torch

from lingvo_b200.core import base_model
from lingvo_b200.core import cluster_factory
from lingvo_b200.core import hyperparams
from lingvo_b200.core import metrics as metrics_lib
from lingvo_b200.core import program_utils
from lingvo_b200.core import py_utils
from lingvo_b200.core import summary_utils
from lingvo_b200.utils import tfevents


class BaseProgram:
  """A unit of work the executor time-slices the devices between."""

  @classmethod
  def Params(cls):
    p = hyperparams.InstantiableParams(cls)
    p.Define('task', None, 'Underlying task params.')
    p.Define('logdir', None, 'Log directory.')
    p.Define('num_splits_per_client', None, 'Kept for parity.')
    p.Define('steps_per_loop', None, 'Steps per device loop.')
    p.Define('dataset_name', None, 'Dataset the program is operating on.')
    p.Define('name', 'base_program', 'Program name.')
    p.Define('task_name', None, 'Task name if multi-task, else None.')
    p.Define('num_threads', 1, 'Background threads.')
    p.Define('spmd', False, 'Kept for parity.')
    p.Define('write_train_input_stats', False, 'Write input stats.')
    p.Define('max_metrics', 256, 'Kept for parity.')
    p.Define('ml_perf', None, 'MLPerf config.')
    return p

  def __init__(self, params, shared_model=None, trial_status_fn=None, **kwargs):
    self.params = params.Copy()
    p = self.params
    self._task_params = p.task
    self._logdir = p.logdir
    self._task_name = p.task_name
    self._program_name = ''
    self._shared_model = shared_model
    self._model = None
    self._task = None
    self._summary_writer = None
    self._program_dir = None
    self._status_fn = trial_status_fn

  def _OutputDir(self) -> str:
    p = self.params
    name = self._program_name + ('_' + p.dataset_name.lower()
                                 if p.dataset_name else '')
    if self._task_name:
      name += '_' + self._task_name
    d = os.path.join(self._logdir, name)
    os.makedirs(d, exist_ok=True)
    return d

  def BuildTpuSubgraph(self):
    """Builds (or adopts) the model for this program (reference :583)."""
    raise NotImplementedError()

  def SetStatusMessage(self, msg):
    logging.info('%s', msg)

  def Compile(self):
    return None

  def Run(self, sess=None, threadpool=None) -> bool:
    """Returns True when the experiment should stop."""
    raise NotImplementedError()

  def Shutdown(self):
    if self._summary_writer:
      self._summary_writer.flush()

  def SaveProgramState(self, sess=None, global_step=None):
    return None

  def _WriteSummaries(self, job_name, global_step, summaries: Dict[str, float]):
    for k, v in summaries.items():
      self._summary_writer.add_scalar(k, float(v), global_step)
    self._summary_writer.flush()
    msg = '%s: step:%6d' % (job_name, global_step)
    for k in sorted(summaries):
      msg += ' %s:%.8g' % (k, summaries[k])
    self.SetStatusMessage(msg)

  def _InstantiateModel(self, do_eval: bool):
    """Own model for this program's dataset (input differs per program)."""
    p = self.params
    cp = p.task.cluster.Copy() if 'cluster' in p.task else (
        cluster_factory.Current().params.Copy())
    cp.do_eval = do_eval
    self._cluster = cluster_factory.Cluster(cp)
    with self._cluster:
      if self._shared_model is not None and not do_eval:
        self._model = self._shared_model
      else:
        self._model = p.task.Instantiate()
        self._model.to(py_utils.CurrentDevice())
    self._task = (self._model.GetTask(self._task_name) if self._task_name
                  else self._model.tasks[0])

  def ShareVariablesFrom(self, src_model):
    """Eval/decode programs alias the train model's Parameters (same GPU)."""
    src = {v.var_name: v for v in src_model.vars.Flatten()}
    for _, layer in self._model.Walk():
      for k, v in list(layer._private_vars.items()):  # pylint: disable=protected-access
        if v.var_name in src:
          layer._private_vars[k] = src[v.var_name]  # pylint: disable=protected-access


class TrainProgram(BaseProgram):
  """Runs `steps_per_loop` train steps per invocation."""

  def __init__(self, params, **kwargs):
    super().__init__(params, **kwargs)
    self._program_name = 'TrainProgram'
    self._step_rate_tracker = summary_utils.StepRateTracker()

  def BuildTpuSubgraph(self):
    self._InstantiateModel(do_eval=False)
    self._program_dir = self._OutputDir()
    self._summary_writer = tfevents.EventFileWriter(self._program_dir)
    return self._model

  @property
  def model(self):
    return self._model

  @property
  def engine(self):
    """DP sync + device prefetch + CUDA-graph replay (`core/train_engine.py`)."""
    if getattr(self, '_engine', None) is None:
      from lingvo_b200.core import train_engine  # pylint: disable=g-import-not-at-top
      with self._cluster:
        self._engine = train_engine.TrainEngine(self._task)
    return self._engine

  def Run(self, sess=None, threadpool=None) -> bool:
    p = self.params
    task = self._task
    acc = metrics_lib.DeviceEvalMetrics()
    t0 = time.time()
    with self._cluster:
      engine = self.engine
      for _ in range(p.steps_per_loop):
        m, _ = engine.Step()
        acc.Update({k: v for k, v in m.items()})
    results = acc.Finalize()
    step = task.global_step
    self.global_step = int(step)
    vals = {k: v for k, (v, _) in results.items()}
    n_ex = vals.get('num_samples_in_batch', 0.0) * p.steps_per_loop
    rate, ex_rate, total = self._step_rate_tracker.ComputeStepRate(step, n_ex)
    vals['global_step/sec'] = rate
    vals['examples/sec'] = ex_rate
    vals['total_samples'] = total
    self._WriteSummaries(os.path.basename(self._program_dir), step, vals)
    tp = task.params.train
    return step >= tp.max_steps


class EvalProgram(BaseProgram):
  """Evaluates `steps_per_loop` batches (or the whole resettable dataset)."""

  def __init__(self, params, **kwargs):
    super().__init__(params, **kwargs)
    self._program_name = 'EvalProgram'

  def BuildTpuSubgraph(self):
    self._InstantiateModel(do_eval=True)
    self._program_dir = self._OutputDir()
    self._summary_writer = tfevents.EventFileWriter(self._program_dir)
    return self._model

  def Run(self, sess=None, threadpool=None) -> bool:
    p = self.params
    task = self._task
    task.input.Reset()
    acc = metrics_lib.DeviceEvalMetrics()
    steps = 0
    with self._cluster:
      while p.steps_per_loop < 0 or steps < p.steps_per_loop:
        try:
          m, _ = task.EvalStep()
        except StopIteration:
          break
        acc.Update(m)
        steps += 1
    results = acc.Finalize()
    step = py_utils.GetGlobalStep()
    vals = {k: v for k, (v, _) in results.items()}
    self.last_metrics = vals
    self._WriteSummaries(os.path.basename(self._program_dir), int(step), vals)
    with open(os.path.join(self._program_dir,
                           'score-{:08d}.txt'.format(int(step))), 'w') as f:
      for k in sorted(vals):
        f.write('%s: %s\n' % (k, vals[k]))
    return False


class DecodeProgram(BaseProgram):
  """Decodes `steps_per_loop` batches and post-processes on the host."""

  def __init__(self, params, **kwargs):
    super().__init__(params, **kwargs)
    self._program_name = 'DecodeProgram'

  def BuildTpuSubgraph(self):
    self._InstantiateModel(do_eval=True)
    self._program_dir = self._OutputDir()
    self._summary_writer = tfevents.EventFileWriter(self._program_dir)
    self._cache = program_utils.DecodeStatusCache(self._program_dir)
    return self._model

  def Run(self, sess=None, threadpool=None) -> bool:
    p = self.params
    task = self._task
    step = int(py_utils.GetGlobalStep())
    if self._cache.TryLoadCache(str(step)):
      logging.info('Decode of step %d already done; skipping.', step)
      return False
    task.input.Reset()
    dec_metrics = task.CreateDecoderMetrics()
    buffered = []
    steps = 0
    start = time.time()
    with self._cluster:
      while p.steps_per_loop < 0 or steps < p.steps_per_loop:
        try:
          out = self._model.ConstructDecodeGraph(self._task_name)
        except StopIteration:
          break
        host = {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor)
                    else (tuple(x.detach().cpu().numpy()
                                if isinstance(x, torch.Tensor) else x
                                for x in v) if isinstance(v, (tuple, list))
                          else v)) for k, v in out.items()}
        post = task.PostProcessDecodeOut(host, dec_metrics)
        if post:
          buffered.extend(post)
        steps += 1
    vals = {k: m.value for k, m in dec_metrics.items()}
    self.last_metrics = dict(vals)
    vals['decode_secs'] = time.time() - start
    self._WriteSummaries(os.path.basename(self._program_dir), step, vals)
    out_path = os.path.join(self._program_dir, 'decoder_out_%09d' % step)
    with open(out_path, 'wb') as f:
      pickle.dump(buffered, f)
    task.DecodeFinalize(base_model.DecodeFinalizeArgs(out_path, buffered))
    self._cache.UpdateCkpt(str(step))
    return False


class MultiInputsDecodeProgram(DecodeProgram):
  """Decodes several datasets with one model (reference :1807)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_params', {}, '{dataset_name: input params}.')
    return p


class HostDrivenTrainProgram(TrainProgram):
  """Train program whose loop is driven step by step from the host (reference :771
  `HostDrivenTrainProgram`): no on-device loop / CUDA-graph replay — every step is an
  eager `TrainStep`, metrics reach the host every `metrics_every_n` steps and per-step
  callbacks may inspect or alter the model in between (debugging, curriculum, custom
  hooks)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('metrics_every_n', 1, 'Fetch metrics to the host every n steps.')
    return p

  def __init__(self, params, **kwargs):
    super().__init__(params, **kwargs)
    self._program_name = 'HostDrivenTrainProgram'
    self._step_callbacks = []

  def AddStepCallback(self, fn):
    """fn(global_step, metrics_dict_or_None) called after every step."""
    self._step_callbacks.append(fn)

  @property
  def engine(self):
    if getattr(self, '_engine', None) is None:
      from lingvo_b200.core import train_engine  # pylint: disable=g-import-not-at-top
      with self._cluster:
        self._engine = train_engine.TrainEngine(self._task, use_cuda_graph='off')
    return self._engine

  def Run(self, sess=None, threadpool=None) -> bool:
    p = self.params
    task = self._task
    acc = metrics_lib.DeviceEvalMetrics()
    with self._cluster:
      engine = self.engine
      for i in range(p.steps_per_loop):
        m, _ = engine.Step()
        acc.Update(dict(m))
        host = None
        if (i + 1) % max(p.metrics_every_n, 1) == 0:
          host = {k: float(v[0]) for k, v in m.items()}
        for fn in self._step_callbacks:
          fn(task.global_step, host)
    results = acc.Finalize()
    step = task.global_step
    self.global_step = int(step)
    vals = {k: v for k, (v, _) in results.items()}
    self._WriteSummaries(os.path.basename(self._program_dir), step, vals)
    return step >= task.params.train.max_steps


class ExperimentalDecodeProgram(DecodeProgram):
  """Decode program that overlaps device decoding with host post-processing (reference
  :1807): batch i+1 is decoded on the device while a worker thread runs
  `PostProcessDecodeOut` (detokenisation, BLEU/WER bookkeeping) on batch i."""

  def __init__(self, params, **kwargs):
    super().__init__(params, **kwargs)
    self._program_name = 'ExperimentalDecodeProgram'

  def Run(self, sess=None, threadpool=None) -> bool:
    import queue  # pylint: disable=g-import-not-at-top
    import threading  # pylint: disable=g-import-not-at-top
    p = self.params
    task = self._task
    step = int(py_utils.GetGlobalStep())
    if self._cache.TryLoadCache(str(step)):
      logging.info('Decode of step %d already done; skipping.', step)
      return False
    task.input.Reset()
    dec_metrics = task.CreateDecoderMetrics()
    buffered = []
    q = queue.Queue(maxsize=4)
    err = []

    def worker():
      while True:
        host = q.get()
        if host is None:
          return
        try:
          post = task.PostProcessDecodeOut(host, dec_metrics)
          if post:
            buffered.extend(post)
        except BaseException as e:  # pylint: disable=broad-except
          err.append(e)

    th = threading.Thread(target=worker, name='decode_postprocess', daemon=True)
    th.start()
    steps = 0
    start = time.time()
    with self._cluster:
      while (p.steps_per_loop < 0 or steps < p.steps_per_loop) and not err:
        try:
          out = self._model.ConstructDecodeGraph(self._task_name)
        except StopIteration:
          break
        # async D2H: the copy of batch i overlaps the device decode of batch i+1
        host = {k: (v.detach().to('cpu', non_blocking=True) if isinstance(v, torch.Tensor)
                    else v) for k, v in out.items()}
        if torch.cuda.is_available():
          torch.cuda.current_stream().synchronize()
        q.put({k: (v.numpy() if isinstance(v, torch.Tensor) else v) for k, v in host.items()})
        steps += 1
    q.put(None)
    th.join()
    if err:
      raise err[0]
    vals = {k: m.value for k, m in dec_metrics.items()}
    self.last_metrics = dict(vals)
    vals['decode_secs'] = time.time() - start
    self._WriteSummaries(os.path.basename(self._program_dir), step, vals)
    out_path = os.path.join(self._program_dir, 'decoder_out_%09d' % step)
    with open(out_path, 'wb') as f:
      pickle.dump(buffered, f, protocol=pickle.HIGHEST_PROTOCOL)
    task.DecodeFinalize(base_model.DecodeFinalizeArgs(out_path, buffered))
    self._cache.UpdateCkpt(str(step))
    return False


class MLPerfTrainDecodeProgram(BaseProgram):
  """One program that alternates `train_steps_per_loop` train steps with
  `decode_steps_per_loop` decode batches on the *same* variables (reference :2037), so an
  MLPerf run needs no checkpoint round-trip between training and scoring."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('train_task', None, 'Train task params.')
    p.Define('decode_task', None, 'Decode task params.')
    p.Define('train_dataset_name', None, 'Train dataset.')
    p.Define('decode_dataset_name', None, 'Decode dataset.')
    p.Define('train_steps_per_loop', 0, 'Train steps per loop.')
    p.Define('decode_steps_per_loop', 0, 'Decode steps per loop.')
    return p

  def __init__(self, params, **kwargs):
    super().__init__(params, **kwargs)
    self._program_name = 'MLPerfTrainDecodeProgram'
    p = self.params
    tp = TrainProgram.Params().Set(
        name='train', task=p.train_task, logdir=p.logdir, task_name=p.task_name,
        dataset_name=p.train_dataset_name, steps_per_loop=p.train_steps_per_loop)
    dp = DecodeProgram.Params().Set(
        name='decode', task=p.decode_task, logdir=p.logdir, task_name=p.task_name,
        dataset_name=p.decode_dataset_name, steps_per_loop=p.decode_steps_per_loop)
    self._train = tp.Instantiate(shared_model=kwargs.get('shared_model'))
    self._decode = dp.Instantiate()

  def BuildTpuSubgraph(self):
    model = self._train.BuildTpuSubgraph()
    self._decode.BuildTpuSubgraph()
    self._decode.ShareVariablesFrom(model)
    self._model = model
    return model

  @property
  def last_metrics(self):
    return getattr(self._decode, 'last_metrics', None)

  def Run(self, sess=None, threadpool=None) -> bool:
    done = self._train.Run(sess)
    self.global_step = self._train.global_step
    self._decode.Run(sess, threadpool)
    return done

  def Shutdown(self):
    self._train.Shutdown()
    self._decode.Shutdown()


class InputBenchmark(BaseProgram):
  """Measures raw input pipeline throughput (reference :2249)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('measurement_type', 'per_batch', 'per_batch|per_example.')
    return p

  def __init__(self, params, **kwargs):
    super().__init__(params, **kwargs)
    self._program_name = 'InputBenchmark'

  def BuildTpuSubgraph(self):
    self._InstantiateModel(do_eval=False)
    self._program_dir = self._OutputDir()
    self._summary_writer = tfevents.EventFileWriter(self._program_dir)

  def Run(self, sess=None, threadpool=None) -> bool:
    p = self.params
    t0 = time.time()
    n = 0
    for _ in range(p.steps_per_loop):
      b = self._task.input.GetPreprocessedInputBatch()
      for t in b.Flatten():
        if hasattr(t, 'shape') and len(t.shape) > 0:
          n += int(t.shape[0])
          break
    dt = time.time() - t0
    self._WriteSummaries('input_benchmark', int(py_utils.GetGlobalStep()),
                         {'batches/sec': p.steps_per_loop / max(dt, 1e-9),
                          'examples/sec': n / max(dt, 1e-9)})
    return True


def _CreateProgramParams(cls, program_name, dataset_name, steps_per_loop,
                         spmd=False):
  p = cls.Params()
  p.name = program_name
  p.dataset_name = dataset_name
  p.steps_per_loop = steps_per_loop
  p.spmd = spmd
  return p


class BaseProgramSchedule(abc.ABC):
  """What the executor drives (:2287): `Run()` advances every program of the schedule by
  its share of steps and returns (done, train seconds, eval seconds)."""

  @classmethod
  def Params(cls):
    return hyperparams.InstantiableParams(cls)

  @abc.abstractmethod
  def Run(self, sess=None, threadpool=None):
    """Runs the programs for some number of steps according to the schedule."""

  @abc.abstractmethod
  def Shutdown(self):
    """Cleans up every program."""

  @abc.abstractmethod
  def Programs(self) -> List['BaseProgram']:
    """The programs managed by the schedule."""


class SimpleProgramSchedule(BaseProgramSchedule):
  """train N steps → [eval datasets] → [decode datasets], repeated (:2329)."""

  @classmethod
  def Params(cls):
    p = hyperparams.InstantiableParams(cls)
    p.Define('task_dict', None, 'dataset_name → task params.')
    p.Define('task_name', None, 'Task name for multi-task models.')
    p.Define('logdir', None, 'Log directory.')
    p.Define('train_program', None, 'Train program params.')
    p.Define('train_executions_per_eval', 1, 'Train loops per eval round.')
    p.Define('eval_programs', [], 'Eval/decode program params.')
    p.Define('num_splits_per_client', None, 'Kept for parity.')
    p.Define('dataset_names', [], 'Dataset names.')
    p.Define('async_postprocess', True, 'Kept for parity.')
    p.Define('emails', [], 'Kept for parity.')
    p.Define('summary_exporter', None, 'Kept for parity.')
    p.Define('eval_program_triggers', None,
             'Optional {dataset: (offset, interval)} to trigger eval programs.')
    p.Define('train_summary_exporter', None, 'Kept for parity.')
    p.Define('ml_perf', None, 'MLPerf config.')
    return p

  def __init__(self, params, shared_model=None, trial_status_fn=None, **kwargs):
    self.params = params.Copy()
    p = self.params
    self._programs: List[BaseProgram] = []
    self.train_program = None
    self.eval_programs = []
    self._triggers = {}
    if p.train_program is not None and p.train_executions_per_eval != 0:
      tp = p.train_program.Copy()
      tp.logdir = p.logdir
      tp.task_name = p.task_name
      if tp.dataset_name not in p.task_dict:
        raise ValueError('could not find train dataset %s in %s' %
                         (tp.dataset_name, list(p.task_dict)))
      tp.task = p.task_dict[tp.dataset_name]
      self.train_program = tp.Instantiate(shared_model=shared_model,
                                          trial_status_fn=trial_status_fn)
      self._programs.append(self.train_program)
    for ep in p.eval_programs:
      ep = ep.Copy()
      ep.logdir = p.logdir
      ep.task_name = p.task_name
      ep.task = p.task_dict[ep.dataset_name]
      prog = ep.Instantiate(shared_model=shared_model,
                            trial_status_fn=trial_status_fn)
      self.eval_programs.append(prog)
      self._programs.append(prog)
      if p.eval_program_triggers and ep.dataset_name in p.eval_program_triggers:
        off, itv = p.eval_program_triggers[ep.dataset_name]
        self._triggers[id(prog)] = program_utils.TriggerScheduler(off, itv)

  def Programs(self):
    return self._programs

  def Run(self, sess=None, threadpool=None):
    p = self.params
    start = time.time()
    done = False
    train_time = 0.0
    for _ in range(p.train_executions_per_eval if self.train_program else 0):
      t0 = time.time()
      done = self.train_program.Run(sess) or done
      train_time += time.time() - t0
      if done:
        break
    eval_time = 0.0
    t0 = time.time()
    for prog in self.eval_programs:
      trig = self._triggers.get(id(prog))
      if trig is not None:
        trig.Trigger()
        if not trig.ShouldRun() and not done:
          continue
      prog.Run(sess, threadpool)
    eval_time = time.time() - t0
    done = self._MlPerfCheck() or done
    return done, train_time, eval_time

  def _MlPerfCheck(self):
    """MLPerf epoch / stop logging; True once the run should stop."""
    mp = self.params.ml_perf
    if mp is None or mp.benchmark_name is None or mp.steps_per_epoch is None:
      return False
    from lingvo_b200.core import ml_perf_log as mlp_log
    step = 0
    if self.train_program is not None:
      step = int(getattr(self.train_program, 'global_step', 0) or 0)
    epoch = int(step / mp.steps_per_epoch) if mp.steps_per_epoch else 0
    if not getattr(self, '_mlperf_started', False):
      self._mlperf_started = True
      for k, v in (mp.submission_metadata or {}).items():
        mlp_log.mlperf_print(k, v)
      mlp_log.mlperf_print('init_stop', None)
      mlp_log.mlperf_print('run_start', None)
    mlp_log.mlperf_print('eval_stop', None, metadata={'epoch_num': epoch})
    value = None
    for prog in self.eval_programs:
      res = getattr(prog, 'last_metrics', None) or {}
      if mp.decoder_metric_name in res:
        value = res[mp.decoder_metric_name]
        if isinstance(value, (tuple, list)):
          value = value[0]
    if value is not None:
      mlp_log.mlperf_print('eval_accuracy', float(value), metadata={'epoch_num': epoch})
      if (mp.decoder_metric_success_threshold is not None and
          float(value) > mp.decoder_metric_success_threshold):
        mlp_log.mlperf_print('run_stop', None, metadata={'status': 'success'})
        return True
    if mp.max_steps_to_train is not None and step >= mp.max_steps_to_train:
      mlp_log.mlperf_print('run_stop', None, metadata={'status': 'abort'})
      return True
    return False

  def Shutdown(self):
    for prog in self._programs:
      prog.Shutdown()

  # -- program state (reference `SaveProgramState` :545): what a resumed executor needs
  #    besides the model checkpoint — trigger counters and decode bookkeeping.
  def SaveProgramState(self, path: str):
    import json  # pylint: disable=g-import-not-at-top
    state = {'triggers': {}, 'programs': [type(pr).__name__ for pr in self._programs]}
    for prog in self.eval_programs:
      trig = self._triggers.get(id(prog))
      if trig is not None:
        state['triggers'][prog.params.dataset_name] = trig.State()
    tmp = path + '.tmp'
    with open(tmp, 'w') as f:
      json.dump(state, f)
    os.replace(tmp, path)

  def LoadProgramState(self, path: str) -> bool:
    import json  # pylint: disable=g-import-not-at-top
    if not os.path.exists(path):
      return False
    with open(path) as f:
      state = json.load(f)
    for prog in self.eval_programs:
      trig = self._triggers.get(id(prog))
      st = state.get('triggers', {}).get(prog.params.dataset_name)
      if trig is not None and st is not None:
        trig.SetState(st)
    return True


class MLPerfProgramSchedule(SimpleProgramSchedule):
  """MLPerf schedule (:2835): ONE `MLPerfTrainDecodeProgram` that trains and scores on the
  same live variables; the compliance log / early stop come from the `ml_perf` params."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.ml_perf = MlPerfParams()
    return p

  def __init__(self, params, shared_model=None, trial_status_fn=None, **kwargs):   # pylint: disable=super-init-not-called
    self.params = params.Copy()
    p = self.params
    tp = p.train_program.Copy()
    for name in (tp.train_dataset_name, tp.decode_dataset_name):
      if name not in p.task_dict:
        raise ValueError('could not find %s in %s' % (name, list(p.task_dict)))
    tp.logdir = p.logdir
    tp.task_name = p.task_name
    tp.train_task = p.task_dict[tp.train_dataset_name]
    tp.decode_task = p.task_dict[tp.decode_dataset_name]
    tp.ml_perf = p.ml_perf.Copy() if p.ml_perf is not None else None
    self.train_program = tp.Instantiate(shared_model=shared_model,
                                        trial_status_fn=trial_status_fn)
    self._programs = [self.train_program]
    # `_MlPerfCheck` reads the decode metrics from the "eval programs"
    self.eval_programs = []
    self._mlperf_metric_sources = [self.train_program]
    self._triggers = {}

  def Run(self, sess=None, threadpool=None):
    start = time.time()
    done = False
    for _ in range(self.params.train_executions_per_eval):
      done = self.train_program.Run(sess, threadpool) or done
      if done:
        break
    train_time = time.time() - start
    self.eval_programs = self._mlperf_metric_sources
    try:
      done = self._MlPerfCheck() or done
    finally:
      self.eval_programs = []
    return done, train_time, 0.0


class MultiTaskProgramSchedule:
  """One `SimpleProgramSchedule` per task of a multi-task model (reference :2319): the
  executor samples a task per loop (`task_scheduler`), runs that task's schedule, and all
  tasks train the shared variables of one `MultiTaskModel`."""

  @classmethod
  def Params(cls):
    p = hyperparams.InstantiableParams(cls)
    p.Define('program_schedule_dict', None, 'task name → SimpleProgramSchedule params.')
    p.Define('logdir', None, 'Log directory.')
    return p

  def __init__(self, params, shared_model=None, **kwargs):
    self.params = params.Copy()
    p = self.params
    assert p.program_schedule_dict
    self.schedules = {}
    self._programs = []
    self.train_program = None
    self.eval_programs = []
    for name in sorted(p.program_schedule_dict):
      sp = p.program_schedule_dict[name].Copy()
      sp.logdir = p.logdir
      sp.task_name = sp.task_name or name
      sched = sp.Instantiate(shared_model=shared_model, **kwargs)
      self.schedules[name] = sched
      self._programs.extend(sched.Programs())
      self.eval_programs.extend(sched.eval_programs)
      if self.train_program is None:
        self.train_program = sched.train_program
    self.steps_run = {name: 0 for name in self.schedules}

  def Programs(self):
    return self._programs

  def Run(self, task_name=None, sess=None, threadpool=None):
    """Runs the schedule of `task_name` (all tasks round-robin when None)."""
    names = [task_name] if task_name is not None else sorted(self.schedules)
    done, train_s, eval_s = False, 0.0, 0.0
    for name in names:
      d, t, e = self.schedules[name].Run(sess, threadpool)
      self.steps_run[name] += 1
      done, train_s, eval_s = done or d, train_s + t, eval_s + e
    return done, train_s, eval_s

  def Shutdown(self):
    for s in self.schedules.values():
      s.Shutdown()


def MlPerfParams():
  """MLPerf run description attached to a schedule (reference :2669-2700): when
  `benchmark_name` and `steps_per_epoch` are set the schedule emits MLPerf log lines and
  stops as soon as `decoder_metric_name` reaches the success threshold."""
  mp = hyperparams.Params()
  mp.Define('submission_metadata', None, 'Dict of static submission fields.')
  mp.Define('benchmark_name', None, 'MLPerf benchmark name, e.g. "bert".')
  mp.Define('steps_per_epoch', None, 'Training steps per (possibly fractional) epoch.')
  mp.Define('decoder_metric_name', None, 'Eval/decode metric compared to the threshold.')
  mp.Define('decoder_metric_success_threshold', None, 'Target quality.')
  mp.Define('max_steps_to_train', None, 'Give up after this many steps.')
  mp.Define('global_batch_size', None, 'Logged.')
  mp.Define('max_sequence_length', None, 'Logged.')
  mp.Define('optimizer_name', None, 'Logged.')
  mp.Define('base_learning_rate', None, 'Logged.')
  mp.Define('warmup_steps', None, 'Logged.')
  return mp


def MLPerfProgramScheduleForTask(train_dataset_name, train_steps_per_loop, decode_dataset_name,
                                 decode_steps_per_loop):
  """`MLPerfProgramSchedule` params for one train and one decode dataset (:2913)."""
  ps = MLPerfProgramSchedule.Params()
  ps.train_program = MLPerfTrainDecodeProgram.Params().Set(
      name='train_and_decode', train_steps_per_loop=train_steps_per_loop,
      decode_steps_per_loop=decode_steps_per_loop, dataset_name=train_dataset_name,
      train_dataset_name=train_dataset_name, decode_dataset_name=decode_dataset_name)
  ps.dataset_names = [train_dataset_name, decode_dataset_name]
  return ps


def SimpleProgramScheduleForTask(train_dataset_name, train_steps_per_loop,
                                 eval_dataset_names, eval_steps_per_loop,
                                 decode_steps_per_loop=None,
                                 experimental_decoder=False,
                                 train_program_cls=TrainProgram,
                                 eval_program_cls=EvalProgram,
                                 async_postprocess=True,
                                 decode_until_out_of_range=False,
                                 postprocess_all_at_once=False,
                                 emails=None, train_summary_exporter=None,
                                 summary_exporter=None, spmd=False):
  """Standard train → eval → decode schedule (reference :2705)."""
  ps = SimpleProgramSchedule.Params()
  ps.train_executions_per_eval = 1
  ps.dataset_names = list(eval_dataset_names)
  ps.ml_perf = MlPerfParams()
  if train_dataset_name:
    ps.train_program = _CreateProgramParams(
        train_program_cls, 'train', train_dataset_name, train_steps_per_loop,
        spmd)

  def per_ds(v, name, idx):
    if isinstance(v, dict):
      return v.get(name)
    if isinstance(v, (list, tuple)):
      return v[idx]
    return v

  for i, name in enumerate(eval_dataset_names):
    n = per_ds(eval_steps_per_loop, name, i)
    if n is not None and n != 0:
      ps.eval_programs.append(_CreateProgramParams(
          eval_program_cls, 'eval_tpu', name, n, spmd))
    d = per_ds(decode_steps_per_loop, name, i)
    if decode_until_out_of_range:
      d = -1
    if d is not None and d != 0:
      ps.eval_programs.append(_CreateProgramParams(
          DecodeProgram, 'decode_tpu', name, d, spmd))
  return ps


def UpdateProgramSchedule(ps_params, dataset_list, train_executions_per_eval,
                          train_steps_per_loop, eval_steps_per_loop,
                          decode_steps_per_loop, multi_inputs_decoder=None,
                          decode_summary_emails=None,
                          oneoff_checkpoint_to_load=None, train_summary_exporter=None):
  """Overrides a schedule from flags (reference :2835)."""
  assert ps_params
  if dataset_list is not None:
    ps_params.dataset_names = dataset_list
    ps_params.eval_programs = [ep for ep in ps_params.eval_programs
                               if ep.dataset_name in dataset_list]
  if train_executions_per_eval is not None:
    ps_params.train_executions_per_eval = train_executions_per_eval
  if train_steps_per_loop is not None and ps_params.train_program is not None:
    ps_params.train_program.steps_per_loop = train_steps_per_loop
  for ep in ps_params.eval_programs:
    if issubclass(ep.cls, DecodeProgram):
      if decode_steps_per_loop is not None:
        ep.steps_per_loop = decode_steps_per_loop
    elif eval_steps_per_loop is not None:
      ep.steps_per_loop = eval_steps_per_loop
  return ps_params
