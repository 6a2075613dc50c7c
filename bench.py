#!/usr/bin/env python
"""Headline benchmark: tokens/s of the GShard-MoE 8-expert LM training step.

  python bench.py --gpus N --steps K --warmup W          (N = 1)
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N \
      --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...   (N > 1)

Metric (BASELINE.json): whole-job tokens/sec, device-timed (CUDA events on the
launching stream, barrier + synchronize on both sides, max over ranks) for
`lm.synthetic_packed_input.MoELm8E` (GShard MoE Transformer LM, 8 experts,
expert-parallel over the ranks), bf16 compute / fp32 master weights,
Adafactor step included, synthetic random-token data, random-init weights.
Weak scaling: 8 sequences × 1024 tokens per GPU.

`--impl reference` runs the stock-PyTorch comparator (`baseline/stock_moe_lm.py`: cuBLAS
matmul/einsum + SDPA + NCCL all_to_all/all_reduce + unfused Adafactor; the reference's dense
GSEC dispatch math) — TF lingvo itself cannot be installed here (DESIGN.md §7).
The measured arm is driven through the product entry point (`trainer.RunnerManager` →
`runners.Trainer` → `TrainEngine`), not a private loop.
"""

import argparse
import json
import os
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

MODEL = 'lm.synthetic_packed_input.MoELm8E'


def _ParseArgs():
  ap = argparse.ArgumentParser()
  ap.add_argument('--gpus', type=int, default=1)
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
  ap.add_argument('--model', default=MODEL)
  ap.add_argument('--comm', default=None, choices=[None, 'fused', 'nccl'],
                  help='fused = hand-written peer-memory kernels (default); '
                  'nccl = stock NCCL+cuBLAS baseline mode.')
  ap.add_argument('--no-e2e', action='store_true')
  ap.add_argument('--no-a2a', action='store_true',
                  help='skip the exposed all-to-all measurement (N > 1)')
  ap.add_argument('--cuda-graph', default='auto', choices=['auto', 'on', 'off'],
                  help='Capture the whole train step into a CUDA graph (auto: fall back '
                  'to eager launches if capture fails).')
  ap.add_argument('--dump-outputs', default=None, metavar='DIR',
                  help='After the timed steps, write what the last timed step returned '
                  '(metrics, per-example outputs) and a fixed sample of the updated '
                  'weights as DIR/<name>.npy.')
  return ap.parse_args()


class ClockSampler:
  """Samples nvidia-smi clocks / throttle reasons during the timed region."""

  Q = ('index,clocks.sm,clocks.max.sm,power.draw,'
       'clocks_event_reasons.hw_slowdown,'
       'clocks_event_reasons.hw_thermal_slowdown,'
       'clocks_event_reasons.sw_thermal_slowdown,'
       'clocks_event_reasons.sw_power_cap')

  def __init__(self, gpu_index=0):
    self._idx = gpu_index
    self._rows = []
    self._stop = threading.Event()
    self._t = None

  def _Run(self):
    while not self._stop.is_set():
      try:
        out = subprocess.run(
            ['nvidia-smi', '--query-gpu=' + self.Q, '--format=csv,noheader,nounits',
             '-i', str(self._idx)], capture_output=True, text=True, timeout=5)
        for line in out.stdout.strip().splitlines():
          self._rows.append([c.strip() for c in line.split(',')])
      except Exception:  # pylint: disable=broad-except
        pass
      self._stop.wait(0.2)

  def __enter__(self):
    self._t = threading.Thread(target=self._Run, daemon=True)
    self._t.start()
    return self

  def __exit__(self, *a):
    self._stop.set()
    self._t.join(timeout=6)

  def Summary(self):
    sm, smax, reasons = [], 0.0, set()
    names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown',
             'sw_power_cap']
    for r in self._rows:
      try:
        sm.append(float(r[1]))
        smax = max(smax, float(r[2]))
        for n, v in zip(names, r[4:8]):
          if v.lower().startswith('active'):
            reasons.add(n)
      except (ValueError, IndexError):
        continue
    sm.sort()
    return {'sm_mhz': sm[len(sm) // 2] if sm else None, 'sm_max_mhz': smax or None,
            'reasons': sorted(reasons), 'samples': len(sm)}


def _Reference(args):
  """Stock-PyTorch comparator (`baseline/stock_moe_lm.py`): nothing of lingvo_b200 —
  no kernels, no engine, no model — is imported on this path."""
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'baseline'))
  import torch
  if not torch.cuda.is_available():
    print(json.dumps({'impl': 'reference', 'unavailable': 'no GPU visible',
                      'n_gpus': args.gpus}))
    return 0
  import stock_moe_lm
  out = stock_moe_lm.RunBenchmark(args, ClockSampler)
  if out is not None:
    print(json.dumps(out), flush=True)
  return 0


def _CreateTrainer(args, logdir):
  """The product entry point: `lingvo_b200.trainer.RunnerManager` builds the same
  `runners.Trainer` that `python -m lingvo_b200.trainer --job=trainer_client` runs."""
  from lingvo_b200 import flags
  from lingvo_b200 import model_imports
  from lingvo_b200 import trainer as trainer_lib
  argv = ['bench', '--model=' + args.model, '--logdir=' + logdir, '--mode=sync',
          '--job=trainer_client', '--worker_gpus=1',
          '--use_cuda_graph=' + args.cuda_graph]
  flags.FLAGS(argv)
  model_imports.ImportParams(args.model)
  mgr = trainer_lib.RunnerManager(args.model)
  mgr.MaybeConfigRunDistributed()
  runner = mgr.CreateRunners(['trainer_client'], logdir)[0]
  return runner


def main():
  args = _ParseArgs()
  if args.impl == 'reference':
    return _Reference(args)
  if args.comm:
    os.environ['LINGVO_B200_COMM'] = args.comm

  import random
  import tempfile
  import numpy as np
  import torch
  import torch.distributed as dist
  # Weight init and the synthetic batches draw from these: same arguments, same inputs.
  random.seed(0)
  np.random.seed(0)
  torch.manual_seed(0)
  world = int(os.environ.get('WORLD_SIZE', '1'))
  rank = int(os.environ.get('RANK', '0'))
  local_rank = int(os.environ.get('LOCAL_RANK', '0'))
  assert torch.cuda.is_available(), 'bench.py needs a GPU'
  torch.cuda.set_device(local_rank)
  if world > 1:
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    dist.init_process_group('nccl', device_id=torch.device('cuda', local_rank))
  assert world == args.gpus, 'WORLD_SIZE %d != --gpus %d' % (world, args.gpus)
  dev = torch.device('cuda', local_rank)

  from lingvo_b200 import ops
  from lingvo_b200.parallel import mesh as mesh_lib
  native = ops.native(required=True)
  mesh_lib.Reset()

  logdir = tempfile.mkdtemp(prefix='lingvo_b200_bench_')
  runner = _CreateTrainer(args, logdir)
  task = runner.task
  with runner._cluster:   # pylint: disable=protected-access
    engine = runner.engine                      # DP attach + prefetcher + graph capture
    tp = task.params
    per_gpu_batch = task.input.InfeedBatchSize()
    seq_len = tp.sequence_length
    tokens_per_step = per_gpu_batch * seq_len * world

    def sync():
      if world > 1:
        dist.barrier()
      torch.cuda.synchronize()

    # ---- device-timed loop: inputs pre-staged on device --------------------
    n_total = args.warmup + args.steps
    batches = [task._MoveBatch(task.input.GetPreprocessedInputBatch(), dev)  # pylint: disable=protected-access
               for _ in range(min(n_total, 8))]

    def timed(n_warm, n_steps, sampler=None):
      for i in range(n_warm):
        engine.Step(batches[i % len(batches)])
      sync()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      ctx = sampler if sampler is not None else _Null()
      with ctx:
        sync()
        e0.record()
        for i in range(n_steps):
          m, per_example = engine.Step(batches[(n_warm + i) % len(batches)])
        e1.record()
        sync()
      ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
      if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
      return float(ms.item()), m, per_example

    # CUDA-graph capture (it runs warm-up steps of its own) happens here, never inside the
    # timed window, so the window holds exactly --steps train steps.
    engine._MaybeCapture(batches[0])   # pylint: disable=protected-access
    launches0 = native.launch_count()
    clocks = ClockSampler(local_rank)
    ms_total, metrics, per_example = timed(args.warmup, args.steps, clocks)
    if args.dump_outputs and rank == 0:
      _DumpOutputs(args.dump_outputs, metrics, per_example, task)
    launches = native.launch_count() - launches0
    if engine.cuda_graph:
      # kernels of ours executed per replay (counted while capturing) × timed steps
      launches = engine.launches_per_step * args.steps
    loss = float(metrics['loss'][0])
    ms_per_step = ms_total / args.steps
    value = tokens_per_step * args.steps / (ms_total / 1e3)

    # ---- end-to-end loop through the public API ----------------------------
    e2e = None
    if not args.no_e2e:
      for _ in range(2):
        engine.Step()
      sync()
      h2d = 0
      d2h = 0
      t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      t0.record()
      for _ in range(args.steps):
        m, _ = engine.Step()               # pinned host → device on a side stream + step
        h2d = engine.h2d_bytes_last
        host_loss = m['loss'][0].detach().float().cpu()   # D2H read of the loss
        d2h = host_loss.numel() * host_loss.element_size()
      t1.record()
      sync()
      ems = torch.tensor([t0.elapsed_time(t1)], device=dev)
      if world > 1:
        dist.all_reduce(ems, op=dist.ReduceOp.MAX)
      e2e = {'value': tokens_per_step * args.steps / (float(ems.item()) / 1e3),
             'unit': 'tokens/s', 'h2d_bytes_per_step': int(h2d),
             'd2h_bytes_per_step': int(d2h)}

    # ---- exposed all-to-all: same step with the EP exchange looped back locally ---------
    exposed_a2a = None
    if world > 1 and not args.no_a2a:
      exposed_a2a = _ExposedA2A(task, engine, batches, ms_per_step, timed, args)

  if rank == 0:
    ctx = mesh_lib.Get()
    out = {
        'metric': 'tokens/sec (whole job, device-timed, max over ranks) '
                  'GShard-MoE 8-expert LM training step',
        'value': value, 'unit': 'tokens/s', 'n_gpus': world,
        'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': ms_per_step,
        'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
        'dtype': 'bf16', 'data': 'synthetic (uniform random token ids, packed '
                                 'LM format; random-init weights)',
        'impl': 'ours', 'comm_mode': ctx.mode,
        'entry_point': 'lingvo_b200.trainer.RunnerManager → runners.Trainer.engine '
                       '(core/train_engine.py)',
        'cuda_graph': engine.cuda_graph,
        'config': {
            'model': args.model, 'global_batch': per_gpu_batch * world,
            'seq_len': seq_len, 'parallelism': 'dp%d+ep%d' % (
                world, min(world, tp.builder.e_dim or 1)),
            'experts': tp.builder.e_dim, 'model_dim': tp.builder.model_dim,
            'layers': tp.num_transformer_layers,
            'optimizer': type(task.learners[0].optimizer).__name__,
            'l2_flush': 'working set (fp32 params + bf16 activations) '
                        'is >> 50 MB L2; no explicit flush',
        },
        'clocks': clocks.Summary(), 'gpu_launches': int(launches),
        'final_loss': loss,
    }
    if e2e is not None:
      out['e2e'] = e2e
    if exposed_a2a is not None:
      out['exposed_a2a_ms_per_step'] = exposed_a2a
    print(json.dumps(out), flush=True)
  if world > 1:
    # Tear-down: a CUDA graph that holds captured NCCL kernels must be gone before the
    # communicator is destroyed, and a stuck destroy must never hold the job open — the
    # measurement is already printed, so a watchdog ends the process if it takes too long.
    import gc
    engine._graphed = None   # pylint: disable=protected-access
    gc.collect()
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    sys.stdout.flush()
    sys.stderr.flush()
    watchdog = threading.Timer(20.0, lambda: os._exit(0))
    watchdog.daemon = True
    watchdog.start()
    dist.destroy_process_group()
    watchdog.cancel()
  import shutil
  shutil.rmtree(logdir, ignore_errors=True)
  return 0


_DUMP_LIMIT_BYTES = 64 << 20
_WEIGHT_SAMPLE = 4096


def _DumpOutputs(out_dir, metrics, per_example, task):
  """Writes the last timed step's results as float32/float64 `.npy` files: every metric
  (value and weight), every per-example output, and for each weight the same seeded sample
  of at most `_WEIGHT_SAMPLE` elements after the update."""
  import numpy as np
  import torch
  os.makedirs(out_dir, exist_ok=True)
  arrays = {}

  def _Add(name, v):
    t = torch.as_tensor(v).detach()
    dtype = torch.float64 if t.dtype == torch.float64 else torch.float32
    arrays[name] = t.to(dtype).cpu().numpy()

  for k, v in sorted(metrics.items()):
    if isinstance(v, (tuple, list)):
      _Add('metric.%s' % k, v[0])
      _Add('metric.%s.weight' % k, v[1])
    else:
      _Add('metric.%s' % k, v)
  if per_example:
    for k, v in per_example.FlattenItems():
      if isinstance(v, torch.Tensor) or np.isscalar(v):
        _Add('per_example.%s' % k, v)
  for k, v in task.vars.FlattenItems():
    flat = v.detach().reshape(-1)
    if flat.numel() > _WEIGHT_SAMPLE:
      gen = torch.Generator().manual_seed(0)
      idx = torch.randperm(flat.numel(), generator=gen)[:_WEIGHT_SAMPLE].sort().values
      flat = flat[idx.to(flat.device)]
    _Add('weight.%s' % k, flat)
  total = sum(a.nbytes for a in arrays.values())
  assert total <= _DUMP_LIMIT_BYTES, 'dump of %d bytes exceeds 64 MB' % total
  for k, a in arrays.items():
    np.save(os.path.join(out_dir, k.replace('/', '.') + '.npy'), a)


class _Null:

  def __enter__(self):
    return self

  def __exit__(self, *a):
    return False


def _ExposedA2A(task, engine, batches, ms_normal, timed, args):
  """ms/step the expert exchange costs on the critical path: step time minus the time of
  the *same* step with every peer store/load redirected to local memory and the peer
  flag waits removed (`MoeExchange.loopback`). NCCL mode: not measured this way."""
  import torch
  from lingvo_b200.core import graph_step
  from lingvo_b200.parallel import mesh as mesh_lib
  ctx = mesh_lib.Get()
  exchanges = [e._fused for e in ctx._ep_engines.values() if getattr(e, '_fused', None)]  # pylint: disable=protected-access
  if not exchanges:
    return None
  saved = engine._graphed   # pylint: disable=protected-access
  try:
    for ex in exchanges:
      ex.loopback = True
    if saved is not None:
      engine._graphed = graph_step.GraphedTrainStep(task, batches[0], warmup=2)  # pylint: disable=protected-access
    ms_lb = timed(2, args.steps)[0]
    return max(0.0, ms_normal - ms_lb / args.steps)
  except Exception as e:  # pylint: disable=broad-except
    sys.stderr.write('exposed-a2a measurement failed: %r\n' % (e,))
    return None
  finally:
    for ex in exchanges:
      ex.loopback = False
    engine._graphed = saved   # pylint: disable=protected-access


if __name__ == '__main__':
  sys.exit(main())
