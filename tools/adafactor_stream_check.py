"""A/B check of the multi-stream Adafactor step (run on a GPU box).

Trains the flagship model for a few steps from identical weights / inputs with the factored
variables on 1 stream and on N streams, eager and graph-replayed, and compares losses and
per-variable checksums. Any cross-stream race shows up as a mismatch far above the
fp32-atomics noise floor (or as NaN).

  python tools/adafactor_stream_check.py [--model lm.synthetic_packed_input.MoELm8E] [--steps 6]
"""
import argparse
import gc
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def Run(model_name, streams, graph, steps):
  from lingvo_b200 import model_registry
  from lingvo_b200.core import cluster_factory, py_utils
  from lingvo_b200.ops import optim
  from lingvo_b200.parallel import mesh as mesh_lib
  import lingvo_b200.models.lm.params.synthetic_packed_input  # noqa: F401
  from lingvo_b200.parallel import symm
  symm._LOCAL.clear()   # per-model exchange buffers of the previous run  # pylint: disable=protected-access
  mesh_lib.Reset()
  optim.Invalidate()
  py_utils.SetGlobalStep(0)
  torch.manual_seed(0)
  cfg = model_registry.GetParams(model_name, 'Train')
  cfg.task.random_seed = 1
  cfg.input.random_seed = 5
  cfg.task.train.optimizer.num_update_streams = streams
  cfg.cluster.worker.gpus_per_replica = 1
  dev = torch.device('cuda', 0)
  with cluster_factory.Cluster(cfg.cluster):
    model = cfg.Instantiate()
    model.to(dev)
    task = model.tasks[0]
    from lingvo_b200.parallel import dp as dp_lib
    dp_lib.Attach(task)
    batches = [task._MoveBatch(task.input.GetPreprocessedInputBatch(), dev) for _ in range(4)]  # pylint: disable=protected-access
    graphed = None
    losses = []
    if graph:
      from lingvo_b200.core import graph_step
      graphed = graph_step.GraphedTrainStep(task, batches[0], warmup=3)
    for i in range(steps):
      b = batches[i % 4]
      metrics, _ = graphed(b) if graphed is not None else task.TrainStep([b])
      losses.append(float(metrics['loss'][0].detach()))
    torch.cuda.synchronize()
    sums = {v.var_name: float(v.detach().double().abs().sum()) for v in task.vars.Flatten()}
  del model, task, graphed, batches
  gc.collect()
  torch.cuda.empty_cache()
  return losses, sums


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--model', default='lm.synthetic_packed_input.MoELm8E')
  ap.add_argument('--steps', type=int, default=6)
  ap.add_argument('--streams', default='1,4,8')
  ap.add_argument('--out', default='gpurun_out/adafactor_stream_check.json')
  args = ap.parse_args()
  report = {}
  ok = True
  for graph in (False, True):
    base = None
    for s in [int(x) for x in args.streams.split(',')]:
      losses, sums = Run(args.model, s, graph, args.steps)
      key = '%s_s%d' % ('graph' if graph else 'eager', s)
      entry = {'losses': losses}
      if base is None:
        base = (losses, sums)
      else:
        rel = max(abs(sums[k] - base[1][k]) / max(abs(base[1][k]), 1e-12) for k in sums)
        worst = max(sums, key=lambda k: abs(sums[k] - base[1][k]) / max(abs(base[1][k]), 1e-12))
        dl = max(abs(a - b) for a, b in zip(losses, base[0]))
        entry.update(max_rel_checksum_diff=rel, worst_var=worst, max_loss_diff=dl)
        finite = all(x == x for x in losses)
        if not finite or rel > 2e-3 or dl > 5e-2:
          ok = False
      report[key] = entry
      print(key, json.dumps(entry), flush=True)
  os.makedirs(os.path.dirname(args.out), exist_ok=True)
  with open(args.out, 'w') as f:
    json.dump(report, f, indent=1)
  print('STREAM_CHECK_OK' if ok else 'STREAM_CHECK_MISMATCH')


if __name__ == '__main__':
  main()
