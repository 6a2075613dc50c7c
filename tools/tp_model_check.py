"""Tensor parallelism through the model API on N GPUs (run under torchrun).

Builds the GShard dense UniTransformer twice in every process with identical (name-seeded)
logical weights:
  * TP:     `device_mesh_shape=[1, N]` → attention heads and FFN hidden dim sharded N ways,
            NCCL all-reduce at the two region boundaries, local wgmma GEMMs;
  * oracle: the same model unsharded on this GPU.
Checks, in bf16 compute with fp32 masters: loss, per-variable gradients (shards gathered),
and 5 Adafactor/Adam steps; then reports ms/step of both for the strong-scaling record.
Prints TP_MODEL_OK on success.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist


def Params(tp, model_dim, heads, ff, layers, vocab):
  from lingvo_b200.core import gshard_builder as gb
  from lingvo_b200.core import optimizer
  from lingvo_b200.core import schedule
  w = dist.get_world_size()
  b = gb.DenseBuilder.Params().Set(
      model_dim=model_dim, attention_num_heads=heads, attention_key_value_dim=128, ff_dim=ff,
      relative_attention_type='bias', relative_attention_num_buckets=32,
      relative_attention_max_distance=128, relative_attention_use_universal_1d_position=True,
      device_mesh_shape=[1, w], dtype=torch.float32, fprop_dtype=torch.bfloat16)
  if not tp:
    b.mhd_w_split = [-1, -1, -1]
    b.mh_wi_split = [-1, -1]
    b.hm_wo_split = [-1, -1]
  p = gb.UniTransformer.Params().Set(
      name='lm', builder=b, vocab_size=vocab, num_transformer_layers=layers, max_length=1024,
      positional_embedding=False, label_smoothing=0.0, z_loss=0.0, gated_gelu=False,
      dtype=torch.float32, fprop_dtype=torch.bfloat16)
  p.random_seed = 4321
  p.train.learning_rate = 1e-3
  p.train.lr_schedule = schedule.Constant.Params()
  p.train.optimizer = optimizer.Adam.Params().Set(beta1=0.9, beta2=0.99, epsilon=1e-6)
  p.train.clip_gradient_norm_to_value = 1.0
  return p


def Batch(bsz, l, vocab, dev):
  from lingvo_b200.core.nested_map import NestedMap
  g = torch.Generator().manual_seed(7)
  ids = torch.randint(2, vocab, (bsz, l), generator=g)
  seg = torch.ones(bsz, l, dtype=torch.long)
  seg[:, l // 2:] = 2
  pos = torch.arange(l).repeat(bsz, 1) % (l // 2)
  return NestedMap(ids=ids, labels=torch.roll(ids, -1, 1), paddings=torch.zeros(bsz, l),
                   segment_ids=seg, segment_pos=pos).Transform(lambda t: t.to(dev))


def Build(tp, dims):
  from lingvo_b200.core import base_model
  from lingvo_b200.core import cluster_factory
  from lingvo_b200.parallel import dp
  with cluster_factory.ForTestingWorker(mode='sync', job='trainer_client', gpus=1):
    model = base_model.SingleTaskModel.Params(Params(tp, *dims)).Instantiate()
    model.to(torch.device('cuda', torch.cuda.current_device()))
    task = model.GetTask()
    if tp:
      dp.Attach(task)
    task.EnableMixedPrecision()
  return task


def LossAndGrads(task, batch, gather):
  from lingvo_b200.parallel import mesh as mesh_lib
  from lingvo_b200.parallel import tp_layers
  ctx = mesh_lib.TensorParallel()
  metrics, _ = task.FPropDefaultTheta(batch)
  loss = metrics['loss'][0]
  loss.backward()
  grads = {}
  for v in task.vars.Flatten():
    src = getattr(v, 'compute', None)
    g = (src.grad if src is not None and src.grad is not None else v.grad)
    g = g.detach().float().clone()
    shard = getattr(v, 'tp_shard', None)
    if gather and shard is not None:
      g = tp_layers.GatherShards(g, ctx, shard[2])
    grads[v.var_name] = g
    v.grad = None
    if src is not None:
      src.grad = None
  task._metrics = None   # pylint: disable=protected-access
  return float(loss), grads


def TimeSteps(task, batch, n=8):
  for _ in range(3):
    task.TrainStep(batch)
  torch.cuda.synchronize()
  dist.barrier()
  t0 = torch.cuda.Event(enable_timing=True)
  t1 = torch.cuda.Event(enable_timing=True)
  t0.record()
  losses = []
  for _ in range(n):
    m, _ = task.TrainStep(batch)
    losses.append(m['loss'][0].detach())
  t1.record()
  torch.cuda.synchronize()
  ms = torch.tensor([t0.elapsed_time(t1) / n], device='cuda')
  dist.all_reduce(ms, op=dist.ReduceOp.MAX)
  return float(ms), [float(x) for x in losses]


def main():
  rank = int(os.environ['RANK'])
  torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', rank)))
  dist.init_process_group('nccl')
  from lingvo_b200.parallel import mesh
  mesh.Reset(mode='nccl')
  w = dist.get_world_size()
  dims = (1024, 8, 4096, 2, 8192)            # model_dim, heads (D=128), ff_dim, layers, vocab
  dev = torch.device('cuda', torch.cuda.current_device())
  batch = Batch(4, 512, dims[-1], dev)
  tp_task = Build(True, dims)
  ctx = mesh.TensorParallel()
  assert ctx is not None and ctx.tp_size == w, 'tensor parallelism did not engage'
  n_sharded = sum(1 for v in tp_task.vars.Flatten() if getattr(v, 'tp_shard', None))
  assert n_sharded >= 6 * dims[3], n_sharded
  ref_task = Build(False, dims)
  assert not any(getattr(v, 'tp_shard', None) for v in ref_task.vars.Flatten())

  l_tp, g_tp = LossAndGrads(tp_task, batch, gather=True)
  l_ref, g_ref = LossAndGrads(ref_task, batch, gather=False)
  assert abs(l_tp - l_ref) < 2e-2 * max(1.0, abs(l_ref)), (l_tp, l_ref)
  worst = (0.0, '')
  for name, want in g_ref.items():
    got = g_tp[name]
    assert got.shape == want.shape, (name, got.shape, want.shape)
    err = float((got - want).norm() / want.norm().clamp_min(1e-6))
    worst = max(worst, (err, name))
    assert err < 6e-2, (name, err)

  ms_tp, loss_tp = TimeSteps(tp_task, batch)
  ms_ref, loss_ref = TimeSteps(ref_task, batch)
  assert all(abs(a - b) < 5e-2 * max(1.0, abs(b)) for a, b in zip(loss_tp, loss_ref)), (
      loss_tp, loss_ref)
  assert loss_tp[-1] < loss_tp[0]
  if rank == 0:
    rec = dict(world=w, dims=dict(model_dim=dims[0], heads=dims[1], ff_dim=dims[2],
                                  layers=dims[3], vocab=dims[4], tokens=4 * 512),
               loss_tp=l_tp, loss_ref=l_ref, worst_grad_rel_err=worst[0], worst_var=worst[1],
               ms_per_step_tp=round(ms_tp, 3), ms_per_step_single_gpu=round(ms_ref, 3),
               sharded_vars=n_sharded)
    os.makedirs('gpurun_out', exist_ok=True)
    with open('gpurun_out/tp_model_check_n%d.json' % w, 'w') as f:
      json.dump(rec, f, indent=1)
    print(json.dumps(rec))
    print('TP_MODEL_OK')
  dist.barrier()
  dist.destroy_process_group()


if __name__ == '__main__':
  main()
