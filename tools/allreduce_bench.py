"""Device-timed benchmark of the peer-memory two-shot all-reduce kernel
(`comm_kernels.cu:allreduce_mean_bf16_kernel`) against NCCL, with NVLink roofline fractions.

Run under torchrun on N GPUs. For every size: time = CUDA events around
[flag sync → kernel → flag sync] (what a gradient bucket costs), max over ranks, median of
`iters`. Traffic model of a two-shot all-reduce of S bytes per rank over W ranks: every rank
*reads* (W−1)/W·S from its peers (reduce-scatter phase) and *writes* (W−1)/W·S to them
(all-gather phase), so per-GPU NVLink traffic is (W−1)/W·S in each direction; the roofline is
that volume over the 450 GB/s per-direction NVLink-4 rate of an H100 SXM. Also reports the capped-grid
variant used while overlapping with backward (`max_blocks=48`) and `dist.all_reduce`.
Writes gpurun_out/allreduce_bench_n<W>.json.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

NVLINK_GBS = 450.0


def Time(fn, iters=20, warmup=5):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  dist.barrier()
  ts = []
  for _ in range(iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))
  t = torch.tensor(sorted(ts)[len(ts) // 2], device='cuda')
  dist.all_reduce(t, op=dist.ReduceOp.MAX)
  return float(t)


def main():
  rank = int(os.environ['RANK'])
  torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', rank)))
  dist.init_process_group('nccl')
  w = dist.get_world_size()
  from lingvo_b200 import ops
  from lingvo_b200.parallel import symm as symm_lib
  from lingvo_b200.parallel import zero as zero_lib
  dev = torch.device('cuda', torch.cuda.current_device())
  sizes_mb = [1, 4, 16, 64, 256, 666]
  max_elems = max(sizes_mb) * (1 << 20) // 2
  max_elems = (max_elems + 8 * w - 1) // (8 * w) * (8 * w)
  arena = symm_lib.SymmArena(max_elems * 2 + (1 << 20), dev)
  off = arena.Alloc(max_elems * 2)
  buf = arena.Local(off, (max_elems,), torch.bfloat16)
  peers = torch.tensor([b + off for b in arena.peer_base], dtype=torch.int64)   # host table
  chan = zero_lib._Channels(arena, w, rank, n=4)   # pylint: disable=protected-access
  dist.barrier()
  nat = ops.native()
  rows = []
  for mb in sizes_mb:
    n = mb * (1 << 20) // 2
    n = n // (8 * w) * (8 * w)
    buf[:n].normal_()

    def Fused(max_blocks=0, n=n):
      chan.Sync(0)
      nat.allreduce_mean_bf16(peers, n // w, rank, w, 1.0 / w, dev.index, True, None, max_blocks)
      chan.Sync(1)

    nccl_buf = torch.randn(n, device=dev, dtype=torch.bfloat16)
    ms = Time(Fused)
    ms_cap = Time(lambda: Fused(48))
    ms_nccl = Time(lambda: dist.all_reduce(nccl_buf))
    link_bytes = (w - 1) / w * n * 2                     # per GPU, per direction
    row = dict(mbytes=mb, us_fused=round(ms * 1e3, 1), us_fused_48cta=round(ms_cap * 1e3, 1),
               us_nccl=round(ms_nccl * 1e3, 1),
               busbw_fused_gbs=round(link_bytes / ms / 1e6, 1),
               busbw_nccl_gbs=round(link_bytes / ms_nccl / 1e6, 1),
               nvlink_fraction_fused=round(link_bytes / ms / 1e6 / NVLINK_GBS, 3),
               nvlink_fraction_48cta=round(link_bytes / ms_cap / 1e6 / NVLINK_GBS, 3))
    rows.append(row)
    if rank == 0:
      print(json.dumps(row))
  # numerics: mean over ranks of rank-dependent data
  n = 8 * w * 1024
  buf[:n] = float(rank + 1)
  chan.Sync(2)
  nat.allreduce_mean_bf16(peers, n // w, rank, w, 1.0 / w, dev.index, True, None, 0)
  chan.Sync(3)
  torch.cuda.synchronize()
  want = (w + 1) / 2.0
  assert abs(float(buf[:n].float().mean()) - want) < 1e-2, (float(buf[:n].float().mean()), want)
  if rank == 0:
    os.makedirs('gpurun_out', exist_ok=True)
    with open('gpurun_out/allreduce_bench_n%d.json' % w, 'w') as f:
      json.dump(dict(world=w, nvlink_gbs_per_direction=NVLINK_GBS, rows=rows), f, indent=1)
    print('ALLREDUCE_BENCH_OK')
  dist.barrier()
  dist.destroy_process_group()


if __name__ == '__main__':
  main()
