"""Multi-GPU check of the fused tensor-parallel FFN (run under torchrun).

Compares `parallel.tp.TpFfn` (collectives inside the wgmma GEMM) against an
fp32 single-device oracle for forward and all gradients, then times it against
the NCCL all_gather + cuBLAS + reduce_scatter baseline.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist


def main():
  rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
  torch.cuda.set_device(int(os.environ['LOCAL_RANK']))
  dev = torch.device('cuda', int(os.environ['LOCAL_RANK']))
  dist.init_process_group('nccl', device_id=dev)
  from lingvo_b200.parallel import tp
  T, M, H = 8192, 2048, 8192
  if len(sys.argv) > 1:
    T, M, H = [int(v) for v in sys.argv[1:4]]
  g = torch.Generator(device='cpu').manual_seed(0)
  x = (torch.randn(T, M, generator=g) * 0.5).to(dev)
  wi = (torch.randn(M, H, generator=g) * M ** -0.5).to(dev)
  wo = (torch.randn(H, M, generator=g) * H ** -0.5).to(dev)
  dy = (torch.randn(T, M, generator=g) * 0.1).to(dev)
  ms, hs = M // world, H // world
  bf = torch.bfloat16
  xs = x[:, rank * ms:(rank + 1) * ms].to(bf).contiguous().requires_grad_()
  wis = wi[:, rank * hs:(rank + 1) * hs].to(bf).contiguous().requires_grad_()
  wos = wo[rank * hs:(rank + 1) * hs].to(bf).contiguous().requires_grad_()
  dys = dy[:, rank * ms:(rank + 1) * ms].to(bf).contiguous()

  # oracle (fp32 on bf16-rounded inputs)
  xr = x.to(bf).float().requires_grad_()
  wir = wi.to(bf).float().requires_grad_()
  wor = wo.to(bf).float().requires_grad_()
  yr = torch.relu(xr @ wir) @ wor
  yr.backward(dy.to(bf).float())

  eng = tp.TpEngine(T, M, H, dev)
  y = tp.TpFfn(eng, xs, wis, wos)
  y.backward(dys)
  torch.cuda.synchronize()

  def rel(a, b):
    return float((a.float() - b).norm() / b.norm())
  errs = {
      'y': rel(y, yr[:, rank * ms:(rank + 1) * ms]),
      'dx': rel(xs.grad, xr.grad[:, rank * ms:(rank + 1) * ms]),
      'dwi': rel(wis.grad, wir.grad[:, rank * hs:(rank + 1) * hs]),
      'dwo': rel(wos.grad, wor.grad[rank * hs:(rank + 1) * hs]),
  }
  # replicated-output (all-reduce) flavour
  y2 = tp.TpFfn(eng, xs.detach(), wis.detach(), wos.detach(), True)
  errs['y_allreduce'] = rel(y2, yr)
  yn = tp.TpFfnNccl(xs.detach(), wis.detach(), wos.detach())
  errs['y_nccl'] = rel(yn, yr[:, rank * ms:(rank + 1) * ms])
  ok = all(v < 2e-2 for v in errs.values())

  def timeit(fn, n=20):
    for _ in range(3):
      fn()
    dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
      fn()
    e1.record(); dist.barrier(); torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / n], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)

  xd, wid, wod = xs.detach(), wis.detach(), wos.detach()
  t_fused = timeit(lambda: tp.TpFfn(eng, xd, wid, wod))
  t_nccl = timeit(lambda: tp.TpFfnNccl(xd, wid, wod))
  def fb():
    xs.grad = wis.grad = wos.grad = None
    tp.TpFfn(eng, xs, wis, wos).backward(dys)
  t_fb = timeit(fb)
  flops = 4.0 * T * M * H / world
  if rank == 0:
    print(json.dumps({'world': world, 'T': T, 'M': M, 'H': H, 'rel_err': errs,
                      'fwd_ms_fused': t_fused, 'fwd_ms_nccl_cublas': t_nccl,
                      'fwd_bwd_ms_fused': t_fb,
                      'fwd_tflops_per_gpu_fused': flops / t_fused / 1e9,
                      'fwd_tflops_per_gpu_nccl': flops / t_nccl / 1e9}))
    print('TP_OK' if ok else 'TP_FAIL')
  dist.barrier()
  dist.destroy_process_group()


if __name__ == '__main__':
  main()
