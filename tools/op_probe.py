"""Device-timed micro-benchmarks of the memory-bound fused ops (run on a GPU box):
norm fwd/bwd, MoE gate logits fwd/bwd vs the stock PyTorch formulation.

  python tools/op_probe.py > gpurun_out/op_probe.json
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def Time(fn, iters=30, warmup=5):
  flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  total = 0.0
  for _ in range(iters):
    flush.zero_()                      # evict L2 between iterations
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    total += e0.elapsed_time(e1)
  return total / iters * 1e3           # µs


def main():
  from lingvo_b200.ops import gate, norm
  out = {}
  t, m, e = 8192, 2048, 8
  x = torch.randn(t, m, device='cuda').to(torch.bfloat16).requires_grad_(True)
  scale = torch.ones(m, device='cuda', requires_grad=True)
  dy = torch.randn(t, m, device='cuda').to(torch.bfloat16)
  y = norm.rms_norm(x, scale, 1e-6)
  us = Time(lambda: norm.rms_norm(x, scale, 1e-6))
  out['rms_norm_fwd'] = {'us': us, 'GBps': 2 * t * m * 2 / us / 1e3}
  us = Time(lambda: torch.autograd.grad(y, [x, scale], dy, retain_graph=True))
  out['rms_norm_bwd'] = {'us': us, 'GBps': 3 * t * m * 2 / us / 1e3}

  gw = (torch.randn(m, e, device='cuda') * 0.05).to(torch.bfloat16).requires_grad_(True)
  dl = torch.randn(t, e, device='cuda')
  yl = gate.gate_logits(x, gw)
  us = Time(lambda: gate.gate_logits(x, gw))
  out['gate_logits_fwd'] = {'us': us, 'GBps': t * m * 2 / us / 1e3}
  us = Time(lambda: torch.autograd.grad(yl, [x, gw], dl, retain_graph=True))
  out['gate_logits_bwd'] = {'us': us, 'GBps': 2 * t * m * 2 / us / 1e3}
  ref = lambda: torch.matmul(x.to(torch.float32), gw.to(torch.float32))
  yr = ref()
  out['gate_logits_fwd_torch'] = {'us': Time(ref)}
  out['gate_logits_bwd_torch'] = {
      'us': Time(lambda: torch.autograd.grad(yr, [x, gw], dl, retain_graph=True))}
  print(json.dumps(out, indent=1))


if __name__ == '__main__':
  main()
