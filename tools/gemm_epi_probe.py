"""Times the wgmma GEMM epilogue variants on FFN shapes (1 GPU)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lingvo_b200.ops import gemm as G

dev = torch.device('cuda')
bf = torch.bfloat16


def timeit(fn, n=30):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(n):
    fn()
  e1.record(); torch.cuda.synchronize()
  return e0.elapsed_time(e1) / n * 1e3

only = sys.argv[1] if len(sys.argv) > 1 else None
res = []
for (m, n, k) in [(8192, 4096, 2048), (8192, 8192, 2048), (8192, 2048, 8192), (16384, 8192, 2048)]:
  x = torch.randn(m, k, device=dev, dtype=bf)
  w = torch.randn(k, n, device=dev, dtype=bf) * 0.02
  h = torch.randn(m, n, device=dev, dtype=bf)
  out = torch.empty(m, n, device=dev, dtype=bf)
  fl = 2.0 * m * n * k
  if only == 'ncu':
    G.gemm(x, w, True, False, act=1, out=out)
    torch.cuda.synchronize()
    break
  r = {'m': m, 'n': n, 'k': k}
  for name, kw in [('act0', {}), ('relu', {'act': 1}),
                   ('relu_mask', {'aux': h, 'aux_mode': 1}), ('bias', {'bias': torch.zeros(n, device=dev)})]:
    us = timeit(lambda: G.gemm(x, w, True, False, out=out, **kw))
    r[name + '_us'] = round(us, 1)
    r[name + '_tf'] = round(fl / us / 1e6, 0)
  us = timeit(lambda: torch.mm(x, w, out=out))
  r['cublas_us'] = round(us, 1); r['cublas_tf'] = round(fl / us / 1e6, 0)
  res.append(r)
  print(json.dumps(r), flush=True)
