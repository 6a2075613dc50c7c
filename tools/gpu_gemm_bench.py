"""Times the wgmma GEMM vs cuBLAS (torch.matmul) with CUDA events."""
import json
import sys
import torch
from lingvo_b200.ops import gemm as G


def bench(fn, iters=20, warm=5):
  flush = torch.empty(256 << 20, dtype=torch.int8, device='cuda')
  for _ in range(warm):
    fn()
  ts = []
  for _ in range(iters):
    flush.zero_()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True)
    a.record(); fn(); b.record(); b.synchronize()
    ts.append(a.elapsed_time(b))
  ts.sort()
  return ts[len(ts) // 2]


def main():
  out = []
  shapes = [(1, 8192, 8192, 8192), (1, 16384, 8192, 2048), (1, 16384, 2048, 8192),
            (8, 4096, 8192, 2048), (8, 4096, 2048, 8192), (1, 4096, 4096, 4096)]
  for g, m, n, k in shapes:
    a = torch.randn(g, m, k, device='cuda').bfloat16()
    b = torch.randn(g, n, k, device='cuda').bfloat16()
    bt = b.transpose(1, 2).contiguous()
    fl = 2.0 * g * m * n * k
    t_nt = bench(lambda: G.gemm(a, b, True, True))
    t_nn = bench(lambda: G.gemm(a, bt, True, False))
    t_cb = bench(lambda: torch.matmul(a, b.transpose(1, 2)))
    rec = dict(g=g, m=m, n=n, k=k, ours_nt_ms=t_nt, ours_nn_ms=t_nn, cublas_ms=t_cb,
               ours_nt_tflops=fl / t_nt / 1e9, ours_nn_tflops=fl / t_nn / 1e9,
               cublas_tflops=fl / t_cb / 1e9)
    print(json.dumps(rec)); sys.stdout.flush()
    out.append(rec)
  with open('gpurun_out/gemm_bench.json', 'w') as f:
    json.dump(out, f, indent=1)


if __name__ == '__main__':
  import os
  os.makedirs('gpurun_out', exist_ok=True)
  main()
