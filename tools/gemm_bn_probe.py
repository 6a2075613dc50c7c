"""Tile-N A/B of the wgmma GEMM on the flagship model's shapes (run on a GPU box; each
setting needs its own process because the override is read once):

  for bn in 256 128; do LINGVO_B200_GEMM_BN=$bn python tools/gemm_bn_probe.py; done
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lingvo_b200.ops import gemm as G


def Bench(fn, iters=20, warm=5):
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
  bn = os.environ.get('LINGVO_B200_GEMM_BN', 'auto')
  # (name, M, N, K, a_kmajor, b_kmajor): fwd x·W (B is [K,N]), dgrad dy·Wᵀ, wgrad xᵀ·dy
  shapes = [('attn_out fwd', 8192, 2048, 2048, True, False), ('qkv dgrad', 8192, 2048, 6144, True, True),
            ('ffn out fwd', 8192, 2048, 8192, True, False), ('ffn dgrad', 8192, 2048, 8192, True, True),
            ('qkv fwd', 8192, 6144, 2048, True, False), ('ffn in fwd', 8192, 8192, 2048, True, False),
            ('attn wgrad', 2048, 2048, 8192, False, False), ('ffn wgrad', 2048, 8192, 8192, False, False)]
  out = {}
  for name, m, n, k, ak, bk in shapes:
    a = torch.randn((m, k) if ak else (k, m), device='cuda').bfloat16()
    b = torch.randn((n, k) if bk else (k, n), device='cuda').bfloat16()
    ms = Bench(lambda: G.gemm(a, b, ak, bk))
    out[name] = {'ms': round(ms, 4), 'tflops': round(2.0 * m * n * k / ms / 1e9, 1)}
  print(json.dumps({'bn': bn, 'shapes': out}))


if __name__ == '__main__':
  main()
