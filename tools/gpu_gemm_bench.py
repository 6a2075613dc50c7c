"""Times the wgmma GEMM on every GEMM of one MoELm8E training step vs torch.matmul.

Each row is one GEMM site of the step (`G x M x N x K`, operand majors, fused epilogue),
timed with CUDA events, L2 flushed before each call. Prints one JSON line per row plus a
header with the card, its power limit and max SM clock, and, given a path, writes them all
there as one JSON list.

  python tools/gpu_gemm_bench.py [OUT.json]
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from lingvo_b200.ops import gemm as G  # noqa: E402

PEAK_TFLOPS = 989.0  # H100 SXM dense BF16 data-sheet figure

# (site, G, M, N, K, A K-major, B K-major, epilogue); epilogue in
# {None, 'residual', 'relu', 'relu_mask', 'row_ptrs', 'row_scale'}.
INVENTORY = [
    ('qkv_fwd', 1, 8192, 6144, 2048, True, False, None),
    ('qkv_dgrad', 1, 8192, 2048, 6144, True, True, None),
    ('qkv_wgrad', 1, 2048, 6144, 8192, False, False, None),
    ('attn_out_fwd', 1, 8192, 2048, 2048, True, False, 'residual'),
    ('attn_out_dgrad', 1, 8192, 2048, 2048, True, True, None),
    ('attn_out_wgrad', 1, 2048, 2048, 8192, False, False, None),
    ('ffn_wi_fwd', 1, 8192, 8192, 2048, True, False, 'relu'),
    ('ffn_wo_fwd', 1, 8192, 2048, 8192, True, False, 'residual'),
    ('ffn_dh', 1, 8192, 8192, 2048, True, True, 'relu_mask'),
    ('ffn_dx', 1, 8192, 2048, 8192, True, True, None),
    ('ffn_dwo', 1, 8192, 2048, 8192, False, False, None),
    ('ffn_dwi', 1, 2048, 8192, 8192, False, False, None),
    ('moe_wi_fwd', 8, 2048, 8192, 2048, True, False, 'relu'),
    ('moe_wo_fwd', 8, 2048, 2048, 8192, True, False, 'row_ptrs'),
    ('moe_dh', 8, 2048, 8192, 2048, True, True, 'relu_mask'),
    ('moe_dx', 8, 2048, 2048, 8192, True, True, 'row_ptrs'),
    ('moe_dwo', 8, 8192, 2048, 2048, False, False, 'row_scale'),
    ('moe_dwi', 8, 2048, 8192, 2048, False, False, 'row_scale'),
    ('lm_logits', 1, 8192, 32000, 2048, True, True, None),
    ('lm_dx', 1, 8192, 2048, 32000, True, False, None),
    ('lm_dw', 1, 32000, 2048, 8192, False, False, None),
]


def _time(fn, flush, iters=10, warm=3):
  for _ in range(warm):
    fn()
  ts = []
  for _ in range(iters):
    flush.zero_()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    ts.append(a.elapsed_time(b))
  ts.sort()
  return ts[len(ts) // 2]


def _card():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                      '--format=csv,noheader'], capture_output=True, text=True)
  return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def main():
  out_path = sys.argv[1] if len(sys.argv) > 1 else None
  assert torch.cuda.is_available(), 'gpu_gemm_bench needs a GPU'
  flush = torch.empty(256 << 20, dtype=torch.int8, device='cuda')
  head = dict(card=_card(), torch_device=torch.cuda.get_device_name(0))
  print(json.dumps(head), flush=True)
  out = [head]
  gen = torch.Generator(device='cuda').manual_seed(0)
  for site, g, m, n, k, ak, bk, epi in INVENTORY:
    def rnd(*shape):
      return torch.randn(*shape, device='cuda', generator=gen).to(torch.bfloat16)
    a = rnd(g, m, k) if ak else rnd(g, k, m)
    b = rnd(g, n, k) if bk else rnd(g, k, n)
    kw = {}
    if epi == 'residual':
      kw = dict(aux=rnd(g, m, n), aux_mode=G.AUX_ADD)
    elif epi == 'relu':
      kw = dict(act=1)
    elif epi == 'relu_mask':
      kw = dict(aux=rnd(g, m, n), aux_mode=G.AUX_RELU_MASK)
    elif epi == 'row_ptrs':
      scratch = torch.empty(g * m, n, device='cuda', dtype=torch.bfloat16)
      perm = torch.randperm(g * m, device='cuda', generator=gen)
      kw = dict(row_ptrs=(scratch.data_ptr() + perm * (n * 2)).to(torch.int64))
    elif epi == 'row_scale':
      kw = dict(row_scale=torch.rand(g, m, device='cuda', generator=gen))
    A = a if ak else a.transpose(1, 2)
    B = b.transpose(1, 2) if bk else b
    fl = 2.0 * g * m * n * k
    t = _time(lambda: G.gemm(a, b, ak, bk, **kw), flush)
    t_ref = _time(lambda: torch.matmul(A, B), flush)
    rec = dict(site=site, g=g, m=m, n=n, k=k, a='K' if ak else 'MN', b='K' if bk else 'MN',
               epilogue=epi, ms=round(t, 4), tflops=round(fl / t / 1e9, 1),
               peak_share=round(fl / t / 1e9 / PEAK_TFLOPS, 3), matmul_ms=round(t_ref, 4),
               vs_matmul=round(t_ref / t, 3))
    print(json.dumps(rec), flush=True)
    out.append(rec)
    del a, b, A, B, kw
  tot = sum(r['ms'] for r in out[1:])
  print(json.dumps(dict(total_ms=round(tot, 3))), flush=True)
  if out_path:
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, 'w') as f:
      json.dump(out, f, indent=1)


if __name__ == '__main__':
  main()
