"""Times the fused GLU + depthwise conv1d kernels (ops/csrc/conv_kernels.cu) with CUDA events
at the Librispeech Conformer's shape, and prints one JSON line.

  python tools/conv_bwd_bench.py [--root TREE] [--b 48 --t 428 --d 512 --k 32] [--causal]

`--root` imports `lingvo_b200` from another checkout with a built extension, so two versions
of the kernel can be compared by alternating runs of this script. The line records the
card's name, power limit and max SM clock next to the times.
"""
import argparse
import json
import os
import subprocess
import sys


def _Card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = ''
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--root', default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
  ap.add_argument('--b', type=int, default=48)
  ap.add_argument('--t', type=int, default=428)
  ap.add_argument('--d', type=int, default=512)
  ap.add_argument('--k', type=int, default=32)
  ap.add_argument('--causal', action='store_true')
  ap.add_argument('--dtype', default='bf16', choices=['bf16', 'fp32'])
  ap.add_argument('--iters', type=int, default=200)
  ap.add_argument('--warmup', type=int, default=20)
  args = ap.parse_args()
  sys.path.insert(0, os.path.abspath(args.root))
  import torch  # pylint: disable=g-import-not-at-top
  from lingvo_b200 import ops  # pylint: disable=g-import-not-at-top
  assert torch.cuda.is_available(), 'conv_bwd_bench needs a GPU'
  nat = ops.native(required=True)
  dtype = torch.bfloat16 if args.dtype == 'bf16' else torch.float32
  g = torch.Generator(device='cuda').manual_seed(0)
  b, t, d, k = args.b, args.t, args.d, args.k
  proj = torch.randn(b, t, 2 * d, device='cuda', generator=g).to(dtype)
  w = torch.randn(k, d, device='cuda', generator=g) / k**0.5
  dy = torch.randn(b, t, d, device='cuda', generator=g).to(dtype)
  lens = torch.randint(t // 2, t + 1, (b,), device='cuda', generator=g)
  pad = (torch.arange(t, device='cuda')[None, :] >= lens[:, None]).float()
  left = k - 1 if args.causal else (k - 1) // 2

  def timed(fn):
    for _ in range(args.warmup):
      fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(args.iters):
      fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) * 1e3 / args.iters

  fwd_us = timed(lambda: nat.glu_dwconv1d_fwd(proj, w, pad, left))
  bwd_us = timed(lambda: nat.glu_dwconv1d_bwd(proj, w, pad, dy, left))
  print(json.dumps({
      'root': os.path.abspath(args.root), 'card': _Card(),
      'shape': dict(b=b, t=t, d=d, k=k, causal=args.causal, dtype=args.dtype),
      'fwd_us': round(fwd_us, 2), 'bwd_us': round(bwd_us, 2)}))


if __name__ == '__main__':
  main()
