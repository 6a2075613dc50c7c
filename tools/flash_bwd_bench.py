"""Times the flash attention backward (`flash_attn_bwd`, csrc/flash_attn.cu) at the shape of
the MoELm8E benchmark step and prints one JSON line.

Shape: B = 8 sequences x L = 1024 tokens, H = 16 query heads x D = 128, causal, with the
[H, 2L-1] relative-bias table and the packed-input metadata the benchmark's synthetic input
produces (one segment per row, positions 0..L-1). Hk = 16 (multi-head) is the benchmark's
case; Hk = 4 and Hk = 1 time the grouped-query path.

For every Hk:
  * `ms`: CUDA events around `--iters` back-to-back `flash_attn_bwd` calls after warm-up,
    divided by the count. This is the whole entry point: the delta, block-summary, dQ fold,
    dRel fold and dK/dV fold kernels and the allocator's fills are all inside it.
  * `fwd_ms`, `fwd_bwd_ms`: the same for `flash_attn_fwd` alone and for a forward followed by
    its backward.
  * `tflops`: the FLOPs of the visible (query block, key block) pairs, counted here from the
    mask (5 products of 2·128^3 per pair and head), over `ms`.
  * `peak_mb`: torch.cuda.max_memory_allocated during one call, above what was allocated
    before it (inputs and forward outputs).
  * `kernels`: with `--profile`, device time per call of each kernel and fill, from
    torch.profiler in a separate pass after the timed one.
The card's name, power limit and SM clock (sampled with nvidia-smi while the timed loop
runs) go in the same line.

`--cap C` soft-caps the logits at C and `--extra X` adds an extra logit X (the specialised
kernels of GShard's `atten_logit_cap` / `attention_extra_logit`); without them the calls pass
neither option, so a checkout that predates them can be timed too.

`--root DIR` imports lingvo_b200 from another checkout (built in place), so two versions can
be timed alternately in one job.
"""
import argparse
import json
import os
import subprocess
import sys


def _Args():
  ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  ap.add_argument('--root', default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
  ap.add_argument('--hk', default='16,4,1', help='comma-separated KV head counts')
  ap.add_argument('--iters', type=int, default=100)
  ap.add_argument('--warmup', type=int, default=10)
  ap.add_argument('--cap', type=float, default=0.0, help='logit_cap (0 = none)')
  ap.add_argument('--extra', type=float, default=None, help='extra_logit (default none)')
  ap.add_argument('--profile', action='store_true', help='add a torch.profiler kernel split')
  ap.add_argument('--out', default=None, help='also write the JSON line to this file')
  return ap.parse_args()


ARGS = _Args()
sys.path.insert(0, os.path.abspath(ARGS.root))

import torch  # noqa: E402

from lingvo_b200 import ops  # noqa: E402

B, L, H, D = 8, 1024, 16, 128
T = 128   # the kernels' block edge


def _Inputs(hk, seed=0):
  gen = torch.Generator().manual_seed(seed)
  randn = lambda *s: torch.randn(*s, generator=gen)
  # q / k / v are column slices of one fused projection, as in the model.
  qkv = (randn(B, L, (H + 2 * hk) * D) * 0.5).bfloat16().cuda()
  q, k, v = qkv.split([H * D, hk * D, hk * D], dim=-1)
  q = q.reshape(B, L, H, D)
  k = k.reshape(B, L, hk, D)
  v = v.reshape(B, L, hk, D)
  rel = randn(H, 2 * L - 1).cuda()
  seg = torch.ones(B, L, dtype=torch.int32, device='cuda')
  pos = torch.arange(L, dtype=torch.int32, device='cuda').expand(B, L).contiguous()
  d_o = (randn(B, L, H, D) * 0.5).bfloat16().cuda()
  return q, k, v, rel, seg, pos, d_o


def _Flops():
  """FLOPs of one backward: 5 products (S, dP, dV, dK, dQ) of 2·T^3 per visible block pair."""
  nblk = L // T
  pairs = sum(1 for i in range(nblk) for j in range(nblk) if j <= i)     # causal
  return pairs * 5 * 2 * T**3 * B * H


def _Smi(fields):
  try:
    r = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()),
                        '--query-gpu=' + fields, '--format=csv,noheader,nounits'],
                       capture_output=True, text=True, timeout=30)
    return [x.strip() for x in r.stdout.strip().split(',')]
  except (OSError, subprocess.SubprocessError):
    return None


def _Time(call, iters):
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  start.record()
  for _ in range(iters):
    call()
  stop.record()
  smi = subprocess.Popen(['nvidia-smi', '-i', str(torch.cuda.current_device()),
                          '--query-gpu=clocks.sm', '--format=csv,noheader,nounits'],
                         stdout=subprocess.PIPE, text=True)
  clock = smi.communicate(timeout=60)[0].strip()
  stop.synchronize()
  return start.elapsed_time(stop) / iters, clock


def _Profile(call, iters):
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(iters):
      call()
    torch.cuda.synchronize()
  out = {}
  for e in prof.key_averages():
    t = getattr(e, 'device_time_total', None)
    if t is None:
      t = e.cuda_time_total
    if t > 0:
      out[e.key[:80]] = round(t / iters / 1e3, 4)      # ms per call
  return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def main():
  assert torch.cuda.is_available(), 'flash_bwd_bench.py needs a GPU'
  nat = ops.native(required=True)
  info = _Smi('name,power.limit,clocks.max.sm') or ['?', '?', '?']
  res = dict(tool='flash_bwd_bench', root=os.path.abspath(ARGS.root), gpu=info[0],
             power_limit_w=info[1], max_sm_clock_mhz=info[2], B=B, L=L, H=H, D=D,
             causal=True, logit_cap=ARGS.cap, extra_logit=ARGS.extra, iters=ARGS.iters,
             gflop=round(_Flops() / 1e9, 2), cases={})
  fwd_opts, bwd_opts = {}, {}
  if ARGS.cap:
    fwd_opts['logit_cap'] = bwd_opts['logit_cap'] = ARGS.cap
  if ARGS.extra is not None:
    fwd_opts['extra_logit'] = ARGS.extra
  for hk in [int(x) for x in ARGS.hk.split(',')]:
    q, k, v, rel, seg, pos, d_o = _Inputs(hk)
    fwd = lambda: nat.flash_attn_fwd(q, k, v, rel, seg, pos, 1.0, True, **fwd_opts)
    out, lse = fwd()
    call = lambda: nat.flash_attn_bwd(q, k, v, out, d_o, lse, rel, seg, pos, 1.0, True, True,
                                      **bwd_opts)

    def fwd_bwd():
      o, l = fwd()
      return nat.flash_attn_bwd(q, k, v, o, d_o, l, rel, seg, pos, 1.0, True, True, **bwd_opts)
    for _ in range(ARGS.warmup):
      fwd()
      fwd_bwd()
    for _ in range(ARGS.warmup):
      call()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    grads = call()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del grads
    ms, clock = _Time(call, ARGS.iters)
    fwd_ms, _ = _Time(fwd, ARGS.iters)
    fwd_bwd_ms, _ = _Time(fwd_bwd, ARGS.iters)
    case = dict(hk=hk, splits=int(nat.flash_attn_bwd_splits(B, L, H, hk)), ms=round(ms, 4),
                fwd_ms=round(fwd_ms, 4), fwd_bwd_ms=round(fwd_bwd_ms, 4),
                tflops=round(_Flops() / (ms * 1e-3) / 1e12, 1),
                peak_mb=round(peak / 2**20, 1), sm_clock_mhz=clock)
    if ARGS.profile:
      case['kernels'] = _Profile(call, 10)
    res['cases'][str(hk)] = case
  line = json.dumps(res)
  print(line)
  if ARGS.out:
    os.makedirs(os.path.dirname(os.path.abspath(ARGS.out)), exist_ok=True)
    with open(ARGS.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
