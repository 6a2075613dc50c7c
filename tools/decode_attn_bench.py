"""Decode-step attention on the GPU: our split-KV kernel against the PyTorch step.

Op level: `decode_attention` (kernel) and `decode_attention_ref` (the fp32 PyTorch step) for
B ∈ {1, 8, 64}, T ∈ {1024, 4096}, t ∈ {T/8, T−1}, H = 16, Hk ∈ {16, 1}. Each call is timed on
its own with CUDA events after an L2 flush (outside the timed window); the median is
reported as `*_call_us` (this includes the host-side cost of the call whenever that exceeds
the kernel's). `kernel_us` is the device time of the kernels alone, from `torch.profiler`,
and is what the bandwidth figures use. Achieved bandwidth counts the bytes the step needs: the
live K/V rows
2·2·B·(t+1)·Hk·128, q, the output and the fp32 split partials (written and read back).

End to end: greedy `gshard_decode.DecodeIds` on a dense LM of MoELm8E's attention shape
(M = 2048, 16×128 heads, 8 layers, FFN 8192, vocab 32000, random weights), B = 8, 512 new
tokens, with the kernel and with `decode_attention_supported` patched to False, alternated.

    python tools/decode_attn_bench.py --out DIR [--e2e-repeats 3] [--skip-e2e]

Writes DIR/decode_attn_bench.json and prints one JSON line per measurement.
"""

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # pylint: disable=g-import-not-at-top

from lingvo_b200 import ops  # pylint: disable=g-import-not-at-top
from lingvo_b200.ops import attention as attention_ops  # pylint: disable=g-import-not-at-top

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def _Card():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                      '--format=csv,noheader'], capture_output=True, text=True, check=False)
  return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip())


def _TimeCalls(fn, iters, warm=5):
  flush = torch.empty(128 << 20, dtype=torch.int8, device='cuda')   # > 50 MB L2
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
    ts.append(a.elapsed_time(b) * 1e3)
  ts.sort()
  return ts[len(ts) // 2]


def _KernelDeviceUs(fn, iters):
  """Mean device time per call of the `decode_attn_*` kernels (split + combine), from
  `torch.profiler`, each call after an L2 flush."""
  from torch.profiler import profile, ProfilerActivity   # pylint: disable=g-import-not-at-top
  flush = torch.empty(128 << 20, dtype=torch.int8, device='cuda')
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(iters):
      flush.zero_()
      fn()
    torch.cuda.synchronize()
  total = sum(e.device_time_total for e in prof.key_averages() if 'decode_attn' in e.key)
  assert total > 0, 'no decode_attn kernels in the trace'
  return total / iters


def _PeakBytes(fn):
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  fn()
  torch.cuda.synchronize()
  return torch.cuda.max_memory_allocated() - base


def _OpLevel(records):
  nat = ops.native()
  h = 16
  for b in (1, 8, 64):
    for tmax in (1024, 4096):
      for hk in (16, 1):
        g = torch.Generator(device='cuda').manual_seed(0)
        ck = torch.randn(b, tmax, hk, 128, generator=g, device='cuda').to(torch.bfloat16)
        cv = torch.randn(b, tmax, hk, 128, generator=g, device='cuda').to(torch.bfloat16)
        q = (torch.randn(b, 1, h, 128, generator=g, device='cuda') * 0.1).to(torch.bfloat16)
        kn = torch.randn(b, 1, hk, 128, generator=g, device='cuda').to(torch.bfloat16)
        vn = torch.randn(b, 1, hk, 128, generator=g, device='cuda').to(torch.bfloat16)
        rel = torch.randn(h, 2 * tmax - 1, generator=g, device='cuda')
        chunk = nat.decode_attn_chunk(b, h, hk, tmax)
        splits = (tmax + chunk - 1) // chunk
        for t in (tmax // 8, tmax - 1):
          tt = torch.tensor(t, device='cuda')
          kern = lambda: attention_ops.decode_attention(q, kn, vn, ck, cv, tt, rel)  # pylint: disable=cell-var-from-loop
          ref = lambda: attention_ops.decode_attention_ref(q, kn, vn, ck, cv, tt, rel)  # pylint: disable=cell-var-from-loop
          err = float((kern().float() - ref().float()).norm() / ref().float().norm())
          call_k = _TimeCalls(kern, 200)
          us_r = _TimeCalls(ref, 20)
          us_k = _KernelDeviceUs(kern, 100)
          live = (t + 1 + chunk - 1) // chunk if splits > 1 else 0
          nbytes = (2 * 2 * b * (t + 1) * hk * 128 + 2 * b * h * 128 * 2 +
                    2 * b * h * live * (128 + 2) * 4)
          rec = dict(kind='op', B=b, T=tmax, t=t, H=h, Hk=hk, chunk=chunk, splits=splits,
                     kernel_us=us_k, kernel_call_us=call_k, ref_call_us=us_r,
                     speedup_per_call=us_r / call_k,
                     kernel_bytes=nbytes, kernel_GBps=nbytes / us_k / 1e3,
                     kernel_share_of_3p35TBps=nbytes / (us_k * 1e-6) / HBM_BYTES_PER_S,
                     kernel_peak_bytes=_PeakBytes(kern), ref_peak_bytes=_PeakBytes(ref),
                     rel_err_vs_ref=err)
          print(json.dumps(rec))
          sys.stdout.flush()
          records.append(rec)
        del ck, cv
        torch.cuda.empty_cache()


def _Lm():
  from lingvo_b200.core import cluster_factory   # pylint: disable=g-import-not-at-top
  from lingvo_b200.core import gshard_builder as gb   # pylint: disable=g-import-not-at-top
  bp = gb.DenseBuilder.Params().Set(
      model_dim=2048, attention_num_heads=16, attention_key_value_dim=128, ff_dim=8192,
      relative_attention_type='bias', relative_attention_num_buckets=32,
      relative_attention_max_distance=128, relative_attention_use_universal_1d_position=True,
      dtype=torch.float32, fprop_dtype=torch.bfloat16, attention_logits_dtype=torch.float32,
      dropout_rate=0.0, attention_dropout_prob=0.0, label_smoothing=0.0)
  # decoder_eos_id = -1: no row stops early, so every run decodes all steps.
  p = gb.UniTransformer.Params().Set(
      name='lm', builder=bp, gated_gelu=True, vocab_size=32000, num_transformer_layers=8,
      max_length=1024, positional_embedding=False, label_smoothing=0.0, z_loss=0.0,
      dtype=torch.float32, fprop_dtype=torch.bfloat16, decoder_eos_id=-1)
  with cluster_factory.ForTestingWorker(mode='sync', job='trainer_client', do_eval=True):
    task = p.Instantiate()
  task.to(torch.device('cuda'))
  return task


def _EndToEnd(records, repeats):
  from lingvo_b200.core import gshard_decode   # pylint: disable=g-import-not-at-top
  from lingvo_b200.core.nested_map import NestedMap   # pylint: disable=g-import-not-at-top
  torch.manual_seed(0)
  task = _Lm()
  b, prefix, steps = 8, 16, 512
  ids = torch.randint(2, 32000, (b, prefix), device='cuda')
  batch = NestedMap(ids=ids, labels=ids, paddings=torch.zeros(b, prefix, device='cuda'))
  supported = attention_ops.decode_attention_supported

  def _Run(kernel):
    attention_ops.decode_attention_supported = supported if kernel else (lambda q, k: False)
    try:
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      out = gshard_decode.DecodeIds(task, task.theta, batch, max_steps=steps)
      torch.cuda.synchronize()
      return time.perf_counter() - t0, out.ids
    finally:
      attention_ops.decode_attention_supported = supported

  _Run(True)
  _Run(False)   # warm-up of both arms
  times = {True: [], False: []}
  ids_of = {}
  for _ in range(repeats):
    for arm in (True, False):
      sec, out_ids = _Run(arm)
      times[arm].append(sec)
      ids_of[arm] = out_ids
  gen = b * (prefix + steps - 1)   # DecodeStep calls × batch (prefix fed one token per step)
  new = slice(prefix, prefix + steps)
  agree = float((ids_of[True][:, new] == ids_of[False][:, new]).float().mean())
  rec = dict(kind='e2e', B=b, prefix=prefix, new_tokens=steps, layers=8, model_dim=2048,
             heads='16x128', kernel_s=times[True], ref_s=times[False],
             kernel_tokens_per_s=gen / min(times[True]), ref_tokens_per_s=gen / min(times[False]),
             speedup=min(times[False]) / min(times[True]), generated_id_agreement=agree)
  print(json.dumps(rec))
  records.append(rec)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', required=True, help='output directory')
  ap.add_argument('--e2e-repeats', type=int, default=3)
  ap.add_argument('--skip-e2e', action='store_true')
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'decode_attn_bench needs a GPU'
  ops.native(required=True)
  os.makedirs(args.out, exist_ok=True)
  records = [dict(kind='card', **_Card())]
  print(json.dumps(records[0]))
  _OpLevel(records)
  if not args.skip_e2e:
    _EndToEnd(records, args.e2e_repeats)
  with open(os.path.join(args.out, 'decode_attn_bench.json'), 'w') as f:
    json.dump(records, f, indent=1)


if __name__ == '__main__':
  main()
