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

With `--beam` it measures flat beam search instead:

  * op level: `flat_beam_attention` (kernel) against `flat_beam_attention_ref` for
    B ∈ {1, 8}, K ∈ {4, 8}, H = 16, Hk ∈ {16, 4, 1}, N ∈ {1024, 4096}, with slot0 = N − K and
    ancestor-shaped masks (a 64-token prompt, then a random parent per step). Bandwidth counts
    the live K/V rows 2·2·B·N·Hk·128, the masks and positions, q, the output and the partials.
  * prefill: `UniTransformer.Prefill` of a P = 512 prompt against feeding the same prompt
    through `DecodeStep` one token at a time, B = 8, on the end-to-end model below.
  * end to end: `BeamDecodeIds` with K = 4 against greedy `DecodeIds`, B = 8, a 16-token
    prompt and at most 256 new tokens, alternated. The model's EOS id is −1, which the beam
    reads as the last vocabulary entry, so it may stop early on its score gap; greedy runs all
    256 steps.

Writes DIR/decode_attn_bench.json (DIR/flat_beam_bench.json with `--beam`) and prints one
JSON line per measurement.
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


def _KernelDeviceUs(fn, iters, name='decode_attn'):
  """Mean device time per call of the kernels whose name contains `name` (split + combine),
  from `torch.profiler`, each call after an L2 flush."""
  from torch.profiler import profile, ProfilerActivity   # pylint: disable=g-import-not-at-top
  flush = torch.empty(128 << 20, dtype=torch.int8, device='cuda')
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(iters):
      flush.zero_()
      fn()
    torch.cuda.synchronize()
  total = sum(e.device_time_total for e in prof.key_averages() if name in e.key)
  assert total > 0, 'no %s kernels in the trace' % name
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


# ------------------------------------------------------------------- flat beam search ----
def _AncestorVis(b, kk, n, slot0, prompt=64, seed=0):
  g = torch.Generator().manual_seed(seed)
  mask = torch.zeros(b, kk, n, dtype=torch.bool)
  mask[:, :, :prompt] = True
  for s0 in range(prompt, slot0, kk):
    mask[:, torch.arange(kk), s0 + torch.arange(kk)] = True
    parent = torch.randint(0, kk, (b, kk), generator=g)
    mask = mask.gather(1, parent.unsqueeze(-1).expand(b, kk, n))
  mask[:, torch.arange(kk), slot0 + torch.arange(kk)] = True
  return attention_ops.pack_visibility(mask).cuda()


def _BeamOpLevel(records):
  nat = ops.native()
  h = 16
  for b in (1, 8):
    for n in (1024, 4096):
      for kk in (4, 8):
        vis = _AncestorVis(b, kk, n, n - kk)
        for hk in (16, 4, 1):
          g = torch.Generator(device='cuda').manual_seed(0)
          ck = torch.randn(b, n, hk, 128, generator=g, device='cuda').to(torch.bfloat16)
          cv = torch.randn(b, n, hk, 128, generator=g, device='cuda').to(torch.bfloat16)
          q = (torch.randn(b, kk, h, 128, generator=g, device='cuda') * 0.1).to(torch.bfloat16)
          kn = torch.randn(b, kk, hk, 128, generator=g, device='cuda').to(torch.bfloat16)
          vn = torch.randn(b, kk, hk, 128, generator=g, device='cuda').to(torch.bfloat16)
          rel = torch.randn(h, 2 * n - 1, generator=g, device='cuda')
          qpos = torch.full((b, kk), n - 1, dtype=torch.int32, device='cuda')
          kpos = torch.arange(n, dtype=torch.int32, device='cuda').repeat(b, 1)
          s0 = torch.tensor(n - kk, device='cuda')
          chunk = nat.flat_beam_attn_chunk(b, kk, h, hk, n)
          splits = (n + chunk - 1) // chunk
          args = (q, kn, vn, ck, cv, s0, vis, qpos, kpos, rel)
          kern = lambda: attention_ops.flat_beam_attention(*args)  # pylint: disable=cell-var-from-loop
          ref = lambda: attention_ops.flat_beam_attention_ref(*args)  # pylint: disable=cell-var-from-loop
          err = float((kern().float() - ref().float()).norm() / ref().float().norm())
          call_k = _TimeCalls(kern, 200)
          us_r = _TimeCalls(ref, 20)
          us_k = _KernelDeviceUs(kern, 100, 'flat_beam_attn')
          nbytes = (2 * 2 * b * n * hk * 128 + b * kk * ((n + 31) // 32) * 4 + b * n * 4 +
                    2 * b * kk * h * 128 * 2 +
                    (2 * b * kk * h * splits * (128 + 2) * 4 if splits > 1 else 0))
          rec = dict(kind='beam_op', B=b, K=kk, N=n, slot0=n - kk, H=h, Hk=hk, chunk=chunk,
                     splits=splits, kernel_us=us_k, kernel_call_us=call_k, ref_call_us=us_r,
                     speedup_per_call=us_r / call_k, kernel_bytes=nbytes,
                     kernel_GBps=nbytes / us_k / 1e3,
                     kernel_share_of_3p35TBps=nbytes / (us_k * 1e-6) / HBM_BYTES_PER_S,
                     kernel_peak_bytes=_PeakBytes(kern), ref_peak_bytes=_PeakBytes(ref),
                     rel_err_vs_ref=err)
          print(json.dumps(rec))
          sys.stdout.flush()
          records.append(rec)
          del ck, cv
          torch.cuda.empty_cache()


def _Timed(fn):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return time.perf_counter() - t0, out


def _BeamPrefill(records, task, repeats):
  b, plen = 8, 512
  ids = torch.randint(2, 32000, (b, plen), device='cuda')
  seg = torch.ones(b, plen, dtype=torch.long, device='cuda')
  pos = torch.arange(plen, device='cuda').repeat(b, 1)

  def Prefill():
    st = task.InitDecodeState(b, plen, ids.device)
    task.Prefill(task.theta, ids, seg, pos, st)
    return st

  def Teacher():
    st = task.InitDecodeState(b, plen, ids.device)
    for t in range(plen):
      task.DecodeStep(task.theta, ids[:, t], st, t)
    return st

  with torch.no_grad():
    a, c = Prefill(), Teacher()
    err = max(float((x.k.float() - y.k.float()).norm() / y.k.float().norm())
              for x, y in zip(a, c) if x is not None)
    times = {'prefill': [], 'decode_steps': []}
    for _ in range(repeats):
      times['prefill'].append(_Timed(Prefill)[0])
      times['decode_steps'].append(_Timed(Teacher)[0])
  rec = dict(kind='beam_prefill', B=b, P=plen, prefill_s=times['prefill'],
             decode_steps_s=times['decode_steps'],
             speedup=min(times['decode_steps']) / min(times['prefill']),
             cache_rel_err_vs_decode_steps=err)
  print(json.dumps(rec))
  records.append(rec)


def _BeamEndToEnd(records, task, repeats):
  from lingvo_b200.core import gshard_decode   # pylint: disable=g-import-not-at-top
  from lingvo_b200.core.nested_map import NestedMap   # pylint: disable=g-import-not-at-top
  b, prefix, steps, kk = 8, 16, 256, 4
  ids = torch.randint(2, 32000, (b, prefix), device='cuda')
  batch = NestedMap(ids=ids, labels=ids, paddings=torch.zeros(b, prefix, device='cuda'))
  run = {
      'beam': lambda: gshard_decode.BeamDecodeIds(task, task.theta, batch, beam_size=kk,
                                                  max_steps=steps),
      'greedy': lambda: gshard_decode.DecodeIds(task, task.theta, batch, max_steps=steps),
  }
  with torch.no_grad():
    for fn in run.values():
      fn()
    times = {k: [] for k in run}
    for _ in range(repeats):
      for k, fn in run.items():
        times[k].append(_Timed(fn)[0])
  rec = dict(kind='beam_e2e', B=b, K=kk, prefix=prefix, new_tokens=steps, layers=8,
             model_dim=2048, heads='16x128', beam_s=times['beam'], greedy_s=times['greedy'],
             beam_over_greedy=min(times['beam']) / min(times['greedy']),
             beam_hyp_tokens_per_s=b * kk * steps / min(times['beam']),
             greedy_tokens_per_s=b * steps / min(times['greedy']))
  print(json.dumps(rec))
  records.append(rec)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', required=True, help='output directory')
  ap.add_argument('--e2e-repeats', type=int, default=3)
  ap.add_argument('--skip-e2e', action='store_true')
  ap.add_argument('--beam', action='store_true', help='measure flat beam search')
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'decode_attn_bench needs a GPU'
  ops.native(required=True)
  os.makedirs(args.out, exist_ok=True)
  records = [dict(kind='card', **_Card())]
  print(json.dumps(records[0]))
  if args.beam:
    _BeamOpLevel(records)
    if not args.skip_e2e:
      torch.manual_seed(0)
      task = _Lm()
      _BeamPrefill(records, task, args.e2e_repeats)
      _BeamEndToEnd(records, task, args.e2e_repeats)
  else:
    _OpLevel(records)
    if not args.skip_e2e:
      _EndToEnd(records, args.e2e_repeats)
  name = 'flat_beam_bench.json' if args.beam else 'decode_attn_bench.json'
  with open(os.path.join(args.out, name), 'w') as f:
    json.dump(records, f, indent=1)


if __name__ == '__main__':
  main()
