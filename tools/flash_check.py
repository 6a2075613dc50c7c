"""GPU check + timing of the wgmma flash attention (csrc/flash_attn.cu).

Numerics against the fp32 oracle for forward, dQ/dK/dV and the bias-table gradient
(several geometries: packed segments, padding, causal / bidirectional, with / without the
relative bias), then timing at the benchmark shape against the cuDNN + rel_bias_grad path
it replaces. Writes gpurun_out/flash_check.json; prints FLASH_OK.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from lingvo_b200.ops import attention as A


def Rel(t, ref):
  return float((t.float() - ref.float()).norm() / (ref.float().norm() + 1e-20))


def RowRel(t, ref):
  """Worst per-row error (rows = all but the last dim), each row normalised by its own norm
  or, for rows with a smaller-than-typical norm, by the median row norm: catches row-local
  mistakes that a whole-tensor norm hides, without dividing bf16 cancellation noise by ~0
  (e.g. dq of the first causal row is exactly 0 in fp32)."""
  t, ref = t.float().reshape(-1, t.shape[-1]), ref.float().reshape(-1, ref.shape[-1])
  num = (t - ref).norm(dim=-1)
  rn = ref.norm(dim=-1)
  den = torch.maximum(rn, rn.median())
  return float((num / den).max())


def Case(b, l, h, use_rel, segs, causal, seed, scale=1.0):
  torch.manual_seed(seed)
  dev = 'cuda'
  d = 128
  qkv = (torch.randn(b, l, 3 * h * d, device=dev) * 0.5).bfloat16()
  q, k, v = [t.reshape(b, l, h, d).detach().requires_grad_(True)
             for t in qkv.split(h * d, dim=-1)]
  rel = (torch.randn(h, 2 * l - 1, device=dev)).requires_grad_(True) if use_rel else None
  seg = pos = None
  if segs:
    # packed rows: `segs` segments + trailing padding in odd rows
    seg = torch.zeros(b, l, dtype=torch.int32, device=dev)
    pos = torch.zeros(b, l, dtype=torch.int32, device=dev)
    for bi in range(b):
      n_valid = l - (37 if bi % 2 else 0)
      cuts = sorted(torch.randperm(n_valid - 1)[:segs - 1].add(1).tolist()) + [n_valid]
      start = 0
      for si, end in enumerate(cuts):
        seg[bi, start:end] = si + 1
        pos[bi, start:end] = torch.arange(end - start, device=dev, dtype=torch.int32)
        start = end
  d_o = (torch.randn(b, l, h, d, device=dev) * 0.5).bfloat16()
  if seg is not None:
    d_o = d_o * (seg != 0)[:, :, None, None].to(d_o.dtype)     # padded rows carry no gradient
  out = A.flash_attention(q, k, v, rel, seg, pos, scale, causal)
  grads = torch.autograd.grad(out, [q, k, v] + ([rel] if use_rel else []), d_o)
  ref = A.flash_attention_ref(q, k, v, rel, seg, pos, scale, causal)
  rgrads = torch.autograd.grad(ref, [q, k, v] + ([rel] if use_rel else []), d_o.float())
  valid = (seg != 0) if seg is not None else torch.ones(b, l, dtype=torch.bool, device=dev)
  o_sel, r_sel = out[valid], ref[valid]
  res = {'cfg': dict(b=b, l=l, h=h, rel=use_rel, segs=segs, causal=causal, scale=scale),
         'out': Rel(o_sel, r_sel), 'out_row': RowRel(o_sel, r_sel)}
  for name, g, rg in zip(['dq', 'dk', 'dv', 'drel'], grads, rgrads):
    res[name] = Rel(g, rg)
    if name != 'drel':
      res[name + '_row'] = RowRel(g[valid], rg[valid])
  return res


def Time(fn, iters=20):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  tot = 0.0
  for _ in range(iters):
    flush.zero_()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    tot += e0.elapsed_time(e1)
  return tot / iters * 1e3


def Bench():
  b, l, h, d = 8, 1024, 16, 128
  dev = 'cuda'
  torch.manual_seed(0)
  qkv = (torch.randn(b, l, 3 * h * d, device=dev) * 0.5).bfloat16()
  q, k, v = [t.reshape(b, l, h, d).detach().requires_grad_(True)
             for t in qkv.split(h * d, dim=-1)]
  rel = torch.randn(h, 2 * l - 1, device=dev).requires_grad_(True)
  seg = torch.ones(b, l, dtype=torch.int32, device=dev)
  pos = torch.arange(l, dtype=torch.int32, device=dev).unsqueeze(0).expand(b, l).contiguous()
  d_o = (torch.randn(b, l, h, d, device=dev) * 0.5).bfloat16()
  out = {}

  def flash_fwd():
    return A.flash_attention(q, k, v, rel, seg, pos, 1.0, True)
  o = flash_fwd()
  out['flash_fwd_us'] = Time(lambda: flash_fwd())
  out['flash_bwd_us'] = Time(lambda: torch.autograd.grad(o, [q, k, v, rel], d_o, retain_graph=True))
  # the path it replaces: build_rel_bias + cuDNN fwd/bwd + rel_bias_grad
  a, c = seg.unsqueeze(-1), seg.unsqueeze(-2)
  mask = (((a != c) | (pos.unsqueeze(-1) < pos.unsqueeze(-2))).float() * -1e9)
  os.environ['LINGVO_B200_ATTN'] = 'cudnn'
  try:
    def cudnn_fwd():
      return A.rel_bias_attention(q, k, v, rel, mask, 1.0, causal=True)
    o2 = cudnn_fwd()
    out['cudnn_path_fwd_us'] = Time(lambda: cudnn_fwd())
    out['cudnn_path_bwd_us'] = Time(
        lambda: torch.autograd.grad(o2, [q, k, v, rel], d_o, retain_graph=True))
    out['fwd_vs_cudnn_path_rel'] = Rel(o, o2)
  finally:
    os.environ['LINGVO_B200_ATTN'] = 'flash'
  flops_fwd = 4.0 * b * h * l * l * d / 2        # causal
  out['flash_fwd_tflops'] = flops_fwd / out['flash_fwd_us'] / 1e6
  out['flash_bwd_tflops'] = 2.5 * flops_fwd / out['flash_bwd_us'] / 1e6
  return out


def main():
  assert torch.cuda.is_available()
  results = []
  cases = [
      (1, 128, 1, False, 0, False, 1),
      (1, 128, 1, False, 0, True, 2),
      (2, 256, 2, True, 0, True, 3),
      (2, 256, 2, True, 0, False, 4),
      (2, 384, 2, True, 3, True, 5),
      (2, 512, 4, True, 2, False, 6),
      (2, 512, 4, False, 4, True, 7),
      (1, 1024, 2, True, 0, True, 8),
  ]
  ok = True
  for c in cases:
    r = Case(*c)
    results.append(r)
    bad = [k for k, v in r.items() if k != 'cfg' and not (v < (0.05 if k.endswith('_row') else 0.02))]
    print(json.dumps(r), 'BAD: %s' % bad if bad else '')
    ok = ok and not bad
  r = Case(2, 256, 2, True, 0, True, 9, scale=0.25)
  results.append(r)
  print(json.dumps(r))
  bench = Bench() if ok or os.environ.get('FLASH_BENCH_ANYWAY') else None
  print(json.dumps(bench))
  os.makedirs('gpurun_out', exist_ok=True)
  json.dump({'cases': results, 'bench': bench, 'ok': ok},
            open('gpurun_out/flash_check.json', 'w'), indent=1)
  if ok:
    print('FLASH_OK')


if __name__ == '__main__':
  main()
