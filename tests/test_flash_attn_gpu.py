"""The wgmma flash attention (ops/csrc/flash_attn.cu) against a float64 oracle written from
the formula, element by element, at the benchmark's shape and at the edges of its tiling.

Contract checked here, for `flash_attention(q, k, v, rel, seg, pos, scale, causal)`:
  * query i sees key j iff seg[i] == seg[j] != 0 and, if causal, pos[j] <= pos[i];
  * for every query that sees at least one key, O and lse (natural log) are those of
    softmax_j(scale·q_i·k_j + rel[h, i-j+L-1]) over the keys it sees;
  * a query that sees no key contributes nothing to the backward: its dO is zero (as the
    model produces it), its dQ is exactly zero, and it adds nothing to dK, dV or d rel. Its
    forward value is unspecified but finite;
  * a key that no query sees has exactly zero dK and dV, and a diagonal of the bias table
    that no visible pair uses has exactly zero d rel.

Every bound has the form |got - want| <= c·2^-8·A + 1 bf16 ulp of want, where A is the
same contraction as the output's, in float64 over absolute values, and c is derived from
where the kernels round (see `_C_*` below).
"""
import math

import pytest
import torch

from lingvo_b200 import ops
from lingvo_b200.core.gshard_builder import RelativePositionBucket, _BucketGather
from lingvo_b200.ops import attention as A

_D = 128
_BENCH = dict(b=8, l=1024, h=16)   # MoELm8E: 8 sequences x 1024 tokens, 16 heads x 128
_BUCKETS, _MAX_DISTANCE = 32, 128

# The forward rounds the unnormalised P to bf16 before P·V (relative 2^-9 of each term of
# P·|V|) and O to bf16 once (the ulp term); l is summed from the unrounded values. c = 2
# leaves a factor 2 for fp32 accumulation and ex2.approx.
_C_O = 2.0
# dV = bf16(P)^T·dO: the same single 2^-9 rounding of every term of P^T·|dO|.
_C_DV = 2.0
# dK, dQ use bf16(scale·dS) (2^-9 of P·(|dP| + |delta|)) where dS carries delta taken from
# the bf16 O (its rounding and the forward's, within 2^-8·Σ_d|dO||O| per row); dQ is folded
# in fp32 over key blocks and rounded once. c = 4 covers the two roundings with a factor 2.
_C_DQK = 4.0
# d rel sums the unrounded fp32 dS, so the only bf16 rounding that reaches it is that of O
# inside delta (c = 4, as for dK/dQ); the fp32 sums of up to a few hundred partials per
# diagonal are covered by a floor of 2^-14 of the sum of the |terms|.
_C_DREL = 4.0
_DREL_FLOOR = 2.0**-14
# lse = (m + lg2(l))·ln 2 with ex2.approx / lg2.approx (2^-22 relative) and fp32 logits
# accumulated over D = 128 products: within 2^-16·(1 + max_j |scale·q_i|·|k_j| + |rel|).
_LSE_REL = 2.0**-16


# ------------------------------------------------------------------ the oracle ----
def _Visible(seg, pos, causal, b, l, dev):
  """[B, L, L] bool: query i sees key j."""
  if seg is None:
    seg = torch.ones(b, l, dtype=torch.int32, device=dev)
  if pos is None:
    pos = torch.arange(l, dtype=torch.int32, device=dev).expand(b, l)
  vis = (seg[:, :, None] == seg[:, None, :]) & (seg[:, :, None] != 0)
  if causal:
    vis = vis & (pos[:, None, :] <= pos[:, :, None])
  return vis


def _Toeplitz(rel, l):
  """rel [H, 2L-1] → [H, L, L] with [h, i, j] = rel[h, i - j + L - 1]."""
  i = torch.arange(l, device=rel.device)
  return rel[:, i[:, None] - i[None, :] + l - 1]


def _DiagSum(x):
  """x [..., L, L] → [..., 2L-1]: out[..., t] = Σ_{i - j + L - 1 = t} x[..., i, j]."""
  l = x.shape[-1]
  y = torch.nn.functional.pad(x.flip(-1), (0, l))              # [.., i, L-1-j] at col i+(L-1-j)
  y = y.reshape(*x.shape[:-2], 2 * l * l)[..., :l * (2 * l - 1)]
  return y.reshape(*x.shape[:-2], l, 2 * l - 1).sum(-2)


def _Forward64(qb, kb, vb, relt, vis, scale):
  """One batch element in float64: qb, kb, vb [H, L, D], relt [H, L, L] or None, vis [L, L].
  Returns (P [H, L, L], O [H, L, D], lse [H, L], S [H, L, L]); rows that see no key have
  P = 0, O = 0 and lse = NaN. Differentiable (used by the self-test's autograd)."""
  s = scale * qb @ kb.transpose(-1, -2)
  if relt is not None:
    s = s + relt
  live = vis.any(-1)
  sm = torch.where(vis, s, -math.inf)
  m = torch.where(live, sm.amax(-1), 0.0).detach()
  e = torch.exp(sm - m[..., None])
  l = e.sum(-1)
  p = e / torch.where(live, l, 1.0)[..., None]
  lse = torch.where(live, m + torch.log(torch.where(live, l, 1.0)), math.nan)
  return p, p @ vb, lse, s


def _Oracle(q, k, v, rel, seg, pos, scale, causal, d_o):
  """Float64 forward and closed-form backward from the kernels' bf16 inputs, one batch element
  at a time, plus the |.| contractions the bounds are made of."""
  b, l, h, d = q.shape
  dev = q.device
  f = lambda t: t.double().permute(1, 0, 2)                     # [L, H, D] → [H, L, D]
  relt = _Toeplitz(rel.double(), l) if rel is not None else None
  vis_all = _Visible(seg, pos, causal, b, l, dev)
  r = {n: torch.zeros(b, l, h, d, dtype=torch.float64, device=dev)
       for n in ('out', 'a_out', 'dq', 'a_dq', 'dk', 'a_dk', 'dv', 'a_dv')}
  r['lse'] = torch.zeros(b, h, l, dtype=torch.float64, device=dev)
  r['a_lse'] = torch.zeros(b, h, l, dtype=torch.float64, device=dev)
  for n in ('drel', 'drel_delta', 'drel_abs'):
    r[n] = torch.zeros(h, 2 * l - 1, dtype=torch.float64, device=dev)
  r['live'] = vis_all.any(-1)                                    # [B, L] query sees a key
  r['seen'] = vis_all.any(-2)                                    # [B, L] key seen by a query
  r['used'] = _DiagSum(vis_all.double()).sum(0) > 0              # [2L-1] diagonal in use
  for bi in range(b):
    qb, kb, vb, dob = f(q[bi]), f(k[bi]), f(v[bi]), f(d_o[bi])
    vis = vis_all[bi]
    p, o, lse, _ = _Forward64(qb, kb, vb, relt, vis, scale)
    a_s = scale * qb.abs() @ kb.abs().transpose(-1, -2)
    if relt is not None:
      a_s = a_s + relt.abs()
    r['a_lse'][bi] = torch.where(vis, a_s, 0.0).amax(-1)
    del a_s
    r['out'][bi] = o.permute(1, 0, 2)
    r['lse'][bi] = lse
    r['a_out'][bi] = (p @ vb.abs()).permute(1, 0, 2)
    r['dv'][bi] = (p.transpose(-1, -2) @ dob).permute(1, 0, 2)
    r['a_dv'][bi] = (p.transpose(-1, -2) @ dob.abs()).permute(1, 0, 2)
    dp = dob @ vb.transpose(-1, -2)
    delta = (dob * o).sum(-1)
    odo = (dob.abs() * o.abs()).sum(-1)
    ds = p * (dp - delta[..., None])
    a_ds = p * (dp.abs() + delta.abs()[..., None] + odo[..., None])
    del dp
    r['dq'][bi] = (scale * ds @ kb).permute(1, 0, 2)
    r['dk'][bi] = (scale * ds.transpose(-1, -2) @ qb).permute(1, 0, 2)
    r['a_dq'][bi] = (scale * a_ds @ kb.abs()).permute(1, 0, 2)
    r['a_dk'][bi] = (scale * a_ds.transpose(-1, -2) @ qb.abs()).permute(1, 0, 2)
    r['drel'] += _DiagSum(ds)
    r['drel_abs'] += _DiagSum(a_ds)
    r['drel_delta'] += _DiagSum(p * odo[..., None])
    del p, ds, a_ds
  return r


# ------------------------------------------------------------------ the bounds ----
def _Bf16Ulp(x):
  """One bf16 ulp of float64 x (0 where x == 0)."""
  e = torch.frexp(x).exponent
  return torch.where(x != 0, torch.ldexp(torch.ones_like(x), e - 8), 0.0)


def _CheckBound(case, name, got, want, bound, where=None):
  """|got - want| <= bound elementwise (over `where`); prints the largest ratio."""
  err = (got.double() - want).abs()
  ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300),
                      torch.where(err > 0, math.inf, 0.0))
  if where is not None:
    ratio = torch.where(where, ratio, 0.0)
  worst = ratio.max().item()
  print('%s %-5s max |got - want| / bound = %.3f' % (case, name, worst))
  if not worst <= 1.0:
    idx = tuple(int(i) for i in (ratio == ratio.max()).nonzero()[0])
    raise AssertionError(
        '%s %s: %d elements out of bounds; worst at %s: got %r, want %r, bound %r' % (
            case, name, int((ratio > 1).sum()), idx, got[idx].item(), want[idx].item(),
            bound[idx].item()))


def _Bits(t):
  return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


# ------------------------------------------------------------------- the cases ----
def _Packed(b, l):
  """seg / pos [b, l] for the packed case: segments crossing 128-row blocks, one ending at a
  multiple of 128, a 1-token segment, trailing padding that makes the last block pure
  padding, and (row 1) a fully padded sequence."""
  layouts = [
      [(0, 100), (100, 256), (256, 257), (257, 700), (700, 880)],   # padding from 880
      [],                                                           # fully padded
      [(0, 384), (384, 385), (385, 1000)],                          # padding from 1000
  ]
  seg = torch.zeros(b, l, dtype=torch.int32)
  pos = torch.zeros(b, l, dtype=torch.int32)
  for bi in range(b):
    for si, (s, e) in enumerate(layouts[bi % len(layouts)]):
      seg[bi, s:e] = si + 1
      pos[bi, s:e] = torch.arange(e - s, dtype=torch.int32)
  return seg, pos


def _BucketTable(h, l, bidirectional, gen):
  """The relative-bias table as the model builds it (`SelfAttentionLayer._RelTable`):
  returns (wrb [H, 32] leaf, bucket [2L-1], rel [H, 2L-1] through `_BucketGather`)."""
  wrb = torch.randn(h, _BUCKETS, generator=gen).cuda().requires_grad_(True)
  bucket = RelativePositionBucket(torch.arange(l - 1, -l, -1, device='cuda'), _BUCKETS,
                                  _MAX_DISTANCE, bidirectional=bidirectional).long()
  return wrb, bucket, _BucketGather.apply(wrb.float(), bucket)


def _Inputs(case, seed):
  """(q, k, v, rel, seg, pos, scale, causal, d_o, extra) for one named case."""
  gen = torch.Generator().manual_seed(seed)
  randn = lambda *s: torch.randn(*s, generator=gen)
  kind = case.split('-')[0]
  extra = {}
  seg = pos = None
  scale = 1.0
  if kind == 'bench':
    b, l, h = _BENCH['b'], _BENCH['l'], _BENCH['h']
    causal = case == 'bench-causal'
    # q/k/v are column slices of the fused QKV projection, row stride 3·H·D.
    qkv = (randn(b, l, 3 * h * _D) * 0.5).bfloat16().cuda()
    q, k, v = [t.reshape(b, l, h, _D) for t in qkv.split(h * _D, dim=-1)]
    seg = torch.ones(b, l, dtype=torch.int32)
    pos = torch.arange(l, dtype=torch.int32).expand(b, l).contiguous()
    wrb, bucket, rel = _BucketTable(h, l, not causal, gen)
    extra.update(wrb=wrb, bucket=bucket)
  else:
    if kind == 'packed':
      b, l, h = 3, 1024, 4
      causal = case.endswith('-causal')
      seg, pos = _Packed(b, l)
    elif kind == 'peaky':
      b, l, h = 2, 512, 4
      causal = case.endswith('-causal')
      scale = _D**-0.5
    else:                                                        # launches-<L>
      l = int(case.split('-')[1])
      b, h = {128: (2, 2), 1152: (1, 2), 2048: (1, 2)}[l]
      causal = l != 1152
      if l == 128:
        seg = torch.ones(b, l, dtype=torch.int32)
        pos = torch.arange(l, dtype=torch.int32).expand(b, l).contiguous()
    std = 2.0 if kind == 'peaky' else 0.5
    q, k, v = [(randn(b, l, h, _D) * std).bfloat16().cuda() for _ in range(3)]
    if kind == 'peaky':
      # Plant k_j = q_i / 2 in the last key block query i sees, so that the running maximum
      # of row i moves in its last block (scale·q_i·k_j ≈ 22 against a spread of ~4).
      for i in (5, 130, 300, 380, 511):
        j = (i // 128) * 128 + (i % 128) // 2 if causal else l - 1 - (i % 128) // 2
        k[:, j] = (q[:, i].float() * 0.5).bfloat16()
    rel = randn(h, 2 * l - 1).cuda().requires_grad_(True)
  if seg is not None:
    seg, pos = seg.cuda(), pos.cuda()
  d_o = (randn(b, l, h, _D) * 0.5).bfloat16().cuda()
  live = _Visible(seg, pos, causal, b, l, 'cuda').any(-1)
  d_o = d_o * live[:, :, None, None].to(d_o.dtype)              # zero where a query sees nothing
  return q, k, v, rel, seg, pos, scale, causal, d_o, extra


_CASES = ['bench-causal', 'bench-bidi', 'packed-causal', 'packed-bidi', 'peaky-causal',
          'peaky-bidi', 'launches-128', 'launches-1152', 'launches-2048']


@pytest.mark.gpu
@pytest.mark.parametrize('case', _CASES)
def test_flash_attention_matches_float64(case):
  """O, lse, dQ, dK, dV, d rel (and d wrb through the bucket gather) within the per-element
  bounds of the float64 oracle, plus the exact zeros of the contract above."""
  q, k, v, rel, seg, pos, scale, causal, d_o, extra = _Inputs(case, _CASES.index(case))
  b, l, h, _ = q.shape
  q, k, v = [t.detach().requires_grad_(True) for t in (q, k, v)]
  assert A.flash_attention_supported(q, k)
  out = A.flash_attention(q, k, v, rel, seg, pos, scale, causal)
  leaf = extra['wrb'] if 'wrb' in extra else rel
  dq, dk, dv, dleaf = torch.autograd.grad(out, [q, k, v, leaf], d_o)
  relv = rel.detach()
  # lse and d rel straight from the kernels (the autograd path does not return them).
  nat = ops.native()
  out2, lse = nat.flash_attn_fwd(q.detach(), k.detach(), v.detach(), relv, seg, pos, scale,
                                 causal)
  drel = nat.flash_attn_bwd(q.detach(), k.detach(), v.detach(), out2, d_o, lse, relv, seg, pos,
                            scale, causal, True)[3]
  assert torch.equal(_Bits(out2), _Bits(out))
  if 'wrb' not in extra:
    assert torch.equal(_Bits(drel), _Bits(dleaf))

  with torch.no_grad():
    r = _Oracle(q.detach(), k.detach(), v.detach(), relv, seg, pos, scale, causal, d_o)
  live, seen = r['live'], r['seen']
  for name, t in [('out', out), ('lse', lse), ('dq', dq), ('dk', dk), ('dv', dv),
                  ('drel', drel)]:
    assert bool(torch.isfinite(t).all()), '%s has non-finite values' % name

  u = 2.0**-8
  rows = live[:, :, None, None].expand_as(out)
  _CheckBound(case, 'out', out, r['out'], _C_O * u * r['a_out'] + _Bf16Ulp(r['out']), rows)
  live_bhl = live[:, None, :].expand(b, h, l)
  _CheckBound(case, 'lse', lse, r['lse'], _LSE_REL * (1 + r['a_lse']), live_bhl)
  _CheckBound(case, 'dv', dv, r['dv'], _C_DV * u * r['a_dv'] + _Bf16Ulp(r['dv']))
  _CheckBound(case, 'dk', dk, r['dk'], _C_DQK * u * r['a_dk'] + _Bf16Ulp(r['dk']))
  _CheckBound(case, 'dq', dq, r['dq'], _C_DQK * u * r['a_dq'] + _Bf16Ulp(r['dq']))
  drel_bound = _C_DREL * u * r['drel_delta'] + _DREL_FLOOR * r['drel_abs']
  _CheckBound(case, 'drel', drel, r['drel'], drel_bound)
  if 'wrb' in extra:
    # d wrb: the kernel's d rel folded by bucket (sorted index_put_, fp32) against the
    # oracle's, folded in float64; each bucket sums up to 2L-1 fp32 values.
    onehot = torch.nn.functional.one_hot(extra['bucket'], _BUCKETS).double()
    fold_abs = r['drel'].abs() @ onehot
    _CheckBound(case, 'dwrb', dleaf, r['drel'] @ onehot,
                drel_bound @ onehot + 2.0**-13 * fold_abs)

  # Exact zeros.
  assert bool((dq[~live] == 0).all()), 'dQ is not 0 at a query that sees no key'
  assert bool((dk[~seen] == 0).all()), 'dK is not 0 at a key that no query sees'
  assert bool((dv[~seen] == 0).all()), 'dV is not 0 at a key that no query sees'
  assert bool((drel[:, ~r['used']] == 0).all()), 'd rel is not 0 on an unused diagonal'
  if causal:              # positions grow with the index in every case: no pair has i < j
    assert not bool(r['used'][:l - 1].any())
  if case.startswith('packed'):
    assert not bool(live[1].any()) and not bool(seen[1].any())   # the fully padded row


def _BenchArgs(seed):
  q, k, v, rel, seg, pos, scale, causal, d_o, _ = _Inputs('bench-causal', seed)
  return q, k, v, rel.detach(), seg, pos, d_o


def _Step(q, k, v, rel, seg, pos, d_o):
  nat = ops.native()
  out, lse = nat.flash_attn_fwd(q, k, v, rel, seg, pos, 1.0, True)
  return (out, lse) + tuple(nat.flash_attn_bwd(q, k, v, out, d_o, lse, rel, seg, pos, 1.0,
                                               True, True))


_NAMES = ['out', 'lse', 'dq', 'dk', 'dv', 'drel']


@pytest.mark.gpu
def test_flash_attention_is_bitwise_reproducible_at_benchmark_shape():
  """The backward folds its dQ and d rel partials in a fixed order: two calls agree bit for
  bit."""
  args = _BenchArgs(11)
  first = _Step(*args)
  again = _Step(*args)
  for name, x, y in zip(_NAMES, first, again):
    assert torch.equal(_Bits(x), _Bits(y)), name


@pytest.mark.gpu
def test_flash_attention_graph_replay_matches_eager():
  """Forward + backward captured once in a CUDA graph and replayed on new q/k/v/rel/dO equals
  the eager call on those inputs bit for bit."""
  static = [t.clone() if t is not None else None for t in _BenchArgs(12)]
  # q/k/v stay column slices of one fused buffer, as in the model.
  qkv = torch.cat([t.reshape(*t.shape[:2], -1) for t in static[:3]], dim=-1)
  h = static[0].shape[2]
  static[:3] = [t.reshape(*t.shape[:2], h, _D) for t in qkv.split(h * _D, dim=-1)]
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    for _ in range(2):
      _Step(*static)
  torch.cuda.current_stream().wait_stream(side)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    captured = _Step(*static)
  new = _BenchArgs(13)
  for i in (3, 6):                                               # rel, dO
    static[i].copy_(new[i])
  qkv.copy_(torch.cat([t.reshape(*t.shape[:2], -1) for t in new[:3]], dim=-1))
  graph.replay()
  eager = _Step(*new)
  torch.cuda.synchronize()
  for name, x, y in zip(_NAMES, captured, eager):
    assert torch.equal(_Bits(x), _Bits(y)), name


# --------------------------------------------------------------- argument checks ----
def _BadFlashCalls():
  """(what, entry point, args) for calls the host-side checks must refuse. The forward takes
  (q, k, v, rel, seg, pos, scale, causal), the backward (q, k, v, out, d_out, lse, rel, seg,
  pos, scale, causal, need_drel)."""
  b, l, h = 2, 256, 3
  q = torch.zeros(b, l, h, _D, dtype=torch.bfloat16, device='cuda')
  rel = torch.zeros(h, 2 * l - 1, device='cuda')
  seg = torch.ones(b, l, dtype=torch.int32, device='cuda')
  lse = torch.zeros(b, h, l, device='cuda')
  fwd = dict(q=q, k=q, v=q, rel=rel, seg=seg, pos=seg)
  bwd = dict(fwd, out=q, d_out=q, lse=lse)
  bad = [('q', q.cpu()), ('k', q.cpu()), ('v', q.cpu()), ('rel', rel.cpu()), ('seg', seg.cpu()),
         ('pos', seg.cpu()), ('seg', seg.reshape(l, b)), ('pos', seg.reshape(1, b * l)),
         ('seg', seg[:1]), ('rel', rel[:, 1:])]
  bad_bwd = [('out', q.cpu()), ('d_out', q.cpu()), ('lse', lse.cpu()),
             ('lse', lse.reshape(b, l, h)), ('lse', lse.reshape(h, b, l)),
             ('lse', lse.reshape(-1))]
  for name, x in bad:
    yield 'fwd %s %s' % (name, _Describe(x)), 'fwd', dict(fwd, **{name: x})
  for name, x in bad + bad_bwd:
    yield 'bwd %s %s' % (name, _Describe(x)), 'bwd', dict(bwd, **{name: x})


def _Describe(t):
  return '%s%s' % (t.device.type, list(t.shape))


@pytest.mark.gpu
def test_flash_attention_rejects_bad_arguments_without_launching():
  nat = ops.native()
  launches = nat.launch_count()
  for what, entry, a in _BadFlashCalls():
    with pytest.raises(RuntimeError, match='flash_attn_%s' % entry):
      if entry == 'fwd':
        nat.flash_attn_fwd(a['q'], a['k'], a['v'], a['rel'], a['seg'], a['pos'], 1.0, True)
      else:
        nat.flash_attn_bwd(a['q'], a['k'], a['v'], a['out'], a['d_out'], a['lse'], a['rel'],
                           a['seg'], a['pos'], 1.0, True, True)
      pytest.fail('accepted: ' + what)
  assert nat.launch_count() == launches


def test_flash_attention_rejects_host_tensors():
  """Runs without a GPU: host tensors are refused before anything is launched."""
  nat = ops.native()
  q = torch.zeros(1, 128, 1, _D, dtype=torch.bfloat16)
  lse = torch.zeros(1, 1, 128)
  with pytest.raises(RuntimeError, match='flash_attn_fwd: q must be a CUDA'):
    nat.flash_attn_fwd(q, q, q, None, None, None, 1.0, True)
  with pytest.raises(RuntimeError, match='flash_attn_bwd: q must be a CUDA'):
    nat.flash_attn_bwd(q, q, q, q, q, lse, None, None, None, 1.0, True, False)


# ------------------------------------------------------------- oracle self-test ----
def test_float64_oracle_matches_fp32_reference_and_autograd():
  """Runs without a GPU. The oracle's forward agrees with `flash_attention_ref` (fp32) on
  every query that sees a key, and its closed-form backward with torch.autograd of its own
  float64 forward, on a packed causal layout with a padded row and a random bias table."""
  gen = torch.Generator().manual_seed(0)
  b, l, h, d, scale = 2, 24, 3, 8, 0.7
  q, k, v, d_o = [torch.randn(b, l, h, d, generator=gen, dtype=torch.float64)
                  for _ in range(4)]
  rel = torch.randn(h, 2 * l - 1, generator=gen, dtype=torch.float64)
  seg = torch.tensor([[1] * 10 + [2] * 9 + [0] * 5, [3] * 24], dtype=torch.int32)
  seg[1, 7] = 4                                                  # a 1-token segment
  pos = torch.cat([torch.arange(10), torch.arange(9), torch.zeros(5, dtype=torch.long)])
  pos = torch.stack([pos, torch.arange(l)]).int()
  for causal in (True, False):
    live = _Visible(seg, pos, causal, b, l, 'cpu').any(-1)
    do = d_o * live[:, :, None, None]
    r = _Oracle(q, k, v, rel, seg, pos, scale, causal, do)
    ref = A.flash_attention_ref(q.float(), k.float(), v.float(), rel.float(), seg, pos, scale,
                                causal)
    torch.testing.assert_close(r['out'][live], ref[live].double(), atol=2e-5, rtol=2e-5)
    assert not bool(live[0, 19:].any()) and bool(live[0, :19].all())

    leaves = [t.clone().requires_grad_(True) for t in (q, k, v, rel)]
    qq, kk, vv, rr = leaves
    vis = _Visible(seg, pos, causal, b, l, 'cpu')
    outs = []
    for bi in range(b):
      f = lambda t: t[bi].permute(1, 0, 2)
      outs.append(_Forward64(f(qq), f(kk), f(vv), _Toeplitz(rr, l), vis[bi], scale)[1]
                  .permute(1, 0, 2))
    grads = torch.autograd.grad(torch.stack(outs), leaves, do)
    for name, g in zip(['dq', 'dk', 'dv', 'drel'], grads):
      torch.testing.assert_close(r[name], g, atol=1e-12, rtol=1e-10, msg=name)
    torch.testing.assert_close(r['out'], torch.stack(outs).detach(), atol=0, rtol=0)
    lse_ref = torch.logsumexp(
        torch.where(vis[:, None], scale * torch.einsum('bihd,bjhd->bhij', q, k) +
                    _Toeplitz(rel, l), -math.inf), -1)
    torch.testing.assert_close(r['lse'][live[:, None].expand(b, h, l)],
                               lse_ref[live[:, None].expand(b, h, l)])
