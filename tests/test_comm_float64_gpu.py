"""The peer-memory all-reduce and ZeRO-Adam kernels (ops/csrc/comm_kernels.cu) against float64
oracles, with W ranks simulated by W buffers on one device.

Both kernels take raw peer pointers, so W local bf16 buffers stand in for the W ranks'
symmetric buffers, and the ranks are launched one after another. That is equivalent to
the concurrent run: rank r reads only its own shard [r·n8, (r+1)·n8) of every buffer, only
rank r writes that shard, and zero_adam reads only the shard it reduced. Every buffer is
padded with a NaN bit pattern on both sides, which must survive.

Contract, u = 2^-24, line numbers comm_kernels.cu's unless adam.cuh is named:

  * allreduce_mean_bf16 (:40-88): y = bf16(fp32(Σ_r x_r in rank order) · fp32(scale)), stored
    into the owner's buffer, or into every buffer with store_all. The sum is a chain of W − 1
    fp32 adds (:57-59, the first add is exact), the product rounds once (:61-64), then one
    round-to-nearest pack. With S = Σ_r x_r in float64 and fs = fp32(scale):

        |y − S·fs| ≤ 2·(½·ulp_bf16(max(|S·fs|, |y|)) + e),   e = ((W − 1)·u·Σ|x_r| + u·|S|)·fs.

    A per-element bound one bf16 ulp wide cannot see a truncating pack or a scale rounded to
    bf16, so a rounding check allows at most 1 % of the elements of a case with ≥ 2^14
    outputs above ⅝ ulp.
  * sumsq (:65-98): it adds Σ_k (a_k·fs)² to the value already there, where a_k·fs is the
    unrounded fp32 mean, not the stored bf16. Each thread chains its squares (8 per 16-byte
    vector, ⌈n8/(blocks·512)⌉ vectors), a warp butterfly adds 32 lanes (5 levels), thread 0
    sums the 16 warps in order into one partial per CTA, and a one-warp fold kernel sums the
    partials (lane l takes l, l + 32, …, then a butterfly) and adds them to sumsq. All terms
    are non-negative, so with q_k = fs·S_k ± e_k:

        |sumsq − v0 − Σ (S_k·fs)²| ≤ Σ e_k·(2·|S_k·fs| + e_k) + L·u·(v0 + Σ (|S_k·fs| + e_k)²),
        L = 8·⌈n8/(blocks·512)⌉ + 1 + 5 + 16 + ⌈blocks/32⌉ + 5 + 1,

    with 1 + 10^-3 for second-order terms. The partials and the fold replace a float
    atomicAdd per warp, whose order changed from run to run; sumsq is now bit-identical, and
    a call with sumsq launches two kernels instead of one.
  * zero_adam (:100-140): g = Σ over grad_world peers (the same chain), gg = g·gs (exactly 0
    when gs = 0, whatever g holds), then `adam_update` (adam.cuh), which adam_flat also
    calls, so its roundings are spelled out once; and bf16(w) stored
    into every peer's replica. The oracle is float64 Adam with the bounds of
    test_adam_flat_matches_float64, widened by the sum's error (1 − β)·e_g. At W = 1 and
    grad_world = 1 the kernel must match adam_flat bit for bit, and every replica must equal
    bf16(master) bit for bit at the rank's shard.

Mutation controls: rank W − 1 dropped; the shard base off by one vector; the scale applied
in bf16; a truncating pack. The kernel's output must fail the bound or the rounding check
against each mutated oracle. The scale control needs bf16(fs) ≠ fs, and the last two need
a case of ≥ 2^14 elements; a control is not built where that does not hold.

Replays. `ZeroAdam.Apply` (parallel/zero.py) at W ∈ {2, 3, 8}, clip off and on: stage the
W gradients, allreduce with store_all = False and sumsq, sum the W sumsq in rank order (for
`dist.all_reduce`), the clip scale as the code computes it, then zero_adam with the rank's
own gradient table and every peer's parameter table. `FusedAllReduce`'s monolithic launch
and its bucketed launches (peer pointers into the middle of the buffer, max_blocks = 48).

Measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock); the inputs are
seeded. Worst err/bound and the largest share above ⅝ ulp:

    allreduce, 110 cases       mean ≤ 0.500, sumsq ≤ 0.062, share ≤ 1.5e-7
    zero_adam, 10 cases       m ≤ 0.477, v ≤ 0.356, w ≤ 0.500
    ZeroAdam.Apply, 6 cases   mean ≤ 0.500, sumsq ≤ 0.031, m ≤ 0.302, v ≤ 0.324, w ≤ 0.492
    FusedAllReduce, 4 cases   mean ≤ 0.500

The mean sits at ½: its error is the final bf16 rounding. Every control was rejected at
every case it applies to. The module runs 140 tests in ~12 s.
"""
import math

import pytest
import torch

from lingvo_b200 import ops

_U = 2.0**-24
_SECOND = 1.0 + 1e-3
_THREADS = 512
_PAD = 64                  # sentinel elements on each side of every buffer (16-byte multiple)
_SENTINEL = 0x7fc1         # a bf16 NaN bit pattern
_ROUND_ULPS = 0.625
_ROUND_FRAC = 0.01
_ROUND_MIN = 2**14
_F32, _BF16 = torch.float32, torch.bfloat16


def _F(x):
  """The fp32 value of a Python float, as the kernels receive it."""
  return float(torch.tensor(x, dtype=_F32))


_B1, _B2, _EPS, _LR = _F(0.9), _F(0.98), _F(1e-8), _F(1e-3)   # the kernels' fp32 values


def _Ulp(t):
  a = t.abs().clamp_min(2.0**-126)
  return torch.exp2(torch.floor(torch.log2(a)) - 7)


def _UlpF32(t):
  a = t.abs().clamp_min(2.0**-126)
  return torch.exp2(torch.floor(torch.log2(a)) - 23)


def _Bits(t):
  t = t.detach().contiguous()
  return t.view(torch.int32) if t.dtype == _F32 else t.view(torch.int16)


def _Truncate(v):
  return (v.float().view(torch.int32) & -65536).view(torch.float32).to(_BF16)


def _Blocks(n8, sms, max_blocks=0):
  """Blocks() of comm_kernels.cu and allreduce_mean_bf16's max_blocks cap."""
  b = max(1, min((n8 + _THREADS - 1) // _THREADS, 4 * sms))
  return min(b, max_blocks) if max_blocks > 0 else b


class _Bufs:
  """W sentinel-padded bf16 buffers of `n` elements each, and their peer-pointer table."""

  def __init__(self, world, n, device='cuda'):
    self.raw = [torch.full((n + 2 * _PAD,), _SENTINEL, dtype=torch.int16,
                           device=device).view(_BF16) for _ in range(world)]
    self.views = [r[_PAD:_PAD + n] for r in self.raw]

  def Table(self, offset=0, ranks=None):
    ranks = range(len(self.views)) if ranks is None else ranks
    return torch.tensor([self.raw[r].data_ptr() + 2 * (_PAD + offset) for r in ranks],
                        dtype=torch.int64)

  def Stage(self, xs):
    for v, x in zip(self.views, xs):
      v.copy_(x)

  def AssertPads(self, what):
    for r, raw in enumerate(self.raw):
      for pad in (raw[:_PAD], raw[-_PAD:]):
        assert bool((_Bits(pad) == _SENTINEL).all()), '%s: buffer %d written outside' % (
            what, r)


class _Result:

  def __init__(self, what):
    self.what, self.worst, self.over, self.total, self.caught = what, {}, 0, 0, {}

  def Finish(self):
    if self.total >= _ROUND_MIN:
      assert self.over <= _ROUND_FRAC * self.total, (
          '%s: %d of %d elements above %g ulp: not rounded to nearest' % (
              self.what, self.over, self.total, _ROUND_ULPS))
    missed = [k for k, v in self.caught.items() if not v]
    assert not missed, '%s: the checks do not reject: %s' % (self.what, ', '.join(missed))
    share = self.over / max(self.total, 1)
    print('%s: worst err/bound %s, share above %g ulp %.1e' % (
        self.what, ' '.join('%s %.3f' % kv for kv in sorted(self.worst.items())),
        _ROUND_ULPS, share))
    return self.worst, share


def _Ratio(res, name, err, bound):
  bad = err > bound
  assert not bool(bad.any()), '%s %s: %d elements outside the bound, worst err/bound %g' % (
      res.what, name, int(bad.sum()), float((err / bound.clamp_min(1e-300))[bad].max()))
  if err.numel():
    res.worst[name] = max(res.worst.get(name, 0.0),
                          float((err / bound.clamp_min(1e-300)).max()))


# ---------------------------------------------------------- the all-reduce check ----
@torch.no_grad()
def _MeanOracle(xs, scale):
  """S·fs and e of the module docstring, float64, from the W staged bf16 inputs."""
  fs = _F(scale)
  x64 = torch.stack([x.double() for x in xs])
  s = x64.sum(0)
  e = ((len(xs) - 1) * _U * x64.abs().sum(0) + _U * s.abs()) * fs
  return s * fs, e, s, x64


def _Rejects(y, ref, e):
  """Whether y fails the bound or the rounding check against the (mutated) oracle ref."""
  err = (y - ref).abs()
  if bool((err > 2 * (0.5 * _Ulp(torch.maximum(ref.abs(), y.abs())) + e)).any()):
    return True
  return y.numel() >= _ROUND_MIN and int((err > _ROUND_ULPS * _Ulp(ref)).sum()) > (
      _ROUND_FRAC * y.numel())


@torch.no_grad()
def _CheckMean(res, y, xs, scale, shard):
  """y: the reduced bf16 values over all W shards, [W·shard]."""
  ref, e, s, x64 = _MeanOracle(xs, scale)
  yd = y.double()
  assert bool(torch.isfinite(yd).all()), '%s: non-finite output' % res.what
  err = (yd - ref).abs()
  _Ratio(res, 'mean', err, 2 * (0.5 * _Ulp(torch.maximum(ref.abs(), yd.abs())) + e))
  res.over += int((err > _ROUND_ULPS * _Ulp(ref)).sum())
  res.total += err.numel()
  if shard == 0:
    return
  fs = _F(scale)
  w = len(xs)
  if w > 1:
    res.caught['rank W-1 dropped'] = res.caught.get('rank W-1 dropped', False) or _Rejects(
        yd, (s - x64[-1]) * fs, e)
  if y.numel() > 8:
    res.caught['shard base off by one vector'] = res.caught.get(
        'shard base off by one vector', False) or _Rejects(yd, torch.roll(ref, -8), e)
  if y.numel() >= _ROUND_MIN:
    bs = float(torch.tensor(fs).bfloat16())
    if bs != fs:
      res.caught['scale in bf16'] = res.caught.get('scale in bf16', False) or _Rejects(
          yd, s * bs, e)
    trunc = _Truncate(ref)
    if not torch.equal(_Bits(trunc), _Bits(ref.float().bfloat16())):   # else a no-op
      res.caught['truncating pack'] = res.caught.get('truncating pack', False) or _Rejects(
          yd, trunc.double(), e)


@torch.no_grad()
def _CheckSumsq(res, got, v0, xs, scale, lo, hi, blocks):
  """got: one rank's sumsq after adding its shard [lo, hi) to v0."""
  ref, e, _, _ = _MeanOracle([x[lo:hi] for x in xs], scale)
  n8 = (hi - lo) // 8
  chain = 8 * -(-n8 // (blocks * _THREADS)) + 1 + 5 + 16 + -(-blocks // 32) + 5 + 1
  want = v0 + float(ref.square().sum())
  bound = (float((e * (2 * ref.abs() + e)).sum()) +
           _SECOND * chain * _U * (v0 + float((ref.abs() + e).square().sum())))
  err = abs(float(got) - want)
  assert err <= bound, '%s: sumsq %r, float64 %r, bound %g' % (res.what, float(got), want, bound)
  res.worst['sumsq'] = max(res.worst.get('sumsq', 0.0), err / bound if bound else 0.0)


def _Inputs(gen, world, n, scale=1.0):
  return [(torch.randn(n, device='cuda', generator=gen) * scale).to(_BF16)
          for _ in range(world)]


def _AllReduce(bufs, shard, world, scale, store_all, sumsq=None, max_blocks=0, offset=0):
  nat = ops.native()
  for r in range(world):
    nat.allreduce_mean_bf16(bufs.Table(offset), shard, r, world, scale, 0, store_all,
                            None if sumsq is None else sumsq[r], max_blocks)


def _ShardSizes(sms):
  cap = 4 * sms * _THREADS * 8
  return {'0': 0, '8': 8, '8x511': 8 * 511, '8x512+8': 8 * 512 + 8,
          'past_grid_cap': cap + 8 * 333}


_SHARD_IDS = list(_ShardSizes(132))


@pytest.mark.gpu
@pytest.mark.parametrize('max_blocks', [0, 1, 48])
@pytest.mark.parametrize('store_all', [False, True], ids=['owner_only', 'store_all'])
@pytest.mark.parametrize('world', [1, 2, 3, 8, 16])
@pytest.mark.parametrize('size', _SHARD_IDS)
def test_allreduce_mean(size, world, store_all, max_blocks):
  if max_blocks and size in ('0', '8'):
    pytest.skip('one CTA either way')
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  shard = _ShardSizes(sms)[size]
  n = world * shard
  gen = torch.Generator(device='cuda').manual_seed(world * 1000 + shard + max_blocks)
  xs = _Inputs(gen, world, n)
  scale = 1.0 / world if world != 2 else 0.3        # 0.3: a scale bf16 cannot hold
  bufs = _Bufs(world, n)
  bufs.Stage(xs)
  v0 = 0.75
  sumsq = [torch.full((1,), v0, device='cuda') for _ in range(world)]
  nat = ops.native()
  before = nat.launch_count()
  _AllReduce(bufs, shard, world, scale, store_all, sumsq, max_blocks)
  assert nat.launch_count() - before == 2 * world     # the all-reduce and the sumsq fold
  bufs.AssertPads('allreduce')
  res = _Result('allreduce %s W=%d store_all=%d max_blocks=%d' % (
      size, world, store_all, max_blocks))
  # Rank r's shard of its own buffer holds the mean; with store_all, every buffer does.
  mine = torch.cat([bufs.views[r][r * shard:(r + 1) * shard] for r in range(world)])
  _CheckMean(res, mine, xs, scale, shard)
  for d in range(world):
    for r in range(world):
      got = bufs.views[d][r * shard:(r + 1) * shard]
      want = mine[r * shard:(r + 1) * shard] if (store_all or d == r) else (
          xs[d][r * shard:(r + 1) * shard])
      assert torch.equal(_Bits(got), _Bits(want)), 'buffer %d, shard %d' % (d, r)
  blocks = _Blocks(shard // 8, sms, max_blocks)
  for r in range(world):
    _CheckSumsq(res, sumsq[r], v0, xs, scale, r * shard, (r + 1) * shard, blocks)
  res.Finish()


@pytest.mark.gpu
@pytest.mark.parametrize('world', [3, 16])
def test_allreduce_is_bitwise_reproducible(world):
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  shard = 4 * sms * _THREADS * 8 + 8 * 333
  gen = torch.Generator(device='cuda').manual_seed(world)
  xs = _Inputs(gen, world, world * shard, scale=3.0)
  outs = []
  for _ in range(3):
    bufs = _Bufs(world, world * shard)
    bufs.Stage(xs)
    sumsq = [torch.zeros(1, device='cuda') for _ in range(world)]
    _AllReduce(bufs, shard, world, 1.0 / world, True, sumsq)
    outs.append((torch.stack(bufs.views), torch.cat(sumsq)))
  for y, s in outs[1:]:
    assert torch.equal(_Bits(y), _Bits(outs[0][0]))
    assert torch.equal(_Bits(s), _Bits(outs[0][1])), 'sumsq differs between calls'


# ------------------------------------------------------------------- zero_adam ----
def _AdamOracle(res, name, w, m, v, w0, m0, v0, s, eg, gs, lr_t):
  """float64 Adam from the float64 gradient sum s (error eg) scaled by gs; the bounds of
  test_adam_flat_matches_float64 widened by the sum's error."""
  gg = s * gs
  mt, vt = _B1 * m0.double(), (1 - _B1) * gg
  _Ratio(res, name + ' m', (m.double() - mt - vt).abs(),
         4 * _U * (mt.abs() + vt.abs()) + (1 - _B1) * eg * gs + 1e-30)
  v_ref = _B2 * v0.double() + (1 - _B2) * gg.square()
  _Ratio(res, name + ' v', (v.double() - v_ref).abs(),
         6 * _U * v_ref + (1 - _B2) * eg * gs * (2 * gg.abs() + eg * gs) + 1e-30)
  delta = lr_t * m.double() / (v.double().sqrt() + _EPS)
  want = w0.double() - delta
  _Ratio(res, name + ' w', (w.double() - want).abs(), 8 * _U * delta.abs() + _UlpF32(want))


def _Adam(world, grad_world, shard, gs_kind, seed, ppeers_offset=0):
  """One zero_adam call per rank on sentinel-padded buffers; returns what the checks need."""
  gen = torch.Generator(device='cuda').manual_seed(seed)
  n = world * shard
  grads = _Bufs(grad_world, n)
  gx = _Inputs(gen, grad_world, n, scale=0.01)
  grads.Stage(gx)
  params = _Bufs(world, n)
  master = [torch.randn(shard, device='cuda', generator=gen) * 0.05 for _ in range(world)]
  m = [torch.randn(shard, device='cuda', generator=gen) * 1e-3 for _ in range(world)]
  v = [torch.rand(shard, device='cuda', generator=gen) * 1e-5 for _ in range(world)]
  w0, m0, v0 = [t.clone() for t in master], [t.clone() for t in m], [t.clone() for t in v]
  if gs_kind == 'scalar':
    gs_arg, gs_t, gs = 0.37, None, _F(0.37)
  else:
    gs_arg, gs_t = 2.0, torch.tensor([0.185], device='cuda')
    gs = _F(2.0 * _F(0.185))
  lr_t = _F(_LR)
  nat = ops.native()
  for r in range(world):
    nat.zero_adam(grads.Table(), params.Table(), master[r], m[r], v[r], r, world, grad_world,
                  gs_arg, gs_t, lr_t, _B1, _B2, _EPS)
  return dict(grads=grads, gx=gx, params=params, master=master, m=m, v=v, w0=w0, m0=m0, v0=v0,
              gs=gs, lr_t=lr_t)


@pytest.mark.gpu
@pytest.mark.parametrize('gs_kind', ['scalar', 'tensor'])
@pytest.mark.parametrize('world,grad_world', [(1, 1), (3, 1), (3, 3), (8, 8), (16, 1)])
def test_zero_adam(world, grad_world, gs_kind):
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  shard = 4 * sms * _THREADS * 8 + 8 * 37 if world <= 3 else 8 * 4099
  k = _Adam(world, grad_world, shard, gs_kind, world * 100 + grad_world)
  res = _Result('zero_adam W=%d grad_world=%d %s' % (world, grad_world, gs_kind))
  g64 = torch.stack([x.double() for x in k['gx']])
  for r in range(world):
    sl = slice(r * shard, (r + 1) * shard)
    s = g64[:, sl].sum(0)
    eg = (grad_world - 1) * _U * g64[:, sl].abs().sum(0) + _U * s.abs()
    _AdamOracle(res, 'rank', k['master'][r], k['m'][r], k['v'][r], k['w0'][r], k['m0'][r],
                k['v0'][r], s, eg, k['gs'], k['lr_t'])
  # Every replica holds bf16(master) at every shard, bit for bit.
  full = torch.cat([t.bfloat16() for t in k['master']])
  for d in range(world):
    assert torch.equal(_Bits(k['params'].views[d]), _Bits(full)), 'replica %d' % d
  k['params'].AssertPads('zero_adam params')
  k['grads'].AssertPads('zero_adam grads')
  for x, got in zip(k['gx'], k['grads'].views):
    assert torch.equal(_Bits(x), _Bits(got)), 'zero_adam wrote a gradient buffer'
  res.Finish()


@pytest.mark.gpu
def test_zero_adam_leaves_other_shards_untouched():
  """Rank 1 of 3 alone: only shard 1 of each replica changes."""
  shard, world = 8 * 1000, 3
  gen = torch.Generator(device='cuda').manual_seed(5)
  grads = _Bufs(1, world * shard)
  grads.Stage(_Inputs(gen, 1, world * shard, 0.01))
  params = _Bufs(world, world * shard)
  before = [p.clone() for p in params.views]
  master = torch.randn(shard, device='cuda', generator=gen)
  m, v = torch.zeros_like(master), torch.zeros_like(master)
  ops.native().zero_adam(grads.Table(), params.Table(), master, m, v, 1, world, 1, 1.0, None,
                         1e-3, _B1, _B2, _EPS)
  for p, b in zip(params.views, before):
    assert torch.equal(_Bits(p[shard:2 * shard]), _Bits(master.bfloat16()))
    for sl in (slice(0, shard), slice(2 * shard, 3 * shard)):
      assert torch.equal(_Bits(p[sl]), _Bits(b[sl]))
  params.AssertPads('zero_adam')


@pytest.mark.gpu
def test_zero_adam_zero_grad_scale_ignores_nonfinite_gradients():
  shard, world = 8 * 4096, 2
  gen = torch.Generator(device='cuda').manual_seed(6)
  g = _Inputs(gen, world, world * shard, 0.01)
  for x in g:
    x[::7] = float('inf')
    x[3::11] = float('nan')
    x[5::13] = float('-inf')
  grads = _Bufs(world, world * shard)
  grads.Stage(g)
  params = _Bufs(world, world * shard)
  for gs_arg, gs_t in ((0.0, None), (1.0, torch.zeros(1, device='cuda'))):
    master = [torch.randn(shard, device='cuda', generator=gen) for _ in range(world)]
    m = [torch.randn(shard, device='cuda', generator=gen) * 1e-3 for _ in range(world)]
    v = [torch.rand(shard, device='cuda', generator=gen) * 1e-5 for _ in range(world)]
    m0, v0, w0 = [t.clone() for t in m], [t.clone() for t in v], [t.clone() for t in master]
    for r in range(world):
      ops.native().zero_adam(grads.Table(), params.Table(), master[r], m[r], v[r], r, world,
                             world, gs_arg, gs_t, _LR, _B1, _B2, _EPS)
    for r in range(world):
      b1, b2 = torch.tensor(_B1), torch.tensor(_B2)
      assert torch.equal(_Bits(m[r]), _Bits(m0[r] * b1)), 'gg is not exactly 0'
      assert torch.equal(_Bits(v[r]), _Bits(v0[r] * b2)), 'gg is not exactly 0'
      assert bool(torch.isfinite(master[r]).all())
      delta = _LR * m[r].double() / (v[r].double().sqrt() + _EPS)
      want = w0[r].double() - delta
      assert bool(((master[r].double() - want).abs() <= 8 * _U * delta.abs() +
                   _UlpF32(want)).all())


@pytest.mark.gpu
@pytest.mark.parametrize('gs_kind', ['scalar', 'tensor'])
def test_zero_adam_matches_adam_flat_bitwise(gs_kind):
  """At W = 1 and grad_world = 1 with finite gradients, the two Adam kernels agree bit for
  bit on w, m, v and the bf16 copy."""
  from lingvo_b200.ops import optim
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  shard = 8 * sms * 256 * 8 * 2 + 8 * 37
  k = _Adam(1, 1, shard, gs_kind, 77)
  w, m, v = k['w0'][0].clone(), k['m0'][0].clone(), k['v0'][0].clone()
  wb = torch.empty(shard, device='cuda', dtype=_BF16)
  gs_arg, gs_t = (0.37, None) if gs_kind == 'scalar' else (2.0,
                                                           torch.tensor([0.185], device='cuda'))
  optim.adam_flat(w, k['gx'][0], m, v, wb, k['lr_t'], _B1, _B2, _EPS, grad_scale=gs_arg,
                  grad_scale_t=gs_t)
  for name, a, b in (('w', k['master'][0], w), ('m', k['m'][0], m), ('v', k['v'][0], v),
                     ('bf16 w', k['params'].views[0], wb)):
    assert torch.equal(_Bits(a), _Bits(b)), '%s differs from adam_flat' % name


# ----------------------------------------------------- the engines' call sequences ----
@pytest.mark.gpu
@pytest.mark.parametrize('clip', [0.0, 0.5], ids=['no_clip', 'clip'])
@pytest.mark.parametrize('world', [2, 3, 8])
def test_zero_adam_engine_step(world, clip):
  """ZeroAdam.Apply, kernel by kernel: reduce-scatter with sumsq, the summed norm, the clip
  scale, then the fused Adam step into every replica."""
  shard = 8 * 9001
  n = world * shard
  gen = torch.Generator(device='cuda').manual_seed(world * 10 + int(clip * 10))
  gx = _Inputs(gen, world, n, scale=0.01)
  gbuf, pbuf = _Bufs(world, n), _Bufs(world, n)
  gbuf.Stage(gx)
  full = torch.randn(n, device='cuda', generator=gen) * 0.05
  for p in pbuf.views:
    p.copy_(full)
  master = [full[r * shard:(r + 1) * shard].clone() for r in range(world)]
  m = [torch.zeros(shard, device='cuda') for _ in range(world)]
  v = [torch.zeros(shard, device='cuda') for _ in range(world)]
  sumsq = [torch.zeros(1, device='cuda') for _ in range(world)]
  nat = ops.native()
  for r in range(world):
    nat.allreduce_mean_bf16(gbuf.Table(), shard, r, world, 1.0 / world, 0, False, sumsq[r])
  total = sumsq[0].clone()
  for s in sumsq[1:]:
    total += s                                         # dist.all_reduce of the partial norms
  gnorm = total.sqrt()
  scale = torch.clamp(clip / gnorm, max=1.0) if clip else torch.ones_like(gnorm)
  scale = torch.where(torch.isfinite(gnorm), scale, torch.zeros_like(scale))
  lr_t = _LR * math.sqrt(1 - _B2) / (1 - _B1)
  for r in range(world):
    nat.zero_adam(gbuf.Table(ranks=[r]), pbuf.Table(), master[r], m[r], v[r], r, world, 1, 1.0,
                  scale, lr_t, _B1, _B2, _EPS)
  res = _Result('ZeroAdam W=%d clip=%g' % (world, clip))
  reduced = torch.cat([gbuf.views[r][r * shard:(r + 1) * shard] for r in range(world)])
  _CheckMean(res, reduced, gx, 1.0 / world, shard)
  blocks = _Blocks(shard // 8, torch.cuda.get_device_properties(0).multi_processor_count)
  for r in range(world):
    _CheckSumsq(res, sumsq[r], 0.0, gx, 1.0 / world, r * shard, (r + 1) * shard, blocks)
  gs = float(scale)
  if clip:
    assert gs < 1.0, 'the clip does not act: raise the gradients'
  for r in range(world):
    s = reduced[r * shard:(r + 1) * shard].double()
    _AdamOracle(res, 'rank', master[r], m[r], v[r], full[r * shard:(r + 1) * shard],
                torch.zeros(shard, device='cuda'), torch.zeros(shard, device='cuda'), s,
                _U * s.abs(), gs, _F(lr_t))
  want = torch.cat([t.bfloat16() for t in master])
  for d in range(world):
    assert torch.equal(_Bits(pbuf.views[d]), _Bits(want)), 'replica %d' % d
  pbuf.AssertPads('ZeroAdam params')
  gbuf.AssertPads('ZeroAdam grads')
  res.Finish()


@pytest.mark.gpu
@pytest.mark.parametrize('bucketed', [False, True], ids=['monolithic', 'bucketed'])
@pytest.mark.parametrize('world', [2, 8])
def test_fused_allreduce_engine(world, bucketed):
  """FusedAllReduce: one launch per rank over the whole buffer, or per bucket with peer
  pointers at the bucket's start and 48 CTAs; every replica must hold the mean."""
  unit = world * 8
  sizes = [unit * 1001, unit * 37, unit * 4096] if bucketed else [unit * 5134]
  n = sum(sizes)
  gen = torch.Generator(device='cuda').manual_seed(world + 10 * bucketed)
  gx = _Inputs(gen, world, n)
  bufs = _Bufs(world, n)
  bufs.Stage(gx)
  start = 0
  for size in sizes:
    _AllReduce(bufs, size // world, world, 1.0 / world, True, None,
               48 if bucketed else 0, offset=start)
    start += size
  res = _Result('FusedAllReduce W=%d bucketed=%d' % (world, bucketed))
  y = bufs.views[0]
  for d in range(1, world):
    assert torch.equal(_Bits(bufs.views[d]), _Bits(y)), 'replica %d differs' % d
  _CheckMean(res, y, gx, 1.0 / world, 0)
  bufs.AssertPads('FusedAllReduce')
  res.Finish()


# -------------------------------------------------------------- argument checks ----
@pytest.mark.gpu
def test_bad_arguments_are_refused_without_launching():
  nat = ops.native()
  world, shard = 4, 8 * 64
  bufs = _Bufs(world, world * shard)
  table = bufs.Table()
  ss = torch.zeros(1, device='cuda')
  master = torch.zeros(shard, device='cuda')
  m, v = torch.zeros_like(master), torch.zeros_like(master)
  odd = torch.zeros(shard + 8, device='cuda')[1:1 + shard]
  launches = nat.launch_count()

  def Ar(**kw):
    args = dict(peer_ptrs_cpu=table, shard_elems=shard, rank=0, world=world, scale=0.25,
                device=0, store_all=True, sumsq=ss, max_blocks=0)
    args.update(kw)
    with pytest.raises(RuntimeError):
      nat.allreduce_mean_bf16(**args)

  def Za(**kw):
    args = dict(g=table, p=table, master=master, m=m, v=v, rank=0, world=world, grad_world=world,
                gs=1.0, gst=None)
    args.update(kw)
    with pytest.raises(RuntimeError):
      nat.zero_adam(args['g'], args['p'], args['master'], args['m'], args['v'], args['rank'],
                    args['world'], args['grad_world'], args['gs'], args['gst'], 1e-3, _B1, _B2,
                    _EPS)

  short = table[:world - 1].clone()
  unaligned = table.clone()
  unaligned[2] += 2
  null = table.clone()
  null[1] = 0
  for bad in (table.cuda(), table.int(), table.view(2, 2), short, unaligned, null,
              torch.zeros(17, dtype=torch.int64)):
    Ar(peer_ptrs_cpu=bad)
    Za(g=bad)
    Za(p=bad)
  for w in (0, 17):
    Ar(world=w)
    Za(world=w)
  for r in (-1, world):
    Ar(rank=r)
    Za(rank=r)
  Za(grad_world=0)
  Za(grad_world=17)
  Za(g=short, grad_world=world)
  for s in (-8, 4):
    Ar(shard_elems=s)
  for bad in (torch.zeros(1, device='cuda', dtype=torch.float64), torch.zeros(1),
              torch.zeros(0, device='cuda')):
    Ar(sumsq=bad)
  if torch.cuda.device_count() > 1:
    Ar(sumsq=torch.zeros(1, device='cuda:1'))
  for name in ('master', 'm', 'v'):
    for bad in (master.double(), master.cpu(), torch.zeros(2 * shard, device='cuda')[::2],
                odd):
      Za(**{name: bad})
  for bad in (torch.ones(1, device='cuda', dtype=torch.float64), torch.ones(1),
              torch.ones(0, device='cuda')):
    Za(gst=bad)
  Za(master=torch.zeros(shard + 4, device='cuda'), m=torch.zeros(shard + 4, device='cuda'),
     v=torch.zeros(shard + 4, device='cuda'))
  assert nat.launch_count() == launches


# ------------------------------------------------------------ the bound on CPU ----
def _MeanStandIn(xs, scale, pack=lambda v: v.to(_BF16)):
  a = torch.zeros_like(xs[0], dtype=_F32)
  for x in xs:
    a = a + x.float()
  return pack(a * _F(scale)), a * _F(scale)


@pytest.mark.parametrize('world,scale', [(3, 1 / 3), (8, 0.125), (2, 0.3)])
def test_bound_and_controls_on_cpu(world, scale):
  """The bound, the rounding check, the sumsq bound and the controls with fp32 emulations of
  the kernels in their place; a truncating pack fails the rounding check."""
  gen = torch.Generator().manual_seed(world)
  shard = 8 * 4096
  xs = [torch.randn(world * shard, generator=gen).to(_BF16) for _ in range(world)]
  y, q = _MeanStandIn(xs, scale)
  res = _Result('cpu W=%d' % world)
  _CheckMean(res, y, xs, scale, shard)
  blocks = 3
  for r in range(world):
    got = torch.tensor(0.5 + float(q[r * shard:(r + 1) * shard].double().square().sum()),
                       dtype=_F32)
    _CheckSumsq(res, got, 0.5, xs, scale, r * shard, (r + 1) * shard, blocks)
  res.Finish()
  yt, _ = _MeanStandIn(xs, scale, _Truncate)
  with pytest.raises(AssertionError, match='not rounded to nearest'):
    bad = _Result('cpu truncating pack')
    _CheckMean(bad, yt, xs, scale, shard)
    bad.Finish()
  # A sumsq that dropped the last CTA's partial is outside the bound.
  qr = q[:shard].double()
  with pytest.raises(AssertionError, match='sumsq'):
    _CheckSumsq(_Result('cpu sumsq'), torch.tensor(float(qr[:-512].square().sum())), 0.0, xs,
                scale, 0, shard, blocks)
