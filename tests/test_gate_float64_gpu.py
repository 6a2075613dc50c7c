"""The MoE router-logit kernels (ops/csrc/gate_kernels.cu) against float64 oracles at the
benchmark's shape, at every instantiation and at the edges of their grids.

Contract, for bf16 x [T, M], gw [M, E] in fp32 or bf16 and fp32 dlogits [T, E]:

    logits = x·gw (fp32),   dx = bf16(dres + dlogits·gwᵀ),   dgw = xᵀ·dlogits (gw's dtype)

with E ∈ {2, 4, 8, 16}, M % 8 == 0 and M·E·4 ≤ 200 KiB. The benchmark (MoELm8E: T = 8192,
M = 2048, E = 8) passes a bf16 gw: its fprop_dtype is bf16, and `BaseLayer._OwnThetaValue`
casts every weight to it before `gate_logits_pass` sees it. Both dtypes are tested there.

The oracle runs in float64 on the device from the same bf16 x and fp32 / bf16 gw values, in
row slabs. Line numbers below are gate_kernels.cu's; u = 2^-24.

  * Forward (:61-108). Lane l of a warp owns columns l·8 + 256·j + i and runs one fma chain
    per (token, expert) over them, j-major, i-minor (:75-95): ⌈M/256⌉·8 terms, M/32 when 256
    divides M. The 32 lane sums meet in a 5-level xor butterfly (:30-33), which adds lane
    groups l mod 16, mod 8, …, mod 1. Every fma and add rounds once to fp32, so

        |y − S| ≤ u·B,   B = Σ_lanes Σ_k |s_k| + Σ_levels Σ_groups |group sum|,

    with s_k the chain's exact partial sums and S = Σ x·w, all computed by the oracle in the
    kernel's order (`_FwdOracle`), times 1 + 10^-3 for the second-order terms. B is at most
    (8⌈M/256⌉ + 5)·P, P = Σ|x·w|, and the oracle asserts that. There is no bf16 rounding:
    the bound rejects gw rounded to bf16 and logits rounded to bf16 at every case.
  * dx (:110-161). Each element is one fma chain that starts from dres and adds dl·w over
    the E experts (:140-148), then one round-to-nearest pack (:153-156):

        |dx − ref| ≤ 2·(½·ulp_bf16(max(|ref|, |dx|)) + E·u·(|dres| + Σ_e |dl·w|)).

  * dgw (:163-230). The host (:357-359) splits the T tokens into `used` ranges of
    tok_per_blk = ⌈T/nblk⌉ tokens, nblk = min(3·SMs, ⌈T/32⌉); CTA (b, y) owns range b and 2048
    columns, and runs one fma chain per (m, e) over its tokens in order (:178-196). The fold
    (:205-230) runs two chains s0 / s1 over the partials k ≡ ky (mod 16) and k ≡ ky + 8,
    adds them, and sums the 8 ky groups in order. So the chain is at most
    L = tok_per_blk + ⌈used/16⌉ + 10 roundings long:

        fp32 gw: |dgw − ref| ≤ L·u·P,   bf16 gw: ≤ 2·(½·ulp_bf16(max(|ref|, |dgw|)) + L·u·P),

    P = Σ_t |x·dl|, with 1 + 10^-3 for second-order terms in the fp32 case.

A per-element bound one bf16 ulp wide cannot see a truncating pack, so a rounding check
allows at most 1 % of the elements of a case with ≥ 2^14 bf16 outputs above ⅝ ulp.

Mutation controls, each applied to the float64 oracle; every case must put some element of
the kernel's output above the bound of each mutated oracle (or, for the truncating pack,
push the rounding share above 1 %):
  * fwd: the last 8-column chunk of M dropped; token t + 1's row used for t; gw rounded to
    bf16 (fp32 gw); the logits rounded to bf16.
  * dx: dres ignored; expert e + 1's weight column used for e; a truncating pack.
  * dgw: the last CTA's partial dropped; partial 0 counted twice; block 0's range shifted by
    one token; the last (ragged) 32-token tile of the last range dropped.
A control that needs two tokens is not built at T = 1; none is built at T = 0, where
the logits and dx are empty and dgw must be exact zeros.

Cases: the benchmark site with both gw dtypes; all 16 fwd / dx instantiations (E × gw
dtype), all 4 dgw kernels and both folds; T ∈ {0, 1, 3, 4, 5, 31, 32, 33, 2·SMs·32 ± a few,
3·SMs·32·k + ragged, 20000}, which reaches the forward's grid-stride loop, the dgw grid's
3·SMs cap, used < nblk and `used % 16` in 1…8 and 9…15; M ∈ {8, 248, 256, 264, 2048, 2056,
4104} (dgw grid.y > 1 from 2056); M·E·4 at 48 KiB and just above (the opt-in shared-memory
path); M at each E's 200 KiB limit. `test_cases_reach_every_path` mirrors the host's
dispatch with the device's SM count and asserts all of this is reached.

Measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock); the inputs are
seeded. Worst err/bound (fwd, dx, dgw) and the largest dx rounding share:

                             fwd     dx      dgw     dx share
    bench, gw fp32           0.054   0.500   0.003   8.3e-7
    bench, gw bf16           0.035   0.500   0.491   6.6e-7
    E ∈ {2, 4, 8, 16}, fp32  ≤ 0.083 ≤ 0.500 ≤ 0.011 ≤ 2.0e-6
    E ∈ {2, 4, 8, 16}, bf16  ≤ 0.055 ≤ 0.500 ≤ 0.497 ≤ 2.0e-6
    T sweep (14 cases)       ≤ 0.110 ≤ 0.500 ≤ 0.500 ≤ 6.3e-6
    M sweep (14 cases)       ≤ 0.481 ≤ 0.500 ≤ 0.497 ≤ 1.5e-6
    shared-memory edges (12) ≤ 0.054 ≤ 0.500 ≤ 0.498 ≤ 2.2e-6
    wrappers                 ≤ 0.089 ≤ 0.500 ≤ 0.494 ≤ 3.9e-6

dx and the bf16 dgw sit at ½: their error is the final bf16 rounding. The fp32 dgw uses
≤ 3 % of its chain bound, and the forward ≤ 11 % of B except at M = 8, where one lane's
8-term chain is the whole sum (0.48). Every control was rejected at every case it applies
to. The module runs 60 tests in ~14 s; the two-GPU refusal test is skipped on one GPU.
"""

import pytest
import torch
import torch.nn.functional as F

from lingvo_b200 import ops
from lingvo_b200.ops import gate

_U = 2.0**-24
_SECOND = 1.0 + 1e-3       # room for the second-order terms of a first-order bound
_WARP_COLS = 256           # columns a warp covers per step: 32 lanes × 8
_WARP_TOKENS = 8 * 4       # kGateWarps × kTok tokens per CTA pass of fwd / dx
_DGW_COLS = 2048           # kDgwCols
_DGW_TILE = 32             # kDgwTile
_SMEM_CAP = 200 * 1024
_SMEM_DEFAULT = 48 * 1024
_SLAB = 2**24              # float64 elements per oracle slab
_ROUND_ULPS = 0.625
_ROUND_FRAC = 0.01
_ROUND_MIN = 2**14
_E_ALL = (2, 4, 8, 16)
_F32, _BF16 = torch.float32, torch.bfloat16


def _Ulp(t):
  """One bf16 ulp at |t| (float64), floored at the smallest normal."""
  a = t.abs().clamp_min(2.0**-126)
  return torch.exp2(torch.floor(torch.log2(a)) - 7)


def _Bits(t):
  t = t.detach().contiguous()
  return t.view(torch.int32) if t.dtype == _F32 else t.view(torch.int16)


def _Truncate(v):
  """fp32 → bf16 by dropping the low 16 bits."""
  return (v.float().view(torch.int32) & -65536).view(torch.float32).to(_BF16)


def _DgwPlan(t, sms):
  """gate_logits_bwd's dgw split (:357-359): (nblk, tok_per_blk, used)."""
  nblk = min(sms * 3, (t + _DGW_TILE - 1) // _DGW_TILE)
  tpb = (t + nblk - 1) // nblk
  return nblk, tpb, (t + tpb - 1) // tpb


def _FwdGrid(t, sms):
  return min((t + _WARP_TOKENS - 1) // _WARP_TOKENS, 2 * sms)


class _Result:
  """Worst err/bound per output, the rounding share, and which controls were caught."""

  def __init__(self, what):
    self.what, self.worst, self.over, self.total, self.caught = what, {}, 0, 0, {}

  def Ratio(self, name, err, bound):
    if err.numel():
      r = float((err / bound.clamp_min(1e-300)).max())
      self.worst[name] = max(self.worst.get(name, 0.0), r)

  def Catch(self, name, hit):
    self.caught[name] = self.caught.get(name, False) or bool(hit)

  def Finish(self):
    if self.total >= _ROUND_MIN:
      assert self.over <= _ROUND_FRAC * self.total, (
          '%s: %d of %d dx elements above %g ulp: not rounded to nearest' % (
              self.what, self.over, self.total, _ROUND_ULPS))
    missed = [k for k, v in self.caught.items() if not v]
    assert not missed, '%s: the bound does not reject: %s' % (self.what, ', '.join(missed))
    share = self.over / max(self.total, 1)
    print('%s: worst err/bound %s, dx share above %g ulp %.1e' % (
        self.what, ' '.join('%s %.3f' % kv for kv in sorted(self.worst.items())),
        _ROUND_ULPS, share))
    return self.worst, share


def _Assert(res, name, y, ref, bound):
  err = (y - ref).abs()
  bad = err > bound
  assert not bool(bad.any()), '%s %s: %d elements outside the bound, worst err/bound %g' % (
      res.what, name, int(bad.sum()), float((err / bound.clamp_min(1e-300))[bad].max()))
  res.Ratio(name, err, bound)


# ------------------------------------------------------------------ the oracles ----
@torch.no_grad()
def _FwdOracle(x, w):
  """S = x·w, P = Σ|x·w| and B (the module docstring), float64 [T, E], in the kernel's
  summation order: lane chains over columns l·8 + 256·j + i, then the xor butterfly."""
  t, m = x.shape
  e = w.shape[1]
  mp = -(-m // _WARP_COLS) * _WARP_COLS
  w64 = F.pad(w.double(), (0, 0, 0, mp - m))
  s = torch.empty(t, e, dtype=torch.float64, device=x.device)
  p, b = torch.empty_like(s), torch.empty_like(s)
  rows = max(1, _SLAB // (mp * e))
  for t0 in range(0, t, rows):
    xs = F.pad(x[t0:t0 + rows].double(), (0, mp - m))
    prod = xs.unsqueeze(2) * w64                                  # [r, mp, E]
    r = prod.shape[0]
    lanes = prod.view(r, mp // _WARP_COLS, 32, 8, e).permute(0, 4, 2, 1, 3).reshape(r, e, 32, -1)
    ps = lanes.cumsum(-1)
    chain = ps.abs().sum(-1).sum(-1)
    v = ps[..., -1]
    tree = torch.zeros_like(chain)
    while v.shape[-1] > 1:
      h = v.shape[-1] // 2
      v = v[..., :h] + v[..., h:]
      tree += v.abs().sum(-1)
    s[t0:t0 + r] = v[..., 0]
    p[t0:t0 + r] = prod.abs().sum(1)
    b[t0:t0 + r] = chain + tree
  assert bool((b <= (8 * (mp // _WARP_COLS) + 5) * p * _SECOND + 1e-300).all())
  return s, p, b


def _Rows(t, m):
  return max(1, _SLAB // max(m, 1))


@torch.no_grad()
def _CheckFwd(res, x, w, y):
  s, p, b = _FwdOracle(x, w)
  y = y.double()
  bound = _SECOND * _U * b
  _Assert(res, 'fwd', y, s, bound)
  t, m = x.shape
  if t == 0:
    return
  x64, w64 = x.double(), w.double()
  def Hit(ref):
    return bool(((y - ref).abs() > bound).any())
  res.Catch('fwd: last 8 columns dropped', Hit(s - x64[:, m - 8:] @ w64[m - 8:]))
  if t > 1:
    res.Catch('fwd: token t + 1', Hit(torch.cat([s[1:], s[-1:]])))
  if w.dtype == _F32:
    res.Catch('fwd: gw rounded to bf16', Hit(x64 @ w.bfloat16().double()))
  res.Catch('fwd: logits rounded to bf16', Hit(s.float().bfloat16().double()))


@torch.no_grad()
def _CheckDx(res, x, w, dl, dres, dx):
  t, m = x.shape
  e = w.shape[1]
  if t == 0:
    assert dx.shape == (0, m)
    return
  w64, dl64 = w.double(), dl.double()
  rows = _Rows(t, m)
  hits = {'dres ignored': False, 'expert e + 1': False, 'truncating pack': False}
  trunc_over = 0
  roll = torch.roll(w64, -1, 1)
  for t0 in range(0, t, rows):
    d = dl64[t0:t0 + rows]
    ref = d @ w64.t()
    a = d.abs() @ w64.abs().t()
    if dres is not None:
      dr = dres[t0:t0 + rows].double()
      ref_nodres = ref
      ref = ref + dr
      a = a + dr.abs()
    y = dx[t0:t0 + rows].double()
    bound = 2 * (0.5 * _Ulp(torch.maximum(ref.abs(), y.abs())) + e * _U * a)
    _Assert(res, 'dx', y, ref, bound)
    err = (y - ref).abs()
    res.over += int((err > _ROUND_ULPS * _Ulp(ref)).sum())
    res.total += err.numel()
    trunc_over += int(((_Truncate(ref).double() - ref).abs() > _ROUND_ULPS * _Ulp(ref)).sum())
    if dres is not None:
      hits['dres ignored'] |= bool(((y - ref_nodres).abs() > bound).any())
    mut = d @ roll.t() + (ref - d @ w64.t())
    hits['expert e + 1'] |= bool(((y - mut).abs() > bound).any())
  if dres is not None:
    res.Catch('dx: dres ignored', hits['dres ignored'])
  res.Catch('dx: expert e + 1', hits['expert e + 1'])
  if t * m >= _ROUND_MIN:
    res.Catch('dx: truncating pack', trunc_over > _ROUND_FRAC * t * m)


@torch.no_grad()
def _CheckDgw(res, x, w, dl, dgw, sms):
  t, m = x.shape
  e = w.shape[1]
  if t == 0:
    assert bool((_Bits(dgw) == 0).all()), '%s: dgw of T = 0 is not +0' % res.what
    return
  _, tpb, used = _DgwPlan(t, sms)
  tp = used * tpb
  xs = F.pad(x.double(), (0, 0, 0, tp - t)).view(used, tpb, m)
  ds = F.pad(dl.double(), (0, 0, 0, tp - t)).view(used, tpb, e)
  part = torch.bmm(xs.transpose(1, 2), ds)                         # [used, M, E]
  ref = part.sum(0)
  p = torch.bmm(xs.abs().transpose(1, 2), ds.abs()).sum(0)
  chain = tpb + (used + 15) // 16 + 10
  y = dgw.double()
  if w.dtype == _F32:
    bound = _SECOND * chain * _U * p
  else:
    bound = 2 * (0.5 * _Ulp(torch.maximum(ref.abs(), y.abs())) + chain * _U * p)
  _Assert(res, 'dgw', y, ref, bound)
  def Hit(mut):
    return bool(((y - mut).abs() > bound).any())
  def Tok(i):
    return torch.outer(xs.view(tp, m)[i], ds.view(tp, e)[i])
  res.Catch('dgw: last partial dropped', Hit(ref - part[used - 1]))
  res.Catch('dgw: partial counted twice', Hit(ref + part[0]))
  res.Catch('dgw: block range shifted', Hit(ref - Tok(0) + (Tok(tpb) if tpb < t else 0)))
  s0 = (used - 1) * tpb
  last = s0 + (t - 1 - s0) // _DGW_TILE * _DGW_TILE
  tile = xs.view(tp, m)[last:t].t() @ ds.view(tp, e)[last:t]
  res.Catch('dgw: last tile dropped', Hit(ref - tile))


# ------------------------------------------------------------------- the runs ----
def _Gen(seed):
  return torch.Generator(device='cuda').manual_seed(seed)


def _Inputs(gen, t, m, e, wdtype, dres=True):
  x = torch.randn(t, m, device='cuda', generator=gen).to(_BF16)
  w = (torch.randn(m, e, device='cuda', generator=gen) * m**-0.5).to(wdtype)
  dl = torch.randn(t, e, device='cuda', generator=gen)
  dr = torch.randn(t, m, device='cuda', generator=gen).to(_BF16) if dres else None
  return x, w, dl, dr


@torch.no_grad()
def _RunCase(what, t, m, e, wdtype, seed, dres=True, repeat=1):
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  x, w, dl, dr = _Inputs(_Gen(seed), t, m, e, wdtype, dres)
  nat = ops.native()
  outs = []
  for _ in range(repeat):
    y = nat.gate_logits_fwd(x, w)
    dx, dgw = nat.gate_logits_bwd(x, w, dl, True, True, dr)
    outs.append((y, dx, dgw))
  for got in outs[1:]:
    for a, b, name in zip(outs[0], got, ('logits', 'dx', 'dgw')):
      assert torch.equal(_Bits(a), _Bits(b)), '%s: %s differs between calls' % (what, name)
  y, dx, dgw = outs[0]
  assert y.dtype == _F32 and dx.dtype == _BF16 and dgw.dtype == wdtype
  res = _Result(what)
  _CheckFwd(res, x, w, y)
  _CheckDx(res, x, w, dl, dr, dx)
  _CheckDgw(res, x, w, dl, dgw, sms)
  return res.Finish()


@pytest.mark.gpu
@pytest.mark.parametrize('wdtype', [_F32, _BF16], ids=['gw_f32', 'gw_bf16'])
def test_benchmark_site(wdtype):
  """MoELm8E's router: T = 8192, M = 2048, E = 8, three identical calls."""
  _RunCase('bench %s' % wdtype, 8192, 2048, 8, wdtype, 1, repeat=3)


@pytest.mark.gpu
@pytest.mark.parametrize('wdtype', [_F32, _BF16], ids=['gw_f32', 'gw_bf16'])
@pytest.mark.parametrize('e', _E_ALL)
def test_every_instantiation(e, wdtype):
  _RunCase('E=%d %s' % (e, wdtype), 1000, 1024, e, wdtype, 10 + e)


def _TokenSweep(sms):
  """name → T: around the fwd grid-stride threshold and past the dgw 3·SMs cap."""
  fwd_cap, dgw_cap = 2 * sms * _WARP_TOKENS, 3 * sms * _DGW_TILE
  cases = {'T%d' % t: t for t in (0, 1, 3, 4, 5, 31, 32, 33, 20000)}
  cases.update({'fwd_cap-3': fwd_cap - 3, 'fwd_cap': fwd_cap, 'fwd_cap+5': fwd_cap + 5,
                'dgw_cap+33': dgw_cap + 33, '2dgw_cap+17': 2 * dgw_cap + 17})
  return cases


_TOKEN_IDS = list(_TokenSweep(132))


@pytest.mark.gpu
@pytest.mark.parametrize('name', _TOKEN_IDS)
def test_token_sweep(name):
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  t = _TokenSweep(sms)[name]
  i = _TOKEN_IDS.index(name)
  _RunCase('T %s=%d' % (name, t), t, 264, 8, (_F32, _BF16)[i % 2], 100 + i, dres=i % 3 != 0)


_M_SWEEP = (8, 248, 256, 264, 2048, 2056, 4104)


@pytest.mark.gpu
@pytest.mark.parametrize('wdtype', [_F32, _BF16], ids=['gw_f32', 'gw_bf16'])
@pytest.mark.parametrize('m', _M_SWEEP)
def test_m_sweep(m, wdtype):
  _RunCase('M=%d %s' % (m, wdtype), 333, m, 4 if m > 4096 else 8, wdtype, 200 + m)


# (E, M): M·E·4 at the 48 KiB default, just above it, and at the 200 KiB cap for each E.
_SMEM_CASES = [(8, 1536), (8, 1544), (16, 3200), (8, 6400), (4, 12800), (2, 25600)]


@pytest.mark.gpu
@pytest.mark.parametrize('e,m', _SMEM_CASES, ids=['E%d_M%d' % c for c in _SMEM_CASES])
def test_shared_memory_edges(e, m):
  for wdtype in (_F32, _BF16):
    _RunCase('smem E=%d M=%d %s' % (e, m, wdtype), 300, m, e, wdtype, 300 + m)


@pytest.mark.gpu
def test_cases_reach_every_path():
  """Mirrors the host's dispatch: every fwd / dx (E, gw dtype) and dgw E, both folds, the
  opt-in shared memory, the forward's grid-stride loop, the dgw grid's 3·SMs cap, used <
  nblk, both halves of the fold's odd tail, and dgw grid.y > 1."""
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  cases = [(8192, 2048, 8, w) for w in (_F32, _BF16)]
  cases += [(1000, 1024, e, w) for e in _E_ALL for w in (_F32, _BF16)]
  cases += [(t, 264, 8, (_F32, _BF16)[i % 2]) for i, t in enumerate(_TokenSweep(sms).values())]
  cases += [(333, m, 4 if m > 4096 else 8, w) for m in _M_SWEEP for w in (_F32, _BF16)]
  cases += [(300, m, e, w) for e, m in _SMEM_CASES for w in (_F32, _BF16)]
  seen = set()
  for t, m, e, w in cases:
    assert gate.supported(torch.empty(1, m, device='cuda', dtype=_BF16),
                          torch.empty(m, e, device='cuda', dtype=w))
    seen.add(('fwd', e, w))
    seen.add(('dgw', e))
    seen.add(('fold', w))
    if m * e * 4 > _SMEM_DEFAULT:
      seen.add('opt-in smem')
    if m * e * 4 == _SMEM_CAP:
      seen.add(('smem cap', e))
    if t > _FwdGrid(t, sms) * _WARP_TOKENS:
      seen.add('fwd grid stride')
    if m > _DGW_COLS:
      seen.add('dgw grid.y > 1')
    if t:
      nblk, _, used = _DgwPlan(t, sms)
      if nblk == 3 * sms:
        seen.add('dgw 3·SMs cap')
      if used < nblk:
        seen.add('used < nblk')
      if 1 <= used % 16 <= 8:
        seen.add('fold tail 1..8')
      if used % 16 > 8:
        seen.add('fold tail 9..15')
  want = {('fwd', e, w) for e in _E_ALL for w in (_F32, _BF16)}
  want |= {('dgw', e) for e in _E_ALL} | {('fold', w) for w in (_F32, _BF16)}
  want |= {('smem cap', e) for e in _E_ALL}
  want |= {'opt-in smem', 'fwd grid stride', 'dgw grid.y > 1', 'dgw 3·SMs cap', 'used < nblk',
           'fold tail 1..8', 'fold tail 9..15'}
  assert seen >= want, sorted(map(str, want - seen))


# ---------------------------------------------------------------- the wrappers ----
@pytest.mark.gpu
def test_gate_logits_wrapper_3d():
  x, w, dl, _ = _Inputs(_Gen(400), 2 * 777, 512, 8, _BF16, dres=False)
  x3 = x.view(2, 777, 512).requires_grad_()
  w = w.requires_grad_()
  y = gate.gate_logits(x3, w)
  assert y.shape == (2, 777, 8)
  nat = ops.native()
  assert torch.equal(_Bits(y.view(-1, 8)), _Bits(nat.gate_logits_fwd(x, w.detach())))
  y.backward(dl.view(2, 777, 8))
  dx, dgw = nat.gate_logits_bwd(x, w.detach(), dl, True, True, None)
  assert x3.grad.shape == x3.shape
  assert torch.equal(_Bits(x3.grad.view(-1, 512)), _Bits(dx))
  assert torch.equal(_Bits(w.grad), _Bits(dgw))
  res = _Result('gate_logits 3-D')
  _CheckFwd(res, x, w.detach(), y.detach().view(-1, 8))
  _CheckDx(res, x, w.detach(), dl, None, x3.grad.view(-1, 512))
  _CheckDgw(res, x, w.detach(), dl, w.grad, torch.cuda.get_device_properties(0)
            .multi_processor_count)
  res.Finish()


@pytest.mark.gpu
@pytest.mark.parametrize('grads', ['dlogits', 'dpass', 'both', 'both_f32_dpass'])
def test_gate_logits_pass_wrapper(grads):
  """dpass alone comes back as dpass itself; with dlogits it is folded into the dx kernel
  (cast to bf16 first when it arrives in fp32), bit for bit a direct gate_logits_bwd."""
  t, m, e = 1000, 512, 8
  x, w, dl, dr = _Inputs(_Gen(401), t, m, e, _BF16)
  nat = ops.native()
  xg = x.clone().requires_grad_()
  wg = w.clone().requires_grad_()
  logits, xp = gate.gate_logits_pass(xg, wg)
  before = nat.launch_count()
  if grads == 'both_f32_dpass':
    # Autograd hands x_pass's gradient over in x's dtype; call backward with an fp32 one.
    dpass = dr.float() * 1.001
    ctx = type('Ctx', (), {})()
    ctx.saved_tensors, ctx.x_shape, ctx.needs_input_grad = (x, w), x.shape, (True, True)
    gx, gw = gate._GateLogitsPassFn.backward(ctx, dl, dpass)  # pylint: disable=protected-access
  else:
    dpass = dr
    outs, grads_in = [], []
    if grads != 'dpass':
      outs.append(logits)
      grads_in.append(dl)
    if grads != 'dlogits':
      outs.append(xp)
      grads_in.append(dpass)
    gx, gw = torch.autograd.grad(outs, [xg, wg], grads_in, allow_unused=True)
  launched = nat.launch_count() - before
  if grads == 'dpass':
    assert gw is None and launched == 0
    assert gx.data_ptr() == dpass.data_ptr() or torch.equal(_Bits(gx), _Bits(dpass))
    return
  assert launched == 3, 'dx, dgw partials and fold: %d launches' % launched
  dres = None if grads == 'dlogits' else dpass.to(_BF16)
  dx, dgw = nat.gate_logits_bwd(x, w, dl, True, True, dres)
  assert torch.equal(_Bits(gx), _Bits(dx)), 'wrapper dx differs from gate_logits_bwd'
  assert torch.equal(_Bits(gw), _Bits(dgw))
  res = _Result('gate_logits_pass %s' % grads)
  _CheckDx(res, x, w, dl, dres, gx)
  res.Finish()


@pytest.mark.gpu
@pytest.mark.parametrize('needs', [(True, False), (False, True), (True, True)],
                         ids=['dx', 'dgw', 'dx_dgw'])
@pytest.mark.parametrize('fn', ['gate_logits', 'gate_logits_pass'])
def test_needs_input_grad_launches_only_what_it_needs(fn, needs):
  t, m, e = 1000, 512, 8
  x, w, dl, _ = _Inputs(_Gen(402), t, m, e, _F32, dres=False)
  nat = ops.native()
  xg = x.clone().requires_grad_(needs[0])
  wg = w.clone().requires_grad_(needs[1])
  out = getattr(gate, fn)(xg, wg)
  logits = out[0] if fn == 'gate_logits_pass' else out
  before = nat.launch_count()
  logits.backward(dl)
  launched = nat.launch_count() - before
  assert launched == needs[0] + 2 * needs[1]          # dx: 1, dgw: partials + fold
  assert (xg.grad is not None) == needs[0] and (wg.grad is not None) == needs[1]
  dx, dgw = nat.gate_logits_bwd(x, w, dl, True, True, None)
  if needs[0]:
    assert torch.equal(_Bits(xg.grad), _Bits(dx))
  if needs[1]:
    assert torch.equal(_Bits(wg.grad), _Bits(dgw))


# -------------------------------------------------------------- argument checks ----
@pytest.mark.gpu
def test_bad_arguments_are_refused_without_launching():
  """x and dres are read with 16-byte loads; E must have an instantiation; gw must fit in
  200 KiB of shared memory; every operand must be on x's device."""
  gen = _Gen(500)
  t, m, e = 64, 256, 8
  x, w, dl, dr = _Inputs(gen, t, m, e, _F32)
  nat = ops.native()
  odd = torch.empty(t * m + 8, device='cuda', dtype=_BF16)
  x_odd = odd[1:1 + t * m].view(t, m)                # contiguous, 2 bytes off 16
  dr_odd = odd[3:3 + t * m].view(t, m)
  assert x_odd.is_contiguous() and x_odd.data_ptr() % 16
  x_odd.copy_(x)
  launches = nat.launch_count()
  with pytest.raises(RuntimeError, match='16-byte aligned'):
    nat.gate_logits_fwd(x_odd, w)
  with pytest.raises(RuntimeError, match='16-byte aligned'):
    nat.gate_logits_bwd(x_odd, w, dl, True, True, None)
  with pytest.raises(RuntimeError, match='16-byte aligned'):
    nat.gate_logits_bwd(x, w, dl, True, False, dr_odd)
  for bad_e in (1, 3, 6, 32):
    for tt in (t, 0):
      wb = torch.zeros(m, bad_e, device='cuda')
      with pytest.raises(RuntimeError, match='expert count'):
        nat.gate_logits_fwd(x[:tt], wb)
      with pytest.raises(RuntimeError, match='expert count'):
        nat.gate_logits_bwd(x[:tt], wb, torch.zeros(tt, bad_e, device='cuda'), True, True, None)
  for e2, m2 in ((16, 3208), (2, 25608)):
    xb = torch.zeros(4, m2, device='cuda', dtype=_BF16)
    with pytest.raises(RuntimeError, match='shared memory'):
      nat.gate_logits_fwd(xb, torch.zeros(m2, e2, device='cuda'))
    assert not gate.supported(xb, torch.zeros(m2, e2, device='cuda'))
  assert nat.launch_count() == launches
  # The wrappers take the matmul path for a misaligned x rather than raising.
  assert not gate.supported(x_odd, w)
  assert gate.supported(x, w)
  # A misaligned dpass is copied before it reaches the kernel.
  xg = x.clone().requires_grad_()
  logits, xp = gate.gate_logits_pass(xg, w)
  (gx,) = torch.autograd.grad([logits, xp], [xg], [dl, dr_odd])
  dx, _ = nat.gate_logits_bwd(x, w, dl, True, False, dr_odd.clone())
  assert torch.equal(_Bits(gx), _Bits(dx))


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_operands_on_another_device_are_refused_without_launching():
  x, w, dl, dr = _Inputs(_Gen(501), 64, 256, 8, _F32)
  other = torch.device('cuda', 1)
  nat = ops.native()
  launches = nat.launch_count()
  with pytest.raises(RuntimeError, match="x's device"):
    nat.gate_logits_fwd(x, w.to(other))
  with pytest.raises(RuntimeError, match="x's device"):
    nat.gate_logits_bwd(x, w, dl.to(other), True, True, None)
  with pytest.raises(RuntimeError, match="x's device"):
    nat.gate_logits_bwd(x, w, dl, True, True, dr.to(other))
  assert nat.launch_count() == launches
  assert not gate.supported(x, w.to(other))


# ------------------------------------------------------------ the bound on CPU ----
def _Fma(a, b, c):
  """fp32 fma from float64 (a·b is exact there for a bf16 a or b)."""
  return (a.double() * b.double() + c.double()).float()


def _FwdStandIn(x, w):
  """The forward's summation order in fp32: lane chains, then the xor butterfly."""
  t, m = x.shape
  e = w.shape[1]
  mp = -(-m // _WARP_COLS) * _WARP_COLS
  xs = F.pad(x.float(), (0, mp - m)).view(t, mp // _WARP_COLS, 32, 8)
  ws = F.pad(w.float(), (0, 0, 0, mp - m)).view(mp // _WARP_COLS, 32, 8, e)
  acc = torch.zeros(t, e, 32)
  for j in range(mp // _WARP_COLS):
    for i in range(8):
      acc = _Fma(xs[:, j, :, i].unsqueeze(1), ws[j, :, i].t().unsqueeze(0), acc)
  for o in (16, 8, 4, 2, 1):
    acc = acc[..., :o] + acc[..., o:2 * o]
  return acc[..., 0]


def _DxStandIn(w, dl, dres, pack=lambda v: v.to(_BF16)):
  t = dl.shape[0]
  o = dres.float() if dres is not None else torch.zeros(t, w.shape[0])
  for k in range(w.shape[1]):
    o = _Fma(dl[:, k:k + 1], w[:, k].float().unsqueeze(0), o)
  return pack(o)


def _DgwStandIn(x, dl, wdtype, sms):
  t, m = x.shape
  e = dl.shape[1]
  _, tpb, used = _DgwPlan(t, sms)
  part = torch.zeros(used, m, e)
  for b in range(used):
    for tok in range(b * tpb, min(t, (b + 1) * tpb)):
      part[b] = _Fma(x[tok].float().unsqueeze(1), dl[tok].unsqueeze(0), part[b])
  red = []
  for ky in range(8):
    s0, s1 = torch.zeros(m, e), torch.zeros(m, e)
    k = ky
    while k + 8 < used:
      s0, s1 = s0 + part[k], s1 + part[k + 8]
      k += 16
    if k < used:
      s0 = s0 + part[k]
    red.append(s0 + s1)
  s = torch.zeros(m, e)
  for r in red:
    s = s + r
  return s.to(wdtype)


@pytest.mark.parametrize('t,m,e,sms', [(300, 264, 4, 3), (1000, 256, 8, 2), (37, 512, 16, 1)])
def test_bound_and_controls_on_cpu(t, m, e, sms):
  """The bounds, controls and rounding check with fp32 emulations of the kernels' order in
  their place (`sms` small, so the dgw split has several ranges and a ragged fold tail).
  gw rounded to bf16 and bf16 logits fail the forward bound; a truncating dx pack fails
  the rounding check."""
  gen = torch.Generator().manual_seed(t + m + e)
  for wdtype in (_F32, _BF16):
    x = torch.randn(t, m, generator=gen).to(_BF16)
    w = (torch.randn(m, e, generator=gen) * m**-0.5).to(wdtype)
    dl = torch.randn(t, e, generator=gen)
    dr = torch.randn(t, m, generator=gen).to(_BF16)
    res = _Result('cpu %s' % wdtype)
    y = _FwdStandIn(x, w)
    _CheckFwd(res, x, w, y)
    _CheckDx(res, x, w, dl, dr, _DxStandIn(w, dl, dr))
    _CheckDgw(res, x, w, dl, _DgwStandIn(x, dl, wdtype, sms), sms)
    res.Finish()
    defects = {'logits rounded to bf16': (y.bfloat16().float(), None),
               'truncating dx pack': (None, _DxStandIn(w, dl, dr, _Truncate))}
    if wdtype == _F32:
      defects['gw rounded to bf16'] = (_FwdStandIn(x, w.bfloat16()), None)
    for name, (yb, dxb) in defects.items():
      bad = _Result('cpu %s' % name)
      with pytest.raises(AssertionError, match='outside the bound|not rounded to nearest'):
        if yb is not None:
          _CheckFwd(bad, x, w, yb)
        else:
          _CheckDx(bad, x, w, dl, dr, dxb)
          bad.Finish()
