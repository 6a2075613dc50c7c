"""The fused MoE exchange (parallel/symm.py: `MoeExchange`, `_MoeFn`) at expert parallelism
ep = 2, 3, 4 and 8, with the ranks simulated on one GPU: bit for bit against the single-rank
exchange, and against a float64 oracle of the expert-parallel MoE FFN.

Contract. Rank r of ep holds the groups [r·G_l, (r+1)·G_l) of the global batch of G = ep·G_l
groups and the experts [r·E_l, (r+1)·E_l) of E = ep·E_l. Its forward `Apply` returns y and aux
of its own tokens. Its gate kernel stores each kept token row into the owner's expert buffer
`xe` [E_l, G·C, M] at row (e_l, g_global, c), the slot convention of parallel/ep.py; the
second expert GEMM's row-pointer epilogue stores each output row back into the source rank's
`yc` [E, G_l·C, M] at row (e·G_l + g_local)·C + c. Backward mirrors that: `dy` scaled by the
gate into the owners' `dye`, and `dxc` rows back to the sources. The semantics are those of
`ExpertParallel.ScaleExpertGrad`: rank r's loss is L_r = ⟨y_r, dy_r⟩ + 0.01·aux_r, with aux_r
taken over its own G_l groups, and rank d's expert-weight gradient is (1/ep)·Σ_r ∂L_r/∂w_d,
the sum over every rank's tokens reaching its experts, scaled by the wgrad epilogue's
`row_scale` (`WgradScale`).

How the ranks are simulated. A `SymmArena` subclass gives each rank a plain device buffer as
its slab, and every rank's peer table holds every slab's address, so the kernels' peer stores
are ordinary stores into another buffer of the same process; no `dist`, no CUDA IPC. Each
rank is a real `MoeExchange` with its own rank id; its arena and layer buffers are built on
the main thread before any rank runs. Each rank then runs forward and backward in its own
Python thread. Backward calls the rank's `_MoeFn` node directly (`y.grad_fn.apply(dy)`): the
autograd engine runs every CUDA backward node on one device thread, so two engine-driven
backwards would queue behind each other and the first would wait for the second forever.
`dlogits` then comes from the recorded gate on the main thread.

`_Sync` is replaced by a host step: `torch.cuda.synchronize()`, then a `threading.Barrier`
wait with a timeout. `moe_sync` itself is never launched: it spin-waits on flags, and two
spinning kernels of simulated ranks on one GPU can each wait for the other forever. The
native entry is wrapped to raise, so a call would fail the test instead. A harness mistake
ends in a `BrokenBarrierError`, not a stuck process. The flag protocol and real NVLink stores
need two GPUs; tests/test_multi_gpu.py checks them.

Every rank's `xe`, `yc`, `dye` and `dxc` (and those of the single-rank run) are filled with a
bf16 NaN before each run, so a row nobody wrote fails.

a. Bit for bit against `MoeExchange(None, E)` run on all G groups with the same logits and the
concatenated expert weights. Routing is per group and capacity per (expert, group), the row
order (g_global, c) of an expert's buffer is the same, every GEMM has the same rows per group
and the same K, and none splits K. So for rank r: index, pos and keep of its groups; y, the
exchange's dx and dgate; `xe` and `dye` of local expert e_l equal the single run's expert
r·E_l + e_l; `yc` and `dxc` viewed [E, G_l, C, M] equal the single run's viewed
[E, ep, G_l, C, M] at [:, r]. dwi and dwo equal 1/ep times the single run's rows of its
experts bit for bit when ep is a power of two: `row_scale` multiplies the fp32 sum by an exact
power of two before the one bf16 rounding. For ep = 3 the two results are two different
roundings of the same fp32 sum S: |dw − dw₁/3| ≤ ½ ulp(dw) + ⅓·½ ulp(dw₁) + 3u·|dw₁/3|
(u = 2^-24, for the fp32 1/3 and the fp32 product). That can reach 7/6 ulp where S/3 falls a
binade below S, so "within one ulp" would not be a bound; the measured worst is below.
The tile width `UseBn256` picks for each GEMM is printed for both runs: the GEMMs see E_l groups
of G·C rows on a rank and E groups on the single run, so the widths can differ.

b. Against float64, with the oracle, bounds and controls of tests/test_moe_exchange_float64_gpu.py
(imported, not copied). Routing through its `_CheckRouting` on every rank. End to end: y, dx,
dlogits and aux of rank r from the oracle on rank r's groups; dwi and dwo of rank d are
(1/ep)·Σ_r of the per-rank oracle gradients, which is the oracle on all groups since the rows
partition by rank, with the bound 3u₈·(A/ep + |dw|) (A the abs-value evaluation summed over
ranks) plus 2u·|dw| where ep is not a power of two. Stages on every rank, through the
buffers: `xe` rows bitwise, from the right source rank's tokens; h, dh, dwo and dwi within the
GEMM bound of tests/test_gemm_float64_gpu.py, the wgrads with a 1/ep row scale the test builds
itself; `yc` and `dxc` within the GEMM bound at the combine layout on the source rank, from the
owners' h and dh rows of that rank; `dye` bitwise bf16(gate·dy).

c. Controls. Two real runs must fail both a and b: every rank with `loopback` (the same stores,
all into the rank's own slab), and rank 0's `row_ptrs_yc` built as if it were rank 1. The
mutated oracles of `_AssertControlsFail` must each put an element above its bound on every rank
of bench_ep8 and skewed_ep4. No rank of bench_ep8 overflows a first choice whose second choice
is kept, so "second dgate dropped" has no token to hit there and four apply (as in the ep = 1
module's bench case); skewed_ep4 rejects all five.

d. Buffer lifetime at ep = 4: forward A, forward B, backward B, backward A is bitwise equal to
each layer run alone; the layers share every rank's `dye` and `dxc`.

e. Without a GPU: for simulated worlds at ep = 2, 3 and 8, every rank's `peer_xe`, `peer_dye`,
`row_ptrs_yc` and `row_ptrs_dxc` (and their loopback forms) hold the address of the row the
slot convention names in the right rank's slab, taken from that slab's own tensor views.

Cases (C = `ExpertCapacity(S, E, 0, factor)`; inputs from the ep = 1 module's `_Inputs` on
all G groups; weight init Uniform(√(3/M)) and Uniform(√(3/H)), logits x·gw):

    case        ep  E (E_l)  G_l  S     M     H     factor  gates
    bench_ep2   2   8 (4)    8    1024  2048  8192  2.0     legacy             2-GPU benchmark
    bench_ep8   8   8 (1)    8    1024  2048  8192  2.0     legacy             8-GPU benchmark;
                                                                               wgrad K = 16384
    skewed_ep4  4   8 (2)    8    1024  2048  8192  2.0     legacy, skewed     both overflow
    padded_ep4  4   16 (4)   3    1000  1024  2048  2.0     renorm, padded     last rank's last
                                                                               group all padding
    many_ep8    8   32 (4)   2    4096  512   1024  2.0     renorm             > 48 KiB smem gate
    ragged_ep3  3   12 (4)   5    77    328   264   0.5     legacy             1/3; ragged dims

Measured on an H100 80GB HBM3 (700 W limit, 1980 MHz max SM clock), seeded so these repeat.
Check a held bit for bit on every rank of every case; ragged_ep3's dw, the one comparison
that is not bitwise, reaches 0.857 of its two-roundings bound. The kernels' choices matched
the float64 ranking on every token. `UseBn256` picked 256-wide tiles for every GEMM of the
single runs (128 at ragged_ep3) but 128 for the ranks' yc and dxc GEMMs at padded_ep4 and for
their wgrads at many_ep8; those outputs are bitwise equal all the same, since the tile width
changes which CTA computes an element, not the order of its accumulation. Worst err/bound of
check b per case, stages then end to end:

                h     yc    dh    dwo   dwi   dxc      y     dx    dlogits aux   dwi   dwo
    bench_ep2   0.484 0.406 0.485 0.467 0.478 0.431    0.042 0.002 0.110   0.004 0.018 0.059
    bench_ep8   0.484 0.405 0.486 0.371 0.378 0.439    0.045 0.003 0.130   0.005 0.008 0.030
    skewed_ep4  0.484 0.405 0.483 0.467 0.465 0.431    0.050 0.004 0.134   0.006 0.034 0.077
    padded_ep4  0.493 0.485 0.493 0.493 0.494 0.488    0.070 0.003 0.128   0.007 0.023 0.108
    many_ep8    0.497 0.494 0.497 0.471 0.475 0.495    0.104 0.028 0.218   0.012 0.030 0.053
    ragged_ep3  0.496 0.498 0.497 0.499 0.499 0.498    0.170 0.008 0.307   0.006 0.034 0.277

The stage ratios sit near ½, the final bf16 rounding, as in the ep = 1 module; the wgrads of
bench_ep8 (K = 16384) sit lower because the accumulation term of the bound grows with K. Both
controls fail check a at rank 0's y and check b at rank 0's xe (loopback: rows never written)
or yc (the shifted row table: rows never written, so non-finite). The whole module takes ~45 s
on the H100.
"""
import gc
import threading
import types

import pytest
import torch

from lingvo_b200.core import gshard_layers
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.ops import gemm
from lingvo_b200.parallel import symm

import test_gemm_float64_gpu as gemm64
import test_moe_exchange_float64_gpu as moe64
import test_moe_routing_gpu as routing

_BARRIER_TIMEOUT = 300.0        # seconds a rank waits for the others at a phase boundary

# name, ep, E, G_l, S, M, H, capacity factor, legacy, padded, skewed
CASES = [
    ('bench_ep2', 2, 8, 8, 1024, 2048, 8192, 2.0, True, False, False),
    ('bench_ep8', 8, 8, 8, 1024, 2048, 8192, 2.0, True, False, False),
    ('skewed_ep4', 4, 8, 8, 1024, 2048, 8192, 2.0, True, False, True),
    ('padded_ep4', 4, 16, 3, 1000, 1024, 2048, 2.0, False, True, False),
    ('many_ep8', 8, 32, 2, 4096, 512, 1024, 2.0, False, False, False),
    ('ragged_ep3', 3, 12, 5, 77, 328, 264, 0.5, True, False, False),
]
_MUTATION_CASES = {'bench_ep8': 4, 'skewed_ep4': 5}    # case → mutations that must apply
_CONTROL_CASES = ('padded_ep4', 'ragged_ep3')
_CASE = {cs[0]: cs for cs in CASES}


# ------------------------------------------------------------ the simulated world ----
class _World:
  """ep simulated ranks of one process: their slabs and the barrier of their lockstep."""

  def __init__(self, ep):
    self.ep = ep
    self.slabs = None
    self.barrier = threading.Barrier(ep, timeout=_BARRIER_TIMEOUT)


class _SimArena(symm.SymmArena):
  """The symmetric arena of a simulated rank: every rank's slab is a device buffer of this
  process, so a peer's address is an ordinary pointer. No `dist`, no IPC, no native call."""

  def __init__(self, nbytes, device, group):
    if group is None:                   # the single-rank exchange: a plain local slab
      super().__init__(nbytes, device, group)
      return
    world = group.world
    if world.slabs is None:
      world.slabs = [torch.zeros(int(nbytes), dtype=torch.uint8, device=device)
                     for _ in range(world.ep)]
    assert all(s.numel() == nbytes for s in world.slabs), (
        'rank %d asks for %d arena bytes, rank 0 for %d' % (group.rank, nbytes,
                                                             world.slabs[0].numel()))
    self.device, self.group, self.nbytes = device, group, int(nbytes)
    self.world, self.rank = world.ep, group.rank
    self._slab = world.slabs[group.rank]
    self.peer_base = [s.data_ptr() for s in world.slabs]
    self._off = 0


def _LockstepSync(self, bufs, phase):
  """Stands in for `MoeExchange._Sync`: once every rank's work so far has finished on the
  device, every peer store of the phase has landed."""
  if self.ep == 1:
    return
  torch.cuda.synchronize(self.device)
  self.group.world.barrier.wait()


def _NoMoeSync(*args, **kw):
  raise AssertionError('moe_sync launched with simulated ranks')


@pytest.fixture
def sim_world(monkeypatch):
  monkeypatch.setattr(symm, 'SymmArena', _SimArena)
  monkeypatch.setattr(symm.dist, 'barrier', lambda *a, **k: None)
  monkeypatch.setattr(symm.MoeExchange, '_Sync', _LockstepSync)
  yield
  gc.collect()
  if torch.cuda.is_available():
    torch.cuda.empty_cache()


@pytest.fixture
def gpu_world(sim_world, monkeypatch):
  from lingvo_b200 import ops
  monkeypatch.setattr(ops.native(), 'moe_sync', _NoMoeSync)
  yield


def _Ranks(ep, e, device, keys, g_l, s, c, m):
  """ep `MoeExchange`s of one simulated world, with the layer buffers of `keys` built."""
  world = _World(ep)
  ranks = []
  for r in range(ep):
    engine = types.SimpleNamespace(ep_size=ep, ep_rank=r, num_experts=e,
                                   group=types.SimpleNamespace(world=world, rank=r))
    ranks.append(symm.MoeExchange(engine, device=device))
  for key in keys:
    for ex in ranks:
      ex._Bufs(key, g_l, s, c, m)
  return world, ranks


_THREAD = threading.local()


def _InRanks(world, fn):
  """fn(r) for every rank r, each in its own thread → [result of rank r]. Re-raises the first
  failure; a failing rank breaks the barrier so that the others stop too."""
  out, err = [None] * world.ep, [None] * world.ep

  def Body(r):
    _THREAD.rank = r
    try:
      out[r] = fn(r)
    except BaseException as e:
      err[r] = e
      world.barrier.abort()
  threads = [threading.Thread(target=Body, args=(r,), name='rank%d' % r)
             for r in range(world.ep)]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  failed = [e for e in err if e is not None]
  if failed:
    root = [e for e in failed if not isinstance(e, threading.BrokenBarrierError)]
    raise (root or failed)[0]
  return out


class _RankSpy:
  """Records, per rank thread, the exchange's GEMM outputs with the tile width the kernel
  picks for each, and the `_MoeFn` inputs (the gate with its graph, the routing, the
  buffers)."""

  def __init__(self, monkeypatch, device):
    self.gemms, self.widths, self.calls = {}, {}, {}
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    real_gemm, real_apply = gemm.gemm, symm._MoeFn.apply

    def Gemm(a, b, a_kmajor=True, b_kmajor=True, *rest, **kw):
      out = real_gemm(a, b, a_kmajor, b_kmajor, *rest, **kw)
      who = getattr(_THREAD, 'rank', None)
      ng = a.shape[0] if a.dim() == 3 else 1
      m = a.shape[-2] if a_kmajor else a.shape[-1]
      n = b.shape[-2] if b_kmajor else b.shape[-1]
      self.gemms.setdefault(who, []).append(out)
      self.widths.setdefault(who, []).append(256 if gemm64._Bn256(ng, m, n, sms) else 128)
      return out

    def Apply(x2d, gate, *rest):
      self.calls.setdefault(getattr(_THREAD, 'rank', None), []).append(
          NestedMap(gate=gate, g=rest[4], bufs=rest[3]))
      return real_apply(x2d, gate, *rest)
    monkeypatch.setattr(gemm, 'gemm', Gemm)
    monkeypatch.setattr(symm._MoeFn, 'apply', staticmethod(Apply))


# ------------------------------------------------------------------------ runs ----
def _Shard(inp, r, g_l, s, e_l):
  gs, ts, es = (slice(r * g_l, (r + 1) * g_l), slice(r * g_l * s, (r + 1) * g_l * s),
                slice(r * e_l, (r + 1) * e_l))
  return NestedMap(x=inp.x[ts], logits=inp.logits[gs], wi=inp.wi[es], wo=inp.wo[es],
                   dy=inp.dy[ts], pad=None if inp.pad is None else inp.pad[gs].contiguous())


def _Forward(ex, key, sh, c, legacy, spy):
  lv = moe64._Leaves(sh)
  lv.y, lv.aux = ex.Apply(key, lv.x, lv.logits, sh.pad, c, legacy, lv.wi, lv.wo)
  lv.rec = spy.calls[getattr(_THREAD, 'rank', None)][-1]
  return lv


def _Backward(lv, dy):
  """The backward of the rank's `_MoeFn` node, called in the rank's thread."""
  dx, dgate, dwi, dwo = lv.y.grad_fn.apply(dy)[:4]
  return NestedMap(dx=dx, dgate=dgate, dwi=dwi, dwo=dwo)


def _Result(ex, lv, grads, with_dlogits):
  bufs, g = lv.rec.bufs, lv.rec.g
  res = NestedMap(y=lv.y.detach(), aux=lv.aux.detach(), gate=lv.rec.gate.detach(),
                  index=g.index, pos=g.pos, keep=g.keep, xe=bufs.xe, yc=bufs.yc, dye=ex.dye,
                  dxc=ex.dxc, **grads)
  if with_dlogits:
    res.dlogits, = torch.autograd.grad(
        [lv.rec.gate, lv.aux], lv.logits,
        [grads.dgate, torch.tensor(moe64._AUX_COEF, device=lv.aux.device)])
  return res


def _Sentinels(ranks, key):
  for ex in ranks:
    moe64._Sentinel(ex._layers[key].xe, ex._layers[key].yc, ex.dye, ex.dxc)


def _RunWorld(world, ranks, key, inp, c, legacy, spy, g_l, s):
  """Forward then backward of one layer on every rank → per-rank results."""
  ep, e_l = len(ranks), ranks[0].e_local
  shards = [_Shard(inp, r, g_l, s, e_l) for r in range(ep)]
  for r in range(ep):
    spy.gemms.pop(r, None)
    spy.widths.pop(r, None)
  fwd = _InRanks(world, lambda r: _Forward(ranks[r], key, shards[r], c, legacy, spy))
  bwd = _InRanks(world, lambda r: _Backward(fwd[r], shards[r].dy))
  outs = []
  for r in range(ep):
    o = _Result(ranks[r], fwd[r], bwd[r], True)
    assert len(spy.gemms[r]) == 6, len(spy.gemms[r])
    o.h, o.dh, o.widths = spy.gemms[r][0], spy.gemms[r][2], spy.widths[r]
    outs.append(o)
  return outs


def _RunSingle(e, device, key, inp, c, legacy, spy, g, s, m):
  ex = symm.MoeExchange(None, e, device)
  bufs = ex._Bufs(key, g, s, c, m)
  moe64._Sentinel(bufs.xe, bufs.yc, ex.dye, ex.dxc)
  _THREAD.rank = 'single'
  try:
    lv = _Forward(ex, key, inp, c, legacy, spy)
    out = _Result(ex, lv, _Backward(lv, inp.dy), False)
  finally:
    del _THREAD.rank
  out.widths = spy.widths.pop('single')
  spy.gemms.pop('single')
  return out


# ------------------------------------------------------------ a: the ep = 1 run ----
def _SameBits(what, got, want):
  it = {torch.bfloat16: torch.int16, torch.float32: torch.int32}[got.dtype]
  assert got.dtype == want.dtype and got.shape == want.shape, (
      what, got.dtype, want.dtype, tuple(got.shape), tuple(want.shape))
  bad = got.contiguous().view(it) != want.contiguous().view(it)
  n = int(bad.sum())
  if n:
    flat = int(bad.reshape(-1).to(torch.int8).argmax())
    first, rest = [], flat
    for d in reversed(got.shape):
      first.append(rest % d)
      rest //= d
    first = tuple(reversed(first))
    raise AssertionError('%s: %d of %d differ; first at %s: got %r, want %r' % (
        what, n, bad.numel(), first, float(got[first]), float(want[first])))


@torch.no_grad()
def _CheckAgainstSingle(outs, single, e_l, g_l, s, c, m):
  """Check a of the module docstring → the worst ratio of dw to its two-roundings bound
  (0 when ep is a power of two, where dw is compared bitwise)."""
  ep = len(outs)
  e = ep * e_l
  worst = 0.0
  for r, o in enumerate(outs):
    gs, ts, es = (slice(r * g_l, (r + 1) * g_l), slice(r * g_l * s, (r + 1) * g_l * s),
                  slice(r * e_l, (r + 1) * e_l))
    what = 'rank %d' % r
    for k in ('index', 'pos', 'keep'):
      routing._AssertEqual('%s %s' % (what, k), o[k], single[k][:, gs])
    _SameBits(what + ' y', o.y, single.y[ts])
    _SameBits(what + ' dx', o.dx, single.dx[ts])
    _SameBits(what + ' dgate', o.dgate, single.dgate[:, ts])
    _SameBits(what + ' xe', o.xe, single.xe[es])
    _SameBits(what + ' dye', o.dye, single.dye[es])
    _SameBits(what + ' yc', o.yc.view(e, g_l, c, m), single.yc.view(e, ep, g_l, c, m)[:, r])
    _SameBits(what + ' dxc', o.dxc.view(e, g_l, c, m), single.dxc.view(e, ep, g_l, c, m)[:, r])
    for k in ('dwi', 'dwo'):
      one = single[k][es]
      if ep & (ep - 1) == 0:
        _SameBits('%s %s' % (what, k), o[k], (one.float() / ep).bfloat16())
        continue
      got, one = o[k].double(), one.double()
      ref = one / ep
      bound = 0.5 * gemm64._Ulp(got) + 0.5 * gemm64._Ulp(one) / ep + 3 * gemm64._U * ref.abs()
      ratio = moe64._Ratio((got - ref).abs(), bound)
      assert bool(torch.isfinite(got).all()), '%s %s: non-finite' % (what, k)
      worst = max(worst, float(ratio.max()))
      assert worst <= 1.0, '%s %s: worst err/bound %g against 1/%d of the single run' % (
          what, k, worst, ep)
  return worst


# -------------------------------------------------------------- b: float64 ----
@torch.no_grad()
def _StageChecks(inp, outs, e_l, g_l, s, c, m, h):
  """The stage checks of b on every rank → worst err/bound per stage."""
  from lingvo_b200.ops import gemm as G
  ep = len(outs)
  e, g = ep * e_l, ep * g_l
  index = torch.cat([o.index for o in outs], 1).cpu()
  pos = torch.cat([o.pos for o in outs], 1).cpu()
  keep = torch.cat([o.keep for o in outs], 1).cpu()
  gate = torch.cat([o.gate.view(2, g_l, s) for o in outs], 1)
  token, choice = routing.ExpectedSlots(index, pos, keep, e, c)
  res = {}

  def Worst(name, v):
    res[name] = max(res.get(name, 0.0), v)
  for d, o in enumerate(outs):
    es = slice(d * e_l, (d + 1) * e_l)
    what = 'rank %d' % d
    routing._AssertRowsBitwise(what + ' xe', o.xe.view(e_l, g, c, m),
                               routing._ExpectedRows(inp.x, token[es]))
    routing._AssertRowsBitwise(what + ' dye', o.dye.view(e_l, g, c, m),
                               routing._ExpectedRows(inp.dy, token[es], choice[es], gate))
    wi, wo = inp.wi[es], inp.wo[es]
    Worst('h', gemm64._Check(o.h, o.xe, wi, True, False, act=1, what=what + ' h')[0])
    Worst('dh', gemm64._Check(o.dh, o.dye, wo, True, True, aux=o.h, aux_mode=G.AUX_RELU_MASK,
                              what=what + ' dh')[0])
    scale = 1.0 / ep
    rs_h = torch.full((e_l, h), scale, dtype=torch.float32, device=o.h.device)
    rs_m = torch.full((e_l, m), scale, dtype=torch.float32, device=o.h.device)
    Worst('dwo', gemm64._Check(o.dwo, o.h, o.dye, False, False, rs=rs_h, what=what + ' dwo')[0])
    Worst('dwi', gemm64._Check(o.dwi, o.xe, o.dh, False, False, rs=rs_m, what=what + ' dwi')[0])
  for r, o in enumerate(outs):
    what = 'rank %d' % r
    # The owners' rows of rank r's tokens, in the combine layout [E, G_l·C, ·].
    h_r = torch.cat([q.h.view(e_l, ep, g_l * c, h)[:, r] for q in outs])
    Worst('yc', gemm64._Check(o.yc, h_r, inp.wo, True, False, what=what + ' yc')[0])
    del h_r
    dh_r = torch.cat([q.dh.view(e_l, ep, g_l * c, h)[:, r] for q in outs])
    Worst('dxc', gemm64._Check(o.dxc, dh_r, inp.wi, True, True, what=what + ' dxc')[0])
    del dh_r
  return res


@torch.no_grad()
def _EndToEndWgrads(acc, outs, e_l):
  """dwi and dwo of every rank against 1/ep of the oracle's gradient over all ranks' tokens."""
  ep = len(outs)
  res = {}
  for k in ('dwi', 'dwo'):
    worst = 0.0
    for d, o in enumerate(outs):
      es = slice(d * e_l, (d + 1) * e_l)
      ref = acc[k][es] / ep
      bound = 3 * moe64._U8 * (acc['a_' + k][es] / ep + ref.abs())
      if ep & (ep - 1):
        bound = bound + 2 * gemm64._U * ref.abs()
      v = o[k].double()
      assert bool(torch.isfinite(v).all()), 'rank %d %s: non-finite' % (d, k)
      r = moe64._Ratio((v - ref).abs(), bound)
      assert float(r.max()) <= 1.0, 'rank %d %s: %d elements outside the bound, worst %g' % (
          d, k, int((r > 1).sum()), float(r.max()))
      worst = max(worst, float(r.max()))
    res[k] = worst
  return res


def _CheckFloat64(name, inp, outs, e_l, g_l, s, c, m, h, legacy, mutations=None):
  """Check b of the module docstring → (stage ratios, end-to-end ratios, tokens ranked
  differently from float64, mutations rejected)."""
  stages = _StageChecks(inp, outs, e_l, g_l, s, c, m, h)
  ends, acc, differ, rejected = {}, None, 0, 0
  for r, o in enumerate(outs):
    what = '%s rank %d' % (name, r)
    sh = _Shard(inp, r, g_l, s, e_l)
    nonpad = moe64._NonPad(sh)
    differ += moe64._CheckRouting(o.index, o.pos, o.keep, sh.logits, nonpad, c, what)
    orc = moe64._Oracle(sh.x, sh.logits, inp.wi, inp.wo, sh.dy, nonpad, o.index, legacy, c)
    moe64._DLogitsBound(orc, o.yc, sh.dy)
    got = NestedMap(y=o.y, dx=o.dx, dlogits=o.dlogits, aux=o.aux)
    for k, v in moe64._EndToEnd(orc, got, what, ('y', 'dx', 'dlogits', 'aux')).items():
      ends[k] = max(ends.get(k, 0.0), v)
    if mutations is not None:
      n = moe64._AssertControlsFail(orc, got, what)
      rejected = max(rejected, n)
    if acc is None:
      acc = NestedMap(dwi=orc.dwi, dwo=orc.dwo, a_dwi=orc.a_dwi, a_dwo=orc.a_dwo)
    else:
      for k in acc:
        acc[k].add_(orc[k])
    del orc
  ends.update(_EndToEndWgrads(acc, outs, e_l))
  if mutations is not None:
    assert rejected >= mutations, '%s: %d mutated oracles applied, want %d' % (
        name, rejected, mutations)
  return stages, ends, differ, rejected


# ------------------------------------------------------------------------ GPU ----
def _Setup(case, monkeypatch):
  name, ep, e, g_l, s, m, h, factor, legacy, padded, skewed = case
  dev = torch.device('cuda', torch.cuda.current_device())
  c = gshard_layers.ExpertCapacity(s, e, 0, factor)
  inp = moe64._Inputs(ep * g_l, s, m, h, e, skewed, padded, dev, 1000 + ep * g_l * s + e)
  spy = _RankSpy(monkeypatch, dev)
  return dev, c, inp, spy


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[cs[0] for cs in CASES])
def test_expert_parallel_exchange(case, gpu_world, monkeypatch):
  name, ep, e, g_l, s, m, h, _, legacy, _, _ = case
  e_l = e // ep
  dev, c, inp, spy = _Setup(case, monkeypatch)
  world, ranks = _Ranks(ep, e, dev, [name], g_l, s, c, m)
  _Sentinels(ranks, name)
  outs = _RunWorld(world, ranks, name, inp, c, legacy, spy, g_l, s)
  single = _RunSingle(e, dev, name, inp, c, legacy, spy, ep * g_l, s, m)
  widths = sorted({tuple(o.widths) for o in outs})
  print('%s tile widths (h, yc, dh, dwo, dwi, dxc): single %s, ranks %s' % (
      name, single.widths, widths))
  dw_ulp = _CheckAgainstSingle(outs, single, e_l, g_l, s, c, m)
  del single
  gc.collect()
  torch.cuda.empty_cache()
  stages, ends, differ, rejected = _CheckFloat64(
      name, inp, outs, e_l, g_l, s, c, m, h, legacy, _MUTATION_CASES.get(name))
  print('%s: bitwise equal to the single-rank exchange%s; %d tokens ranked differently '
        'from float64' % (name, '' if not dw_ulp else
                          ' (dw within %.3f of its two-roundings bound)' % dw_ulp, differ))
  print('%s stages: %s' % (name, ' '.join('%s %.3f' % kv for kv in stages.items())))
  print('%s end to end: %s' % (name, ' '.join('%s %.3f' % kv for kv in ends.items())))
  if rejected:
    print('%s: all %d mutated oracles rejected on every rank' % (name, rejected))


def _Refused(check):
  """Runs a check that must fail → its message."""
  with pytest.raises(AssertionError) as info:
    check()
  return str(info.value).splitlines()[0]


@pytest.mark.gpu
@pytest.mark.parametrize('control', ['loopback', 'row table of rank 1'])
@pytest.mark.parametrize('name', _CONTROL_CASES)
def test_controls_fail_both_checks(name, control, gpu_world, monkeypatch):
  """Real runs with a wrong peer address must fail checks a and b."""
  case = _CASE[name]
  _, ep, e, g_l, s, m, h, _, legacy, _, _ = case
  e_l = e // ep
  dev, c, inp, spy = _Setup(case, monkeypatch)
  world, ranks = _Ranks(ep, e, dev, [name], g_l, s, c, m)
  if control == 'loopback':
    for ex in ranks:
      ex.loopback = True
  else:
    ex = ranks[0]
    bufs = ex._layers[name]
    ex.rank = 1
    try:
      bufs._row_ptrs_yc[False] = ex.RowPtrTable(bufs.yc_off, g_l, c, m)
    finally:
      ex.rank = 0
  _Sentinels(ranks, name)
  outs = _RunWorld(world, ranks, name, inp, c, legacy, spy, g_l, s)
  single = _RunSingle(e, dev, name, inp, c, legacy, spy, ep * g_l, s, m)
  a = _Refused(lambda: _CheckAgainstSingle(outs, single, e_l, g_l, s, c, m))
  b = _Refused(lambda: _CheckFloat64(name, inp, outs, e_l, g_l, s, c, m, h, legacy))
  print('%s, %s: check a rejects it (%s); check b rejects it (%s)' % (name, control, a, b))


_LIFE_EP = 4


@pytest.mark.gpu
def test_two_layers_interleaved_match_running_each_alone(gpu_world, monkeypatch):
  """Forward A, forward B, backward B, backward A on four ranks equals each layer alone."""
  g_l, s, m, h, e, factor = moe64._LIFE
  ep = _LIFE_EP
  dev = torch.device('cuda', torch.cuda.current_device())
  c = gshard_layers.ExpertCapacity(s, e, 0, factor)
  inp = {k: moe64._Inputs(ep * g_l, s, m, h, e, False, False, dev, seed)
         for k, seed in (('A', 1), ('B', 2))}
  spy = _RankSpy(monkeypatch, dev)
  world, ranks = _Ranks(ep, e, dev, ['A', 'B'], g_l, s, c, m)
  shards = {k: [_Shard(v, r, g_l, s, e // ep) for r in range(ep)] for k, v in inp.items()}

  def Fwd(k):
    return _InRanks(world, lambda r: _Forward(ranks[r], k, shards[k][r], c, True, spy))

  def Bwd(k, fwd):
    grads = _InRanks(world, lambda r: _Backward(fwd[r], shards[k][r].dy))
    return [NestedMap(y=f.y, **g) for f, g in zip(fwd, grads)]
  _Sentinels(ranks, 'A')
  _Sentinels(ranks, 'B')
  alone = {'A': Bwd('A', Fwd('A'))}
  alone['B'] = Bwd('B', Fwd('B'))
  fa = Fwd('A')
  fb = Fwd('B')
  got = {'B': Bwd('B', fb)}
  got['A'] = Bwd('A', fa)
  for k in ('A', 'B'):
    for r in range(ep):
      for name in ('y', 'dx', 'dgate', 'dwi', 'dwo'):
        _SameBits('layer %s rank %d %s' % (k, r, name), got[k][r][name].detach(),
                  alone[k][r][name].detach())


# ------------------------------------------------------------------------ CPU ----
@pytest.mark.parametrize('ep', [2, 3, 8])
def test_peer_tables_address_the_slot_convention_rows(ep, sim_world):
  """Every rank's peer and row-pointer tables, built by the real `MoeExchange` in a simulated
  world, against addresses taken from the destination slabs' own views."""
  e_l, g_l, s, c, m = 2, 3, 16, 4, 24
  e = ep * e_l
  _, ranks = _Ranks(ep, e, torch.device('cpu'), ['A'], g_l, s, c, m)
  xe = [ex._layers['A'].xe for ex in ranks]
  yc = [ex._layers['A'].yc for ex in ranks]
  for d, ex in enumerate(ranks):
    bufs = ex._layers['A']
    for loopback in (False, True):
      ex.loopback = loopback
      src = [d] * ep if loopback else list(range(ep))
      assert bufs.peer_xe.tolist() == [xe[j].data_ptr() for j in src], (d, loopback)
      assert ex.peer_dye.tolist() == [ranks[j].dye.data_ptr() for j in src], (d, loopback)
      for table, dst in ((bufs.row_ptrs_yc, yc), (ex.row_ptrs_dxc, [q.dxc for q in ranks])):
        # Local expert e_l of rank d is expert d·E_l + e_l; its row (g_global, c) holds
        # token slot c of group g_global mod G_l of rank g_global // G_l.
        want = torch.tensor([[[dst[src[gg // g_l]][d * e_l + el, (gg % g_l) * c + cc].data_ptr()
                               for cc in range(c)] for gg in range(ep * g_l)]
                             for el in range(e_l)], dtype=torch.int64)
        assert table.shape == (e_l, ep * g_l * c), tuple(table.shape)
        routing._AssertEqual('rank %d row table (loopback %s)' % (d, loopback),
                             table.view(e_l, ep * g_l, c), want)
    ex.loopback = False
