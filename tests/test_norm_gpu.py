"""The fused RMS norm / LayerNorm kernels (ops/csrc/norm_kernels.cu) against a float64 oracle
written from the formula, at the benchmark's shape and at the edges of the kernels' tiling.

Contract checked here, for bf16 x [R, D] (D a multiple of 8) and the fp32 scale / bias the
kernel reads (a bf16 parameter is widened exactly):
  * forward: y = x̂·scale (+ bias) with x̂ = (x − mean)·rstd, rstd = (var + eps)^-½; RMS norm
    has mean = 0 and var = E[x²]; `stats` holds (mean, rstd) per row, mean = 0 exactly for RMS;
  * backward: dx = rstd·(g − mean(g) − x̂·mean(g·x̂)) with g = dy·scale (RMS: no mean(g)),
    plus the residual-stream gradient when one is given, rounded to bf16 once;
    dscale = Σ_rows dy·x̂ and dbias = Σ_rows dy in fp32, folded in a fixed order, so every
    output is bit-identical from run to run.

Where the kernels round, and the bounds that follow (u = 2^-24, n = 8·⌈D/256⌉ + 5 the length
of the longest fp32 summation chain of a row: a lane's sequential terms plus 5 shuffle levels):
  * mean = s1/D: |Δmean| ≤ (n + 1)·u·mean|x|.
  * var = s2/D − mean² in one pass: |Δvar| ≤ (n + 3)·u·(E[x²] + 3·|mean|·mean|x|), and
    rstd = rsqrtf (2 ulp): |Δrstd|/rstd ≤ ½|Δvar|/(var + eps) + 2^-22 + u. For RMS norm
    this is ½(n + 5)·u + 2^-22 ≤ 2^-16 up to D = 8192. For LayerNorm it grows with the
    rows' mean offset: E[x²]/var = 1 + offset²/σ². A CPU emulation of the kernel's fp32
    summation order (not a GPU measurement) puts the worst relative rstd error at D = 1024 at

        | mean offset | 8σ   | 64σ  | 256σ |
        | rstd error  | 4e-6 | 3e-4 | 3e-3 |

    The worst-case bound above is 20–70x larger; the `stats` check uses it. y stays within
    1 bf16 ulp while the rstd error is below 2^-9 (half a bf16 ulp, relative), which holds
    up to 64σ and fails near 256σ, so the LayerNorm tests go up to 64σ.
  * y is rounded to bf16 once: within 1 ulp of the oracle, except where x − mean nearly
    cancels, where the mean's error (rstd·|scale|·|Δmean|) may exceed an ulp, and where a
    bias cancels x̂·scale, where the rstd's error (taken from the kernel's own `stats`,
    which are checked against the bound above) times |x̂·scale| may.
  * dx: g·x̂ products (2u), fp32 sums of D terms for mean(g), mean(g·x̂) (n·u), x̂ from the
    kernel's rstd and mean, then one bf16 rounding: within 1 ulp, or where the three terms
    cancel, within rstd·(|g| + mean|g| + (|x̂| + 1)·mean|g·x̂|)·(2·ε_rstd + rstd·|Δmean| +
    (n + 6)·u) of the oracle.
  * dscale / dbias: fmaf chains of 16 rows per partial (kDsRows), then the fold's chain of
    ⌈P/16⌉ + 1 partials and 8 row groups: m = 16 + ⌈P/16⌉ + 9 roundings of running sums,
    so |Δ| ≤ m·u·Σ|dy·x̂| plus the x̂ error carried by Σ|dy|·|Δx̂|.
Every bound carries a factor _C = 2 over the sum of the worst cases. At the benchmark's
shape, losing one of the 512 dscale partials moves dscale by ~1e-3 of Σ|dy·x̂|; the bound
there is ~1e-5.
"""
import math

import pytest
import torch

from lingvo_b200 import ops
from lingvo_b200.ops import norm

pytestmark = pytest.mark.gpu

_U = 2.0**-24
_RSQRT = 2.0**-22          # rsqrtf: 2 ulp
_C = 2.0
_DS_ROWS = 16              # rows per dscale partial (kDsRows)
_EPS = 1e-6
_BENCH = (8192, 2048)      # MoELm8E: 8 x 1024 tokens, M = 2048


def _Chain(dim):
  return 8 * math.ceil(dim / 256) + 5


def _Ulp(t):
  """One bf16 ulp at |t| (float64), floored at the smallest normal."""
  a = t.abs().clamp_min(2.0**-126)
  return torch.exp2(torch.floor(torch.log2(a)) - 7)


def _Ordered(b):
  i = b.contiguous().view(torch.int16).int()
  return torch.where(i < 0, -(i & 0x7fff), i)


def _AssertBf16(got, want, slack, what):
  """bf16 `got` within 1 ulp of float64 `want` rounded to bf16, or within `slack` of it."""
  assert got.dtype == torch.bfloat16 and got.shape == want.shape, what
  if got.numel() == 0:
    return
  ulps = (_Ordered(got) - _Ordered(want.bfloat16())).abs()
  bad = (ulps > 1) & ~((got.double() - want).abs() <= slack)
  assert not bool(bad.any()), '%s: %d elements outside the bound, worst %g at %s' % (
      what, int(bad.sum()), float(((got.double() - want).abs() - slack)[bad].max()),
      tuple(bad.nonzero()[0].tolist()))


def _AssertWithin(got, want, bound, what):
  err = (got.double() - want).abs()
  bad = err > bound
  assert not bool(bad.any()), '%s: %d elements outside the bound, worst excess %g' % (
      what, int(bad.sum()), float((err - bound)[bad].max()))


# ------------------------------------------------------------------ the oracle ----
def _Oracle(x, dy, scale, bias, center, dres=None):
  """Float64 forward and backward from the kernel's inputs, with the error bounds of the
  module docstring. x, dy, dres bf16 [R, D]; scale / bias the fp32 vectors the kernel reads."""
  r, dim = x.shape
  n = _Chain(dim)
  xd = x.double()
  mabs = xd.abs().mean(-1, keepdim=True)
  mean = xd.mean(-1, keepdim=True) if center else torch.zeros_like(mabs)
  xc = xd - mean
  var = (xc * xc).mean(-1, keepdim=True)
  rstd = (var + _EPS).rsqrt()
  xhat = xc * rstd
  sc = scale.double() if scale is not None else torch.ones(dim, dtype=torch.float64,
                                                           device=x.device)
  o = {'mean': mean[:, 0], 'rstd': rstd[:, 0]}
  o['xs'] = xhat * sc
  o['y'] = o['xs'] + (bias.double() if bias is not None else 0.0)
  d_mean = (n + 1) * _U * mabs if center else torch.zeros_like(mabs)
  ex2 = (xd * xd).mean(-1, keepdim=True)
  d_var = (n + 3) * _U * (ex2 + 3 * mean.abs() * mabs)
  e_r = 0.5 * d_var / (var + _EPS) + _RSQRT + _U                   # relative rstd error
  o['d_mean'] = _C * d_mean[:, 0]
  o['d_rstd'] = _C * (e_r * rstd)[:, 0]
  d_xhat = rstd * d_mean                                            # absolute, from the mean
  o['slack_y'] = _C * (sc.abs() * (d_xhat + 3 * _U * xhat.abs()) +
                       (2 * _U * bias.double().abs() if bias is not None else 0.0))
  if dy is None:
    return o
  dyd = dy.double()
  g = dyd * sc
  c1 = g.mean(-1, keepdim=True) if center else 0.0
  c2 = (g * xhat).mean(-1, keepdim=True)
  dx = rstd * (g - c1 - xhat * c2)
  a_g = g.abs().mean(-1, keepdim=True) if center else 0.0
  a_gx = (g * xhat).abs().mean(-1, keepdim=True)
  slack = rstd * (g.abs() + a_g + (xhat.abs() + 1) * a_gx) * (2 * e_r + d_xhat + (n + 6) * _U)
  if dres is not None:
    dx = dx + dres.double()
    slack = slack + _U * dres.double().abs()
  o['dx'] = dx
  o['slack_dx'] = _C * slack
  nblk = math.ceil(r / _DS_ROWS)
  m = _DS_ROWS + math.ceil(nblk / 16) + 9
  o['ds'] = (dyd * xhat).sum(0)
  o['d_ds'] = _C * (m * _U * (dyd * xhat).abs().sum(0) +
                    (dyd.abs() * (xhat.abs() * (e_r + 2 * _U) + d_xhat)).sum(0))
  o['db'] = dyd.sum(0)
  o['d_db'] = _C * m * _U * dyd.abs().sum(0)
  return o


def _Inputs(rows, dim, seed, offset=0.0):
  """x = offset_r + N(0, 1) with row offsets spread over [-offset, offset]; dy = N(0, 1)."""
  g = torch.Generator(device='cuda').manual_seed(seed)
  x = torch.randn(rows, dim, device='cuda', generator=g)
  if offset and rows:
    x = x + torch.linspace(-offset, offset, rows, device='cuda')[:, None]
  dy = torch.randn(rows, dim, device='cuda', generator=g).bfloat16()
  scale = torch.rand(dim, device='cuda', generator=g) + 0.5
  bias = torch.randn(dim, device='cuda', generator=g)
  return x.bfloat16(), dy, scale, bias


def _CheckNative(x, dy, scale, bias, center, need_ds=True, need_db=True, what=''):
  """norm_fwd + norm_bwd through the bindings against the oracle; returns the outputs."""
  nat = ops.native()
  y, stats, _ = nat.norm_fwd(x, None, scale, bias, _EPS, center, False)
  o = _Oracle(x, dy, scale, bias, center)
  assert stats.shape == (x.shape[0], 2) and stats.dtype == torch.float32
  # where a bias cancels x̂·scale, the rstd's own error (bounded below) may exceed an ulp of y
  rel_rstd = ((stats[:, 1].double() - o['rstd']).abs() / o['rstd'])[:, None]
  _AssertBf16(y, o['y'], o['slack_y'] + _C * rel_rstd * o['xs'].abs() + _Ulp(o['y']),
              what + ' y')
  if center:
    _AssertWithin(stats[:, 0], o['mean'], o['d_mean'], what + ' mean')
  else:
    assert bool((stats[:, 0] == 0).all()), what + ' RMS mean must be 0 exactly'
  _AssertWithin(stats[:, 1], o['rstd'], o['d_rstd'], what + ' rstd')
  dx, ds, db = nat.norm_bwd(x, dy, None, scale, stats, center, need_ds, need_db)
  _AssertBf16(dx, o['dx'], o['slack_dx'] + _Ulp(o['dx']), what + ' dx')
  if need_ds:
    assert ds.dtype == torch.float32 and ds.shape == (x.shape[1],)
    _AssertWithin(ds, o['ds'], o['d_ds'], what + ' dscale')
  else:
    assert ds is None
  if need_db:
    assert db.dtype == torch.float32 and db.shape == (x.shape[1],)
    if center:
      _AssertWithin(db, o['db'], o['d_db'], what + ' dbias')
    else:
      assert bool((db == 0).all())
  else:
    assert db is None
  return y, stats, dx, ds, db


# ------------------------------------------------------ RMS norm at the bench shape ----
@pytest.mark.parametrize('scale_dtype', [torch.float32, torch.bfloat16])
def test_rms_norm_benchmark_shape(scale_dtype):
  """8192 x 2048: 512 dscale partials of 16 rows; the forward and backward through autograd."""
  rows, dim = _BENCH
  x, dy, scale, _ = _Inputs(rows, dim, 1)
  scale = scale.to(scale_dtype)
  xg = x.clone().requires_grad_()
  sg = scale.clone().requires_grad_()
  y = norm.rms_norm(xg, sg, _EPS)
  y.backward(dy)
  o = _Oracle(x, dy, scale.float(), None, False)
  assert y.dtype == torch.bfloat16
  _AssertBf16(y.detach(), o['y'], o['slack_y'] + _Ulp(o['y']), 'y')
  _AssertBf16(xg.grad, o['dx'], o['slack_dx'] + _Ulp(o['dx']), 'dx')
  # the fp32 dscale the kernels fold, and its single rounding to the parameter's dtype
  _, stats, _ = ops.native().norm_fwd(x, None, scale, None, _EPS, False, False)
  assert bool((stats[:, 0] == 0).all())
  _AssertWithin(stats[:, 1], o['rstd'], o['d_rstd'], 'rstd')
  assert float((o['d_rstd'] / o['rstd']).max()) <= 2 * 2.0**-16
  _, ds, _ = ops.native().norm_bwd(x, dy, None, scale, stats, False, True, False)
  _AssertWithin(ds, o['ds'], o['d_ds'], 'dscale')
  assert sg.grad.dtype == scale_dtype
  assert torch.equal(sg.grad, ds.to(scale_dtype))
  # losing one 16-row partial must be far outside the bound
  lost = (dy[:_DS_ROWS].double() * x[:_DS_ROWS].double() *
          o['rstd'][:_DS_ROWS, None]).sum(0).abs()
  assert float((lost > o['d_ds']).double().mean()) > 0.9


def test_rms_norm_pass_benchmark_shape():
  """(norm(x), x) as one node: both branches, the normalised branch only, the residual only."""
  rows, dim = _BENCH
  x, dy, scale, _ = _Inputs(rows, dim, 2)
  g = torch.Generator(device='cuda').manual_seed(3)
  dres = torch.randn(rows, dim, device='cuda', generator=g).bfloat16()
  xg = x.clone().requires_grad_()
  sg = scale.clone().requires_grad_()
  yn, xp = norm.rms_norm_pass(xg, sg, _EPS)
  assert torch.equal(xp, x)
  o = _Oracle(x, None, scale, None, False)
  _AssertBf16(yn.detach(), o['y'], o['slack_y'] + _Ulp(o['y']), 'y')
  # both branches: the residual gradient is added before the one bf16 rounding
  gx, gs = torch.autograd.grad([yn, xp], [xg, sg], [dy, dres])
  o = _Oracle(x, dy, scale, None, False, dres=dres)
  _AssertBf16(gx, o['dx'], o['slack_dx'] + _Ulp(o['dx']), 'dx with dres')
  _AssertWithin(gs, o['ds'], o['d_ds'], 'dscale with dres')
  # the normalised branch only: dx is the plain norm gradient, the same bits as rms_norm's
  yn, xp = norm.rms_norm_pass(xg, sg, _EPS)
  gx1, gs1 = torch.autograd.grad(yn, [xg, sg], dy)
  o1 = _Oracle(x, dy, scale, None, False)
  _AssertBf16(gx1, o1['dx'], o1['slack_dx'] + _Ulp(o1['dx']), 'dx without dres')
  gx2, gs2 = torch.autograd.grad(norm.rms_norm(xg, sg, _EPS), [xg, sg], dy)
  assert torch.equal(gx1, gx2) and torch.equal(gs1, gs2)
  assert torch.equal(gs1, gs)
  # the residual branch only: the gradient passes through exactly
  yn, xp = norm.rms_norm_pass(xg, sg, _EPS)
  (gx3,) = torch.autograd.grad(xp, xg, dres)
  assert torch.equal(gx3, dres)


@pytest.mark.parametrize('center', [False, True])
def test_backward_is_bitwise_reproducible(center):
  rows, dim = _BENCH
  x, dy, scale, bias = _Inputs(rows, dim, 4)
  dres = _Inputs(rows, dim, 5)[1]
  nat = ops.native()
  _, stats, _ = nat.norm_fwd(x, None, scale, bias if center else None, _EPS, center, False)
  runs = [nat.norm_bwd(x, dy, dres, scale, stats, center, True, center) for _ in range(3)]
  for dx, ds, db in runs[1:]:
    assert torch.equal(dx, runs[0][0]) and torch.equal(ds, runs[0][1])
    if center:
      assert torch.equal(db, runs[0][2])


# ------------------------------------------------------------- tiling edges ----
# 8: lanes 1-31 hold no columns; 264: not a multiple of 256; 5120: the dscale kernel has 3
# column chunks of 2048, the last partial. 20000 rows: every warp goes round the persistent
# grid (132 SMs x 8 CTAs x 8 warps = 8448 rows) more than twice.
_DIMS = [8, 264, 1024, 2048, 5120, 8192]
_ROWS = [0, 1, 7, 16 * 5 + 3, 20000]


@pytest.mark.parametrize('rows', _ROWS)
@pytest.mark.parametrize('dim', _DIMS)
@pytest.mark.parametrize('center', [False, True], ids=['rms', 'ln'])
def test_tiling_edges(center, dim, rows):
  assert ops.native().norm_fwd is not None
  x, dy, scale, bias = _Inputs(rows, dim, 10 + dim + rows)
  y, stats, dx, ds, db = _CheckNative(x, dy, scale, bias if center else None, center,
                                      True, center, what='%dx%d' % (rows, dim))
  if rows == 0:
    assert y.shape == (0, dim) and dx.shape == (0, dim)
    assert bool((ds == 0).all()) and (db is None or bool((db == 0).all()))


# ------------------------------------------------------------------ LayerNorm ----
@pytest.mark.parametrize('has_scale,has_bias,need_grads', [
    (True, True, True), (True, False, True), (False, True, True), (True, True, False)],
    ids=['scale+bias', 'scale', 'bias', 'no-param-grads'])
@pytest.mark.parametrize('offset', [0.0, 8.0, 64.0])
def test_layer_norm_variants_and_mean_offsets(has_scale, has_bias, need_grads, offset):
  """Row means spread over [-offset, offset] (σ = 1): y stays within 1 bf16 ulp."""
  rows, dim = 4099, 1024
  x, dy, scale, bias = _Inputs(rows, dim, 20, offset)
  _CheckNative(x, dy, scale if has_scale else None, bias if has_bias else None, True,
               need_grads and has_scale, need_grads and has_bias,
               what='offset %g' % offset)


# ----------------------------------------------------------- the layer on CUDA ----
def _LayerNormLayer(dim, center, bias, dtype):
  from lingvo_b200.core import layers
  p = layers.LayerNorm.Params().Set(name='ln', input_dim=dim, center=center, bias=bias)
  p.fprop_dtype = dtype
  l = p.Instantiate().cuda()
  g = torch.Generator(device='cuda').manual_seed(30)
  with torch.no_grad():
    for v in l.vars.Flatten():
      v.copy_(torch.randn(v.shape, device='cuda', generator=g) * 0.5)
  return l


def _LayerOracle(l, x, center, dy=None):
  """Float64 y of the layer's formula from the scale / bias values it uses; with dy, also
  the float64 autograd gradients of x and of every variable (by name)."""
  scale, bias = l._GetScaleAndBias(l.theta)  # pylint: disable=protected-access
  xd = x.double()
  xc = xd - xd.mean(-1, keepdim=True) if center else xd
  y = xc * ((xc * xc).mean(-1, keepdim=True) + l.params.epsilon).rsqrt() * scale.double()
  y = y + bias.double() if bias is not None else y
  if dy is None:
    return y
  vr = {n: v.detach().double().requires_grad_() for n, v in l.vars.FlattenItems()}
  xr = x.detach().double().requires_grad_()
  sc = vr['scale'] if l.params.direct_scale else 1.0 + vr['scale']
  xc = xr - xr.mean(-1, keepdim=True) if center else xr
  yr = xc * ((xc * xc).mean(-1, keepdim=True) + l.params.epsilon).rsqrt() * sc
  if 'bias' in vr:
    yr = yr + vr['bias']
  yr.backward(dy.double())
  return y, xr.grad, {n: v.grad for n, v in vr.items()}


@pytest.mark.parametrize('center,bias', [(True, True), (True, False), (False, True),
                                         (False, False)])
def test_layer_fp32_input_stays_fp32(center, bias):
  """An fp32 activation is normalised in fp32 and returned as fp32, to fp32 accuracy."""
  dim = 1024
  l = _LayerNormLayer(dim, center, bias, torch.float32)
  x = (torch.randn(333, dim, device='cuda') * 3 + 1).requires_grad_()
  y = l.FPropDefaultTheta(x)
  assert y.dtype == torch.float32
  dy = torch.randn_like(y)
  y.backward(dy)
  want, dx, dvars = _LayerOracle(l, x.detach(), center, dy)
  tol = 2e-5
  torch.testing.assert_close(y.detach().double(), want, rtol=tol,
                             atol=tol * float(want.abs().max()))
  assert x.grad.dtype == torch.float32
  torch.testing.assert_close(x.grad.double(), dx, rtol=tol, atol=tol * float(dx.abs().max()))
  for n, v in l.vars.FlattenItems():
    r = dvars[n]
    torch.testing.assert_close(v.grad.double(), r, rtol=tol, atol=tol * float(r.abs().max()),
                               msg=n)


@pytest.mark.parametrize('center,bias', [(True, True), (True, False), (False, True),
                                         (False, False)])
def test_layer_bf16_input(center, bias):
  """bf16 input: the kernel's bf16 output within 1 ulp of the oracle (for center=False with
  a bias, within the two roundings of the norm and the bias add), and every parameter's
  gradient is that of the float64 formula."""
  dim, rows = 1024, 517
  l = _LayerNormLayer(dim, center, bias, torch.bfloat16)
  x = torch.randn(rows, dim, device='cuda').bfloat16().requires_grad_()
  launches = ops.native().launch_count()
  y = l.FPropDefaultTheta(x)
  assert ops.native().launch_count() > launches, 'the fused kernel was not taken'
  assert y.dtype == torch.bfloat16
  want = _LayerOracle(l, x.detach(), center)
  scale, b = l._GetScaleAndBias(l.theta)  # pylint: disable=protected-access
  slack = _Ulp(want)
  if b is not None and not center:
    slack = slack + _Ulp(want - b.double())          # the norm's own bf16 rounding
  _AssertBf16(y.detach(), want, 2 * 2.0**-16 * (want.abs() + 1) + slack, 'y')
  dy = torch.randn(rows, dim, device='cuda').bfloat16()
  y.backward(dy)
  _, dx, dvars = _LayerOracle(l, x.detach(), center, dy)
  assert x.grad.dtype == torch.bfloat16
  torch.testing.assert_close(x.grad.double(), dx, rtol=2.0**-6,
                             atol=2.0**-6 * float(dx.abs().max()))
  for n, v in l.vars.FlattenItems():
    r = dvars[n]
    assert v.grad is not None, n
    torch.testing.assert_close(v.grad.double(), r, rtol=2.0**-7,
                               atol=2.0**-7 * float(r.abs().max()), msg=n)


def test_layer_not_centred_adds_and_trains_bias():
  """center=False with a bias: y = x̂·scale + bias on the GPU as on the CPU, and the bias
  receives Σ dy."""
  dim = 256
  for dtype in (torch.float32, torch.bfloat16):
    l = _LayerNormLayer(dim, False, True, dtype)
    x = torch.randn(64, dim, device='cuda').to(dtype)
    y = l.FPropDefaultTheta(x)
    want = _LayerOracle(l, x, False)
    tol = 2.0**-6 if dtype == torch.bfloat16 else 1e-5
    torch.testing.assert_close(y.double(), want, rtol=tol, atol=tol * 4)
    dy = torch.randn_like(y)
    y.backward(dy)
    bias_grad = l.vars.bias.grad
    torch.testing.assert_close(bias_grad.double(), dy.double().sum(0), rtol=2.0**-8,
                               atol=1e-3)


# ------------------------------------------------------------- refusals ----
def _Refused(fn, match):
  before = ops.native().launch_count()
  with pytest.raises(RuntimeError, match=match):
    fn()
  assert ops.native().launch_count() == before


def test_norm_fwd_refusals():
  nat = ops.native()
  x = torch.randn(16, 64, device='cuda').bfloat16()
  s = torch.ones(64, device='cuda')
  _Refused(lambda: nat.norm_fwd(x.float(), None, s, None, _EPS, True, False), 'bf16')
  _Refused(lambda: nat.norm_fwd(x[:, :60].contiguous(), None, None, None, _EPS, True, False),
           'multiple of 8')
  _Refused(lambda: nat.norm_fwd(x, None, s[:56], None, _EPS, True, False), 'scale')
  _Refused(lambda: nat.norm_fwd(x, None, s, torch.ones(72, device='cuda'), _EPS, True, False),
           'bias')
  _Refused(lambda: nat.norm_fwd(x, x[:8], None, None, _EPS, False, False), 'res')
  # a contiguous bf16 view at a storage offset of 4 elements (8 bytes)
  flat = torch.randn(16 * 64 + 8, device='cuda').bfloat16()
  xv = flat[4:4 + 16 * 64].view(16, 64)
  assert xv.is_contiguous() and xv.data_ptr() % 16 == 8
  _Refused(lambda: nat.norm_fwd(xv, None, s, None, _EPS, True, False), 'aligned')
  _Refused(lambda: nat.norm_fwd(x, xv, s, None, _EPS, True, False), 'res')
  sflat = torch.ones(72, device='cuda')
  _Refused(lambda: nat.norm_fwd(x, None, sflat[2:66], None, _EPS, True, False), 'aligned')


def test_norm_bwd_refusals():
  nat = ops.native()
  x = torch.randn(16, 64, device='cuda').bfloat16()
  s = torch.ones(64, device='cuda')
  _, stats, _ = nat.norm_fwd(x, None, s, None, _EPS, False, False)
  dy = torch.randn_like(x)
  flat = torch.randn(16 * 64 + 8, device='cuda').bfloat16()
  xv = flat[4:4 + 16 * 64].view(16, 64)
  cases = [
      (lambda: nat.norm_bwd(x.float(), dy, None, s, stats, False, True, False), 'bf16'),
      (lambda: nat.norm_bwd(x, dy.float(), None, s, stats, False, True, False), 'dy'),
      (lambda: nat.norm_bwd(x, dy[:8], None, s, stats, False, True, False), 'dy'),
      (lambda: nat.norm_bwd(x.view(16, 8, 8).reshape(16, 8, 8)[:, :, :4].contiguous(),
                            dy, None, None, stats, False, True, False), 'multiple of 8'),
      (lambda: nat.norm_bwd(x, dy, dy[:8], s, stats, False, True, False), 'dres'),
      (lambda: nat.norm_bwd(x, dy, None, s, stats[:8], False, True, False), 'stats'),
      (lambda: nat.norm_bwd(x, dy, None, s, stats.reshape(-1), False, True, False), 'stats'),
      (lambda: nat.norm_bwd(x, dy, None, s, stats.double(), False, True, False), 'stats'),
      (lambda: nat.norm_bwd(x, dy, None, s[:32], stats, False, True, False), 'scale'),
      (lambda: nat.norm_bwd(xv, dy, None, s, stats, False, True, False), 'aligned'),
      (lambda: nat.norm_bwd(x, xv, None, s, stats, False, True, False), 'aligned'),
      (lambda: nat.norm_bwd(x, dy, xv, s, stats, False, True, False), 'dres'),
  ]
  for fn, match in cases:
    _Refused(fn, match)
