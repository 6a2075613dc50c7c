"""The Conformer's fused GLU + padding mask + depthwise conv1d (ops/csrc/conv_kernels.cu)
against a float64 oracle written from the formula in the kernel file's header, with the
gradients taken by float64 autograd.

Contract checked here, for proj = (gated | act) [B, T, 2D], w [K, D], pad [B, T] in {0, 1}
and left = K − 1 (causal) or ⌊(K − 1)/2⌋ (SAME):
  * g[b, t, d] = act·σ(gated)·(1 − pad[b, t]) and
    y[b, t, d] = (1 − pad[b, t])·Σ_k w[k, d]·g[b, t + k − left, d] (g = 0 outside [0, T));
  * d proj and d w are the gradients of that formula; y and d proj are exactly zero at
    padded frames; d w is folded in a fixed order, so every output is bit-identical from
    run to run.

Where the kernels round (u = 2^-24): σ uses __expf, whose error is (2 + 1.173·|x|) ulp, so
σ(x) carries ε_σ(x) = (2 + 1.173·|x|)·2^-23 + 3u. g is one product more (2u). y is a chain
of K fp32 products and sums ((K + 1)·u), so |Δy| ≤ Σ_k |w|·|g|·(ε_σ + (K + 4)·u). d g is a
chain of K terms of w·dy', and d act = d g·σ, d gated = d g·act·σ·(1 − σ), whose
derivative in σ is at most 1, so both are within σ·(|act| + 1)·Σ_k |w|·|dy'|·(ε_σ + (K + 6)·u).
d w sums dy'·act·σ in fp32: 32 frames of a tile, the kRun = 2 tiles of a block in order,
then the fold of the P = B·⌈T/64⌉ block partials over 8 row groups: a chain of
m = 32 + 3 + 2 + ⌈P/8⌉ + 8 roundings, so |Δdw| ≤ Σ|dy'·g|·(ε_σ + m·u). Every output is
also rounded once to its dtype (1 bf16 ulp, or u in fp32). Each bound carries a factor
_C = 2 over the sum of the worst cases.
"""
import math

import pytest
import torch

from lingvo_b200 import ops
from lingvo_b200.ops import conv as C

pytestmark = pytest.mark.gpu

_U = 2.0**-24
_C = 2.0
_TT, _RUN = 32, 2
_MAX_K = 86                 # (220 KiB / 512 B − 93) / 4: the backward's shared memory


# ------------------------------------------------------------------ the oracle ----
def _Conv(x, w, left):
  """x [B, T, D] float64, w [K, D] → Σ_k w[k]·x[t + k − left] (zero outside [0, T))."""
  k, d = w.shape
  xp = torch.nn.functional.pad(x.transpose(1, 2), (left, k - 1 - left))
  return torch.nn.functional.conv1d(xp, w.t().unsqueeze(1), groups=d).transpose(1, 2)


def _ConvT(x, w, left):
  """Adjoint of _Conv: Σ_k w[k]·x[t − k + left]."""
  return _Conv(x, w.flip(0), w.shape[0] - 1 - left)


def _Oracle(proj, w, pad, dy, left):
  """Float64 y, d proj, d w from the kernel's inputs, with the bounds of the docstring."""
  pd = proj.double().requires_grad_()
  wd = w.double().requires_grad_()
  m = (1.0 - pad.double()).unsqueeze(-1)
  gated, act = pd.chunk(2, -1)
  g = act * torch.sigmoid(gated) * m
  y = _Conv(g, wd, left) * m
  y.backward(dy.double())
  k = w.shape[0]
  with torch.no_grad():
    gt, at = proj.double().chunk(2, -1)
    sig = torch.sigmoid(gt)
    e_s = (2 + 1.173 * gt.abs()) * 2.0**-23 + 3 * _U
    ga = (at * sig * m).abs()
    wa = w.double().abs()
    o = {'y': y.detach(), 'dproj': pd.grad, 'dw': wd.grad}
    o['d_y'] = _C * _Conv(ga * (e_s + (k + 4) * _U), wa, left) * m
    dya = (dy.double() * m).abs()
    adg = _ConvT(dya, wa, left)
    e_max = float(e_s.max()) if e_s.numel() else 0.0
    d_dg = adg * (e_max + (k + 6) * _U) * sig * m
    o['d_dproj'] = _C * torch.cat([d_dg * (at.abs() + 1), d_dg], -1)
    b, t, _ = proj.shape
    nparts = b * math.ceil(t / (_TT * _RUN))
    mm = _TT + 3 + _RUN + math.ceil(nparts / 8) + 8
    # Σ_{b,t} |dy'[t]|·|g[t + k − left]| for every k: correlate |dy'| with shifted |g|
    gpad = torch.nn.functional.pad(ga, (0, 0, left, k - 1 - left))
    a_dw = torch.stack([(dya * gpad[:, j:j + t]).sum((0, 1)) for j in range(k)])
    o['d_dw'] = _C * a_dw * (e_max + mm * _U)
  return o


def _Ulp(t, dtype):
  if dtype == torch.float32:
    return t.abs() * _U * 2
  a = t.abs().clamp_min(2.0**-126)
  return torch.exp2(torch.floor(torch.log2(a)) - 7)


def _Assert(got, want, slack, dtype, what):
  assert got.dtype == dtype and got.shape == want.shape, what
  if got.numel() == 0:
    return
  err = (got.double() - want).abs()
  bad = err > slack + _Ulp(want, dtype)
  if dtype == torch.bfloat16:   # within 1 ulp of want rounded to bf16 always passes
    i = got.contiguous().view(torch.int16).int()
    j = want.bfloat16().contiguous().view(torch.int16).int()
    oi = torch.where(i < 0, -(i & 0x7fff), i)
    oj = torch.where(j < 0, -(j & 0x7fff), j)
    bad = bad & ((oi - oj).abs() > 1)
  assert not bool(bad.any()), '%s: %d elements outside the bound, worst excess %g' % (
      what, int(bad.sum()), float((err - slack - _Ulp(want, dtype))[bad].max()))


def _Pads(b, t, seed):
  """Ragged paddings: trailing pads of different lengths, a fully padded row and a row with
  padding in the middle."""
  pad = torch.zeros(b, t)
  for i in range(b):
    n = (i * 37 + seed) % max(t, 1)
    if n:
      pad[i, t - n:] = 1
  if b > 2:
    pad[1] = 1
  if b > 3 and t > 4:
    pad[2, :] = 0
    pad[2, t // 3:t // 3 + max(1, t // 5)] = 1
  return pad.cuda()


def _Run(b, t, d, k, causal, dtype, seed=0):
  g = torch.Generator(device='cuda').manual_seed(seed)
  proj = (torch.randn(b, t, 2 * d, device='cuda', generator=g) * 1.5).to(dtype)
  w = torch.randn(k, d, device='cuda', generator=g) * (1.0 / math.sqrt(k))
  dy = torch.randn(b, t, d, device='cuda', generator=g).to(dtype)
  pad = _Pads(b, t, seed)
  left = k - 1 if causal else (k - 1) // 2
  pg = proj.clone().requires_grad_()
  wg = w.clone().requires_grad_()
  y = C.glu_dwconv1d(pg, wg, pad, causal)
  y.backward(dy)
  return proj, w, pad, dy, left, y.detach(), pg.grad, wg.grad


def _Check(b, t, d, k, causal, dtype, seed=0):
  proj, w, pad, dy, left, y, dproj, dw = _Run(b, t, d, k, causal, dtype, seed)
  o = _Oracle(proj, w, pad, dy, left)
  what = 'B%d T%d D%d K%d %s %s' % (b, t, d, k, 'causal' if causal else 'same', dtype)
  _Assert(y, o['y'], o['d_y'], dtype, what + ' y')
  _Assert(dproj, o['dproj'], o['d_dproj'], dtype, what + ' dproj')
  _Assert(dw, o['dw'], o['d_dw'], torch.float32, what + ' dw')
  padded = pad.bool()
  assert bool((y[padded] == 0).all()), what + ' y at padded frames'
  assert bool((dproj[padded] == 0).all()), what + ' dproj at padded frames'
  return y, dproj, dw


# ----------------------------------------------------------- Librispeech shape ----
@pytest.mark.parametrize('causal', [False, True], ids=['same', 'causal'])
def test_librispeech_shape_bf16(causal):
  """B = 48, T = 428 (the longest bucket after 4x subsampling), D = 512, K = 32 (SAME is
  left 15, right 16)."""
  _Check(48, 428, 512, 32, causal, torch.bfloat16)


@pytest.mark.parametrize('causal', [False, True], ids=['same', 'causal'])
def test_smaller_shape_fp32(causal):
  _Check(6, 150, 384, 32, causal, torch.float32, seed=1)


def test_backward_is_bitwise_reproducible():
  proj, w, pad, dy, left = _Run(48, 428, 512, 32, False, torch.bfloat16)[:5]
  nat = ops.native()
  runs = [nat.glu_dwconv1d_bwd(proj, w, pad, dy, left) for _ in range(3)]
  for dproj, dw in runs[1:]:
    assert torch.equal(dproj, runs[0][0])
    assert torch.equal(dw, runs[0][1])


# ------------------------------------------------------------------- edges ----
# K = 2 SAME is left 0, right 1; at K = 33 the halo (32 + K − 1 = 64 frames) is two whole
# tiles; K = 86 is the largest backward that fits. T = 5 is shorter than K; T = 33 leaves a
# one-frame tile. D = 513 leaves a one-channel block.
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('causal', [False, True], ids=['same', 'causal'])
@pytest.mark.parametrize('d', [1, 200, 513])
@pytest.mark.parametrize('t', [1, 5, 32, 33])
@pytest.mark.parametrize('k', [1, 2, 31, 33, 86])
def test_edges(k, t, d, causal, dtype):
  _Check(5, t, d, k, causal, dtype, seed=k + t + d)


def test_run_of_tiles_and_empty():
  """T = 129 and 513: a one-frame last tile in a partial last run; T = 0 returns empty outputs and zero dw."""
  _Check(3, 129, 128, 9, False, torch.float32)
  _Check(2, 513, 256, 4, True, torch.float32)
  proj = torch.randn(2, 0, 16, device='cuda')
  w = torch.randn(3, 8, device='cuda')
  pad = torch.zeros(2, 0, device='cuda')
  nat = ops.native()
  assert nat.glu_dwconv1d_fwd(proj, w, pad, 1).shape == (2, 0, 8)
  dproj, dw = nat.glu_dwconv1d_bwd(proj, w, pad, torch.zeros(2, 0, 8, device='cuda'), 1)
  assert dproj.shape == proj.shape and bool((dw == 0).all())


# ------------------------------------------------------------ the layer ----
@pytest.mark.parametrize('causal', [False, True], ids=['same', 'causal'])
def test_lconv_layer_fused_matches_unfused(causal, monkeypatch):
  """LConvLayer in fp32 at K = 32 with ragged paddings: the fused kernel and the unfused
  GLU + depthwise conv layer give the same outputs and parameter gradients."""
  from lingvo_b200.core import conformer_layer
  from lingvo_b200.core import layers
  monkeypatch.setattr(torch.backends.cudnn, 'allow_tf32', False)
  monkeypatch.setattr(torch.backends.cuda.matmul, 'allow_tf32', False)
  b, t, d, k = 4, 97, 64, 32
  p = conformer_layer.LConvLayer.CommonParams(input_dim=d, kernel_size=k, is_causal=causal)
  p.name = 'lconv'
  p.conv_norm_layer_tpl = layers.LayerNorm.Params()
  l = p.Instantiate().cuda()
  g = torch.Generator(device='cuda').manual_seed(7)
  with torch.no_grad():
    for v in l.vars.Flatten():
      v.copy_(torch.randn(v.shape, device='cuda', generator=g) * 0.3)
  x = torch.randn(b, t, d, device='cuda', generator=g)
  pad = _Pads(b, t, 5)
  dy = torch.randn(b, t, d, device='cuda', generator=g)
  names = [n for n, _ in l.vars.FlattenItems()]

  def run(disable):
    if disable:
      monkeypatch.setenv('LINGVO_B200_DISABLE_FUSED_CONV', '1')
    else:
      monkeypatch.delenv('LINGVO_B200_DISABLE_FUSED_CONV', raising=False)
    assert C.glu_dwconv1d_supported(x, l.depthwise_conv1d) == (not disable)
    for v in l.vars.Flatten():
      v.grad = None
    xg = x.clone().requires_grad_()
    launches = ops.native().launch_count()
    y, _ = l.FPropDefaultTheta(xg, pad)
    y.backward(dy)
    return (y.detach(), xg.grad, [v.grad.clone() for v in l.vars.Flatten()],
            ops.native().launch_count() - launches)

  yf, dxf, gf, nf = run(False)
  yu, dxu, gu, nu = run(True)
  assert nf > nu                     # the fused path launched the conv kernels
  tol = 1e-5
  torch.testing.assert_close(yf, yu, rtol=tol, atol=tol * float(yu.abs().max()))
  torch.testing.assert_close(dxf, dxu, rtol=tol, atol=tol * float(dxu.abs().max()))
  for n, a, r in zip(names, gf, gu):
    torch.testing.assert_close(a, r, rtol=tol, atol=tol * float(r.abs().max()), msg=n)


# ------------------------------------------------------------- refusals ----
def _Refused(fn, match):
  before = ops.native().launch_count()
  with pytest.raises(RuntimeError, match=match):
    fn()
  assert ops.native().launch_count() == before


def test_kernel_size_limit_refused_without_launch():
  nat = ops.native()
  assert nat.glu_dwconv_max_k == _MAX_K
  b, t, d = 2, 40, 128
  pad = torch.zeros(b, t, device='cuda')
  proj = torch.randn(b, t, 2 * d, device='cuda').bfloat16()
  dy = torch.randn(b, t, d, device='cuda').bfloat16()
  for k in range(_MAX_K + 1, 131):
    w = torch.randn(k, d, device='cuda')
    _Refused(lambda: nat.glu_dwconv1d_bwd(proj, w, pad, dy, (k - 1) // 2), 'kernel size')
    _Refused(lambda: nat.glu_dwconv1d_fwd(proj, w, pad, k - 1), 'kernel size')
  w = torch.randn(9, d, device='cuda')
  _Refused(lambda: nat.glu_dwconv1d_bwd(proj, w, pad, dy[:, :-1].contiguous(), 4), 'dy')
  _Refused(lambda: nat.glu_dwconv1d_bwd(proj, w, pad, dy.float(), 4), 'dy')
  _Refused(lambda: nat.glu_dwconv1d_bwd(proj, w, pad, dy, 9), 'left')
  _Refused(lambda: nat.glu_dwconv1d_fwd(proj, w, pad, -1), 'left')
  _Refused(lambda: nat.glu_dwconv1d_fwd(proj, w[:0], pad, 0), 'kernel size')


@pytest.mark.parametrize('causal', [False, True], ids=['same', 'causal'])
def test_supported_agrees_with_the_kernel_limit(causal):
  """A layer whose K the kernel refuses takes the unfused path instead of failing."""
  from lingvo_b200.core import conv_layers_with_time_padding as conv_lib
  cls = conv_lib.CausalDepthwiseConv2DLayer if causal else conv_lib.DepthwiseConv2DLayer
  x = torch.randn(2, 8, 16, device='cuda')
  for k, want in ((1, True), (_MAX_K, True), (_MAX_K + 1, False), (128, False)):
    l = cls.Params().Set(name='dw', filter_shape=(k, 1, 16, 1)).Instantiate()
    assert C.glu_dwconv1d_supported(x, l) == want, k
