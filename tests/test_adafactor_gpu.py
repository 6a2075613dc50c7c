"""Fused Adafactor and Adam kernels (ops/csrc/optim_kernels.cu) against float64 oracles.

The oracle is the Adafactor step of the `XLAShardingAdafactor` docstring, written out in float64
independently of the optimizer's own PyTorch path. Every check starts from the kernel's own state
before the step (fp32 weights and slots), so each step is compared on its own and an error cannot
hide in the drift of a long run.

Op-level cases run `adafactor_stats` + `adafactor_update` at the MoELm8E benchmark's variable
shapes and at ragged ones; the learner-level cases run `Learner.ScaleGradients` →
`XLAShardingAdafactor.PreGradStats` → `Apply(grad_scale=...)` over a full-size variable set, eager
and graph-captured.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

EPS1, EPS2 = 1e-30, 1e-3
POW = 0.8            # decay_exponent_pow of the MoELm8E optimizer
U = 2.0**-24         # fp32 unit roundoff


def _decay(step):
  return 1.0 - (step + 1.0)**-POW


def _ulp(x):
  """fp32 ulp at |x| (float64 result)."""
  a = x.abs().float()
  return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


def _cleanup(*variables):
  from lingvo_b200.ops import optim
  for v in variables:
    optim._SCRATCH.pop(id(v), None)   # pylint: disable=protected-access


def _grad(shape, gen, dtype, mult=1.0):
  """Gradient with a spread of row and column magnitudes, so that the two factors differ."""
  r, c = shape[-2] if len(shape) > 1 else 1, shape[-1]
  rs = torch.exp(torch.randn(shape[:-2] + (r, 1) if len(shape) > 1 else (1,), device='cuda',
                             generator=gen) * 0.5)
  cs = torch.exp(torch.randn(c, device='cuda', generator=gen) * 0.5)
  g = torch.randn(shape, device='cuda', generator=gen) * 0.01 * mult
  if len(shape) > 1:
    g = g * rs * cs
  return g.to(dtype)


# ---------------------------------------------------------------------------- oracles --
def _factored_ref(w, g, vr, vc, vr_is_rows, lr, decay, clip, mult, gs):
  """One factored Adafactor step in float64 on fp32 state viewed as [B, R, C].

  Returns (vr_new, vc_new, [(w_new_b, delta_b) per slice b], clipped). gs=None means 1;
  gs == 0 drops the gradient (it may hold Inf/NaN): the EMAs only decay toward eps1."""
  b_, r_, c_ = w.shape
  mix = 1.0 - decay
  gs = 1.0 if gs is None else float(gs)
  vr_new = torch.empty(vr.shape, dtype=torch.float64, device=w.device)
  vc_new = torch.empty(vc.shape, dtype=torch.float64, device=w.device)
  fr = torch.empty(b_, r_, dtype=torch.float64, device=w.device)
  fc = torch.empty(b_, c_, dtype=torch.float64, device=w.device)

  def scaled(b):
    if gs == 0:
      return torch.zeros(r_, c_, dtype=torch.float64, device=w.device)
    return g[b].double() * gs

  xsq, wsq = 0.0, 0.0
  for b in range(b_):
    gb = scaled(b)
    g2 = gb.square()
    row_mean = g2.mean(1) + EPS1          # [R]: mean over C
    col_mean = g2.mean(0) + EPS1          # [C]: mean over R
    if vr_is_rows:                        # vr [R] (C is d0), vc [C]
      nvr = vr[b].double() * decay + row_mean * mix
      nvc = vc[b].double() * decay + col_mean * mix
      fr[b] = torch.rsqrt(nvr / nvr.mean())
      fc[b] = torch.rsqrt(nvc)
    else:                                 # vr [C] (R is d0), vc [R]
      nvr = vr[b].double() * decay + col_mean * mix
      nvc = vc[b].double() * decay + row_mean * mix
      fc[b] = torch.rsqrt(nvr / nvr.mean())
      fr[b] = torch.rsqrt(nvc)
    vr_new[b], vc_new[b] = nvr, nvc
    xsq += float((gb * fr[b][:, None] * fc[b][None, :]).square().sum())
    wsq += float(w[b].double().square().sum())
  n = w.numel()
  scale = lr
  if mult:
    scale *= max(math.sqrt(wsq / n), EPS2)
  clipped = clip > 0 and math.sqrt(xsq / n) > clip
  if clip > 0:
    scale /= max(1.0, math.sqrt(xsq / n) / clip)
  out = []
  for b in range(b_):
    delta = scaled(b) * fr[b][:, None] * fc[b][None, :] * scale
    out.append((w[b].double() - delta, delta))
  return vr_new, vc_new, out, clipped


def _small_ref(w, g, v, lr, decay, clip, mult, gs):
  """Non-factored Adafactor step in float64: (v_new, w_new, delta)."""
  gs = 1.0 if gs is None else float(gs)
  g64 = torch.zeros_like(w, dtype=torch.float64) if gs == 0 else g.double() * gs
  v_new = v.double() * decay + (g64.square() + EPS1) * (1.0 - decay)
  x = g64 * torch.rsqrt(v_new)
  scale = lr
  if mult:
    scale *= max(math.sqrt(float(w.double().square().mean())), EPS2)
  if clip > 0:
    scale /= max(1.0, math.sqrt(float(x.square().mean())) / clip)
  delta = x * scale
  return v_new, w.double() - delta, delta


def _assert_w(got, want, delta, rel, what):
  err = (got.double() - want).abs()
  bad = err > rel * delta.abs() + _ulp(want)
  assert not bool(bad.any()), '%s: %d of %d weights off (worst excess %g)' % (
      what, int(bad.sum()), bad.numel(), float((err - rel * delta.abs()).max()))


def _assert_rel(got, want, rel, what):
  err = (got.double() - want).abs()
  bad = err > rel * want.abs()
  assert not bool(bad.any()), '%s: %d of %d off by more than %g relative (worst %g)' % (
      what, int(bad.sum()), bad.numel(), rel, float((err / want.abs()).max()))


def _assert_scalar(got, want, rel, what):
  got = float(got)
  assert abs(got - want) <= rel * abs(want), '%s: %r vs float64 %r' % (what, got, want)


def _sum_bound(r, c):
  """Relative error bounds (second moments, weights) from the kernels' summation lengths.

  Every sum is of non-negative terms, so n sequential fp32 adds stay within n·2⁻²⁴ relative.
  A row sum (over C) is 8 adds per lane, a 5-level warp fold, 8 strips and one add per
  2048-column chunk. A column sum (over R) is 32 rows per CTA and then ⌈R/32⌉/4 adds in
  each lane of the 4-way fold plus 2; at R = 32000 that is 284 adds, 1.7e-5. The EMA adds
  a few more operations. The floor is 3e-5; only [540736, 8] (4260 adds, 2.5e-4) is above it.
  The weight tolerance keeps the same ratio to it as 5e-5 to 3e-5: the factors are rsqrt of
  the second moments and of their mean."""
  nchunk = (c + 2047) // 2048
  n_row = 8 + 5 + 8 + nchunk
  n_col = 32 + ((r + 31) // 32 + 3) // 4 + 2
  v = max(3e-5, (max(n_row, n_col) + 8) * U)
  return v, 5e-5 * v / 3e-5


def _carried_bound(b, r, c):
  """Σw² left by the apply kernel: each lane sums its 8 columns of 64 rows for every work
  item its warp visits in the grid-stride loop, then a 5-level warp fold and the ordered
  fold of the warp partials (≤ 32 per thread and an 8-level tree)."""
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  items = b * ((c + 255) // 256) * ((r + 63) // 64)
  grid = min((items + 7) // 8, sms * 8)
  per_warp = (items + grid * 8 - 1) // (grid * 8)
  n = per_warp * 64 * 8 + 5 + (grid * 8 + 255) // 256 + 8
  return max(5e-5, n * U)


# ------------------------------------------------------------------------- op level --
_BF16, _F32 = torch.bfloat16, torch.float32
# shape, gradient dtype, bf16 copy, clip, param scale, device hyper, grad-scale schedule, lr,
# weight scale
_OP_CASES = [
    ((8, 2048, 8192), _BF16, True, 1.0, True, False, 'scaled', 0.01, 0.05),
    ((8, 8192, 2048), _BF16, True, 1.0, True, True, 'skip', 0.01, 0.05),
    ((2048, 8192), _F32, False, 0.0, True, False, 'one', 0.5, 0.05),
    ((8192, 2048), _BF16, True, 0.25, False, False, 'skip', 0.01, 1.0),
    ((32000, 2048), _BF16, True, 1.0, True, False, 'scaled', 0.01, 0.05),
    ((2048, 2048), _F32, True, 100.0, True, True, 'none', 0.5, 0.05),
    ((3, 131, 2056), _BF16, False, 1.0, True, False, 'skip', 0.5, 1e-5),
    ((33, 2056), _F32, True, 0.25, True, False, 'scaled', 0.01, 0.05),
    ((540736, 8), _BF16, True, 1.0, True, False, 'scaled', 0.01, 0.05),
]
_GS = {'none': [None] * 4, 'one': [1.0] * 4, 'scaled': [0.37] * 4,
       'skip': [1.0, 0.37, 0.0, 0.37]}   # step 2 of 'skip' carries Inf/NaN in its gradient


def _op_id(case):
  shape, gd, copy, clip, mult, hyper, gs, lr, ws = case
  return '%s-%s-%s-clip%g-%s-%s-gs_%s-lr%g-w%g' % (
      'x'.join(map(str, shape)), 'bf16' if gd == _BF16 else 'f32', 'copy' if copy else 'nocopy',
      clip, 'pscale' if mult else 'nopscale', 'hyper' if hyper else 'args', gs, lr, ws)


def _run_op_case(shape, gdtype, copy, clip, mult, use_hyper, gs_mode, lr, wscale, vr_is_rows,
                 slice_of=None):
  from lingvo_b200.ops import optim
  dev = torch.device('cuda')
  gen = torch.Generator(device=dev)
  gen.manual_seed(hash((shape, vr_is_rows)) % (1 << 31))
  r, c = shape[-2], shape[-1]
  b = math.prod(shape[:-2])
  nd = len(shape)
  d0, d1 = (nd - 1, nd - 2) if vr_is_rows else (nd - 2, nd - 1)
  w = torch.nn.Parameter(torch.randn(shape, device=dev, generator=gen) * wscale)
  if copy:
    w.compute = w.data.bfloat16()
  vr = torch.zeros((b, r) if vr_is_rows else (b, c), device=dev)
  vc = torch.zeros((b, c) if vr_is_rows else (b, r), device=dev)
  tol_v, tol_w = _sum_bound(r, c)
  tol_carry = _carried_bound(b, r, c)
  hyper = torch.zeros(2, device=dev) if use_hyper else None
  big = None
  if slice_of is not None:
    big = torch.empty(slice_of, device=dev, dtype=gdtype)
  clipped = []
  try:
    for step, gs in enumerate(_GS[gs_mode]):
      decay = _decay(step)
      if big is not None:
        big.copy_(_grad(slice_of, gen, gdtype))
        g = big[:, c:2 * c]
        assert not g.is_contiguous() and g.stride(0) != c
      else:
        g = _grad(shape, gen, gdtype)
      if gs == 0:
        g.view(-1)[7] = math.inf
        g.view(-1)[g.numel() // 2 + 3] = math.nan
      gst = None if gs is None else torch.tensor([gs], device=dev)
      if hyper is not None:
        hyper.copy_(torch.tensor([lr, decay]))
      w_old, vr_old, vc_old = w.data.clone(), vr.clone(), vc.clone()
      wb_old = w.compute.clone() if copy else None
      total = torch.zeros(1, device=dev)
      fresh = optim.adafactor_stats(w, g, d0, d1, mult, total, 0)
      assert fresh == (step == 0)
      g3 = g.reshape(b, r, c) if g.is_contiguous() else g.unsqueeze(0)
      # Σg² of the raw gradient (no grad scale, no eps1).
      g_sq = sum(float(g3[i].double().square().sum()) for i in range(b))
      if gs == 0:
        assert not math.isfinite(float(total))
      else:
        _assert_scalar(total, g_sq, 5e-5, 'sum(g^2) step %d' % step)
      # Between the two phases the carried Σw² is that of the weights being updated.
      w_sq = float(w_old.double().square().sum())
      _assert_scalar(optim.carried_sumsq(w), w_sq, tol_carry, 'carried sum(w^2) before step %d' % step)
      # With a device hyper tensor the lr / decay arguments must be ignored.
      optim.adafactor_update(w, g, vr, vc, d0, d1, 123.0 if hyper is not None else lr,
                             0.123 if hyper is not None else decay, EPS1, EPS2, clip, mult, gst,
                             fresh, hyper)
      vr_ref, vc_ref, out, clp = _factored_ref(w_old.view(b, r, c), g3, vr_old, vc_old,
                                               vr_is_rows, lr, decay, clip, mult,
                                               None if gst is None else float(gst))
      clipped.append(clp)
      _assert_rel(vr, vr_ref, tol_v, 'vr step %d' % step)
      _assert_rel(vc, vc_ref, tol_v, 'vc step %d' % step)
      wn = w.data.view(b, r, c)
      if gs == 0:
        assert torch.equal(w.data, w_old), 'skipped step changed the weights'
        if copy:
          assert torch.equal(w.compute, wb_old), 'skipped step changed the bf16 copy'
      for i, (w_ref, delta) in enumerate(out):
        _assert_w(wn[i], w_ref, delta, tol_w, 'w step %d slice %d' % (step, i))
      if copy:
        assert torch.equal(w.compute, w.data.bfloat16()), 'bf16 copy step %d' % step
      _assert_scalar(optim.carried_sumsq(w), float(w.data.double().square().sum()), tol_carry,
                     'carried sum(w^2) after step %d' % step)
  finally:
    _cleanup(w)
  return clipped


@pytest.mark.parametrize('vr_is_rows', [True, False], ids=['vr_rows', 'vr_cols'])
@pytest.mark.parametrize('case', _OP_CASES, ids=[_op_id(c) for c in _OP_CASES])
def test_adafactor_ops_match_float64(case, vr_is_rows):
  shape, gdtype, copy, clip, mult, hyper, gs_mode, lr, ws = case
  clipped = _run_op_case(shape, gdtype, copy, clip, mult, hyper, gs_mode, lr, ws, vr_is_rows)
  if clip == 0.25:
    assert any(clipped), 'the clipping case never clipped'
  if clip == 100.0:
    assert not any(clipped)


@pytest.mark.parametrize('vr_is_rows', [True, False], ids=['vr_rows', 'vr_cols'])
def test_adafactor_ops_column_slice_gradient(vr_is_rows):
  """The middle third of a [2048, 3·4104] bf16 gradient: row stride ≠ C with three 2048-column
  chunks, the last of them 8 columns wide."""
  _run_op_case((2048, 4104), _BF16, True, 1.0, True, False, 'scaled', 0.01, 0.05, vr_is_rows,
               slice_of=(2048, 3 * 4104))


# -------------------------------------------------------------------- learner level --
# name, shape, expert parallel, gradient dtype, bf16 compute copy
_VARS = [
    ('emb/var', (32000, 2048), False, _F32, True),
    ('moe/wi/var', (8, 2048, 8192), True, _BF16, True),
    ('moe/wo/var', (8, 8192, 2048), True, _BF16, True),
    ('ffw/wi/var', (2048, 8192), False, _BF16, True),
    ('ffw/wo/var', (8192, 2048), False, _BF16, False),
    ('atten/w/var', (2048, 2048), False, _BF16, True),
    ('moe/gw/var', (2048, 8), False, _F32, True),
    ('ln/scale/var', (2048,), False, _F32, False),
    ('atten/wrb/var', (16, 32), False, _BF16, True),
]
_LR = 0.01
_GRAD_MULT = [1.0, 0.2, 1.0, 3.0]     # with clip_gradient_norm_to_value=100: scale < 1, 1, skip, < 1
_BAD_STEP = 2


def _optimizer_params(streams=8):
  from lingvo_b200.core import optimizer
  return optimizer.XLAShardingAdafactor.Params().Set(
      beta1=0.0, beta2=0.99, multiply_by_parameter_scale=True, clipping_threshold=1.0,
      factored=True, decay_exponent_pow=POW, num_update_streams=streams)


def _make_vars():
  gen = torch.Generator(device='cuda')
  gen.manual_seed(11)
  out = []
  for name, shape, ep, _, copy in _VARS:
    v = torch.nn.Parameter(torch.randn(shape, device='cuda', generator=gen) * 0.05)
    v.var_name = name
    if ep:
      v.expert_parallel = True
    if copy:
      v.compute = v.data.bfloat16()
    out.append(v)
  return out


def _step_grads(step):
  gen = torch.Generator(device='cuda')
  gen.manual_seed(1000 + step)
  grads = [_grad(shape, gen, gd, _GRAD_MULT[step]) for _, shape, _, gd, _ in _VARS]
  if step == _BAD_STEP:
    grads[2].view(-1)[5] = math.inf
    grads[7][3] = math.nan
  return grads


def _slots(opt, v):
  from lingvo_b200.core import optimizer
  return opt._slots.get(optimizer._VarKey(v), {})   # pylint: disable=protected-access


def _state(opt, variables):
  """Every weight, slot and compute copy, cloned."""
  out = []
  for v in variables:
    out.append(v.data.clone())
    if getattr(v, 'compute', None) is not None:
      out.append(v.compute.clone())
    out.extend(t.clone() for _, t in sorted(_slots(opt, v).items()))
  return out


def _check_learner_step(opt, variables, grads, before, gs, step):
  decay = _decay(step)
  for v, g, (w_old, slots_old) in zip(variables, grads, before):
    name = v.var_name
    dims = opt._FactoredDims(list(v.shape))   # pylint: disable=protected-access
    slots = _slots(opt, v)
    if dims is None:
      v_old = slots_old.get('v', torch.zeros_like(w_old))
      v_ref, w_ref, delta = _small_ref(w_old, g, v_old, _LR, decay, 1.0, True, gs)
      _assert_rel(slots['v'], v_ref, 3e-5, '%s v step %d' % (name, step))
      _assert_w(v.data, w_ref, delta, 5e-5, '%s w step %d' % (name, step))
    else:
      nd = v.dim()
      r, c = v.shape[-2], v.shape[-1]
      b = v.numel() // (r * c)
      vr_is_rows = dims[0] == nd - 1
      vr_old = slots_old.get('vr', torch.zeros_like(slots['vr'])).view(b, -1)
      vc_old = slots_old.get('vc', torch.zeros_like(slots['vc'])).view(b, -1)
      vr_ref, vc_ref, out, _ = _factored_ref(w_old.view(b, r, c), g.reshape(b, r, c), vr_old,
                                             vc_old, vr_is_rows, _LR, decay, 1.0, True, gs)
      tol_v, tol_w = _sum_bound(r, c)
      _assert_rel(slots['vr'].view(b, -1), vr_ref, tol_v, '%s vr step %d' % (name, step))
      _assert_rel(slots['vc'].view(b, -1), vc_ref, tol_v, '%s vc step %d' % (name, step))
      wn = v.data.view(b, r, c)
      for i, (w_ref, delta) in enumerate(out):
        _assert_w(wn[i], w_ref, delta, tol_w, '%s w step %d slice %d' % (name, step, i))
    if gs == 0:
      assert torch.equal(v.data, w_old), '%s changed on a skipped step' % name
    if getattr(v, 'compute', None) is not None:
      assert torch.equal(v.compute, v.data.bfloat16()), '%s bf16 copy step %d' % (name, step)


def _run_learner(streams, check):
  from lingvo_b200.core import learner as learner_lib
  from lingvo_b200.core import py_utils
  from lingvo_b200.core.nested_map import NestedMap
  lrn = learner_lib.Learner.Params().Set(
      name='loss', learning_rate=1.0, clip_gradient_norm_to_value=100.0,
      optimizer=_optimizer_params(streams)).Instantiate()
  opt = lrn.optimizer
  variables = _make_vars()
  metrics = []
  try:
    for step in range(4):
      py_utils.SetGlobalStep(step)
      grads = _step_grads(step)
      before = [(v.data.clone(), {k: t.clone() for k, t in _slots(opt, v).items()})
                for v in variables] if check else None
      vg = NestedMap({v.var_name.replace('/', '_'): py_utils.VarGrad(v, g)
                      for v, g in zip(variables, grads)})
      scaled = lrn.ScaleGradients(vg, defer_scale=True)
      gs_t = lrn._deferred_scale   # pylint: disable=protected-access
      assert gs_t is not None
      opt.Apply(_LR, scaled.final_var_grads, grad_scale=gs_t)
      st = scaled.stats
      metrics.append([st[k][0].clone() for k in ('grad_norm/all', 'var_norm/all')] + [gs_t.clone()])
      if not check:
        continue
      gsq = [float(g.double().square().sum()) for g in grads]
      ep_sq = sum(s for s, (_, _, ep, _, _) in zip(gsq, _VARS) if ep)
      wsq = sum(float(w.double().square().sum()) for w, _ in before)
      gnorm = float(st['grad_norm/all'][0])
      if step == _BAD_STEP:
        assert not math.isfinite(gnorm)
        assert float(gs_t) == 0.0
      else:
        _assert_scalar(gnorm**2, sum(gsq), 5e-5, 'grad_norm/all^2 step %d' % step)
        ep_got = float(opt._pre_ep_sumsq)   # pylint: disable=protected-access
        _assert_scalar(ep_got, ep_sq, 5e-5, 'expert-parallel sum(g^2) step %d' % step)
        _assert_scalar(gnorm**2 - ep_got, sum(gsq) - ep_sq, 5e-5,
                       'dense sum(g^2) step %d' % step)
        _assert_scalar(gs_t, min(1.0, 100.0 / math.sqrt(sum(gsq))), 5e-5,
                       'grad scale step %d' % step)
      _assert_scalar(float(st['var_norm/all'][0])**2, wsq, 5e-5, 'var_norm/all^2 step %d' % step)
      _check_learner_step(opt, variables, grads, before, float(gs_t), step)
    return _state(opt, variables), metrics
  finally:
    _cleanup(*variables)


def test_learner_adafactor_steps_match_float64():
  """Four learner steps (global-norm clip, one non-finite step) over one full-size variable of
  each benchmark kind; the same run on a single stream is bitwise identical."""
  state8, metrics8 = _run_learner(8, check=True)
  state1, metrics1 = _run_learner(1, check=False)
  assert len(state8) == len(state1)
  for a, b in zip(state8, state1):
    assert torch.equal(a, b)
  for a, b in zip(metrics8, metrics1):     # grad norm, var norm, grad scale: bitwise
    for x, y in zip(a, b):
      assert torch.equal(x.reshape(1).view(torch.int32), y.reshape(1).view(torch.int32))


def test_graphed_adafactor_step_matches_eager_device_hyper():
  """One captured PreGradStats + Apply step, replayed with changing SetHyper(lr, step), equals
  the same steps run eagerly with device hyper-parameters, bitwise, slots included."""
  from lingvo_b200.core import py_utils
  from lingvo_b200.core.nested_map import NestedMap
  dev = torch.device('cuda')
  lrs = [0.01, 0.02, 0.005, 0.01]

  def setup():
    opt = _optimizer_params().Set(name='adafactor').Instantiate()
    opt.EnableDeviceHyper(dev)
    variables = _make_vars()
    grads = [torch.empty(s, device=dev, dtype=gd) for _, s, _, gd, _ in _VARS]
    gs = torch.ones(1, device=dev)
    vg = NestedMap({v.var_name.replace('/', '_'): py_utils.VarGrad(v, g)
                    for v, g in zip(variables, grads)})
    return opt, variables, grads, gs, vg

  def feed(grads, gs, step):
    for dst, src in zip(grads, _step_grads(step)):
      dst.copy_(src)
    gs.fill_(0.0 if step == _BAD_STEP else 0.37 + 0.1 * step)

  def step_fn(opt, variables, grads, gs, vg):
    opt.PreGradStats([(v, g) for v, g in zip(variables, grads)])
    opt.Apply(_LR, vg, grad_scale=gs)

  eager = setup()
  graphed = setup()
  try:
    # step 0: eager on both (the graphed one on a side stream, as capture requires)
    py_utils.SetGlobalStep(0)
    feed(eager[2], eager[3], 0)
    eager[0].SetHyper(lrs[0], 0)
    step_fn(*eager)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      feed(graphed[2], graphed[3], 0)
      graphed[0].SetHyper(lrs[0], 0)
      step_fn(*graphed)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode='thread_local'):
      step_fn(*graphed)
    torch.cuda.synchronize()
    for a, b in zip(_state(eager[0], eager[1]), _state(graphed[0], graphed[1])):
      assert torch.equal(a, b)
    for step in range(1, 4):
      py_utils.SetGlobalStep(step)
      feed(eager[2], eager[3], step)
      eager[0].SetHyper(lrs[step], step)
      step_fn(*eager)
      feed(graphed[2], graphed[3], step)
      graphed[0].SetHyper(lrs[step], step)
      graph.replay()
      sa, sb = _state(eager[0], eager[1]), _state(graphed[0], graphed[1])
      assert len(sa) == len(sb)
      for i, (a, b) in enumerate(zip(sa, sb)):
        assert torch.equal(a, b), 'state tensor %d differs after replayed step %d' % (i, step)
  finally:
    _cleanup(*eager[1], *graphed[1])


# ------------------------------------------------------------------------------ Adam --
@pytest.mark.parametrize('gdtype', [_BF16, _F32], ids=['bf16', 'f32'])
@pytest.mark.parametrize('scale_kind', ['scalar', 'tensor'])
@pytest.mark.parametrize('size', ['n8', 'grid_stride'])
def test_adam_flat_matches_float64(size, scale_kind, gdtype):
  from lingvo_b200.ops import optim
  dev = torch.device('cuda')
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  # Past the capped grid (8 CTAs per SM of 256 threads, 8 elements each) with a ragged tail.
  n = 8 if size == 'n8' else 2 * sms * 8 * 256 * 8 + 8 * 37
  gen = torch.Generator(device=dev)
  gen.manual_seed(n)
  w = torch.randn(n, device=dev, generator=gen) * 0.05
  m = torch.zeros(n, device=dev)
  v = torch.zeros(n, device=dev)
  wb = torch.empty(n, device=dev, dtype=_BF16)
  f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))   # the kernel's fp32 arguments
  b1, b2, eps, lr_t = f32(0.9), f32(0.98), f32(1e-8), f32(1e-3)
  for step in range(3):
    g = (torch.randn(n, device=dev, generator=gen) * 0.01).to(gdtype)
    if scale_kind == 'scalar':
      gs_arg, gs_t, gs = 0.37, None, f32(0.37)
    else:
      gs_arg, gs_t = 2.0, torch.tensor([0.185], device=dev)
      gs = f32(2.0 * f32(0.185))
    w0, m0, v0 = w.clone(), m.clone(), v.clone()
    optim.adam_flat(w, g, m, v, wb, lr_t, b1, b2, eps, grad_scale=gs_arg, grad_scale_t=gs_t)
    gg = g.double() * gs
    mt, vt = b1 * m0.double(), (1 - b1) * gg
    m_ref = mt + vt
    assert bool(((m.double() - m_ref).abs() <= 4 * U * (mt.abs() + vt.abs()) + 1e-30).all())
    v_ref = b2 * v0.double() + (1 - b2) * gg.square()
    _assert_rel(v, v_ref, 6 * U, 'adam v step %d' % step)
    # The weight update from the kernel's own m and v: a few roundings of |Δ|.
    delta = lr_t * m.double() / (v.double().sqrt() + eps)
    _assert_w(w, w0.double() - delta, delta, 8 * U, 'adam w step %d' % step)
    assert torch.equal(wb, w.bfloat16())
