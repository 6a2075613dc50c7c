"""Fused sm_90a kernels vs plain PyTorch fp32 references."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
  """Worst of (i) the whole-tensor relative error and (ii) the worst *per-row* error, each
  row normalised by its own norm (rows with a smaller-than-median norm by the median) — so
  a mistake confined to a few rows cannot hide behind the tensor's largest entries."""
  a, b = a.float(), b.float()
  whole = ((a - b).abs().max() / (b.abs().max() + 1e-6)).item()
  if a.dim() < 2 or a.shape[-1] < 8:
    return whole
  a2, b2 = a.reshape(-1, a.shape[-1]), b.reshape(-1, b.shape[-1])
  rn = b2.norm(dim=-1)
  den = torch.maximum(rn, rn.median()) + 1e-12
  rows = ((a2 - b2).norm(dim=-1) / den).max().item()
  return max(whole, rows)


@pytest.mark.parametrize('dim', [256, 2048, 4096])
def test_rms_norm(dim):
  from lingvo_b200.ops import norm
  x = torch.randn(300, dim, device='cuda').bfloat16().requires_grad_()
  scale = (torch.rand(dim, device='cuda') + 0.5).requires_grad_()
  y = norm.rms_norm(x, scale, 1e-6)
  dy = torch.randn_like(y)
  y.backward(dy)
  xr = x.detach().float().requires_grad_()
  sr = scale.detach().clone().requires_grad_()
  yr = xr * torch.rsqrt(xr.square().mean(-1, keepdim=True) + 1e-6) * sr
  yr.backward(dy.float())
  assert _rel(y, yr) < 2e-2
  assert _rel(x.grad, xr.grad) < 3e-2
  assert _rel(scale.grad, sr.grad) < 3e-2


def test_layer_norm():
  from lingvo_b200.ops import norm
  dim = 1024
  x = torch.randn(200, dim, device='cuda').bfloat16().requires_grad_()
  scale = (torch.rand(dim, device='cuda') + 0.5).requires_grad_()
  bias = torch.randn(dim, device='cuda').requires_grad_()
  y = norm.layer_norm(x, scale, bias, 1e-6)
  dy = torch.randn_like(y)
  y.backward(dy)
  xr = x.detach().float().requires_grad_()
  sr = scale.detach().clone().requires_grad_()
  br = bias.detach().clone().requires_grad_()
  yr = torch.nn.functional.layer_norm(xr, (dim,), sr, br, 1e-6)
  yr.backward(dy.float())
  assert _rel(y, yr) < 2e-2
  assert _rel(x.grad, xr.grad) < 3e-2
  assert _rel(scale.grad, sr.grad) < 3e-2
  assert _rel(bias.grad, br.grad) < 3e-2


@pytest.mark.parametrize('shape', [(512, 1024), (1024, 256), (4, 256, 512)])
@pytest.mark.parametrize('gdtype', [torch.bfloat16, torch.float32])
def test_adafactor_matches_reference(shape, gdtype):
  from lingvo_b200.core import optimizer, py_utils
  torch.manual_seed(0)
  w0 = torch.randn(shape, device='cuda')
  grads = [torch.randn(shape, device='cuda').to(gdtype) * 0.1 for _ in range(3)]

  def run(fused):
    p = optimizer.XLAShardingAdafactor.Params().Set(
        name='adafactor', beta1=0.0, beta2=0.99, clipping_threshold=1.0,
        factored=True, decay_exponent_pow=0.8, fused=fused)
    opt = p.Instantiate()
    w = torch.nn.Parameter(w0.clone())
    w.var_name = 'w/var'
    if gdtype == torch.bfloat16:
      w.compute = w.data.bfloat16().requires_grad_()
    for step, g in enumerate(grads):
      with py_utils.GlobalStepContext(step):
        opt.Apply(0.01, [py_utils.VarGrad(w, g)])
    return w

  a, b = run(True), run(False)
  assert _rel(a, b) < 1e-4
  if gdtype == torch.bfloat16:
    assert torch.equal(a.compute.data, a.data.bfloat16())


def _ordered_bf16(b):
  """bf16 bit patterns mapped to integers that are consecutive for adjacent bf16 values."""
  i = b.contiguous().view(torch.int16).int()
  return torch.where(i < 0, -(i & 0x7fff), i)


def _assert_within_bf16_ulp(got, want, slack):
  """bf16 `got` is fp32 `want` rounded to bf16 up to one ulp. Where the fp32 terms of an
  element nearly cancel, `got` may instead be within `slack` of `want`."""
  ulps = (_ordered_bf16(got) - _ordered_bf16(want.bfloat16())).abs()
  bad = (ulps > 1) & ~((got.float() - want).abs() <= slack)
  assert not bool(bad.any()), '%d elements off by more than 1 bf16 ulp' % int(bad.sum())


def test_ffn_relu():
  from lingvo_b200.ops import gemm
  x = torch.randn(384, 256, device='cuda').bfloat16().requires_grad_()
  wi = (torch.randn(256, 512, device='cuda') * 0.05).bfloat16().requires_grad_()
  wo = (torch.randn(512, 256, device='cuda') * 0.05).bfloat16().requires_grad_()
  y = gemm.ffn_relu(x, wi, wo)
  dy = torch.randn_like(y)
  y.backward(dy)
  xr, wir, wor = [t.detach().float().requires_grad_() for t in (x, wi, wo)]
  yr = torch.relu(xr @ wir) @ wor
  yr.backward(dy.float())
  for a, b in ((y, yr), (x.grad, xr.grad), (wi.grad, wir.grad), (wo.grad, wor.grad)):
    assert _rel(a, b) < 3e-2


@pytest.mark.parametrize('causal', [False, True])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
def test_glu_dwconv1d_kernel(causal, dtype):
  from lingvo_b200.ops import conv as C
  torch.manual_seed(0)
  dev = torch.device('cuda')
  b, t, d, k = 3, 77, 200, 9
  proj = torch.randn(b, t, 2 * d, device=dev).to(dtype).requires_grad_()
  w = (torch.randn(k, d, device=dev) * 0.3).requires_grad_()
  pad = torch.zeros(b, t, device=dev)
  pad[1, 50:] = 1
  pad[2, 10:] = 1
  dy = torch.randn(b, t, d, device=dev).to(dtype)
  y = C.glu_dwconv1d(proj, w, pad, causal)
  y.backward(dy)
  got = [y.detach().float(), proj.grad.float().clone(), w.grad.clone()]
  proj.grad = None; w.grad = None
  pr = proj.detach().float().requires_grad_()
  wr = w.detach().clone().requires_grad_()
  yr = C.glu_dwconv1d_ref(pr, wr, pad, causal)
  yr.backward(dy.float())
  tol = 3e-2 if dtype == torch.bfloat16 else 1e-4
  for name, g, r in zip(['y', 'dproj', 'dw'], got, [yr.detach(), pr.grad, wr.grad]):
    err = float((g - r).norm() / r.norm().clamp_min(1e-6))
    assert err < tol, (name, err)


def test_adafactor_small_multi_tensor_matches_python_path():
  """One-launch non-factored Adafactor == the per-variable PyTorch implementation."""
  from lingvo_b200.core import optimizer as opt_lib
  from lingvo_b200.core import py_utils
  from lingvo_b200.core.nested_map import NestedMap
  dev = torch.device('cuda')
  torch.manual_seed(0)
  shapes = [(2048,), (16, 32), (2048, 8), (77,)]

  def make():
    vs = [torch.nn.Parameter(torch.randn(s, device=dev) * 0.5) for s in shapes]
    for i, v in enumerate(vs):
      v.var_name = 'v%d/var' % i
    return vs
  a, b = make(), make()
  for x, y in zip(a, b):
    y.data.copy_(x.data)
  pa = opt_lib.XLAShardingAdafactor.Params().Set(
      name='a', beta1=0.0, beta2=0.99, multiply_by_parameter_scale=True,
      clipping_threshold=1.0, factored=True, decay_exponent_pow=0.8)
  fa = pa.Instantiate()
  fb = pa.Copy().Set(fused=False).Instantiate()
  for step in range(3):
    py_utils.SetGlobalStep(step)
    grads = [torch.randn_like(v) * (0.1 + step) for v in a]
    fa.Apply(0.01, NestedMap({'v%d' % i: py_utils.VarGrad(v, g.to(torch.bfloat16) if i % 2 else g)
                              for i, (v, g) in enumerate(zip(a, grads))}))
    fb.Apply(0.01, NestedMap({'v%d' % i: py_utils.VarGrad(v, (g.to(torch.bfloat16).float() if i % 2 else g))
                              for i, (v, g) in enumerate(zip(b, grads))}))
  for x, y in zip(a, b):
    torch.testing.assert_close(x.data, y.data, atol=2e-5, rtol=2e-4)


def test_graphed_train_step_matches_eager():
  """CUDA-graph replay of the whole train step reproduces the eager losses."""
  from lingvo_b200 import model_registry
  from lingvo_b200.core import cluster_factory
  from lingvo_b200.core import graph_step
  import lingvo_b200.models.lm.params.synthetic_packed_input  # noqa: F401
  dev = torch.device('cuda', 0)

  def build():
    cfg = model_registry.GetParams('lm.synthetic_packed_input.MoELm8ETiny', 'Train')
    cfg.task.random_seed = 3
    cfg.input.random_seed = 9
    cfg.cluster.worker.gpus_per_replica = 1
    return cfg
  losses = {}
  for mode in ('eager', 'graph'):
    cfg = build()
    with cluster_factory.Cluster(cfg.cluster):
      m = cfg.Instantiate()
      m.to(dev)
      task = m.tasks[0]
      batch = task._MoveBatch(task.input.GetPreprocessedInputBatch(), dev)
      out = []
      if mode == 'eager':
        for _ in range(6):
          mt, _ = task.TrainStep([batch])
          out.append(float(mt['loss'][0]))
        out = out[3:]
      else:
        g = graph_step.GraphedTrainStep(task, batch, warmup=3)
        assert g.launches_per_step > 10
        for _ in range(3):
          mt, _ = g(batch)
          out.append(float(mt['loss'][0]))
      losses[mode] = out
  for x, y in zip(losses['eager'], losses['graph']):
    assert abs(x - y) < 2e-3 * max(1.0, abs(x)), losses
  assert losses['graph'][-1] < losses['graph'][0]


@pytest.mark.parametrize('t,m,e,wdtype', [(8192, 2048, 8, torch.bfloat16), (1000, 1024, 4, torch.float32),
                                          (37, 2056, 16, torch.bfloat16), (3, 64, 2, torch.float32)])
def test_gate_logits_matches_fp32_oracle(t, m, e, wdtype):
  from lingvo_b200.ops import gate
  torch.manual_seed(0)
  x = torch.randn(t, m, device='cuda').to(torch.bfloat16).requires_grad_(True)
  gw = (torch.randn(m, e, device='cuda') * 0.05).to(wdtype).requires_grad_(True)
  assert gate.supported(x, gw)
  y = gate.gate_logits(x, gw)
  assert y.dtype == torch.float32 and y.shape == (t, e)
  dl = torch.randn(t, e, device='cuda')
  dx, dgw = torch.autograd.grad(y, [x, gw], dl)
  xr = x.detach().float().requires_grad_(True)
  gr = gw.detach().float().requires_grad_(True)
  yr = gate.gate_logits_ref(xr, gr)
  dxr, dgr = torch.autograd.grad(yr, [xr, gr], dl)
  torch.testing.assert_close(y, yr, atol=2e-3, rtol=1e-3)
  torch.testing.assert_close(dx.float(), dxr, atol=2e-2, rtol=2e-2)       # bf16 output
  tol = 3e-2 if wdtype == torch.bfloat16 else 2e-3
  torch.testing.assert_close(dgw.float(), dgr, atol=tol * dgr.abs().max().item(), rtol=tol)
  # 3-D input keeps its leading dims
  y3 = gate.gate_logits(x.detach().reshape(1, t, m), gw.detach())
  assert y3.shape == (1, t, e)


def test_adafactor_accepts_column_slice_gradients():
  """dwq/dwk/dwv arrive as column slices of the fused qkv gradient: the fused kernels read
  them in place and must match the step taken on contiguous copies."""
  from lingvo_b200.core import optimizer, py_utils
  torch.manual_seed(1)
  k, n = 512, 256
  fused_grads = [torch.randn(k, 3 * n, device='cuda').to(torch.bfloat16) * 0.1 for _ in range(3)]
  w0 = [torch.randn(k, n, device='cuda') for _ in range(3)]

  def run(slice_views):
    opt = optimizer.XLAShardingAdafactor.Params().Set(
        name='adafactor', beta1=0.0, beta2=0.99, clipping_threshold=1.0, factored=True,
        decay_exponent_pow=0.8, fused=True).Instantiate()
    ws = []
    for i, w in enumerate(w0):
      p = torch.nn.Parameter(w.clone())
      p.var_name = 'w%d/var' % i
      p.compute = p.data.bfloat16().requires_grad_()
      ws.append(p)
    for step, fg in enumerate(fused_grads):
      views = [fg[:, i * n:(i + 1) * n] for i in range(3)]
      assert not views[1].is_contiguous()
      gs = views if slice_views else [v.contiguous() for v in views]
      with py_utils.GlobalStepContext(step):
        opt.Apply(0.01, [py_utils.VarGrad(w, g) for w, g in zip(ws, gs)])
    return ws

  a, b = run(True), run(False)
  for x, y in zip(a, b):
    assert _rel(x, y) < 1e-6
    assert torch.equal(x.compute.data, x.data.bfloat16())


def test_embed_rows_backward_matches_dense_embedding_backward():
  from lingvo_b200.core import gshard_builder
  import torch.nn.functional as F
  torch.manual_seed(0)
  w = torch.randn(1000, 64, device='cuda').to(torch.bfloat16).requires_grad_(True)
  ids = torch.randint(0, 50, (4, 128), device='cuda')          # many duplicates
  dy = torch.randn(4, 128, 64, device='cuda').to(torch.bfloat16)
  out = gshard_builder._EmbedRows.apply(w, ids)
  (dw,) = torch.autograd.grad(out, w, dy)
  w2 = w.detach().float().requires_grad_(True)
  ref = F.embedding(ids, w2)
  (dw2,) = torch.autograd.grad(ref, w2, dy.float())
  assert torch.equal(out, F.embedding(ids, w.detach()))
  torch.testing.assert_close(dw.float(), dw2, atol=2e-2, rtol=1e-2)


def test_rms_norm_pass_fuses_residual_gradient():
  """x_pass + f(norm(x)) through `_NormPassFn` == the plain two-branch graph."""
  from lingvo_b200.ops import norm
  torch.manual_seed(0)
  x = (torch.randn(512, 1024, device='cuda')).to(torch.bfloat16).requires_grad_(True)
  scale = torch.rand(1024, device='cuda').add(0.5).requires_grad_(True)
  w = (torch.randn(1024, 1024, device='cuda') * 0.03).to(torch.bfloat16)
  dy = torch.randn(512, 1024, device='cuda').to(torch.bfloat16)
  xn, xp = norm.rms_norm_pass(x, scale, 1e-6)
  y = xp + xn @ w
  gx, gs = torch.autograd.grad(y, [x, scale], dy)
  xr = x.detach().float().requires_grad_(True)
  sr = scale.detach().clone().requires_grad_(True)
  yr = xr + (norm.rms_norm_ref(xr, sr, 1e-6) @ w.float())
  gxr, gsr = torch.autograd.grad(yr, [xr, sr], dy.float())
  torch.testing.assert_close(y.float(), yr, atol=5e-2, rtol=2e-2)
  torch.testing.assert_close(gx.float(), gxr, atol=6e-2, rtol=3e-2)
  torch.testing.assert_close(gs, gsr, atol=0.5, rtol=3e-2)
  # only the residual branch used → gradient passes straight through
  xn2, xp2 = norm.rms_norm_pass(x, scale, 1e-6)
  (g_only,) = torch.autograd.grad(xp2, x, dy)
  assert torch.equal(g_only, dy)


def test_gate_logits_pass_adds_the_other_branch_gradient():
  from lingvo_b200.ops import gate
  torch.manual_seed(0)
  t, m, e = 777, 512, 8
  x = torch.randn(t, m, device='cuda').to(torch.bfloat16).requires_grad_(True)
  gw = (torch.randn(m, e, device='cuda') * 0.05).to(torch.bfloat16).requires_grad_(True)
  w2 = (torch.randn(m, m, device='cuda') * 0.03).to(torch.bfloat16)
  dl = torch.randn(t, e, device='cuda')
  dy = torch.randn(t, m, device='cuda').to(torch.bfloat16)
  logits, xp = gate.gate_logits_pass(x, gw)
  other = xp @ w2                                   # second consumer of x
  gx, ggw = torch.autograd.grad([logits, other], [x, gw], [dl, dy])
  xr = x.detach().float().requires_grad_(True)
  gr = gw.detach().float().requires_grad_(True)
  gxr, ggr = torch.autograd.grad([gate.gate_logits_ref(xr, gr), xr @ w2.float()], [xr, gr], [dl, dy.float()])
  torch.testing.assert_close(gx.float(), gxr, atol=6e-2, rtol=3e-2)
  torch.testing.assert_close(ggw.float(), ggr, atol=3e-2 * ggr.abs().max().item(), rtol=3e-2)


@pytest.mark.parametrize('b,l,h,use_rel,segs,causal', [
    (1, 128, 1, False, 0, True),
    (2, 256, 2, True, 0, True),
    (2, 256, 2, True, 0, False),
    (2, 384, 2, True, 3, True),
    (2, 512, 4, False, 4, False),
])
def test_flash_attention_wgmma_matches_fp32_oracle(b, l, h, use_rel, segs, causal):
  """Our flash attention (fwd, dQ/dK/dV, d rel-bias) vs the plain fp32 softmax oracle, with
  packed segments + padding, causal and bidirectional."""
  from lingvo_b200.ops import attention as A
  torch.manual_seed(b * 1000 + l + h)
  d = 128
  qkv = (torch.randn(b, l, 3 * h * d, device='cuda') * 0.5).bfloat16()
  q, k, v = [t.reshape(b, l, h, d).detach().requires_grad_(True)
             for t in qkv.split(h * d, dim=-1)]          # strided views of a fused projection
  assert A.flash_attention_supported(q, k)
  rel = torch.randn(h, 2 * l - 1, device='cuda').requires_grad_(True) if use_rel else None
  seg = pos = None
  if segs:
    seg = torch.zeros(b, l, dtype=torch.int32, device='cuda')
    pos = torch.zeros(b, l, dtype=torch.int32, device='cuda')
    for bi in range(b):
      n_valid = l - (37 if bi % 2 else 0)
      cuts = sorted(torch.randperm(n_valid - 1)[:segs - 1].add(1).tolist()) + [n_valid]
      start = 0
      for si, end in enumerate(cuts):
        seg[bi, start:end] = si + 1
        pos[bi, start:end] = torch.arange(end - start, device='cuda', dtype=torch.int32)
        start = end
  d_o = (torch.randn(b, l, h, d, device='cuda') * 0.5).bfloat16()
  valid = (seg != 0) if seg is not None else torch.ones(b, l, dtype=torch.bool, device='cuda')
  d_o = d_o * valid[:, :, None, None].to(d_o.dtype)
  wrt = [q, k, v] + ([rel] if use_rel else [])
  out = A.flash_attention(q, k, v, rel, seg, pos, 1.0, causal)
  grads = torch.autograd.grad(out, wrt, d_o)
  ref = A.flash_attention_ref(q, k, v, rel, seg, pos, 1.0, causal)
  rgrads = torch.autograd.grad(ref, wrt, d_o.float())
  assert _rel(out[valid], ref[valid]) < 2e-2
  for name, g, rg in zip(['dq', 'dk', 'dv'], grads, rgrads):
    assert _rel(g[valid], rg[valid]) < 4e-2, name
  if use_rel:
    err = ((grads[3] - rgrads[3]).norm() / rgrads[3].norm()).item()
    assert err < 1e-2, err


def test_flash_attention_backward_is_reproducible_across_key_block_launches():
  """L = 1280 spans two backward launches of key blocks. The gradients match the oracle, and
  repeated runs on the same inputs give bit-identical dQ, dK, dV and d rel-bias: the partial
  sums are folded in a fixed order, not by atomics."""
  from lingvo_b200.ops import attention as A
  torch.manual_seed(7)
  b, l, h, d = 1, 1280, 2, 128
  q, k, v = [(torch.randn(b, l, h, d, device='cuda') * 0.5).bfloat16().requires_grad_(True)
             for _ in range(3)]
  rel = torch.randn(h, 2 * l - 1, device='cuda').requires_grad_(True)
  seg = torch.ones(b, l, dtype=torch.int32, device='cuda')
  seg[:, 700:] = 2
  pos = torch.cat([torch.arange(700), torch.arange(l - 700)]).int().cuda().unsqueeze(0)
  d_o = (torch.randn(b, l, h, d, device='cuda') * 0.5).bfloat16()
  wrt = [q, k, v, rel]
  runs = []
  for _ in range(3):
    out = A.flash_attention(q, k, v, rel, seg, pos, 1.0, True)
    runs.append(torch.autograd.grad(out, wrt, d_o))
  for again in runs[1:]:
    for name, g0, g1 in zip(['dq', 'dk', 'dv', 'drel'], runs[0], again):
      assert torch.equal(g0, g1), name
  ref = A.flash_attention_ref(q, k, v, rel, seg, pos, 1.0, True)
  rgrads = torch.autograd.grad(ref, wrt, d_o.float())
  for name, g, rg in zip(['dq', 'dk', 'dv'], runs[0], rgrads):
    assert _rel(g, rg) < 4e-2, name
  err = ((runs[0][3] - rgrads[3]).norm() / rgrads[3].norm()).item()
  assert err < 1e-2, err


def test_flash_attention_reference_quirk_positions_are_not_assumed_causal():
  """`segment_pos` all equal (the reference's synthetic input) makes every key visible even
  in a decoder: block skipping must come from the data, not from the index."""
  from lingvo_b200.ops import attention as A
  torch.manual_seed(3)
  b, l, h, d = 1, 256, 1, 128
  q, k, v = [(torch.randn(b, l, h, d, device='cuda') * 0.5).bfloat16() for _ in range(3)]
  seg = torch.ones(b, l, dtype=torch.int32, device='cuda')
  pos = torch.ones(b, l, dtype=torch.int32, device='cuda')
  out = A.flash_attention(q, k, v, None, seg, pos, 1.0, True)
  ref = A.flash_attention_ref(q, k, v, None, seg, pos, 1.0, True)
  assert _rel(out, ref) < 2e-2


@pytest.mark.parametrize('k,v,dtype', [(4, 1000, torch.float32), (8, 32000, torch.float32),
                                       (3, 4099, torch.bfloat16), (16, 515, torch.float32)])
def test_beam_topk_kernel_matches_torch_oracle(k, v, dtype):
  """K13: fused score-add + EOS mask + per-hyp top-K vs the plain PyTorch formulation,
  including the (score desc, word id asc) tie order."""
  from lingvo_b200.ops import beam_search as bs
  torch.manual_seed(k + v)
  n = 24
  lp = torch.log_softmax(torch.randn(n, v, device='cuda') * 3, -1)
  lp[:, 7] = lp[:, 11]                                   # exact ties
  lp = lp.to(dtype)
  cum = torch.randn(n, device='cuda')
  active = torch.rand(n, device='cuda') > 0.2
  got = bs._TopK(lp, cum, active, k, 2)
  want = bs._TopKRef(lp, cum, active, k, 2)
  torch.testing.assert_close(got[0], want[0])
  assert torch.equal(got[1], want[1])
  for a, b in zip(got[2:], want[2:]):
    torch.testing.assert_close(a, b)


def test_moe_row_movers_match_oracles():
  """ops/moe.py: token-major combine / gather / gate-gradient kernels vs fp32 oracles, on
  random slots (which may collide)."""
  torch.manual_seed(0)
  e, g, c, m, s = 8, 4, 64, 512, 96
  t = g * s
  dev = 'cuda'
  yc = torch.randn(e, g, c, m, device=dev).bfloat16()
  index = torch.randint(0, e, (2, t), device=dev, dtype=torch.int32)
  pos = torch.randint(0, c, (2, t), device=dev, dtype=torch.int32)
  gate = torch.rand(2, t, device=dev)
  gate[torch.rand(2, t, device=dev) < 0.2] = 0.0                 # dropped choices
  _check_row_movers(yc, index, pos, gate, s, g, c)


@pytest.mark.parametrize('m', [2048, 328])    # 328: not a multiple of the 256-column lane stride
def test_moe_row_movers_on_gate_kernel_routing(m):
  """The row movers on the (index, pos, gate) `moe_gate_dispatch` itself produces, at the
  benchmark's MoE geometry (E = 8, G = 8 groups of S = 1024 tokens, C = 256)."""
  from lingvo_b200 import ops
  torch.manual_seed(0)
  e, g, c, s = 8, 8, 256, 1024
  t = g * s
  dev = 'cuda'
  yc = torch.randn(e, g, c, m, device=dev).bfloat16()
  logits = torch.randint(-256, 257, (g, s, e), device=dev).float() / 64
  logits[..., 1] += 2.0                                           # overflows capacity
  no_peers = torch.zeros(1, dtype=torch.int64, device=dev)
  index, pos, gate, _ = ops.native().moe_gate_dispatch(logits, None, None, no_peers, c, e, 0, 1,
                                                        False)
  index, pos, gate = index.view(2, t), pos.view(2, t), gate.view(2, t)
  assert bool((gate == 0).any()) and bool((gate != 0).any())
  _check_row_movers(yc, index, pos, gate, s, g, c)


def _check_row_movers(yc, index, pos, gate, s, g, c):
  """combine / gather_rows to one bf16 ulp of the fp32 oracles, combine_bwd_gate to 1e-5 of
  the sum of |products|; dropped choices give exactly 0."""
  from lingvo_b200.ops import moe
  t, m = index.shape[-1], yc.shape[-1]
  slack = 2.0**-22 * moe.combine_ref(yc.abs(), index, pos, gate.abs(), s, g, c)
  y = moe.combine(yc, index, pos, gate, s, g, c)
  want = moe.combine_ref(yc, index, pos, gate, s, g, c)
  assert _rel(y, want) < 1e-2
  _assert_within_bf16_ulp(y, want, slack)
  ga = moe.gather_rows(yc, index, pos, gate, s, g, c)
  want = moe.gather_rows_ref(yc, index, pos, gate, s, g, c)
  assert _rel(ga, want) < 1e-2
  _assert_within_bf16_ulp(ga, want, 2.0**-22 * moe.gather_rows_ref(yc.abs(), index, pos, gate,
                                                                   s, g, c))
  dy = torch.randn(t, m, device=yc.device).bfloat16()
  dg = moe.combine_bwd_gate(yc, dy, index, pos, gate, s, g, c)
  ref = moe.combine_bwd_gate_ref(yc, dy, index, pos, gate, s, g, c)
  assert _rel(dg, ref) < 1e-2 and bool((dg[gate == 0] == 0).all())
  bound = 1e-5 * moe.combine_bwd_gate_ref(yc.abs(), dy.abs(), index, pos, gate, s, g, c)
  assert bool(((dg - ref).abs() <= bound).all())
