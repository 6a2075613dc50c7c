"""Soft-capped logits and an extra logit in the wgmma flash attention (ops/csrc/flash_attn.cu),
against a float64 oracle written from the formula, and the decode steps of a capped,
extra-logit LM against its forward.

Contract checked here, for `flash_attention(q, k, v, rel, seg, pos, scale, causal, logit_cap,
extra_logit)` with s_ij = scale·q_i·k_j:
  * z_ij = (cap > 0 ? cap·tanh(s_ij / cap) : s_ij) + rel[h, i-j+L-1] on the pairs i sees (the
    mask of `test_flash_attn_gpu.py`); the bias and the mask come after the cap;
  * O_i = Σ_j softmax(z_i ∪ {extra})_j · v_j, the extra slot having value 0, and
    lse_i = log(Σ_j exp z_ij + [extra given]·exp(extra));
  * with an extra logit, a query that sees no key returns exactly 0 and lse == extra; without
    one, such a query's forward is unspecified but finite. Either way it contributes nothing
    to the backward, a key no query sees has zero dK and dV, and an unused diagonal has zero
    d rel;
  * d rel is built from dS = P∘(dP - delta), dQ and dK from dS∘(1 - tanh²)·scale.

The bounds are those of `test_flash_attn_gpu.py` (c·2^-8·A + 1 bf16 ulp) plus the error of
the kernels' tanh, 1 - 2/(1 + 2^(2u·log2e)) with ex2.approx and rcp.approx: it is within 2^-20
of tanh(u) for every u, so a logit moves by at most cap·2^-20, which changes P by that much
relative, and 1 - tanh² moves by at most 2^-20 absolute. `_TANH` = 2^-18 covers both terms with
a factor 4.

The CPU tests check the oracle itself against `flash_attention_ref` and fp32 autograd, and
that a capped, extra-logit decoder LM decodes, token by token and by flat beam search, what
its teacher-forced forward computes.
"""
import math

import pytest
import torch

import test_flash_attn_gpu as TF
from lingvo_b200 import ops
from lingvo_b200.core import cluster_factory
from lingvo_b200.core import gshard_builder as gb
from lingvo_b200.core import gshard_decode
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.ops import attention as A

_D = 128
_TANH = 2.0**-18
# (logit_cap, extra_logit): the reference's cap of 50, the extra logit alone, both, and a small
# cap (most scores beyond it) with a negative extra logit.
_OPTIONS = [(50.0, None), (0.0, 0.0), (50.0, 0.0), (5.0, -2.0)]
_OPTION_IDS = ['cap50', 'extra0', 'cap50-extra0', 'cap5-extra-2']


# ------------------------------------------------------------------ the oracle ----
def _Oracle(q, k, v, rel, seg, pos, scale, causal, d_o, cap, extra):
  """Float64 forward and closed-form backward, one batch element at a time, plus the |.|
  contractions of the bounds. k, v have Hk heads; dK, dV are summed over each group."""
  b, l, h, d = q.shape
  hk = k.shape[2]
  g = h // hk
  dev = q.device
  f = lambda t: t.double().permute(1, 0, 2)                     # [L, H, D] → [H, L, D]
  fk = lambda t: f(t).repeat_interleave(g, dim=0)               # KV head h // G
  relt = TF._Toeplitz(rel.double(), l) if rel is not None else None
  vis_all = TF._Visible(seg, pos, causal, b, l, dev)
  r = {n: torch.zeros(b, l, h, d, dtype=torch.float64, device=dev)
       for n in ('out', 'a_out', 'dq', 'a_dq', 'a_dq0')}
  for n in ('dk', 'a_dk', 'a_dk0', 'dv', 'a_dv'):
    r[n] = torch.zeros(b, l, hk, d, dtype=torch.float64, device=dev)
  r['lse'] = torch.zeros(b, h, l, dtype=torch.float64, device=dev)
  r['a_lse'] = torch.zeros(b, h, l, dtype=torch.float64, device=dev)
  for n in ('drel', 'drel_delta', 'drel_abs'):
    r[n] = torch.zeros(h, 2 * l - 1, dtype=torch.float64, device=dev)
  r['live'] = vis_all.any(-1)
  r['seen'] = vis_all.any(-2)
  r['used'] = TF._DiagSum(vis_all.double()).sum(0) > 0
  fold = lambda t: t.reshape(hk, g, l, d).sum(1).permute(1, 0, 2)   # [H, L, D] → [L, Hk, D]
  for bi in range(b):
    qb, kb, vb, dob = f(q[bi]), fk(k[bi]), fk(v[bi]), f(d_o[bi])
    vis = vis_all[bi]
    s = scale * qb @ kb.transpose(-1, -2)
    a_s = scale * qb.abs() @ kb.abs().transpose(-1, -2)
    if cap > 0:
      t = torch.tanh(s / cap)
      z, a_z, dz = cap * t, (cap * t).abs(), 1 - t * t
      del t
    else:
      z, a_z, dz = s, a_s, torch.ones_like(s)
    del s
    if relt is not None:
      z, a_z = z + relt, a_z + relt.abs()
    r['a_lse'][bi] = torch.where(vis, torch.maximum(a_s, a_z), 0.0).amax(-1)
    del a_s, a_z
    zm = torch.where(vis, z, -math.inf)
    del z
    if extra is None:
      live = vis.any(-1)
      m = torch.where(live, zm.amax(-1), 0.0)
      e = torch.exp(zm - m[..., None])
      lsum = e.sum(-1)
      p = e / torch.where(live, lsum, 1.0)[..., None]
      lse = torch.where(live, m + torch.log(torch.where(live, lsum, 1.0)), math.nan)
    else:
      m = torch.maximum(zm.amax(-1), torch.full_like(zm[..., 0], extra))
      e = torch.exp(zm - m[..., None])
      lsum = e.sum(-1) + torch.exp(extra - m)
      p = e / lsum[..., None]
      lse = m + torch.log(lsum)
    del zm, e
    o = p @ vb
    r['out'][bi] = o.permute(1, 0, 2)
    r['lse'][bi] = lse
    r['a_out'][bi] = (p @ vb.abs()).permute(1, 0, 2)
    r['dv'][bi] = fold(p.transpose(-1, -2) @ dob)
    r['a_dv'][bi] = fold(p.transpose(-1, -2) @ dob.abs())
    dp = dob @ vb.transpose(-1, -2)
    delta = (dob * o).sum(-1)
    odo = (dob.abs() * o.abs()).sum(-1)
    ds = p * (dp - delta[..., None])
    a_ds = p * (dp.abs() + delta.abs()[..., None] + odo[..., None])
    del dp
    r['drel'] += TF._DiagSum(ds)
    r['drel_abs'] += TF._DiagSum(a_ds)
    r['drel_delta'] += TF._DiagSum(p * odo[..., None])
    dsc, a_dsc = ds * dz, a_ds * dz
    del ds, dz
    r['dq'][bi] = (scale * dsc @ kb).permute(1, 0, 2)
    r['dk'][bi] = fold(scale * dsc.transpose(-1, -2) @ qb)
    r['a_dq'][bi] = (scale * a_dsc @ kb.abs()).permute(1, 0, 2)
    r['a_dk'][bi] = fold(scale * a_dsc.transpose(-1, -2) @ qb.abs())
    r['a_dq0'][bi] = (scale * a_ds @ kb.abs()).permute(1, 0, 2)
    r['a_dk0'][bi] = fold(scale * a_ds.transpose(-1, -2) @ qb.abs())
    del p, dsc, a_dsc, a_ds
  return r


# ------------------------------------------------------------- the oracle on the CPU ----
def _SmallInputs(hk, extra, seed=0):
  gen = torch.Generator().manual_seed(seed)
  b, l, h, d = 3, 48, 4, 16
  seg = torch.tensor([[1] * 20 + [2] * 20 + [0] * 8, [0] * l, [1] * l], dtype=torch.int32)
  pos = torch.cat([torch.arange(20), torch.arange(20), torch.zeros(8, dtype=torch.long)])
  pos = torch.stack([pos, torch.zeros(l, dtype=torch.long), torch.arange(l)]).to(torch.int32)
  q = torch.randn(b, l, h, d, generator=gen)
  k = torch.randn(b, l, hk, d, generator=gen)
  v = torch.randn(b, l, hk, d, generator=gen)
  rel = torch.randn(h, 2 * l - 1, generator=gen)
  d_o = torch.randn(b, l, h, d, generator=gen)
  if extra is None:       # a query that sees nothing gets no gradient from the model
    d_o = d_o * TF._Visible(seg, pos, True, b, l, 'cpu').any(-1)[:, :, None, None]
  return q, k, v, rel, seg, pos, d_o


@pytest.mark.parametrize('hk', [4, 2])
@pytest.mark.parametrize('cap,extra', _OPTIONS, ids=_OPTION_IDS)
def test_oracle_matches_reference_and_fp32_autograd(cap, extra, hk):
  """The float64 oracle against `flash_attention_ref` (the CPU path of `flash_attention`) and
  the fp32 autograd of it: forward, lse from the fp32 logits, and dQ, dK, dV, d rel, which
  exercise the cap's derivative and the extra logit."""
  q, k, v, rel, seg, pos, d_o = _SmallInputs(hk, extra)
  scale = 0.5                            # |scale·q·k| ~ 2, well past a cap of 5 in the tails
  leaves = [t.clone().requires_grad_(True) for t in (q, k, v, rel)]
  out = A.flash_attention(*leaves[:3], leaves[3], seg, pos, scale, True, cap, extra)
  assert torch.equal(out, A.flash_attention_ref(q, k, v, rel, seg, pos, scale, True, cap, extra))
  dq, dk, dv, drel = torch.autograd.grad(out, leaves, d_o)
  r = _Oracle(q, k, v, rel, seg, pos, scale, True, d_o, cap, extra)
  live = r['live']
  if extra is None:
    rows = live[:, :, None, None].expand_as(out)
    torch.testing.assert_close(out[rows].double(), r['out'][rows], atol=1e-5, rtol=1e-5)
  else:
    torch.testing.assert_close(out.double(), r['out'], atol=1e-5, rtol=1e-5)
    assert bool((r['out'][~live] == 0).all()) and bool((r['lse'].transpose(1, 2)[~live] == extra).all())
  for name, got in [('dq', dq), ('dk', dk), ('dv', dv), ('drel', drel)]:
    torch.testing.assert_close(got.double(), r[name], atol=2e-5, rtol=1e-4, msg=name)
  # lse of the live rows from fp32 logits built the way the contract states them.
  s = scale * torch.einsum('blhd,bmhd->bhlm', q, k.repeat_interleave(4 // hk, dim=2))
  z = cap * torch.tanh(s / cap) if cap else s
  z = z + TF._Toeplitz(rel, q.shape[1])
  vis = TF._Visible(seg, pos, True, *q.shape[:2], 'cpu')[:, None]
  z = z.masked_fill(~vis, -math.inf)
  if extra is not None:
    z = torch.cat([z, torch.full_like(z[..., :1], extra)], -1)
  lse = torch.logsumexp(z, -1)
  live_bhl = live[:, None, :].expand_as(lse)
  torch.testing.assert_close(lse[live_bhl].double(), r['lse'][live_bhl], atol=1e-5, rtol=1e-5)


# ------------------------------------------------- decoding a capped LM on the CPU ----
def _CappedTask(cap=2.0, extra=0.0, kv_heads=None):
  bp = gb.DenseBuilder.Params().Set(
      model_dim=16, attention_num_heads=4, attention_num_memory_heads=kv_heads,
      attention_key_value_dim=8, ff_dim=32, relative_attention_type='bias',
      relative_attention_num_buckets=8, relative_attention_max_distance=16,
      atten_logit_cap=cap, attention_extra_logit=extra, fprop_dtype=torch.float32,
      dtype=torch.float32, label_smoothing=0.0)
  p = gb.UniTransformer.Params().Set(
      name='lm', builder=bp, vocab_size=40, num_transformer_layers=2, max_length=64,
      positional_embedding=False, label_smoothing=0.0, z_loss=0.0, decoder_eos_id=1,
      fprop_dtype=torch.float32)
  p.random_seed = 5
  with cluster_factory.ForTestingWorker(mode='sync', job='trainer_client', do_eval=True):
    task = p.Instantiate()
  with torch.no_grad():
    task.dec_emb.theta.embedding.mul_(4.0)
    for name, t in task.theta.FlattenItems():
      if name.endswith('.wq'):          # logits of several units: the cap of 2 bends them
        t.mul_(4.0)
  return task


def _TeacherForced(task, ids):
  bsz, l = ids.shape
  batch = NestedMap(ids=ids, labels=ids, paddings=torch.zeros(bsz, l),
                    segment_ids=torch.ones(bsz, l, dtype=torch.long),
                    segment_pos=torch.arange(l).repeat(bsz, 1))
  pred = task.ComputePredictions(task.theta, batch)
  return task._ComputeLogits(task.theta, pred.dec_outputs).float()   # pylint: disable=protected-access


@pytest.mark.parametrize('kv_heads', [None, 2])
def test_capped_decode_step_matches_teacher_forced_forward(kv_heads):
  """Token-by-token `DecodeStep` of a decoder LM with relative bias, a cap of 2 (tanh far
  from linear) and an extra logit of 0 equals its teacher-forced forward in fp32."""
  torch.manual_seed(0)
  task = _CappedTask(kv_heads=kv_heads)
  bsz, l, tmax = 2, 12, 16
  ids = torch.randint(2, 40, (bsz, l))
  with torch.no_grad():
    full = _TeacherForced(task, ids)
    # The options change the result by far more than the tolerance below.
    plain = _TeacherForced(_CappedTask(cap=0.0, extra=None, kv_heads=kv_heads), ids)
    assert float((plain - full).abs().max()) > 0.1
    st = task.InitDecodeState(bsz, tmax, ids.device)
    for i in range(l):
      got = task.DecodeStep(task.theta, ids[:, i], st, i).float()
      torch.testing.assert_close(got, full[:, i], atol=2e-4, rtol=2e-4, msg='step %d' % i)


def test_capped_beam_step_after_prefill_matches_teacher_forced_forward(monkeypatch):
  """A K = 1 flat-beam search of the same LM (one-pass `Prefill` of the prompt, then beam
  steps): every step's logits equal the forward of the sequence it extends."""
  torch.manual_seed(0)
  task = _CappedTask()
  steps = []
  real = task.BeamDecodeStep

  def Record(theta, ids, pos, state, slot0, vis):
    logits = real(theta, ids, pos, state, slot0, vis)
    steps.append((ids.clone(), int(pos[0, 0]), logits.clone()))
    return logits
  monkeypatch.setattr(task, 'BeamDecodeStep', Record)
  prompt = [5, 9, 3, 7, 2]
  batch = NestedMap(tgt=NestedMap(ids=torch.tensor([prompt]), paddings=torch.zeros(1, 5)))
  with torch.no_grad():
    gshard_decode.BeamDecodeIds(task, task.theta, batch, beam_size=1, max_steps=5)
    assert len(steps) == 5
    seq = prompt[:-1]
    for ids, pos, logits in steps:
      seq = seq + [int(ids[0, 0])]
      assert pos == len(seq) - 1
      want = _TeacherForced(task, torch.tensor([seq]))[0, -1]
      torch.testing.assert_close(logits[0, 0].float(), want, atol=2e-4, rtol=2e-4)


def test_moe_lm_8e_softcap_config():
  from lingvo_b200 import model_registry
  import lingvo_b200.models.lm.params.synthetic_packed_input as spi
  assert model_registry.GetParams('lm.synthetic_packed_input.MoELm8ESoftCap', 'Train') is not None
  bp = spi.MoELm8ESoftCap()._Builder()
  assert bp.atten_logit_cap == 50.0 and bp.attention_extra_logit == 0.0
  base = spi.MoELm8E()._Builder()
  assert not base.atten_logit_cap and base.attention_extra_logit is None


# ----------------------------------------------------------------- on the H100 ----
def _BenchInputs(hk, extra, seed):
  """B = 8, L = 1024, H = 16, D = 128 with the packed layouts of `test_flash_attn_gpu.py`
  (rows 1, 4 and 7 fully padded), causal, the model's bucketed bias table. scale = 2 puts
  |scale·q·k| (std ≈ 5.7) beyond a cap of 5 for ~40% of the pairs."""
  gen = torch.Generator().manual_seed(seed)
  b, l, h = 8, 1024, 16
  q = (torch.randn(b, l, h, _D, generator=gen) * 0.5).bfloat16().cuda()
  k = (torch.randn(b, l, hk, _D, generator=gen) * 0.5).bfloat16().cuda()
  v = (torch.randn(b, l, hk, _D, generator=gen) * 0.5).bfloat16().cuda()
  seg, pos = TF._Packed(b, l)
  seg, pos = seg.cuda(), pos.cuda()
  wrb, bucket, rel = TF._BucketTable(h, l, False, gen)
  d_o = (torch.randn(b, l, h, _D, generator=gen) * 0.5).bfloat16().cuda()
  if extra is None:
    d_o = d_o * TF._Visible(seg, pos, True, b, l, 'cuda').any(-1)[:, :, None, None].to(d_o.dtype)
  return q, k, v, rel.detach(), seg, pos, 2.0, d_o


@pytest.mark.gpu
@pytest.mark.parametrize('hk', [16, 4, 1])
@pytest.mark.parametrize('cap,extra', _OPTIONS, ids=_OPTION_IDS)
def test_softcap_flash_attention_matches_float64(cap, extra, hk):
  """O, lse, dQ, dK, dV and d rel at the benchmark's shape within the oracle's bounds, and
  the exact values of the contract: zeros for what nothing sees and, with an extra logit,
  O = 0 and lse == extra for a query that sees no key."""
  q, k, v, rel, seg, pos, scale, d_o = _BenchInputs(hk, extra, 100 + hk)
  b, l, h, _ = q.shape
  leaves = [t.detach().requires_grad_(True) for t in (q, k, v, rel)]
  assert A.flash_attention_supported(q, k)
  out = A.flash_attention(*leaves[:3], leaves[3], seg, pos, scale, True, cap, extra)
  dq, dk, dv, drel = torch.autograd.grad(out, leaves, d_o)
  out2, lse = ops.native().flash_attn_fwd(q, k, v, rel, seg, pos, scale, True, cap, extra)
  assert torch.equal(TF._Bits(out2), TF._Bits(out))
  for name, t in [('out', out), ('lse', lse), ('dq', dq), ('dk', dk), ('dv', dv),
                  ('drel', drel)]:
    assert bool(torch.isfinite(t).all()), '%s has non-finite values' % name
  with torch.no_grad():
    r = _Oracle(q, k, v, rel, seg, pos, scale, True, d_o, cap, extra)
  live, seen = r['live'], r['seen']
  case = 'hk%d-cap%g-extra%s' % (hk, cap, extra)
  u, tc = 2.0**-8, _TANH * cap
  ulp = TF._Bf16Ulp
  rows = live[:, :, None, None].expand_as(out) if extra is None else None
  TF._CheckBound(case, 'out', out, r['out'], (TF._C_O * u + tc) * r['a_out'] + ulp(r['out']),
                 rows)
  live_bhl = live[:, None, :].expand(b, h, l)
  TF._CheckBound(case, 'lse', lse, r['lse'], TF._LSE_REL * (1 + r['a_lse']) + 4 * tc,
                 live_bhl)
  TF._CheckBound(case, 'dv', dv, r['dv'], (TF._C_DV * u + tc) * r['a_dv'] + ulp(r['dv']))
  TF._CheckBound(case, 'dk', dk, r['dk'],
                 (TF._C_DQK * u + tc) * r['a_dk'] + _TANH * r['a_dk0'] + ulp(r['dk']))
  TF._CheckBound(case, 'dq', dq, r['dq'],
                 (TF._C_DQK * u + tc) * r['a_dq'] + _TANH * r['a_dq0'] + ulp(r['dq']))
  TF._CheckBound(case, 'drel', drel, r['drel'],
                 TF._C_DREL * u * r['drel_delta'] + (TF._DREL_FLOOR + tc) * r['drel_abs'])

  # Exact values.
  assert not bool(live[1].any()) and not bool(seen[1].any())     # a fully padded row
  if extra is not None:
    assert bool((out[~live] == 0).all()), 'O is not 0 at a query that sees no key'
    dead = ~live[:, None, :].expand(b, h, l)
    assert bool((lse[dead] == extra).all()), 'lse is not the extra logit where nothing is seen'
  assert bool((dq[~live] == 0).all()), 'dQ is not 0 at a query that sees no key'
  assert bool((dk[~seen] == 0).all()), 'dK is not 0 at a key that no query sees'
  assert bool((dv[~seen] == 0).all()), 'dV is not 0 at a key that no query sees'
  assert bool((drel[:, ~r['used']] == 0).all()), 'd rel is not 0 on an unused diagonal'


def _Step(q, k, v, rel, seg, pos, d_o, cap=50.0, extra=0.0):
  nat = ops.native()
  out, lse = nat.flash_attn_fwd(q, k, v, rel, seg, pos, 1.0, True, cap, extra)
  return (out, lse) + tuple(nat.flash_attn_bwd(q, k, v, out, d_o, lse, rel, seg, pos, 1.0,
                                               True, True, cap))


def _StepArgs(seed, hk=16):
  q, k, v, rel, seg, pos, _, d_o = _BenchInputs(hk, 0.0, seed)
  return [q, k, v, rel, seg, pos, d_o]


@pytest.mark.gpu
@pytest.mark.parametrize('hk', [16, 4])
def test_softcap_flash_attention_is_bitwise_reproducible(hk):
  args = _StepArgs(11, hk)
  first, again = _Step(*args), _Step(*args)
  for name, x, y in zip(TF._NAMES, first, again):
    assert torch.equal(TF._Bits(x), TF._Bits(y)), name


@pytest.mark.gpu
def test_softcap_flash_attention_graph_replay_matches_eager():
  """A capped, extra-logit forward + backward captured once in a CUDA graph and replayed on
  new inputs equals the eager call on them bit for bit."""
  static = [t.clone() for t in _StepArgs(12)]
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    for _ in range(2):
      _Step(*static)
  torch.cuda.current_stream().wait_stream(side)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    captured = _Step(*static)
  new = _StepArgs(13)
  for dst, src in zip(static, new):
    dst.copy_(src)
  graph.replay()
  eager = _Step(*new)
  torch.cuda.synchronize()
  for name, x, y in zip(TF._NAMES, captured, eager):
    assert torch.equal(TF._Bits(x), TF._Bits(y)), name


@pytest.mark.gpu
@pytest.mark.parametrize('hk', [16, 1])
def test_default_options_are_the_plain_kernels_bitwise(hk):
  """Passing logit_cap = 0 and extra_logit = None explicitly is the call without them."""
  q, k, v, rel, seg, pos, d_o = _StepArgs(14, hk)
  nat = ops.native()
  plain_fwd = nat.flash_attn_fwd(q, k, v, rel, seg, pos, 1.0, True)
  opt_fwd = nat.flash_attn_fwd(q, k, v, rel, seg, pos, 1.0, True, logit_cap=0.0,
                               extra_logit=None)
  out, lse = plain_fwd
  plain_bwd = nat.flash_attn_bwd(q, k, v, out, d_o, lse, rel, seg, pos, 1.0, True, True)
  opt_bwd = nat.flash_attn_bwd(q, k, v, out, d_o, lse, rel, seg, pos, 1.0, True, True,
                               logit_cap=0.0)
  for x, y in zip(list(plain_fwd) + list(plain_bwd), list(opt_fwd) + list(opt_bwd)):
    assert torch.equal(TF._Bits(x), TF._Bits(y))
  leaves = [t.detach().requires_grad_(True) for t in (q, k, v, rel)]
  a = A.flash_attention(*leaves[:3], leaves[3], seg, pos, 1.0, True)
  ga = torch.autograd.grad(a, leaves, d_o)
  c = A.flash_attention(*leaves[:3], leaves[3], seg, pos, 1.0, True, 0.0, None)
  gc = torch.autograd.grad(c, leaves, d_o)
  for x, y in zip([a, *ga], [c, *gc]):
    assert torch.equal(TF._Bits(x), TF._Bits(y))


@pytest.mark.gpu
def test_bad_logit_options_are_refused_without_launching():
  b, l, h = 2, 256, 2
  q = torch.zeros(b, l, h, _D, dtype=torch.bfloat16, device='cuda')
  lse = torch.zeros(b, h, l, device='cuda')
  nat = ops.native()
  launches = nat.launch_count()
  torch.cuda.synchronize()
  bad = [dict(logit_cap=-1.0), dict(logit_cap=math.nan), dict(logit_cap=math.inf),
         dict(extra_logit=math.nan), dict(extra_logit=math.inf), dict(extra_logit=-math.inf)]
  for kw in bad:
    with pytest.raises(RuntimeError, match='logit'):
      nat.flash_attn_fwd(q, q, q, None, None, None, 1.0, True, **kw)
  for cap in (-1.0, math.nan, math.inf):
    with pytest.raises(RuntimeError, match='logit_cap'):
      nat.flash_attn_bwd(q, q, q, q, q, lse, None, None, None, 1.0, True, False, cap)
  torch.cuda.synchronize()
  assert nat.launch_count() == launches


@pytest.mark.gpu
def test_moe_lm_8e_softcap_attention_layer_takes_flash(monkeypatch):
  """The bf16 `SelfAttentionLayer` of MoELm8ESoftCap (cap 50, extra logit 0, relative bias,
  decoder) runs the flash kernel, never `_AttentionCore`, and its output and the gradients of
  wq, wk, wv, wo and wrb match the same weights run through the layer's fp32 path."""
  import lingvo_b200.models.lm.params.synthetic_packed_input as spi
  bp = spi.MoELm8ESoftCap()._Builder()
  lp = gb.SelfAttentionLayer.Params().Set(name='sa', b=bp, relative_bias=True, decoder=True)
  lp.random_seed = 5
  layer = lp.Instantiate().cuda()
  b, l = 2, 1024
  gen = torch.Generator().manual_seed(7)
  x = torch.randn(b, l, bp.model_dim, generator=gen).cuda()
  seg, pos = TF._Packed(b, l)
  seg, pos = seg.cuda(), pos.cuda()
  w = torch.randn(b, l, bp.model_dim, generator=gen).cuda() * (seg != 0)[:, :, None].float()
  names = ['wq', 'wk', 'wv', 'wo', 'wrb']
  leaves = [layer.theta[n] for n in names]

  def _Run(xx):
    out, _ = layer.FProp(layer.theta, xx, seg, pos)
    return out, torch.autograd.grad((out.float() * w).sum(), leaves)

  calls = []
  real_flash, real_core = A.flash_attention, gb._AttentionCore

  def _NoCore(*a, **kw):
    raise AssertionError('the bf16 layer fell back to _AttentionCore')
  monkeypatch.setattr(A, 'flash_attention',
                      lambda *a, **kw: calls.append((a[7], kw)) or real_flash(*a, **kw))
  monkeypatch.setattr(gb, '_AttentionCore', _NoCore)
  out16, g16 = _Run(x.bfloat16())
  assert calls == [(True, dict(logit_cap=50.0, extra_logit=0.0))], calls
  monkeypatch.setattr(gb, '_AttentionCore', real_core)
  out32, g32 = _Run(x)
  assert len(calls) == 1, 'the fp32 layer took the flash branch'

  def _Rel(a, ref):
    return float((a.detach().float() - ref.detach()).norm() / ref.detach().norm())
  rows = seg != 0
  assert _Rel(out16[rows], out32[rows]) < 2e-2
  for n, a, ref in zip(names, g16, g32):
    assert _Rel(a, ref) < 3e-2, (n, _Rel(a, ref))
