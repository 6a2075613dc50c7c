"""Grouped-query and multi-query attention through the wgmma flash kernels
(ops/csrc/flash_attn.cu): k and v carry Hk heads with H % Hk == 0, and query head h reads KV
head h // (H/Hk).

The contract of `test_flash_attn_gpu.py` holds head by head; dK and dV of a KV head are the
sums over the G = H/Hk query heads that read it. The float64 oracle is that file's, run on
K/V expanded to H heads, with dK, dV and their |.| contractions summed over each group. The
bounds have the same form and constants.
"""
import pytest
import torch

import test_flash_attn_gpu as TF
from lingvo_b200 import ops
from lingvo_b200.core import gshard_builder as gb
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.ops import attention as A

_D = 128


def _Splits(b, l, h, hk):
  return ops.native().flash_attn_bwd_splits(b, l, h, hk)


# ------------------------------------------------------------------- the cases ----
def _PackedBert(b, l):
  """seg / pos [b, l] for L = 512 encoder rows: segments crossing 128-row blocks, a 1-token
  segment, trailing padding (a pure-padding last block in row 0) and a fully padded row."""
  layouts = [
      [(0, 200), (200, 333), (333, 380)],                           # padding from 380
      [(0, 128), (128, 129), (129, 512)],
      [],                                                           # fully padded
      [(0, 500)],                                                   # padding from 500
  ]
  seg = torch.zeros(b, l, dtype=torch.int32)
  pos = torch.zeros(b, l, dtype=torch.int32)
  for bi in range(b):
    for si, (s, e) in enumerate(layouts[bi % len(layouts)]):
      seg[bi, s:e] = si + 1
      pos[bi, s:e] = torch.arange(e - s, dtype=torch.int32)
  return seg, pos


# name: (b, l, h, hk, causal, packing)
_SHAPES = {
    'moe-kv8': (8, 1024, 16, 8, True, 'moe'),      # MoELm8E's shape with grouped KV heads
    'moe-kv4': (8, 1024, 16, 4, True, 'moe'),
    'moe-kv1': (8, 1024, 16, 1, True, 'moe'),
    'bert': (4, 512, 8, 1, False, 'bert'),         # wiki_bert: multi-query encoder, L = 512
    'small': (2, 128, 2, 1, True, None),           # one block, G = 2
}
_CASES = list(_SHAPES)


def _Inputs(case, seed):
  """(q, k, v, rel, seg, pos, scale, causal, d_o) with k, v [B, L, Hk, 128]; q/k/v are
  column slices of one fused projection, as in a layer."""
  b, l, h, hk, causal, packing = _SHAPES[case]
  gen = torch.Generator().manual_seed(seed)
  qkv = (torch.randn(b, l, (h + 2 * hk) * _D, generator=gen) * 0.5).bfloat16().cuda()
  q, k, v = qkv.split([h * _D, hk * _D, hk * _D], dim=-1)
  q, k, v = q.reshape(b, l, h, _D), k.reshape(b, l, hk, _D), v.reshape(b, l, hk, _D)
  seg = pos = None
  if packing == 'moe':
    seg, pos = TF._Packed(b, l)
  elif packing == 'bert':
    seg, pos = _PackedBert(b, l)
  if seg is not None:
    seg, pos = seg.cuda(), pos.cuda()
  rel = torch.randn(h, 2 * l - 1, generator=gen).cuda()
  d_o = (torch.randn(b, l, h, _D, generator=gen) * 0.5).bfloat16().cuda()
  live = TF._Visible(seg, pos, causal, b, l, 'cuda').any(-1)
  d_o = d_o * live[:, :, None, None].to(d_o.dtype)              # zero where a query sees nothing
  return q, k, v, rel, seg, pos, 1.0, causal, d_o


def _Expand(t, h):
  return t.repeat_interleave(h // t.shape[2], dim=2)


def _GqaOracle(q, k, v, rel, seg, pos, scale, causal, d_o):
  """The float64 oracle on K/V expanded to H heads; dK, dV and their bounds' contractions
  summed over the query heads of each group."""
  b, l, h, _ = q.shape
  hk = k.shape[2]
  r = TF._Oracle(q, _Expand(k, h), _Expand(v, h), rel, seg, pos, scale, causal, d_o)
  for n in ('dk', 'a_dk', 'dv', 'a_dv'):
    r[n] = r[n].reshape(b, l, hk, h // hk, _D).sum(3)
  return r


# ------------------------------------------------------------ float64 oracle ----
def test_cases_cover_both_backward_layouts():
  """Runs without a GPU when the extension is built: among the cases, some keep dK/dV in
  bf16 straight from registers (S = 1) and some split the group (S > 1)."""
  splits = {c: _Splits(*_SHAPES[c][:4]) for c in _CASES}
  assert splits['moe-kv8'] == 1 and splits['moe-kv4'] > 1 and splits['moe-kv1'] > 1, splits
  for c, s in splits.items():
    g = _SHAPES[c][2] // _SHAPES[c][3]
    assert g % s == 0, (c, s)
  # Multi-head attention is never split, and the rule depends on the shapes only.
  for b, l, h in [(8, 1024, 16), (1, 128, 1), (2, 4096, 40)]:
    assert _Splits(b, l, h, h) == 1


@pytest.mark.gpu
@pytest.mark.parametrize('case', _CASES)
def test_gqa_flash_attention_matches_float64(case):
  """O, lse, dQ, dK, dV and d rel within the per-element bounds of the float64 oracle, plus
  the exact zeros: unseen keys get zero dK/dV, dead queries zero dQ, unused diagonals zero
  d rel."""
  q, k, v, rel, seg, pos, scale, causal, d_o = _Inputs(case, 100 + _CASES.index(case))
  b, l, h, _ = q.shape
  hk = k.shape[2]
  q, k, v = [t.detach().requires_grad_(True) for t in (q, k, v)]
  rel = rel.requires_grad_(True)
  assert A.flash_attention_supported(q, k)
  out = A.flash_attention(q, k, v, rel, seg, pos, scale, causal)
  dq, dk, dv, drel = torch.autograd.grad(out, [q, k, v, rel], d_o)
  assert out.shape == (b, l, h, _D) and dq.shape == q.shape
  assert dk.shape == (b, l, hk, _D) and dv.shape == (b, l, hk, _D)
  nat = ops.native()
  out2, lse = nat.flash_attn_fwd(q.detach(), k.detach(), v.detach(), rel.detach(), seg, pos,
                                 scale, causal)
  assert torch.equal(TF._Bits(out2), TF._Bits(out))

  with torch.no_grad():
    r = _GqaOracle(q.detach(), k.detach(), v.detach(), rel.detach(), seg, pos, scale, causal,
                   d_o)
  live, seen = r['live'], r['seen']
  for name, t in [('out', out), ('lse', lse), ('dq', dq), ('dk', dk), ('dv', dv),
                  ('drel', drel)]:
    assert bool(torch.isfinite(t).all()), '%s has non-finite values' % name

  u = 2.0**-8
  rows = live[:, :, None, None].expand_as(out)
  TF._CheckBound(case, 'out', out, r['out'], TF._C_O * u * r['a_out'] + TF._Bf16Ulp(r['out']),
                 rows)
  live_bhl = live[:, None, :].expand(b, h, l)
  TF._CheckBound(case, 'lse', lse, r['lse'], TF._LSE_REL * (1 + r['a_lse']), live_bhl)
  TF._CheckBound(case, 'dv', dv, r['dv'], TF._C_DV * u * r['a_dv'] + TF._Bf16Ulp(r['dv']))
  TF._CheckBound(case, 'dk', dk, r['dk'], TF._C_DQK * u * r['a_dk'] + TF._Bf16Ulp(r['dk']))
  TF._CheckBound(case, 'dq', dq, r['dq'], TF._C_DQK * u * r['a_dq'] + TF._Bf16Ulp(r['dq']))
  TF._CheckBound(case, 'drel', drel, r['drel'],
                 TF._C_DREL * u * r['drel_delta'] + TF._DREL_FLOOR * r['drel_abs'])

  assert bool((dq[~live] == 0).all()), 'dQ is not 0 at a query that sees no key'
  assert bool((dk[~seen] == 0).all()), 'dK is not 0 at a key that no query sees'
  assert bool((dv[~seen] == 0).all()), 'dV is not 0 at a key that no query sees'
  assert bool((drel[:, ~r['used']] == 0).all()), 'd rel is not 0 on an unused diagonal'
  if seg is not None:
    assert not bool(seen.all()), 'the case has no unseen key'


# ------------------------------------------------------- bitwise equal to MHA ----
def _Step(q, k, v, rel, seg, pos, scale, causal, d_o):
  """(out, lse, dq, dk, dv, drel) straight from the kernels."""
  nat = ops.native()
  out, lse = nat.flash_attn_fwd(q, k, v, rel, seg, pos, scale, causal)
  return (out, lse) + tuple(nat.flash_attn_bwd(q, k, v, out, d_o, lse, rel, seg, pos, scale,
                                               causal, True))


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['moe-kv4', 'moe-kv1', 'bert', 'small'])
def test_gqa_equals_mha_on_expanded_kv_bitwise(case):
  """Hk KV heads give the same out, lse, dQ and d rel, bit for bit, as the multi-head call
  on K/V repeated to H heads: this pins the head mapping. dK/dV are summed over the group
  in fp32 before rounding, so they are checked against the oracle above instead."""
  q, k, v, rel, seg, pos, scale, causal, d_o = _Inputs(case, 200 + _CASES.index(case))
  h = q.shape[2]
  gqa = _Step(q, k, v, rel, seg, pos, scale, causal, d_o)
  mha = _Step(q, _Expand(k, h), _Expand(v, h), rel, seg, pos, scale, causal, d_o)
  for name, x, y in zip(TF._NAMES, gqa, mha):
    if name not in ('dk', 'dv'):
      assert torch.equal(TF._Bits(x), TF._Bits(y)), name


# ------------------------------------------------- reproducibility, graph replay ----
@pytest.mark.gpu
def test_gqa_backward_is_bitwise_reproducible_when_split():
  args = _Inputs('moe-kv1', 11)
  assert _Splits(*_SHAPES['moe-kv1'][:4]) > 1
  first = _Step(*args)
  again = _Step(*args)
  for name, x, y in zip(TF._NAMES, first, again):
    assert torch.equal(TF._Bits(x), TF._Bits(y)), name


@pytest.mark.gpu
def test_gqa_graph_replay_matches_eager():
  """Forward + backward at a split case, captured once in a CUDA graph and replayed on new
  q/k/v/rel/dO, equals the eager call on those inputs bit for bit."""
  assert _Splits(*_SHAPES['moe-kv4'][:4]) > 1
  static = list(_Inputs('moe-kv4', 12))
  q, k, v = static[:3]
  qkv = torch.cat([t.reshape(*t.shape[:2], -1) for t in (q, k, v)], dim=-1)   # one buffer
  h, hk = q.shape[2], k.shape[2]
  parts = qkv.split([h * _D, hk * _D, hk * _D], dim=-1)
  static[:3] = [t.reshape(*t.shape[:2], -1, _D) for t in parts]
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    for _ in range(2):
      _Step(*static)
  torch.cuda.current_stream().wait_stream(side)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    captured = _Step(*static)
  new = _Inputs('moe-kv4', 13)
  for i in (3, 8):                                               # rel, dO
    static[i].copy_(new[i])
  qkv.copy_(torch.cat([t.reshape(*t.shape[:2], -1) for t in new[:3]], dim=-1))
  graph.replay()
  eager = _Step(*new)
  torch.cuda.synchronize()
  for name, x, y in zip(TF._NAMES, captured, eager):
    assert torch.equal(TF._Bits(x), TF._Bits(y)), name


# ------------------------------------------------------------- argument checks ----
@pytest.mark.gpu
def test_gqa_rejects_bad_head_layouts_without_launching():
  nat = ops.native()
  b, l, h = 2, 256, 4
  z = lambda *s: torch.zeros(*s, dtype=torch.bfloat16, device='cuda')
  q = z(b, l, h, _D)
  lse = torch.zeros(b, h, l, device='cuda')
  rel = torch.zeros(h, 2 * l - 1, device='cuda')
  bad = [
      ('H % Hk != 0', z(b, l, 3, _D), z(b, l, 3, _D), rel, False),
      ('v heads != k heads', z(b, l, 2, _D), z(b, l, 1, _D), rel, True),
      ('k length != q length', z(b, l - 128, 2, _D), z(b, l - 128, 2, _D), rel, False),
      ('rel with Hk rows', z(b, l, 2, _D), z(b, l, 2, _D), rel[:2].contiguous(), True),
  ]
  launches = nat.launch_count()
  for what, k, v, r, qk_ok in bad:
    with pytest.raises(RuntimeError, match='flash_attn_fwd: '):
      nat.flash_attn_fwd(q, k, v, r, None, None, 1.0, True)
      pytest.fail('fwd accepted: ' + what)
    with pytest.raises(RuntimeError, match='flash_attn_bwd: '):
      nat.flash_attn_bwd(q, k, v, q, q, lse, r, None, None, 1.0, True, True)
      pytest.fail('bwd accepted: ' + what)
    # The front end sees q and k only; a v or rel that does not match k / q is a caller's
    # mistake that the kernels refuse rather than a shape to fall back on.
    assert A.flash_attention_supported(q, k) == qk_ok, what
  assert nat.launch_count() == launches


# ----------------------------------------------------------------------- layer ----
def _Layer(hk, decoder, fprop_dtype):
  bp = gb.DenseBuilder.Params().Set(
      model_dim=512, attention_num_heads=16, attention_num_memory_heads=hk,
      attention_key_value_dim=_D, relative_attention_num_buckets=32,
      relative_attention_max_distance=128, relative_attention_use_universal_1d_position=True,
      dtype=torch.float32, fprop_dtype=fprop_dtype, attention_combine_dims=True)
  lp = gb.SelfAttentionLayer.Params().Set(name='sa', b=bp, relative_bias=True, decoder=decoder)
  lp.random_seed = 5
  return lp.Instantiate().cuda()


@pytest.mark.gpu
@pytest.mark.parametrize('hk', [1, 4])
@pytest.mark.parametrize('decoder', [True, False], ids=['decoder', 'encoder'])
def test_self_attention_layer_takes_flash_with_grouped_kv(hk, decoder, monkeypatch):
  """bf16 layer (flash) against the same weights run in fp32 (`_AttentionCore` on K/V
  expanded to H heads): output and the gradients of wq, wk, wv, wo and wrb."""
  calls = []
  real = A.flash_attention

  def _Counted(*a, **kw):
    calls.append(a[1].shape)
    return real(*a, **kw)
  monkeypatch.setattr(A, 'flash_attention', _Counted)

  layer = _Layer(hk, decoder, torch.bfloat16)
  b, l = 2, 1024
  gen = torch.Generator().manual_seed(7)
  x = torch.randn(b, l, 512, generator=gen).bfloat16().cuda()
  seg, pos = TF._Packed(b, l)
  seg, pos = seg.cuda(), pos.cuda()
  live = (seg != 0)[:, :, None].float()
  w = torch.randn(b, l, 512, generator=gen).cuda() * live
  names = ['wq', 'wk', 'wv', 'wo', 'wrb']
  leaves = [layer.theta[n] for n in names]

  def _Run(xx):
    out, _ = layer.FProp(layer.theta, xx, seg, pos)
    return out, torch.autograd.grad((out.float() * w).sum(), leaves)

  out16, g16 = _Run(x)
  assert calls == [(b, l, hk, _D)], calls
  out32, g32 = _Run(x.float())
  assert len(calls) == 1, 'the fp32 layer took the flash branch'
  assert leaves[1].shape == (512, hk * _D)

  def _Rel(a, ref):
    return float((a.detach().float() - ref.detach()).norm() / ref.detach().norm())
  rows = seg != 0
  assert _Rel(out16[rows], out32[rows]) < 2e-2
  for n, a, ref in zip(names, g16, g32):
    assert _Rel(a, ref) < 3e-2, (n, _Rel(a, ref))


@pytest.mark.gpu
@pytest.mark.parametrize('hk', [1, 2])
def test_gqa_decoder_fprop_matches_extend_step(hk, monkeypatch):
  """Train and serve agree: the decoder stack's FProp (flash, L = 128) equals ExtendStep
  (decode_attn.cu) position by position, with grouped and multi-query KV heads at D = 128."""
  calls = []
  real = A.flash_attention
  monkeypatch.setattr(A, 'flash_attention', lambda *a, **kw: calls.append(1) or real(*a, **kw))
  bp = gb.DenseBuilder.Params().Set(
      model_dim=256, attention_num_heads=4, attention_num_memory_heads=hk,
      attention_key_value_dim=_D, ff_dim=512, relative_attention_type='bias',
      relative_attention_num_buckets=32, relative_attention_max_distance=128,
      relative_attention_use_universal_1d_position=True,
      fprop_dtype=torch.bfloat16, dtype=torch.float32, label_smoothing=0.0)
  bld = bp.Instantiate()
  lp = bld.DecoderLayerStack(
      'dec', [bld.DecSelfAttentionRelativeBias('self'), bld.DenseReluDense('ffn')], num=2)
  lp.random_seed = 3
  stack = lp.Instantiate()
  stack.InstantiateVariables()
  stack = stack.cuda()
  bsz, l = 2, 128
  x = torch.randn(bsz, l, 256, generator=torch.Generator().manual_seed(1)).bfloat16().cuda()
  seg = torch.ones(bsz, l, dtype=torch.int32, device='cuda')
  pos = torch.arange(l, dtype=torch.int32, device='cuda').unsqueeze(0).expand(bsz, l)
  with torch.no_grad():
    out = stack.FProp(stack.theta, NestedMap(vec=x, segment_id=seg, segment_pos=pos,
                                             aux_loss=torch.zeros((), device='cuda'))).vec
    assert len(calls) == 2, 'FProp did not take the flash branch'
    state = stack.InitDecodeState(bsz, l, x.device, x.dtype)
    assert state[0].k.shape == (bsz, l, hk, _D)
    steps = torch.cat([stack.ExtendStep(stack.theta, x[:, t:t + 1], state, t)
                       for t in range(l)], 1)
  err = (steps.float() - out.float()).norm(dim=-1) / out.float().norm(dim=-1)
  assert float(err.max()) < 3e-2, float(err.max())


# ------------------------------------------------------------------------- CPU ----
def test_cpu_flash_attention_with_grouped_kv_is_the_reference():
  gen = torch.Generator().manual_seed(0)
  b, l, h, hk = 2, 16, 4, 2
  q = torch.randn(b, l, h, 8, generator=gen).requires_grad_(True)
  k = torch.randn(b, l, hk, 8, generator=gen).requires_grad_(True)
  v = torch.randn(b, l, hk, 8, generator=gen).requires_grad_(True)
  rel = torch.randn(h, 2 * l - 1, generator=gen)
  seg = torch.tensor([[1] * 10 + [2] * 6, [1] * 12 + [0] * 4], dtype=torch.int32)
  pos = torch.cat([torch.arange(10), torch.arange(6)]).expand(b, l).int()
  assert not A.flash_attention_supported(q, k)
  out = A.flash_attention(q, k, v, rel, seg, pos, 0.5, True)
  want = A.flash_attention_ref(q, k, v, rel, seg, pos, 0.5, True)
  assert torch.equal(out, want)
  dq, dk, dv = torch.autograd.grad(out.sum(), [q, k, v])
  assert dq.shape == q.shape and dk.shape == k.shape and dv.shape == v.shape
  # The reference expands K/V the way the kernels read them: query head h uses KV head h // 2.
  want = A.flash_attention_ref(q, _Expand(k, h), _Expand(v, h), rel, seg, pos, 0.5, True)
  assert torch.equal(out, want)


def test_moe_lm_8e_kv4_has_grouped_kv_heads():
  from lingvo_b200 import model_registry
  import lingvo_b200.models.lm.params.synthetic_packed_input as spi
  cfg = model_registry.GetParams('lm.synthetic_packed_input.MoELm8EKv4', 'Train')
  assert cfg is not None
  bp = spi.MoELm8EKv4()._Builder()
  assert bp.attention_num_memory_heads == 4 and bp.attention_num_heads == 16
  assert spi.MoELm8E()._Builder().attention_num_memory_heads is None
  layer = gb.SelfAttentionLayer.Params().Set(name='sa', b=bp, relative_bias=True).Instantiate()
  assert tuple(layer.theta.wk.shape) == (2048, 512)
  assert tuple(layer.theta.wv.shape) == (2048, 512)
  assert tuple(layer.theta.wq.shape) == (2048, 2048)
