"""Decode-step attention with the KV-cache append (`ops.attention.decode_attention`): the CPU
path against the original step formula, grouped KV heads in `ExtendStep`, and on the GPU the
split-KV kernel against the fp32 oracle, its determinism, CUDA-graph replay over `t` and the
`UniTransformer.DecodeStep` it serves."""

import pytest
import torch

from lingvo_b200.core import cluster_factory
from lingvo_b200.core import gshard_builder as gb
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.ops import attention as attention_ops


def _StepFormula(q, k, v, cache_k, cache_v, t, wrb=None, num_buckets=8, max_distance=16):
  """The decode step's attention as it was written inline in `_SelfAttentionExtendStep`
  (MHA / MQA only: `expand` cannot broadcast grouped KV heads)."""
  bsz, _, h, d = q.shape
  hk = cache_k.shape[2]
  tmax = cache_k.shape[1]
  xd = q.dtype
  dev = q.device
  tt = torch.as_tensor(t, device=dev).reshape(())
  onehot = (torch.arange(tmax, device=dev) == tt).to(xd).reshape(1, tmax, 1, 1)
  cache_k.mul_(1 - onehot).add_(k * onehot)
  cache_v.mul_(1 - onehot).add_(v * onehot)
  kk, vv = cache_k, cache_v
  if hk != h:
    kk, vv = kk.expand(bsz, tmax, h, d), vv.expand(bsz, tmax, h, d)
  logits = torch.einsum('bqhd,bkhd->bhqk', q.float(), kk.float())
  key_pos = torch.arange(tmax, device=dev)
  if wrb is not None:
    bucket = gb.RelativePositionBucket(key_pos - tt, num_buckets, max_distance,
                                       bidirectional=False)
    logits = logits + wrb.float()[:, bucket.long()].reshape(1, h, 1, tmax)
  logits = logits + ((key_pos > tt).float() * -1e9).reshape(1, 1, 1, tmax)
  probs = torch.softmax(logits, -1)
  return torch.einsum('bhqk,bkhd->bqhd', probs, vv.float()).to(xd)


def _RelTable(wrb, tmax, num_buckets=8, max_distance=16):
  bucket = gb.RelativePositionBucket(torch.arange(tmax - 1, -tmax, -1, device=wrb.device),
                                     num_buckets, max_distance, bidirectional=False)
  return wrb.float()[:, bucket.long()]


@pytest.mark.parametrize('hk', [4, 1])
@pytest.mark.parametrize('use_rel', [False, True])
def test_cpu_decode_attention_equals_step_formula(hk, use_rel):
  g = torch.Generator().manual_seed(0)
  b, h, d, tmax = 2, 4, 8, 11
  wrb = torch.randn(h, 8, generator=g) if use_rel else None
  ck = torch.randn(b, tmax, hk, d, generator=g)
  cv = torch.randn(b, tmax, hk, d, generator=g)
  ck2, cv2 = ck.clone(), cv.clone()
  for t in (0, 5, tmax - 1):
    q = torch.randn(b, 1, h, d, generator=g)
    k = torch.randn(b, 1, hk, d, generator=g)
    v = torch.randn(b, 1, hk, d, generator=g)
    want = _StepFormula(q, k, v, ck, cv, t, wrb)
    rel = _RelTable(wrb, tmax) if use_rel else None
    got = attention_ops.decode_attention(q, k, v, ck2, cv2, torch.tensor(t), rel)
    assert got.shape == (b, 1, h, d)
    assert torch.equal(got, want)
    assert torch.equal(ck2, ck) and torch.equal(cv2, cv)
    assert torch.equal(ck2[:, t], k[:, 0]) and torch.equal(cv2[:, t], v[:, 0])


def test_grouped_kv_heads_extend_step_matches_fprop():
  bp = gb.DenseBuilder.Params().Set(
      model_dim=16, attention_num_heads=4, attention_num_memory_heads=2,
      attention_key_value_dim=8, ff_dim=32, relative_attention_type='bias',
      relative_attention_num_buckets=8, relative_attention_max_distance=16,
      fprop_dtype=torch.float32, dtype=torch.float32, label_smoothing=0.0)
  b = bp.Instantiate()
  lp = b.DecoderLayerStack(
      'dec', [b.DecSelfAttentionRelativeBias('self'), b.DenseReluDense('ffn')], num=2)
  lp.random_seed = 3
  stack = lp.Instantiate()
  stack.InstantiateVariables()
  assert isinstance(stack.layers[0].layer, gb.SelfAttentionLayer)
  bsz, l = 2, 7
  x = torch.randn(bsz, l, 16, generator=torch.Generator().manual_seed(1))
  seg = torch.ones(bsz, l, dtype=torch.long)
  pos = torch.arange(l).unsqueeze(0).expand(bsz, l)
  with torch.no_grad():
    out = stack.FProp(stack.theta, NestedMap(vec=x, segment_id=seg, segment_pos=pos,
                                             aux_loss=torch.zeros(())))
    state = stack.InitDecodeState(bsz, l + 3, x.device, x.dtype)
    assert state[0].k.shape == (bsz, l + 3, 2, 8)
    steps = [stack.ExtendStep(stack.theta, x[:, t:t + 1], state, t) for t in range(l)]
  torch.testing.assert_close(torch.cat(steps, 1), out.vec, atol=2e-4, rtol=2e-4)


# ----------------------------------------------------------------------------- GPU ----
def _RelErr(a, b):
  a, b = a.float(), b.float()
  return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _Inputs(b, tmax, h, hk, use_rel, seed=0):
  g = torch.Generator(device='cuda').manual_seed(seed)

  def _Bf16(*shape):
    return torch.randn(*shape, generator=g, device='cuda').to(torch.bfloat16)
  q, kn, vn = _Bf16(b, 1, h, 128) * 0.1, _Bf16(b, 1, hk, 128), _Bf16(b, 1, hk, 128)
  ck, cv = _Bf16(b, tmax, hk, 128), _Bf16(b, tmax, hk, 128)
  rel = torch.randn(h, 2 * tmax - 1, generator=g, device='cuda') if use_rel else None
  return q, kn, vn, ck, cv, rel


def _Chunk(b, h, hk, tmax):
  from lingvo_b200 import ops
  return ops.native().decode_attn_chunk(b, h, hk, tmax)


@pytest.mark.gpu
@pytest.mark.parametrize('use_rel', [False, True])
@pytest.mark.parametrize('h,hk', [(16, 16), (16, 4), (16, 1)])
@pytest.mark.parametrize('where', ['zero', 'chunk-1', 'chunk', 'last', 'past-end'])
@pytest.mark.parametrize('tmax', [100, 1024, 4096])
@pytest.mark.parametrize('b', [1, 3])
def test_kernel_matches_reference(b, tmax, where, h, hk, use_rel):
  q, kn, vn, ck, cv, rel = _Inputs(b, tmax, h, hk, use_rel)
  assert attention_ops.decode_attention_supported(q, ck)
  chunk = _Chunk(b, h, hk, tmax)
  t = {'zero': 0, 'chunk-1': min(chunk - 1, tmax - 1), 'chunk': min(chunk, tmax - 1),
       'last': tmax - 1, 'past-end': tmax}[where]
  ck0, cv0 = ck.clone(), cv.clone()
  rk, rv = ck.float(), cv.float()
  want = attention_ops.decode_attention_ref(q.float(), kn.float(), vn.float(), rk, rv, t, rel)
  got = attention_ops.decode_attention(q, kn, vn, ck, cv, torch.tensor(t, device='cuda'), rel)
  assert got.shape == (b, 1, h, 128) and got.dtype == torch.bfloat16
  assert _RelErr(got, want) < 5e-3
  rows = torch.arange(tmax, device='cuda') != t
  assert torch.equal(ck[:, rows], ck0[:, rows]) and torch.equal(cv[:, rows], cv0[:, rows])
  if t < tmax:
    assert torch.equal(ck[:, t], kn[:, 0]) and torch.equal(cv[:, t], vn[:, 0])


@pytest.mark.gpu
@pytest.mark.parametrize('h,hk', [(16, 16), (16, 1), (32, 1), (12, 4)])
def test_kernel_is_deterministic_and_accepts_int32_t(h, hk):
  q, kn, vn, ck, cv, rel = _Inputs(3, 4096, h, hk, True, seed=1)
  t = torch.tensor(3000, device='cuda', dtype=torch.int32)
  outs = [attention_ops.decode_attention(q, kn, vn, ck, cv, t, rel) for _ in range(3)]
  assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
  want = attention_ops.decode_attention_ref(q.float(), kn.float(), vn.float(), ck.float(),
                                            cv.float(), 3000, rel)
  assert _RelErr(outs[0], want) < 5e-3


@pytest.mark.gpu
def test_kernel_replays_in_cuda_graph_for_every_t():
  b, tmax, h, hk, n = 2, 1024, 16, 4, 300
  _, _, _, ck, cv, rel = _Inputs(b, tmax, h, hk, True, seed=2)
  g = torch.Generator(device='cuda').manual_seed(3)
  seq = [tuple(torch.randn(b, 1, x, 128, generator=g, device='cuda').to(torch.bfloat16)
               for x in (h, hk, hk)) for _ in range(n)]
  eager_k, eager_v = ck.clone(), cv.clone()
  eager = [attention_ops.decode_attention(qi * 0.1, ki, vi, eager_k, eager_v, i, rel)
           for i, (qi, ki, vi) in enumerate(seq)]

  sq, sk, sv = (x.clone() for x in seq[0])
  sq.mul_(0.1)
  gk, gv = ck.clone(), cv.clone()
  st = torch.zeros((), dtype=torch.long, device='cuda')
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    attention_ops.decode_attention(sq, sk, sv, gk, gv, st, rel)   # warm-up (writes row 0)
  torch.cuda.current_stream().wait_stream(side)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    out = attention_ops.decode_attention(sq, sk, sv, gk, gv, st, rel)
  gk.copy_(ck)
  gv.copy_(cv)
  for i, (qi, ki, vi) in enumerate(seq):
    sq.copy_(qi * 0.1)
    sk.copy_(ki)
    sv.copy_(vi)
    st.fill_(i)
    graph.replay()
    assert torch.equal(out, eager[i]), i
  assert torch.equal(gk, eager_k) and torch.equal(gv, eager_v)


def _Lm():
  bp = gb.DenseBuilder.Params().Set(
      model_dim=128, attention_num_heads=2, attention_key_value_dim=128, ff_dim=256,
      relative_attention_type='bias', relative_attention_num_buckets=32,
      relative_attention_max_distance=128, label_smoothing=0.0)
  gb.DenseBuilder.SetFPropDtype(bp, torch.bfloat16)
  p = gb.UniTransformer.Params().Set(
      name='lm', builder=bp, vocab_size=64, num_transformer_layers=2, max_length=64,
      positional_embedding=False, label_smoothing=0.0, z_loss=0.0, fprop_dtype=torch.bfloat16)
  with cluster_factory.ForTestingWorker(mode='sync', job='trainer_client', do_eval=True):
    task = p.Instantiate()
  task.to(torch.device('cuda'))
  return task


@pytest.mark.gpu
def test_decode_step_matches_full_forward_and_cuda_graph():
  torch.manual_seed(0)
  task = _Lm()
  bsz, l, tmax = 3, 24, 40
  ids = torch.randint(2, 64, (bsz, l), device='cuda')
  batch = NestedMap(ids=ids, labels=ids, paddings=torch.zeros(bsz, l, device='cuda'),
                    segment_ids=torch.ones(bsz, l, dtype=torch.long, device='cuda'),
                    segment_pos=torch.arange(l, device='cuda').repeat(bsz, 1))
  with torch.no_grad():
    pred = task.ComputePredictions(task.theta, batch)
    full = task._ComputeLogits(task.theta, pred.dec_outputs).float()   # pylint: disable=protected-access
    st = task.InitDecodeState(bsz, tmax, ids.device)
    assert st[0].k.dtype == torch.bfloat16 and st[0].k.shape[-1] == 128
    eager = []
    for i in range(l):
      eager.append(task.DecodeStep(task.theta, ids[:, i], st, i))
      assert _RelErr(eager[-1], full[:, i]) < 2e-2, i

    # the same step captured once, replayed with t as a device scalar
    gst = task.InitDecodeState(bsz, tmax, ids.device)
    sid = ids[:, 0].clone()
    t = torch.zeros((), dtype=torch.long, device='cuda')
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      task.DecodeStep(task.theta, sid, gst, t)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
      logits = task.DecodeStep(task.theta, sid, gst, t)
    for c in gst:
      if c is not None:
        c.k.zero_()
        c.v.zero_()
    for i in range(l):
      sid.copy_(ids[:, i])
      t.fill_(i)
      graph.replay()
      assert _RelErr(logits, eager[i]) < 1e-3, i
