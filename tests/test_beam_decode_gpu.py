"""The flat-beam-search attention kernel (`ops.attention.flat_beam_attention`, csrc/decode_attn.cu)
on the GPU: against the fp32 oracle over head layouts, beam sizes, buffer lengths, masks and
slot0 at chunk boundaries; its cache writes; bitwise reproducibility and CUDA-graph replay
over slot0; argument refusals before any launch; and the bf16 beam step of a UniTransformer
against the full forward of each hypothesis's sequence."""

import pytest
import torch

from lingvo_b200.core import cluster_factory
from lingvo_b200.core import gshard_builder as gb
from lingvo_b200.core import gshard_decode
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.ops import attention as attention_ops

pytestmark = pytest.mark.gpu


def _RelErr(a, b):
  a, b = a.float(), b.float()
  return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _Native():
  from lingvo_b200 import ops
  return ops.native()


def _AncestorMask(b, kk, n, slot0, prompt, g):
  """The masks a flat beam search builds: a right-aligned prompt of `prompt` rows, then one
  row per earlier step (each hypothesis inherits a random parent's path) and its own row."""
  mask = torch.zeros(b, kk, n, dtype=torch.bool)
  if prompt:
    plen = torch.randint(1, prompt + 1, (b,), generator=g)
    for i in range(b):
      mask[i, :, prompt - int(plen[i]):prompt] = True
  for s0 in range(prompt, slot0, kk):
    mask[:, torch.arange(kk), s0 + torch.arange(kk)] = True
    parent = torch.randint(0, kk, (b, kk), generator=g)
    mask = mask.gather(1, parent.unsqueeze(-1).expand(b, kk, n))
  mask[:, torch.arange(kk), slot0 + torch.arange(kk)] = True
  return mask


def _Inputs(b, kk, n, h, hk, use_rel, mask_kind, slot0, seed=0):
  g = torch.Generator().manual_seed(seed)
  gd = torch.Generator(device='cuda').manual_seed(seed)

  def _Bf16(*shape):
    return torch.randn(*shape, generator=gd, device='cuda').to(torch.bfloat16)
  q = _Bf16(b, kk, h, 128) * 0.1
  kn, vn = _Bf16(b, kk, hk, 128), _Bf16(b, kk, hk, 128)
  ck, cv = _Bf16(b, n, hk, 128), _Bf16(b, n, hk, 128)
  if mask_kind == 'random':
    mask = torch.rand(b, kk, n, generator=g) < 0.3
    mask[:, torch.arange(kk), slot0 + torch.arange(kk)] = True
  else:
    mask = _AncestorMask(b, kk, n, slot0, min(slot0, 64), g)
  vis = attention_ops.pack_visibility(mask).cuda()
  qpos = torch.randint(0, n, (b, kk), generator=g).int().cuda()
  kpos = torch.randint(0, n, (b, n), generator=g).int().cuda()
  rel = torch.randn(h, 2 * n - 1, generator=gd, device='cuda') if use_rel else None
  return q, kn, vn, ck, cv, vis, qpos, kpos, rel


@pytest.mark.parametrize('where', ['chunk-edge', 'last'])
@pytest.mark.parametrize('mask_kind', ['random', 'ancestor'])
@pytest.mark.parametrize('use_rel', [False, True])
@pytest.mark.parametrize('n', [100, 1280, 4096])
@pytest.mark.parametrize('kk', [1, 4, 8])
@pytest.mark.parametrize('h,hk', [(16, 16), (16, 4), (16, 1)])
def test_kernel_matches_reference(h, hk, kk, n, use_rel, mask_kind, where):
  b = 2
  chunk = _Native().flat_beam_attn_chunk(b, kk, h, hk, n)
  # 'chunk-edge': the K written rows straddle the first chunk boundary (or start on it)
  slot0 = {'chunk-edge': max(0, min(chunk - kk // 2, n - kk)), 'last': n - kk}[where]
  q, kn, vn, ck, cv, vis, qpos, kpos, rel = _Inputs(b, kk, n, h, hk, use_rel, mask_kind, slot0)
  assert attention_ops.flat_beam_attention_supported(q, ck)
  ck0, cv0 = ck.clone(), cv.clone()
  rk, rv = ck.float(), cv.float()
  want = attention_ops.flat_beam_attention_ref(q.float(), kn.float(), vn.float(), rk, rv,
                                               slot0, vis, qpos, kpos, rel)
  got = attention_ops.flat_beam_attention(q, kn, vn, ck, cv,
                                          torch.tensor(slot0, device='cuda'), vis, qpos, kpos,
                                          rel)
  assert got.shape == (b, kk, h, 128) and got.dtype == torch.bfloat16
  assert _RelErr(got, want) < 5e-3
  rows = torch.arange(n, device='cuda')
  new = (rows >= slot0) & (rows < slot0 + kk)
  assert torch.equal(ck[:, ~new], ck0[:, ~new]) and torch.equal(cv[:, ~new], cv0[:, ~new])
  assert torch.equal(ck[:, new], kn) and torch.equal(cv[:, new], vn)


@pytest.mark.parametrize('h,hk,kk', [(16, 16, 4), (16, 1, 16), (12, 4, 5)])
def test_kernel_is_deterministic(h, hk, kk):
  q, kn, vn, ck, cv, vis, qpos, kpos, rel = _Inputs(3, kk, 4096, h, hk, True, 'random', 3000,
                                                    seed=1)
  s0 = torch.tensor(3000, device='cuda', dtype=torch.int32)
  outs = [attention_ops.flat_beam_attention(q, kn, vn, ck, cv, s0, vis, qpos, kpos, rel)
          for _ in range(3)]
  assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
  want = attention_ops.flat_beam_attention_ref(q.float(), kn.float(), vn.float(), ck.float(),
                                               cv.float(), 3000, vis, qpos, kpos, rel)
  assert _RelErr(outs[0], want) < 5e-3


def test_kernel_replays_in_cuda_graph_for_every_slot0():
  b, kk, n, h, hk = 2, 4, 1024, 16, 4
  *_, ck, cv, _, _, _, rel = _Inputs(b, kk, n, h, hk, True, 'random', 0, seed=2)
  g = torch.Generator().manual_seed(3)
  gd = torch.Generator(device='cuda').manual_seed(3)
  slots = list(range(0, n - kk + 1, kk))[:200]
  seq = []
  for s in slots:
    qkv = tuple(torch.randn(b, kk, x, 128, generator=gd, device='cuda').to(torch.bfloat16)
                for x in (h, hk, hk))
    mask = _AncestorMask(b, kk, n, s, min(s, 32), g)
    seq.append(qkv + (attention_ops.pack_visibility(mask).cuda(),
                      torch.randint(0, n, (b, kk), generator=g).int().cuda()))
  kpos = torch.arange(n, device='cuda', dtype=torch.int32).repeat(b, 1)
  eager_k, eager_v = ck.clone(), cv.clone()
  eager = [attention_ops.flat_beam_attention(qi * 0.1, ki, vi, eager_k, eager_v, s, visi, qp,
                                             kpos, rel)
           for s, (qi, ki, vi, visi, qp) in zip(slots, seq)]

  sq, sk, sv, svis, sqp = (x.clone() for x in seq[0])
  gk, gv = ck.clone(), cv.clone()
  st = torch.zeros((), dtype=torch.long, device='cuda')
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    attention_ops.flat_beam_attention(sq, sk, sv, gk, gv, st, svis, sqp, kpos, rel)   # warm-up
  torch.cuda.current_stream().wait_stream(side)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    out = attention_ops.flat_beam_attention(sq, sk, sv, gk, gv, st, svis, sqp, kpos, rel)
  gk.copy_(ck)
  gv.copy_(cv)
  for i, (s, (qi, ki, vi, visi, qp)) in enumerate(zip(slots, seq)):
    sq.copy_(qi * 0.1)
    sk.copy_(ki)
    sv.copy_(vi)
    svis.copy_(visi)
    sqp.copy_(qp)
    st.fill_(s)
    graph.replay()
    assert torch.equal(out, eager[i]), i
  assert torch.equal(gk, eager_k) and torch.equal(gv, eager_v)


def test_bad_arguments_are_refused_before_any_launch():
  mod = _Native()
  b, kk, n, h, hk = 2, 4, 256, 8, 2
  q, kn, vn, ck, cv, vis, qpos, kpos, rel = _Inputs(b, kk, n, h, hk, True, 'random', 8)
  s0 = torch.tensor(8, device='cuda')
  good = dict(q=q, k_new=kn, v_new=vn, k_cache=ck, v_cache=cv, slot0=s0, vis=vis, qpos=qpos,
              kpos=kpos, rel=rel, scale=1.0)
  bad = {
      'q': q.float(), 'k_new': kn[:, :2], 'v_new': vn.transpose(1, 2),
      'k_cache': ck[:, :, :1], 'v_cache': cv[..., :64],
      'slot0': torch.tensor(8), 'vis': vis[..., :1], 'qpos': qpos.long(), 'kpos': kpos.cpu(),
      'rel': rel[:, :-1],
  }
  before = mod.launch_count()
  for name, value in bad.items():
    with pytest.raises(RuntimeError, match='flat_beam_attn'):
      mod.flat_beam_attn_fwd(**dict(good, **{name: value}))
  q17 = torch.zeros(1, 17, 1, 128, dtype=torch.bfloat16, device='cuda')
  k17 = torch.zeros(1, 17, 1, 128, dtype=torch.bfloat16, device='cuda')
  c = torch.zeros(1, 64, 1, 128, dtype=torch.bfloat16, device='cuda')
  with pytest.raises(RuntimeError, match='K <= 16'):
    mod.flat_beam_attn_fwd(q17, k17, k17, c, c, s0, torch.zeros(1, 17, 2, dtype=torch.int32,
                                                                 device='cuda'),
                           torch.zeros(1, 17, dtype=torch.int32, device='cuda'),
                           torch.zeros(1, 64, dtype=torch.int32, device='cuda'), None, 1.0)
  torch.cuda.synchronize()
  assert mod.launch_count() == before
  mod.flat_beam_attn_fwd(**good)
  assert mod.launch_count() > before


def _Lm():
  bp = gb.DenseBuilder.Params().Set(
      model_dim=128, attention_num_heads=4, attention_num_memory_heads=2,
      attention_key_value_dim=128, ff_dim=256, relative_attention_type='bias',
      relative_attention_num_buckets=32, relative_attention_max_distance=128,
      relative_attention_use_universal_1d_position=True, label_smoothing=0.0)
  gb.DenseBuilder.SetFPropDtype(bp, torch.bfloat16)
  p = gb.UniTransformer.Params().Set(
      name='lm', builder=bp, vocab_size=64, num_transformer_layers=2, max_length=64,
      positional_embedding=False, label_smoothing=0.0, z_loss=0.0, fprop_dtype=torch.bfloat16)
  with cluster_factory.ForTestingWorker(mode='sync', job='trainer_client', do_eval=True):
    task = p.Instantiate()
  task.to(torch.device('cuda'))
  return task


def test_beam_step_runs_our_kernel_and_matches_the_full_forward(monkeypatch):
  torch.manual_seed(0)
  task = _Lm()
  prompts = [[5, 9, 3, 17, 40], [7, 2, 8, 4, 6, 11, 13, 50, 21, 22, 23], [12]]
  kk, steps_n = 4, 6
  width = max(len(x) for x in prompts)
  ids = torch.zeros(len(prompts), width, dtype=torch.long, device='cuda')
  pad = torch.ones(len(prompts), width, device='cuda')
  for i, x in enumerate(prompts):
    ids[i, :len(x)] = torch.tensor(x)
    pad[i, :len(x)] = 0.0
  batch = NestedMap(tgt=NestedMap(ids=ids, paddings=pad))

  def Refuse(*args, **kwargs):
    raise AssertionError('the beam step fell back to the fp32 oracle')
  monkeypatch.setattr(attention_ops, 'flat_beam_attention_ref', Refuse)
  from lingvo_b200 import ops
  recorded = []
  real = task.BeamDecodeStep

  def Record(theta, tid, pos, state, slot0, vis):
    before = ops.native().launch_count()
    logits = real(theta, tid, pos, state, slot0, vis)
    torch.cuda.synchronize()
    recorded.append((tid.clone(), slot0, vis.clone(), logits.clone(),
                     ops.native().launch_count() - before))
    return logits
  monkeypatch.setattr(task, 'BeamDecodeStep', Record)
  with torch.no_grad():
    res = gshard_decode.BeamDecodeIds(task, task.theta, batch, beam_size=kk, max_steps=steps_n)
  assert res.topk_ids.shape == (3, kk, steps_n)
  pmax = 12
  n = pmax + kk * steps_n
  fed = torch.zeros(len(prompts), n, dtype=torch.long, device='cuda')
  assert recorded
  for tid, slot0, vis, logits, launches in recorded:
    assert launches > 0
    fed[:, slot0:slot0 + kk] = tid
    mask = attention_ops.unpack_visibility(vis, n)
    for b, prompt in enumerate(prompts):
      for k in range(kk):
        gen = [int(fed[b, s]) for s in mask[b, k].nonzero().flatten() if s >= pmax]
        seq = prompt[:-1] + gen
        l = len(seq)
        sid = torch.tensor([seq], device='cuda')
        full = NestedMap(ids=sid, labels=sid, paddings=torch.zeros(1, l, device='cuda'),
                         segment_ids=torch.ones(1, l, dtype=torch.long, device='cuda'),
                         segment_pos=torch.arange(l, device='cuda').unsqueeze(0))
        with torch.no_grad():
          pred = task.ComputePredictions(task.theta, full)
          want = task._ComputeLogits(task.theta, pred.dec_outputs).float()[0, -1]   # pylint: disable=protected-access
        assert _RelErr(logits[b, k], want) < 2e-2, (slot0, b, k)
