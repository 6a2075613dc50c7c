"""Flat beam-search decoding of GShard LMs on the CPU (fp32): the `flat_beam_attention` oracle
against a dense masked softmax, one-pass prompt prefill plus beam steps against the full
forward of each hypothesis's own sequence, the search results of `BeamDecodeIds`, and the
refusals of unsupported stacks and arguments."""

import pytest
import torch

from lingvo_b200.core import cluster_factory
from lingvo_b200.core import flat_beam_search_helper as fbs
from lingvo_b200.core import gshard_builder as gb
from lingvo_b200.core import gshard_decode
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.ops import attention as attention_ops


# ------------------------------------------------------------------------------ op ----
def _DenseMaskedAttention(q, k_cache, v_cache, vis, qpos, kpos, rel):
  """Per (b, k, h) the softmax over the visible rows, written out with explicit loops."""
  bsz, kk, h, d = q.shape
  n, hk = k_cache.shape[1], k_cache.shape[2]
  out = torch.zeros(bsz, kk, h, d, dtype=torch.float64)
  for b in range(bsz):
    for k in range(kk):
      rows = [j for j in range(n) if vis[b, k, j]]
      for hh in range(h):
        kv = hh // (h // hk)
        logits = torch.stack([
            (q[b, k, hh].double() * k_cache[b, j, kv].double()).sum() +
            (rel[hh, min(max(int(qpos[b, k]) - int(kpos[b, j]) + n - 1, 0), 2 * n - 2)].double()
             if rel is not None else 0.0) for j in rows])
        p = torch.softmax(logits, 0)
        out[b, k, hh] = (p.unsqueeze(1) * v_cache[b, rows, kv].double()).sum(0)
  return out


@pytest.mark.parametrize('hk', [4, 2, 1])
@pytest.mark.parametrize('use_rel', [False, True])
def test_reference_equals_dense_masked_softmax(hk, use_rel):
  g = torch.Generator().manual_seed(0)
  bsz, kk, h, d, n, slot0 = 2, 3, 4, 8, 45, 33     # rows 33..35 are written by the call
  q = torch.randn(bsz, kk, h, d, generator=g)
  kn, vn = torch.randn(bsz, kk, hk, d, generator=g), torch.randn(bsz, kk, hk, d, generator=g)
  ck, cv = torch.randn(bsz, n, hk, d, generator=g), torch.randn(bsz, n, hk, d, generator=g)
  vis = torch.rand(bsz, kk, n, generator=g) < 0.5
  vis[:, :, slot0 + kk:] = False
  vis[:, torch.arange(kk), slot0 + torch.arange(kk)] = True        # each sees its own row
  vis[0, 1, slot0:slot0 + kk] = True                                 # and one sees siblings
  qpos = torch.randint(0, n, (bsz, kk), generator=g).int()
  kpos = torch.randint(0, n, (bsz, n), generator=g).int()
  rel = torch.randn(h, 2 * n - 1, generator=g) if use_rel else None
  ck0, cv0 = ck.clone(), cv.clone()
  packed = attention_ops.pack_visibility(vis)
  assert packed.shape == (bsz, kk, 2) and packed.dtype == torch.int32
  assert torch.equal(attention_ops.unpack_visibility(packed, n), vis)
  got = attention_ops.flat_beam_attention(q, kn, vn, ck, cv, slot0, packed, qpos, kpos, rel)
  rows = torch.arange(n)
  new = (rows >= slot0) & (rows < slot0 + kk)
  assert torch.equal(ck[:, ~new], ck0[:, ~new]) and torch.equal(cv[:, ~new], cv0[:, ~new])
  assert torch.equal(ck[:, new], kn) and torch.equal(cv[:, new], vn)
  want = _DenseMaskedAttention(q, ck, cv, vis, qpos, kpos, rel)
  torch.testing.assert_close(got.double(), want, atol=1e-5, rtol=1e-5)
  # rows at or past slot0 + K are never visible, whatever the mask says
  vis_all = attention_ops.pack_visibility(torch.ones(bsz, kk, n, dtype=torch.bool))
  got = attention_ops.flat_beam_attention(q, kn, vn, ck, cv, slot0, vis_all, qpos, kpos, rel)
  live = (rows < slot0 + kk).expand(bsz, kk, n)
  torch.testing.assert_close(got.double(),
                             _DenseMaskedAttention(q, ck, cv, live, qpos, kpos, rel),
                             atol=1e-5, rtol=1e-5)


# --------------------------------------------------------------------------- model ----
def _Task(rope=False, kv_heads=None, vocab=40, eos=1):
  bp = gb.DenseBuilder.Params().Set(
      model_dim=16, attention_num_heads=4, attention_num_memory_heads=kv_heads,
      attention_key_value_dim=8, ff_dim=32, relative_attention_type='bias',
      relative_attention_num_buckets=8, relative_attention_max_distance=16,
      use_rotary_position_emb=rope, fprop_dtype=torch.float32, dtype=torch.float32,
      label_smoothing=0.0)
  p = gb.UniTransformer.Params().Set(
      name='lm', builder=bp, vocab_size=vocab, num_transformer_layers=2, max_length=64,
      positional_embedding=rope, label_smoothing=0.0, z_loss=0.0, decoder_eos_id=eos,
      fprop_dtype=torch.float32)
  p.random_seed = 5
  with cluster_factory.ForTestingWorker(mode='sync', job='trainer_client', do_eval=True):
    task = p.Instantiate()
  # spread the weights so that the beam branches
  with torch.no_grad():
    task.dec_emb.theta.embedding.mul_(4.0)
  return task


def _Batch(prompts, width=None):
  width = width or max(len(x) for x in prompts)
  ids = torch.zeros(len(prompts), width, dtype=torch.long)
  pad = torch.ones(len(prompts), width)
  for i, x in enumerate(prompts):
    ids[i, :len(x)] = torch.tensor(x)
    pad[i, :len(x)] = 0.0
  return NestedMap(tgt=NestedMap(ids=ids, paddings=pad))


def _FullLogits(task, seq):
  l = len(seq)
  ids = torch.tensor([seq])
  batch = NestedMap(ids=ids, labels=ids, paddings=torch.zeros(1, l),
                    segment_ids=torch.ones(1, l, dtype=torch.long),
                    segment_pos=torch.arange(l).unsqueeze(0))
  pred = task.ComputePredictions(task.theta, batch)
  return task._ComputeLogits(task.theta, pred.dec_outputs)[0, -1].float()   # pylint: disable=protected-access


def _RecordSteps(task, monkeypatch):
  steps = []
  real = task.BeamDecodeStep

  def Record(theta, ids, pos, state, slot0, vis):
    logits = real(theta, ids, pos, state, slot0, vis)
    steps.append((ids.clone(), pos.clone(), slot0, vis.clone(), logits.clone()))
    return logits
  monkeypatch.setattr(task, 'BeamDecodeStep', Record)
  return steps


@pytest.mark.parametrize('rope,kv_heads', [(False, 2), (True, None)])
def test_every_hypothesis_sees_exactly_its_own_sequence(rope, kv_heads, monkeypatch):
  torch.manual_seed(0)
  task = _Task(rope=rope, kv_heads=kv_heads)
  prompts = [[5, 9, 3], [7, 2, 8, 4, 6, 11, 13], [12], [3, 3, 20, 21, 22]]
  kk = 4
  steps = _RecordSteps(task, monkeypatch)
  with torch.no_grad():
    gshard_decode.BeamDecodeIds(task, task.theta, _Batch(prompts), beam_size=kk, max_steps=6)
    pmax = 8                                            # 7 rounded up to a multiple of K
    n = pmax + kk * 6
    assert len(steps) == 6
    fed = torch.zeros(len(prompts), n, dtype=torch.long)
    branched = False
    for ids, pos, slot0, vis, logits in steps:
      fed[:, slot0:slot0 + kk] = ids
      mask = attention_ops.unpack_visibility(vis, n)
      for b, prompt in enumerate(prompts):
        for k in range(kk):
          slots = mask[b, k].nonzero().flatten()
          assert int(slots[-1]) == slot0 + k                # it sees itself last
          gen = [int(fed[b, s]) for s in slots if s >= pmax]
          seq = prompt[:-1] + gen
          assert gen[0] == prompt[-1] and int(pos[b, k]) == len(seq) - 1
          want = _FullLogits(task, seq)
          torch.testing.assert_close(logits[b, k], want, atol=2e-4, rtol=2e-4)
        branched |= len({tuple(mask[b, k].tolist()) for k in range(kk)}) > 2
    assert branched


def test_beam_search_with_prefix_finds_the_most_likely_sequence():
  # A fixed first-order model: after token t the next-token log-probs are row t of `table`.
  v, eos = 6, 2
  table = torch.full((v, v), -4.0)
  table[5, 3] = 0.0      # prompt … 5 → 3
  table[3, 4] = 0.0      # 3 → 4
  table[4, eos] = 0.0    # 4 → </s>
  table[5, 4] = -0.5     # a tempting but worse branch: 5 → 4 → </s>
  calls = []

  def Callback(ids, pos, seg, mask, state, t):
    calls.append((ids.shape, mask is None, t))
    return (None if mask is None else table[ids]), state

  prefix = torch.tensor([[0, 0, 1, 5], [0, 0, 0, 5]])
  (ids, lens, scores), _ = fbs.flat_beam_search(
      2, 2, 5, Callback, None, eos_id=eos, beam_gap=None, prefix=prefix,
      prefix_len=torch.tensor([3, 1]))
  assert calls[0] == ((2, 4), True, 0) and calls[1] == ((2, 2), False, 2)
  assert ids.shape == (2, 2, 5)
  for b in range(2):
    assert ids[b, 0, :int(lens[b, 0])].tolist() == [3, 4, eos]
    assert ids[b, 1, :int(lens[b, 1])].tolist() == [4, eos]
    assert scores[b, 0] >= scores[b, 1]


def test_ragged_batch_gives_the_same_nbest_as_each_row_alone():
  torch.manual_seed(0)
  task = _Task(kv_heads=2)
  prompts = [[5, 9, 3], [7, 2, 8, 4, 6, 11, 13], [12]]
  with torch.no_grad():
    together = gshard_decode.BeamDecodeIds(task, task.theta, _Batch(prompts), beam_size=4,
                                           max_steps=7)
    for b, prompt in enumerate(prompts):
      alone = gshard_decode.BeamDecodeIds(task, task.theta, _Batch([prompt]), beam_size=4,
                                          max_steps=7)
      assert torch.equal(alone.topk_lens[0], together.topk_lens[b])
      for n in range(4):
        ln = int(alone.topk_lens[0, n])
        assert torch.equal(alone.topk_ids[0, n, :ln], together.topk_ids[b, n, :ln])
      torch.testing.assert_close(alone.topk_scores[0], together.topk_scores[b], atol=1e-4,
                                 rtol=1e-4)
  assert together.topk_ids.shape == (3, 4, 7)
  assert together.prefix_lens.tolist() == [3, 7, 1]
  assert bool((together.topk_scores[:, :-1] >= together.topk_scores[:, 1:]).all())


def test_beam_of_one_follows_greedy_until_greedy_stops(monkeypatch):
  torch.manual_seed(0)
  task = _Task(kv_heads=2, vocab=24, eos=1)
  prompts = [[5, 9, 3], [7, 2, 8, 4, 6], [12]]
  batch = _Batch(prompts)
  with torch.no_grad():
    greedy = gshard_decode.DecodeIds(task, task.theta, batch, max_steps=10)
  steps = _RecordSteps(task, monkeypatch)
  with torch.no_grad():
    gshard_decode.BeamDecodeIds(task, task.theta, batch, beam_size=1, max_steps=10)
  beam = torch.stack([ids[:, 0] for ids, *_ in steps[1:]], 1)   # the tokens chosen at 0..
  compared = 0
  for b, prompt in enumerate(prompts):
    gen = greedy.ids[b, len(prompt):int(greedy.lens[b])].tolist()
    if 1 in gen:
      gen = gen[:gen.index(1)]
    gen = gen[:beam.shape[1]]
    assert beam[b, :len(gen)].tolist() == gen, (b, gen, beam[b])
    compared += len(gen)
  assert compared >= 5


def test_refusals():
  bp = gb.DenseBuilder.Params().Set(
      model_dim=16, attention_num_heads=2, attention_key_value_dim=8, ff_dim=32,
      fprop_dtype=torch.float32, dtype=torch.float32)
  b = bp.Instantiate()
  for sub in (b.DecMultiDconvHeadAttention('mdha'), b.DecEncAttention('cross')):
    lp = b.DecoderLayerStack('dec', [sub, b.DenseReluDense('ffn')], num=1)
    lp.random_seed = 1
    stack = lp.Instantiate()
    stack.InstantiateVariables()
    state = stack.InitDecodeState(1, 16, torch.device('cpu'), torch.float32)
    with pytest.raises(NotImplementedError, match='cannot be prefilled or beam-stepped'):
      stack.Prefill(stack.theta, torch.zeros(1, 4, 16), torch.ones(1, 4, dtype=torch.long),
                    torch.arange(4).unsqueeze(0), state)
    with pytest.raises(NotImplementedError, match='cannot be prefilled or beam-stepped'):
      stack.BeamExtendStep(stack.theta, torch.zeros(1, 2, 16), state, 4,
                           torch.zeros(1, 2, 1, dtype=torch.int32),
                           torch.zeros(1, 2, dtype=torch.int32))

  def Callback(*args):
    raise AssertionError('no call expected')
  with pytest.raises(ValueError, match='multiple of beam_size'):
    fbs.flat_beam_search(1, 4, 3, Callback, None, prefix=torch.ones(1, 6, dtype=torch.long),
                         prefix_len=torch.tensor([2]))
  with pytest.raises(ValueError, match='prefix_len'):
    fbs.flat_beam_search(1, 2, 3, Callback, None, prefix=torch.ones(1, 4, dtype=torch.long),
                         prefix_len=torch.tensor([0]))

  from lingvo_b200 import ops
  mod = ops.native(required=False)
  if mod is not None and hasattr(mod, 'flat_beam_attn_fwd'):
    q = torch.zeros(1, 2, 2, 128, dtype=torch.bfloat16)
    kv = torch.zeros(1, 2, 2, 128, dtype=torch.bfloat16)
    cache = torch.zeros(1, 64, 2, 128, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match='flat_beam_attn'):
      mod.flat_beam_attn_fwd(q, kv, kv, cache, cache, torch.tensor(0),
                             torch.zeros(1, 2, 2, dtype=torch.int32),
                             torch.zeros(1, 2, dtype=torch.int32),
                             torch.zeros(1, 64, dtype=torch.int32), None, 1.0)


def test_decode_tool_writes_the_best_hypothesis(tmp_path):
  from lingvo_b200.models.lm.tools import gshard_lm_decode
  import lingvo_b200.models.lm.params.synthetic_packed_input  # noqa: F401
  f = tmp_path / 'prompts.tsv'
  f.write_text('5 6 7\n8 9\n10 11 12 13\n')
  dec = gshard_lm_decode.GShardLMDecodeBatch(
      'lm.synthetic_packed_input.DenseLmTiny', prefix_max_len=8, batch_size=2,
      max_decode_steps=4, device='cpu', beam_size=2)
  outs = dec.DecodeFiles([str(f)], str(tmp_path / 'out'))
  dec.stop()
  lines = [l.split('\t') for l in open(outs[0]).read().strip().split('\n')]
  assert [l[0] for l in lines] == ['5 6 7', '8 9', '10 11 12 13']
  with torch.no_grad():
    ids, pad = dec.MakeBatch(['5 6 7', '8 9'])
    want = gshard_decode.BeamDecodeIds(dec.task, dec.task.theta,
                                       NestedMap(ids=torch.as_tensor(ids),
                                                 paddings=torch.as_tensor(pad)), beam_size=2)
  for r in range(2):
    n = int(want.topk_lens[r, 0])
    assert lines[r][1] == ' '.join(str(int(i)) for i in want.topk_ids[r, 0, :n])
    assert abs(float(lines[r][2]) - float(want.topk_scores[r, 0])) < 1e-4
