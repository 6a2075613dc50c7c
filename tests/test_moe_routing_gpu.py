"""The fused MoE gate + dispatch and the slot-major scatter (ops/csrc/moe_kernels.cu), called
directly and checked exactly against the fp32 gating oracle `moe.top2_gate_ref`.

Logits are multiples of 1/64 in [-4, 4], with +2 on one or two experts so that first and
second choices overflow capacity. Two distinct logits then differ by at least a factor
e^(1/64) after the softmax, so the kernel's `__expf` and the oracle's `torch.softmax` rank
every token alike, while the many exact ties check that both pick the lowest expert id. So
index, pos, keep and the slot table must match exactly, and every expert-buffer row bitwise.

The expert buffers are filled with a NaN bit pattern beforehand, so a row the kernel never
wrote cannot pass for a zero row.
"""
import pytest
import torch

from lingvo_b200 import ops
from lingvo_b200.core import gshard_layers
from lingvo_b200.ops import moe

_SENTINEL = 0x7fc1          # a bf16 NaN

# (G, S, E, capacity factor); C = gshard_layers.ExpertCapacity(S, E, 0, factor).
_SHAPES = [
    pytest.param(8, 1024, 8, 2.0, id='g8s1024e8'),      # the benchmark's groups: 4 scan chunks
    pytest.param(3, 1000, 16, 2.0, id='g3s1000e16'),    # S not a multiple of 32 or 256
    pytest.param(2, 4096, 32, 2.0, id='g2s4096e32'),    # > 48 KiB shared memory, 32 experts
    pytest.param(5, 77, 2, 0.5, id='g5s77e2'),          # both choices overflow heavily
    pytest.param(4, 1, 32, 2.0, id='g4s1e32'),          # the smallest group
]


def _Logits(g, s, e, seed):
  gen = torch.Generator().manual_seed(seed)
  logits = torch.randint(-256, 257, (g, s, e), generator=gen).float() / 64
  logits[..., 1 % e] += 2.0
  if e > 2:
    logits[..., e // 2] += 2.0
  return logits


def _Paddings(g, s, seed):
  """Two random padded spans in each group but the last, which is fully padded."""
  gen = torch.Generator().manual_seed(seed)
  pad = torch.zeros(g, s)
  for gi in range(g - 1):
    for _ in range(2):
      start = int(torch.randint(0, s, (1,), generator=gen))
      n = int(torch.randint(0, s // 4 + 2, (1,), generator=gen))
      pad[gi, start:start + n] = 1.0
  pad[g - 1] = 1.0
  return pad


def ExpectedSlots(index, pos, gate, e, c):
  """The slot tables `[E, G, C]` a dispatch of (index, pos, gate) `[2, G, S]` must fill: the
  token id g·S + t and the choice k of every choice with a nonzero gate, -1 elsewhere."""
  _, _, s = index.shape
  token = torch.full((e, index.shape[1], c), -1, dtype=torch.int32)
  choice = torch.full_like(token, -1)
  k, g, t = torch.nonzero(gate != 0, as_tuple=True)
  slot = (index[k, g, t].long(), g, pos[k, g, t].long())
  token[slot] = (g * s + t).int()
  choice[slot] = k.int()
  assert int((token >= 0).sum()) == k.numel(), 'two kept choices share a slot'
  return token, choice


def _AssertEqual(name, got, want):
  got, want = got.cpu(), want.cpu()
  assert got.shape == want.shape, (name, tuple(got.shape), tuple(want.shape))
  bad = got != want
  if bool(bad.any()):
    first = tuple(int(i) for i in bad.nonzero()[0])
    raise AssertionError('%s: %d of %d differ; first at %s: got %s, want %s' % (
        name, int(bad.sum()), bad.numel(), first, got[first].item(), want[first].item()))


def _AssertRowsBitwise(name, got, want):
  """bf16 `got` == `want` bit for bit; reports rows still holding the sentinel."""
  gi, wi = got.view(torch.int16), want.view(torch.int16)
  unwritten = int((gi.reshape(-1, gi.shape[-1]) == _SENTINEL).all(-1).sum())
  assert unwritten == 0, '%s: %d rows were never written' % (name, unwritten)
  _AssertEqual(name, gi, wi)


def _SentinelBuffer(*shape):
  return torch.full(shape, _SENTINEL, dtype=torch.int16, device='cuda').view(torch.bfloat16)


def _PeerTable(bufs):
  return torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device='cuda')


def _GateDispatch(logits, pad, x, peers, c, e_local, rank, ep, legacy):
  return ops.native().moe_gate_dispatch(
      logits.cuda().contiguous(), None if pad is None else pad.cuda(), x, peers, c, e_local,
      rank, ep, legacy)


def _CheckGate(got, ref, e, c):
  """Compares the kernel's (index, pos, gate, slot_token) with the oracle; returns the
  expected slot tables."""
  index, pos, gate, slot_token = [t.cpu() for t in got]
  _AssertEqual('index', index, ref.index)
  _AssertEqual('pos', pos, ref.pos)
  _AssertEqual('keep', gate != 0, ref.gate != 0)
  torch.testing.assert_close(gate, ref.gate, atol=1e-6, rtol=1e-5)
  token, choice = ExpectedSlots(ref.index, ref.pos, ref.gate, e, c)
  _AssertEqual('slot_token', slot_token, token)
  return token, choice


def _ExpectedRows(src, token, choice=None, gate=None):
  """`[E, G, C, M]`: src[token] (times the gate of the choice in that slot), 0 where -1."""
  tok = token.long().cuda()
  t = tok.clamp_min(0)
  rows = src[t]
  if gate is not None:
    scale = gate.reshape(2, -1)[choice.long().cuda().clamp_min(0), t]
    rows = (rows.float() * scale.unsqueeze(-1)).bfloat16()
  return torch.where((tok >= 0).unsqueeze(-1), rows, torch.zeros_like(rows))


def _Capacity(s, e, factor):
  return gshard_layers.ExpertCapacity(s, e, 0, factor)


# ------------------------------------------------------------------------ CPU --
@pytest.mark.parametrize('legacy', [True, False])
def test_expected_slot_table_matches_dense_dispatch(legacy):
  """The oracle side of the GPU tests: the slot table built from `top2_gate_ref` marks the
  same (token, expert, slot) triples as the dense dispatch tensor of `Top2GatingOnLogits`,
  at a capacity small enough that both choices overflow."""
  g, s, e, c = 3, 40, 4, 8
  logits, pad = _Logits(g, s, e, 5), _Paddings(g, s, 6)
  ref = moe.top2_gate_ref(logits, pad, c, legacy)
  assert ref.capacity == c
  token, _ = ExpectedSlots(ref.index, ref.pos, ref.gate, e, c)
  _, _, dispatch = gshard_layers.Top2GatingOnLogits(
      None, pad, logits, 1, e, c, torch.float32, False, 'all', 0.0, legacy, None)
  dense = torch.zeros(g, s, e, c)
  ei, gi, ci = torch.nonzero(token >= 0, as_tuple=True)
  dense[gi, token[ei, gi, ci].long() - gi * s, ei, ci] = 1.0
  assert torch.equal(dense, dispatch)
  nonpad = int((pad == 0).sum())
  assert 0 < int((ref.gate[0] != 0).sum()) < nonpad       # some first choices dropped
  assert 0 < int((ref.gate[1] != 0).sum()) < nonpad       # and some second choices


# ------------------------------------------------------------------------ GPU --
@pytest.mark.gpu
@pytest.mark.parametrize('m', [2048, 328])
@pytest.mark.parametrize('padded', [False, True], ids=['nopad', 'pad'])
@pytest.mark.parametrize('legacy', [True, False], ids=['legacy', 'renorm'])
@pytest.mark.parametrize('g,s,e,factor', _SHAPES)
def test_gate_dispatch_matches_oracle(g, s, e, factor, legacy, padded, m):
  c = _Capacity(s, e, factor)
  seed = g * 1000 + s + e
  logits = _Logits(g, s, e, seed)
  pad = _Paddings(g, s, seed + 1) if padded else None
  ref = moe.top2_gate_ref(logits, pad, c, legacy)
  gen = torch.Generator(device='cuda').manual_seed(seed)
  x = torch.randn(g * s, m, device='cuda', generator=gen).bfloat16()
  xe = _SentinelBuffer(e, g, c, m)
  got = _GateDispatch(logits, pad, x, _PeerTable([xe]), c, e, 0, 1, legacy)
  token, _ = _CheckGate(got, ref, e, c)
  _AssertRowsBitwise('expert rows', xe, _ExpectedRows(x, token))

  # Without x a single CTA per group computes the gate: it must agree bit for bit.
  alone = _GateDispatch(logits, pad, None, _PeerTable([xe]), c, e, 0, 1, legacy)
  for name, a, b in zip(['index', 'pos', 'gate', 'slot_token'], alone, got):
    _AssertEqual(name + ' (x=None)', a.view(torch.int32), b.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize('gated', [False, True], ids=['ungated', 'gated'])
@pytest.mark.parametrize('m', [2048, 328])
@pytest.mark.parametrize('g,s,e,factor', _SHAPES)
def test_scatter_rows_matches_oracle(g, s, e, factor, m, gated):
  """`moe_scatter_rows` with the kernel's own slot table: row (e, g, c) = src[token] times the
  gate of the choice that landed there, rounded once to bf16, or zeros."""
  c = _Capacity(s, e, factor)
  seed = g * 1000 + s + e
  logits, pad = _Logits(g, s, e, seed), _Paddings(g, s, seed + 1)
  ref = moe.top2_gate_ref(logits, pad, c, False)
  peers = _PeerTable([_SentinelBuffer(1, 8)])
  got = _GateDispatch(logits, pad, None, peers, c, e, 0, 1, False)
  token, choice = _CheckGate(got, ref, e, c)
  index, gate, slot_token = got[0].view(2, -1), got[2].view(2, -1), got[3]
  gen = torch.Generator(device='cuda').manual_seed(seed + 2)
  src = torch.randn(g * s, m, device='cuda', generator=gen).bfloat16()
  dst = _SentinelBuffer(e, g, c, m)
  ops.native().moe_scatter_rows(src, slot_token, index, gate if gated else None,
                                _PeerTable([dst]), e, 0, 1)
  want = _ExpectedRows(src, token, choice, gate) if gated else _ExpectedRows(src, token)
  _AssertRowsBitwise('scattered rows', dst, want)


@pytest.mark.gpu
@pytest.mark.parametrize('m', [2048, 328])
@pytest.mark.parametrize('g_l,s,e,factor', [
    pytest.param(4, 1024, 8, 2.0, id='g4s1024e8'),
    pytest.param(3, 1000, 16, 2.0, id='g3s1000e16'),
])
def test_two_rank_dispatch_and_scatter_address_every_row(g_l, s, e, factor, m):
  """ep = 2 on one device: two local buffers stand for the two ranks' expert buffers. Each
  rank dispatches its own groups into both; buffer d then holds, at row
  (e_l·G_t + r·G_l + g)·C + c, rank r's slot (d·E_l + e_l, g, c)."""
  ep, e_l, c = 2, e // 2, _Capacity(s, e, factor)
  bufs = [_SentinelBuffer(e_l, ep, g_l, c, m) for _ in range(ep)]
  dyes = [_SentinelBuffer(e_l, ep, g_l, c, m) for _ in range(ep)]
  ranks = []
  for r in range(ep):
    seed = 77 + r
    logits, pad = _Logits(g_l, s, e, seed), _Paddings(g_l, s, seed + 1)
    ref = moe.top2_gate_ref(logits, pad, c, False)
    gen = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(g_l * s, m, device='cuda', generator=gen).bfloat16()
    dy = torch.randn(g_l * s, m, device='cuda', generator=gen).bfloat16()
    got = _GateDispatch(logits, pad, x, _PeerTable(bufs), c, e_l, r, ep, False)
    token, choice = _CheckGate(got, ref, e, c)
    ops.native().moe_scatter_rows(dy, got[3], got[0].view(2, -1), got[2].view(2, -1),
                                  _PeerTable(dyes), e_l, r, ep)
    ranks.append((_ExpectedRows(x, token),
                  _ExpectedRows(dy, token, choice, got[2].view(2, -1))))
  for name, out, which in (('dispatch', bufs, 0), ('scatter', dyes, 1)):
    for d in range(ep):
      want = torch.stack([ranks[r][which].view(ep, e_l, g_l, c, m)[d] for r in range(ep)], 1)
      _AssertRowsBitwise('%s into rank %d' % (name, d), out[d], want)
