"""`xent_stats` / `xent_bwd` (ops/csrc/xent_kernels.cu) on given bf16 logits against float64
math on the same bf16 values, with no GEMM in between.

One CTA of 256 threads works on a row and each thread reads 8 columns per pass, so a pass
covers 2048 columns. The widths give one thread with data (8), mostly idle threads (1000),
exactly one pass (2048), a second pass of a single vector (2056) and the benchmark's
vocabulary (32000, 15.6 passes).
"""
import pytest
import torch

from lingvo_b200 import ops

_VS = [8, 1000, 2048, 2056, 32000]
_T = 300


def _Logits(t, v, seed, layout):
  """bf16 `[t, v]` logits: multiples of 1/8 in [-8, 8], so every row's maximum is tied many
  times and the lowest index must win, plus rows that stress the online softmax. With
  layout 'slice' they are columns [8, 8 + v) of a `[t, v + 32]` buffer; returns (logits,
  buffer)."""
  gen = torch.Generator().manual_seed(seed)
  x = torch.randint(-64, 65, (t, v), generator=gen).float() / 8
  x[0] = 0.375                                   # constant row
  x[1] += 60.0
  x[2] -= 60.0
  if v >= 16:                                    # one aligned 8-wide block of -inf
    blk = (v // 16) * 8
    x[3, blk:blk + 8] = -float('inf')
  x[4, v - 1] = 9.0                              # unique maximum in the last vector
  x[5, v // 3] = x[5, v - 1] = 9.0               # maximum tied across passes
  if layout == 'dense':
    buf = x.bfloat16().cuda()
    return buf, buf
  buf = torch.randn(t, v + 32, generator=gen).bfloat16().cuda()
  buf[:, 8:8 + v] = x.bfloat16().cuda()
  return buf[:, 8:8 + v], buf


def _Labels(t, v, seed):
  gen = torch.Generator().manual_seed(seed)
  labels = torch.randint(0, v, (t,), generator=gen)
  labels[0] = 0
  labels[1] = v - 1
  labels[-1] = v - 1
  labels[3] = (v // 16) * 8                      # the -inf block (column 0 when v = 8)
  return labels.cuda()


def _Ordered(b):
  """bf16 bit patterns mapped to integers that are consecutive for adjacent bf16 values."""
  i = b.contiguous().view(torch.int16).int()
  return torch.where(i < 0, -(i & 0x7fff), i)


def _AssertWithinBf16Ulp(got, want, slack):
  """bf16 `got` is float64 `want` rounded to bf16 up to one ulp. Where the fp32 terms of an
  element nearly cancel, `got` may instead be within `slack` of `want`."""
  ulps = (_Ordered(got) - _Ordered(want.bfloat16())).abs()
  err = (got.double() - want).abs()
  bad = (ulps > 1) & ~(err <= slack)
  if bool(bad.any()):
    r, c = (int(i) for i in bad.nonzero()[0])
    raise AssertionError('%d elements off by more than 1 bf16 ulp; first [%d, %d]: got %r, '
                         'want %r' % (int(bad.sum()), r, c, got[r, c].item(), want[r, c].item()))


@pytest.mark.gpu
@pytest.mark.parametrize('layout', ['dense', 'slice'])
@pytest.mark.parametrize('v', _VS)
def test_xent_stats_matches_float64(v, layout):
  logits, _ = _Logits(_T, v, v, layout)
  labels = _Labels(_T, v, v + 1)
  lse, true_logit, sum_logits, argmax = ops.native().xent_stats(logits, labels)
  x = logits.double()
  torch.testing.assert_close(lse.double(), torch.logsumexp(x, -1), atol=1e-4, rtol=0)
  assert torch.equal(true_logit.double(), x.gather(1, labels[:, None])[:, 0])
  want_sum, abs_sum = x.sum(-1), x.abs().sum(-1)
  finite = torch.isfinite(want_sum)
  assert torch.equal(sum_logits[~finite].double(), want_sum[~finite])
  err = (sum_logits.double() - want_sum)[finite].abs()
  assert bool((err <= 1e-6 * abs_sum[finite]).all()), err.max().item()
  want_argmax = x.cpu().argmax(-1).cuda()        # the first of tied maxima
  bad = (argmax != want_argmax).nonzero()
  assert bad.numel() == 0, 'argmax differs in %d rows, first %d: got %d, want %d' % (
      bad.numel(), bad[0, 0], argmax[bad[0, 0]], want_argmax[bad[0, 0]])


@pytest.mark.gpu
@pytest.mark.parametrize('layout', ['dense', 'slice'])
@pytest.mark.parametrize('v', _VS)
def test_xent_bwd_matches_float64(v, layout):
  """dlogits = exp(logit - lse)·a - b - onehot(label)·c, written over the logits in place;
  columns outside the logits' slice stay bit for bit as they were."""
  logits, buf = _Logits(_T, v, v, layout)
  labels = _Labels(_T, v, v + 1)
  nat = ops.native()
  lse = nat.xent_stats(logits, labels)[0]
  gen = torch.Generator(device='cuda').manual_seed(v)
  a = torch.rand(_T, device='cuda', generator=gen) + 0.5
  b = torch.rand(_T, device='cuda', generator=gen) / v
  c = torch.rand(_T, device='cuda', generator=gen) + 0.5
  x = logits.double()
  before = buf.clone()
  p_a = torch.exp(x - lse.double()[:, None]) * a.double()[:, None]
  c_hot = torch.zeros_like(x).scatter_(1, labels[:, None], c.double()[:, None])
  want = p_a - b.double()[:, None] - c_hot
  nat.xent_bwd(logits, labels, lse, a, b, c)
  _AssertWithinBf16Ulp(logits, want, 2.0**-18 * (p_a + b.double()[:, None] + c_hot))
  if layout == 'slice':
    assert torch.equal(buf[:, :8].view(torch.int16), before[:, :8].view(torch.int16))
    assert torch.equal(buf[:, 8 + v:].view(torch.int16), before[:, 8 + v:].view(torch.int16))


def _BadXentCalls():
  """(what, position of the bad argument, (logits, labels, lse, a, b, c)) for calls that the
  host-side checks must refuse."""
  t, v = 16, 64
  logits = torch.zeros(t, v, dtype=torch.bfloat16, device='cuda')
  labels = torch.zeros(t, dtype=torch.int64, device='cuda')
  f = torch.zeros(t, device='cuda')
  ok = (logits, labels, f, f, f, f)
  bad = {
      0: [('fp32 logits', logits.float()),
          ('1-D logits', logits.view(-1)),
          ('column stride 2', torch.zeros(t, 2 * v, dtype=torch.bfloat16,
                                          device='cuda')[:, ::2]),
          ('V % 8 != 0', logits[:, :60]),
          ('row stride % 8 != 0', torch.zeros(t, 68, dtype=torch.bfloat16,
                                              device='cuda')[:, :64])],
      1: [('int32 labels', labels.int()),
          ('short labels', labels[:-1]),
          ('strided labels', torch.zeros(2 * t, dtype=torch.int64, device='cuda')[::2]),
          ('labels on the host', labels.cpu())],
  }
  for i, name in enumerate(['lse', 'a', 'b', 'c'], start=2):
    bad[i] = [('bf16 ' + name, f.bfloat16()),
              ('long ' + name, torch.zeros(t + 1, device='cuda')),
              ('strided ' + name, torch.zeros(2 * t, device='cuda')[::2]),
              (name + ' on the host', f.cpu())]
  for i, cases in bad.items():
    for what, x in cases:
      yield what, i, ok[:i] + (x,) + ok[i + 1:]


def _Refusal(fn, *args):
  try:
    fn(*args)
  except RuntimeError as e:
    return str(e)
  return 'accepted'


def test_xent_rejects_host_tensors():
  """Runs without a GPU: host tensors are refused before anything is launched."""
  nat = ops.native()
  logits = torch.zeros(4, 64, dtype=torch.bfloat16)
  labels = torch.zeros(4, dtype=torch.int64)
  f = torch.zeros(4)
  assert 'xent_stats: logits' in _Refusal(nat.xent_stats, logits, labels)
  assert 'xent_bwd: logits' in _Refusal(nat.xent_bwd, logits, labels, f, f, f, f)


@pytest.mark.gpu
def test_xent_rejects_bad_arguments_without_launching():
  """xent_bwd writes 16-byte vectors into the logits in place, so it checks its arguments
  as xent_stats does; a refused call launches nothing."""
  nat = ops.native()
  launches = nat.launch_count()
  for what, i, args in _BadXentCalls():
    assert 'xent_bwd:' in _Refusal(nat.xent_bwd, *args), what
    if i < 2:
      assert 'xent_stats:' in _Refusal(nat.xent_stats, *args[:2]), what
  assert nat.launch_count() == launches
