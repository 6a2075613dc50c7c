"""The decode-attention, flat-beam-attention and beam top-K kernels against float64 and exact
oracles at the serving shapes and at the edges of their tiling.

Kernels: `decode_attn_fwd` and `flat_beam_attn_fwd` (ops/csrc/decode_attn.cu) and `beam_topk`
(ops/csrc/beam_kernels.cu). Line numbers below are decode_attn.cu's.

The contract, for bf16 q, keys and values (D = 128), an fp32 `rel` table and a float scale:

    y = bf16( Σ_j p_j·v_j ),   p = softmax_j over the visible keys of x_j,
    x_j = scale·q·k_j + rel[h, idx_j]

Decode: idx = t − j + T − 1, visible ⇔ j ≤ t for t in [0, T), every key otherwise; key t is
k_new / v_new. Flat beam: idx = qpos[k] − kpos[j] + N − 1, visible ⇔ mask bit j of the
hypothesis ∧ j < min(slot0 + K, N); rows slot0 + k are k_new / v_new[:, k]. Both clamp idx to
[0, 2T−2] / [0, 2N−2]. A query that sees no key returns exact zeros.

The oracle computes x in float64 from the same bf16 inputs, the softmax with masks (no −1e9
additions), ref = Σ p_j·v_j and A = Σ p_j·|v_j| ≥ |ref|. It runs on the device in slabs of
batch rows holding at most 2^25 float64 cache elements (268 MB per operand), so it adds a
few hundred MB at B = 64, T = 4096, where each bf16 cache is 1.07 GB.

Where the kernels round (u = 2^-24):

  * Logits: one fp32 fma chain of 128 terms per (query, key), in head-dim order 0…127
    (`TileLogits`, :109, and its inline copy at :243). bf16 products are exact in fp32, so
    the chain's error is at most u·Σ_k |s_k|, the magnitudes of its 128 partial sums, which
    the oracle computes (`_PartialSums`). Then `× scale` and `+ rel` (:263-264) round once
    each. So δ_j = u·(scale·Σ_k|s_k| + scale·|s_j| + |x_j|).
  * Weights: `__expf(x − m)` (:267-268, :647-648) rounds x − m (u·|x − m|), multiplies by
    log2(e) in fp32 (the constant and the product: 2u·|x − m| more) and takes
    `ex2.approx.ftz.f32`, whose maximum relative error PTX states as at most 2^-22 = 4u. m
    only grows, and the running max, the warp fold's max (:326, :682) and the split fold's
    max (:355, :713) telescope: the arguments a key's weight passes through sum to M − x_j,
    M the row's largest logit. Every `alpha` rescale (one per tile a warp streams, n_w =
    chunk/128 at most), the warp fold and the split fold add one ex2 (4u) and one multiply
    (u). A weight below 2^-126 relative to the running max is flushed: keys with
    x_j < M − 60 count as wholly lost. So a key's weight is off by a relative
    ε_j = δ_j + 3u·(M − x_j) + 5u·(n_w + 3), or 1 where flushed. A relative weight error ε_j
    moves the output by Σ_j p_j·ε_j·|v_j − ref| ≤ Σ_j p_j·ε_j·|v_j| + |ref|·Σ_j p_j·ε_j,
    which is ≤ 2·max ε·A; the oracle uses the left side.
  * Accumulation: each lane accumulates o over the keys its warp streams, round robin over
    32-key tiles (:228, :617), so the fma chain is 32·n_w = chunk/4 long, not T; ℓ is one
    fma per tile per lane (:270) and a 5-level shuffle sum (:305). The warp fold adds 4
    terms (:323-344, :679-702) and the split fold S (:348-363, :706-722), each a multiply and
    an add. One IEEE division. Together the absolute error after normalisation is at most
    u·L·A with L = 33·n_w + 4·S + 22.
  * One `__float2bfloat16_rn` (:336, :362, :694, :721): ½ ulp.

So every element must satisfy

    |y − ref| ≤ C·(½·ulp_bf16(max(|ref|, |y|)) + E),   C = 2,
    E = u·L·A + Σ_j p_j·ε_j·|v_j| + |ref|·Σ_j p_j·ε_j.

There is no blanket T·u·A term: with random V, |ref| ≈ A/50, and T·u·A at T = 4096 is as
large as one key's contribution. The real chain lengths keep one key dropped or doubled
above the bound at T = 4096.

Exact parts, checked bitwise: zeros (not NaN) for a flat-beam query that sees no key; cache
rows other than the written ones untouched, the written rows equal to k_new / v_new, and
nothing written for t ∉ [0, T) or rows ≥ N; three calls identical, and an int32 t / slot0
identical to an int64 one. A per-element bound one ulp wide cannot see a truncating bf16
pack, so a rounding check allows at most 1 % of the elements of a case with ≥ 2^14 outputs
above ⅝ ulp of |ref|.

Mutation controls. Every case builds mutated float64 oracles from the same pieces and each
must put some element above the bound. Decode: key t read from the stale cache row instead
of k_new / v_new; the first key of split 1 (j = chunk; with one live split, the first key of
the last tile) dropped, and counted twice; the rel index off by one for key t only; for
G > 16, the second query-head group given the first group's rel rows. Flat beam: the mask
bit of row 32·w + 31 read from word w + 1; the last of the fresh rows below N read from the
cache; qpos of hypothesis k + 1 used for k; the first tile a hypothesis sees skipped. A
control whose mutation cannot change the result is not built: no t row for t ∉ [0, T); no
rel; K = 1 for the qpos control; a K = 1 ancestor mask, whose bits are all set, for the
mask-word control; counting the only visible key twice; a bias change that is constant
over every query's visible keys (one visible key, or every index clamped to one end).

Peaky logits (q·1) put almost all the weight on a few keys, where dropping a fixed key
changes nothing visible. So every decode case sets the key rows of j = chunk (or its
single-split stand-in) and of t, in every batch row and KV head, to a multiple of the
group's first query head, chosen so that head scores the key 1 below its largest other
logit (`_Boost`). Flat-beam cases use q·0.1, or q·1 with scale 1/√128, where no key
dominates, and a fresh row has its own query's position. In the flat-beam cases with a
±30 table (+30 on every other run of 32 indices from N − 1, −30 on 5 %), all hypotheses
share one position, as in a real step, so every fresh row sits in a +30 run for every
hypothesis; otherwise a fresh row in a −30 run would carry no weight anywhere.

Cases. Serving shapes (DESIGN.md decode and flat-beam benchmarks, H = 16, D = 128, rel
present): decode B ∈ {1, 8, 64} × T ∈ {1024, 4096} × Hk ∈ {16, 4, 1} at t = T − 1 and at t
in the middle of a chunk; flat beam B = 8, N = 4096, K ∈ {4, 8}, Hk ∈ {16, 4, 1} and B = 1,
K = 16, Hk ∈ {16, 1}, slot0 = N − K, ancestor masks with a 64-row prompt. The edge sweep
covers G ∈ {1, 2, 3, 5, 8, 16, 20, 32}, T ∈ {1, 31, 32, 33, 127, 128, 129, 4097}, t ∈ {0,
31, 32, chunk − 1, chunk, chunk + 1, T − 1, T, −1, 10·T}, K ∈ {1, 2, 3, 5, 16}, slot0 ∈ {0,
straddling the first chunk boundary, on it, N − K, N − K + 2}, scale ∈ {1, 1/√128}, flat
and peaky logits, a rel table with ±30 entries (a later tile raises the running max, and
`alpha` rescales), positions that hit both clamp ends, and masks: random 30 %, ancestor,
all visible rows in one split, a hypothesis that sees no row, one that sees only itself,
bits set at rows ≥ slot0 + K and bits past N in the last word. `test_cases_reach_every_path`
mirrors the host's dispatch with the device's own chunk and asserts that the cases reach
all five instantiations of each kernel with S > 1, S == 1 for each kernel, and more than one
query-head group with a partial last group.

beam_topk: every score is one fp32 add, so it is compared bit for bit with an explicit
(score desc, word id asc) ordering computed on the host, on all five outputs.

Measured once on an H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock); the inputs
are seeded. Worst err/bound and the share of elements above ⅝ ulp, serving shapes:

    decode, H = 16        Hk = 16                Hk = 4                 Hk = 1
                          t=T−1     mid          t=T−1     mid          t=T−1     mid
    B=1   T=1024     0.490 0      0.492 0      0.487 0      0.493 0      0.486 4.9e-4 0.494 0
    B=1   T=4096     0.475 4.9e-4 0.486 0      0.468 4.9e-4 0.491 0      0.476 0      0.492 0
    B=8   T=1024     0.492 0      0.491 0      0.489 6.1e-5 0.494 0      0.489 6.1e-5 0.495 6.1e-5
    B=8   T=4096     0.461 0      0.472 6.1e-5 0.476 6.1e-5 0.488 0      0.481 6.1e-5 0.492 6.1e-5
    B=64  T=1024     0.485 5.3e-5 0.487 7.6e-5 0.486 9.9e-5 0.488 8.4e-5 0.491 5.3e-5 0.494 5.3e-5
    B=64  T=4096     0.458 1.1e-4 0.461 1.3e-4 0.460 1.2e-4 0.462 1.1e-4 0.477 3.8e-5 0.486 6.1e-5

    flat beam, N = 4096   Hk = 16        Hk = 4         Hk = 1
    B=8  K=4              0.479 6.1e-5   0.485 3.1e-5   0.486 1.5e-5
    B=8  K=8              0.481 9.9e-5   0.485 4.6e-5   0.487 6.9e-5
    B=1  K=16             0.491 3.1e-5   —              0.492 0

    edge sweeps: decode (88 cases) ≤ 0.497 and ≤ 3.9e-3; flat beam (83 cases) ≤ 0.498 and
    ≤ 7.8e-4. (Shares at cases below 2^14 outputs are printed but not checked.)

Every ratio is below ½: the error is the final bf16 rounding, and the accumulation and
weight terms are headroom. Every control was rejected at every case. The CPU test finds
bf16 P rejected at every shape it runs (worst err/bound 5–52), so a tensor-core P·V with
bf16 P needs a bound of its own. The whole module takes ~16 s of test time on the H100.
"""
import pytest
import torch

from lingvo_b200.ops import attention as A
from lingvo_b200.ops import beam_search as bs

_U = 2.0**-24
_C = 2.0
_D = 128
_MAXG = 16                 # query heads / pairs per CTA
_CTA_KEYS = 128            # the chunk is a multiple of this
_ELEMS = 2**25             # float64 cache elements per oracle slab
_FLUSH = -60.0             # keys this far below the max count as lost
_ROUND_ULPS = 0.625
_ROUND_FRAC = 0.01
_ROUND_MIN = 2**14
_NEG = bs.NEG


def _Ulp(t):
  """One bf16 ulp at |t| (float64), floored at the smallest normal."""
  a = t.abs().clamp_min(2.0**-126)
  return torch.exp2(torch.floor(torch.log2(a)) - 7)


def _Bits(t):
  return t.detach().contiguous().view(torch.int16)


def _Bound(ref, y, e):
  return _C * (0.5 * _Ulp(torch.maximum(ref.abs(), y.abs())) + e)


# ------------------------------------------------------------------ the oracle ----
def _PartialSums(qg, kc):
  """Σ_k |s_k| over the 128 partial sums of each logit's fma chain, head dims in order.
  qg [b, c, p, D], kc [b, n, c, D] float64 → [b, c, p, n]."""
  b, c, p, d = qg.shape
  n = kc.shape[1]
  step = max(1, _ELEMS // (b * c * p * d))
  out = torch.empty(b, c, p, n, dtype=torch.float64, device=qg.device)
  kt = kc.permute(0, 2, 1, 3)
  for j0 in range(0, n, step):
    prod = qg.unsqueeze(3) * kt[:, :, j0:j0 + step].unsqueeze(2)     # [b, c, p, nj, D]
    out[..., j0:j0 + step] = prod.cumsum_(-1).abs_().sum(-1)
  return out


def _Softmax(x, vis, v, kw=None):
  """ref = Σ p·v over the visible keys (weights times `kw`), the weights p and the max.
  x [b, c, p, n], vis bool broadcastable to x, v [b, n, c, D]. No visible key: ref = 0."""
  xm = x.masked_fill(~vis, float('-inf'))
  m = xm.amax(-1, keepdim=True)
  m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
  e = torch.exp(xm - m)
  if kw is not None:
    e = e * kw
  w = e / e.sum(-1, keepdim=True).clamp_min(1e-300)
  return torch.einsum('bcpn,bncd->bcpd', w, v), w, m


class _Result:
  """Worst err/bound, elements above the rounding threshold, and which controls were caught."""

  def __init__(self):
    self.worst, self.over, self.total, self.caught = 0.0, 0, 0, {}

  def Finish(self, what):
    if self.total >= _ROUND_MIN:
      assert self.over <= _ROUND_FRAC * self.total, (
          '%s: %d of %d elements above %g ulp: not rounded to nearest from fp32' % (
              what, self.over, self.total, _ROUND_ULPS))
    missed = [k for k, v in self.caught.items() if not v]
    assert not missed, '%s: the bound does not reject: %s' % (what, ', '.join(missed))
    share = self.over / max(self.total, 1)
    print('%s: worst err/bound %.4f, share above %g ulp %.1e' % (what, self.worst, _ROUND_ULPS,
                                                                  share))
    return self.worst, share


@torch.no_grad()
def _CheckSlab(res, sl, scale, chunk, n_split, what):
  """Asserts the bound and the exact zeros for one slab, and runs its controls.

  `sl`: qg [b, c, p, D], kc / vc [b, n, c, D] (float64, the written rows in place), bias
  broadcastable to [b, c, p, n] or None, vis bool broadcastable to it, y [b, c, p, D] bf16,
  and `controls`: name → function(pieces) → mutated pieces."""
  qg, kc, vc, bias, vis, y = sl['qg'], sl['kc'], sl['vc'], sl['bias'], sl['vis'], sl['y']
  s = torch.einsum('bcpd,bncd->bcpn', qg, kc)
  x = scale * s if bias is None else scale * s + bias
  ref, w, m = _Softmax(x, vis, vc)
  n_w = chunk // _CTA_KEYS
  big_l = 33 * n_w + 4 * n_split + 22
  delta = _U * (scale * _PartialSums(qg, kc) + scale * s.abs() + x.abs())
  eps = delta + 3 * _U * (m - x) + 5 * _U * (n_w + 3)
  eps = torch.where(x - m < _FLUSH, torch.ones_like(eps), eps)
  we = w * eps
  va = vc.abs()
  e = (_U * big_l * torch.einsum('bcpn,bncd->bcpd', w, va) +
       torch.einsum('bcpn,bncd->bcpd', we, va) + ref.abs() * we.sum(-1, keepdim=True))
  yd = y.double()
  assert bool(torch.isfinite(yd).all()), '%s: non-finite output' % what
  err = (yd - ref).abs()
  bound = _Bound(ref, yd, e)
  bad = err > bound
  assert not bool(bad.any()), '%s: %d elements outside the bound, worst err/bound %g' % (
      what, int(bad.sum()), float((err / bound)[bad].max()))
  res.worst = max(res.worst, float((err / bound).max()))
  blind = ~vis.expand_as(x).any(-1)
  assert bool((_Bits(y)[blind] == 0).all()), '%s: a query that sees no key is not +0' % what
  res.over += int((err > _ROUND_ULPS * _Ulp(ref)).sum())
  res.total += err.numel()
  pieces = dict(x=x, s=s, vis=vis, v=vc, kw=None)
  for name, fn in sl['controls'].items():
    mut = fn(dict(pieces))
    if mut is None:
      continue
    ref2, _, _ = _Softmax(mut['x'], mut['vis'], mut['v'], mut['kw'])
    hit = bool(((yd - ref2).abs() > _Bound(ref2, yd, e)).any())
    res.caught[name] = res.caught.get(name, False) or hit


def _Moves(d, vis):
  """Whether adding d to the logits can change the softmax: d is not constant over the
  visible keys of some query."""
  d, vis = torch.broadcast_tensors(d, vis)
  inf = torch.full_like(d, float('inf'))
  hi = torch.where(vis, d, -inf).amax(-1)
  lo = torch.where(vis, d, inf).amin(-1)
  return bool((hi > lo).any())


def _RowX(qg, k_row, scale, bias_col):
  """Logits of every query of the slab against one key row k_row [b, c, D]."""
  s = torch.einsum('bcpd,bcd->bcp', qg, k_row)
  return scale * s if bias_col is None else scale * s + bias_col


# --------------------------------------------------------------------- decode ----
def _DecodeSlabs(q, kn, vn, ck0, cv0, y, t, rel, scale, chunk, controls=True):
  """Oracle pieces of `decode_attn_fwd` per slab of batch rows. q / y [B, H, D], kn / vn
  [B, Hk, D], ck0 / cv0 the caches before the call."""
  bsz, h, _ = q.shape
  tmax, hk = ck0.shape[1], ck0.shape[2]
  g = h // hk
  dev = q.device
  wr = t if 0 <= t < tmax else None
  n_vis = t + 1 if wr is not None else tmax
  j = torch.arange(tmax, device=dev)
  relw = 2 * tmax - 1
  bias = None
  if rel is not None:
    idx = (t - j + tmax - 1).clamp(0, relw - 1)
    bias = rel.double()[:, idx].view(1, hk, g, tmax)
  vis = (j < n_vis).view(1, 1, 1, tmax)
  j1 = chunk if chunk < n_vis else (n_vis - 1) // 32 * 32
  rows = max(1, _ELEMS // (tmax * hk * _D))
  for b0 in range(0, bsz, rows):
    b1 = min(bsz, b0 + rows)
    nb = b1 - b0
    qg = q[b0:b1].double().view(nb, hk, g, _D)
    kc, vc = ck0[b0:b1].double(), cv0[b0:b1].double()
    if wr is not None:
      kc[:, wr] = kn[b0:b1].double()
      vc[:, wr] = vn[b0:b1].double()
    ctl = {}
    if controls:
      def KeyWeight(c, f):
        if f == 2.0 and n_vis == 1:
          return None
        kw = torch.ones(tmax, dtype=torch.float64, device=dev)
        kw[j1] = f
        return dict(c, kw=kw)
      ctl['split-1 key dropped'] = lambda c: KeyWeight(c, 0.0)
      ctl['split-1 key twice'] = lambda c: KeyWeight(c, 2.0)
      if wr is not None:
        def Stale(c, b0=b0, b1=b1, qg=qg):
          x = c['x'].clone()
          x[..., wr] = _RowX(qg, ck0[b0:b1, wr].double(), scale,
                             None if bias is None else bias[..., wr])
          v = c['v'].clone()
          v[:, wr] = cv0[b0:b1, wr].double()
          return dict(c, x=x, v=v)
        ctl['key t from the stale row'] = Stale
      if wr is not None and rel is not None and tmax > 1:
        def RelOff(c):
          x = c['x'].clone()
          x[..., wr] = scale * c['s'][..., wr] + rel.double()[:, tmax].view(1, hk, g)
          return dict(c, x=x) if _Moves(x - c['x'], vis) else None
        ctl['rel index off by one at t'] = RelOff
      if g > _MAXG and rel is not None:
        def Group(c):
          b2 = bias.clone()
          b2[:, :, _MAXG:2 * _MAXG] = bias[:, :, :min(g, 2 * _MAXG) - _MAXG]
          return dict(c, x=scale * c['s'] + b2) if _Moves(b2 - bias, vis) else None
        ctl['group 1 with group 0 rel rows'] = Group
    yield dict(qg=qg, kc=kc, vc=vc, bias=bias, vis=vis, y=y[b0:b1].view(nb, hk, g, _D),
               controls=ctl)


def _Boost(q, kn, ck, t, rel, scale, keys):
  """Sets key row j of every batch row and KV head, for j in `keys`, to a multiple of the
  group's first query head such that this head scores it 1 below its largest logit over
  the other visible keys. Row t is set in k_new."""
  bsz, h, _ = q.shape
  tmax, hk = ck.shape[1], ck.shape[2]
  g = h // hk
  wr = t if 0 <= t < tmax else None
  n_vis = t + 1 if wr is not None else tmax
  j = torch.arange(tmax, device=q.device)
  qh = q.view(bsz, hk, g, _D)[:, :, 0].float()                       # [B, Hk, D]
  bias = None
  if rel is not None:
    idx = (t - j + tmax - 1).clamp(0, 2 * tmax - 2)
    bias = rel.float()[::g][:, idx]                                    # [Hk, T]
  others = (j < n_vis)
  for k in keys:
    others = others & (j != k)
  rows = max(1, _ELEMS // (tmax * hk * _D))
  for b0 in range(0, bsz, rows):
    b1 = min(bsz, b0 + rows)
    x = scale * torch.einsum('bcd,bjcd->bcj', qh[b0:b1], ck[b0:b1].float())
    if bias is not None:
      x = x + bias
    m = x.masked_fill(~others, float('-inf')).amax(-1)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    nq = (qh[b0:b1] * qh[b0:b1]).sum(-1)
    for k in keys:
      bk = 0.0 if bias is None else bias[:, k]
      row = (((m - 1.0 - bk) / (scale * nq)).unsqueeze(-1) * qh[b0:b1]).to(torch.bfloat16)
      if k == wr:
        kn[b0:b1] = row
      else:
        ck[b0:b1, k] = row


_MODES = {   # name: (q scale, logit scale, rel kind)
    'flat': (0.1, 1.0, 'randn'),
    'peaky': (1.0, 1.0, 'randn'),
    'scaled': (1.0, _D**-0.5, 'randn'),
    'rel30': (0.1, 1.0, 'pm30'),
    'half30': (0.1, 1.0, 'half30'),  # flat beam: +30 on every other run of 32 indices from N − 1
    'norel': (0.1, 1.0, None),
    'clamp': (0.1, 1.0, 'randn'),    # flat beam: positions past both ends of the table
}


def _Rel(gen, h, width, kind):
  if kind is None:
    return None
  rel = torch.randn(h, width, device=gen.device, generator=gen)
  pick = torch.rand(h, width, device=gen.device, generator=gen)
  if kind == 'pm30':
    rel = torch.where(pick < 0.05, torch.full_like(rel, 30.0), rel)
  if kind == 'half30':
    run = (torch.arange(width, device=gen.device) - (width - 1) // 2).div(32, rounding_mode='floor')
    rel = torch.where(run % 2 == 0, rel + 30.0, rel)
  if kind in ('pm30', 'half30'):
    rel = torch.where(pick > 0.95, torch.full_like(rel, -30.0), rel)
  return rel


def _Gen(seed, dev='cuda'):
  return torch.Generator(device=dev).manual_seed(seed)


def _Rnd(gen, *shape, scale=1.0):
  return (torch.randn(*shape, device=gen.device, generator=gen) * scale).to(torch.bfloat16)


def _DecodeT(where, tmax, chunk):
  return {'0': 0, '31': 31, '32': 32, 'chunk-1': chunk - 1, 'chunk': chunk,
          'chunk+1': chunk + 1, 'mid': chunk // 2 + 5, 'T-1': tmax - 1, 'T': tmax, '-1': -1,
          '10T': 10 * tmax}[where]


def _Native():
  from lingvo_b200 import ops
  return ops.native()


def _RunDecode(seed, bsz, tmax, h, hk, where, mode):
  """One decode case on the GPU: inputs, three calls (int64, int64, int32 t), the exact
  checks and the bound with its controls."""
  what = 'decode B=%d T=%d H=%d Hk=%d t=%s %s' % (bsz, tmax, h, hk, where, mode)
  gen = _Gen(seed)
  qs, scale, rk = _MODES[mode]
  chunk = _Native().decode_attn_chunk(bsz, h, hk, tmax)
  n_split = (tmax + chunk - 1) // chunk
  t = _DecodeT(where, tmax, chunk)
  q = _Rnd(gen, bsz, h, _D, scale=qs)
  kn, vn = _Rnd(gen, bsz, hk, _D), _Rnd(gen, bsz, hk, _D)
  ck, cv = _Rnd(gen, bsz, tmax, hk, _D), _Rnd(gen, bsz, tmax, hk, _D)
  rel = _Rel(gen, h, 2 * tmax - 1, rk)
  wr = t if 0 <= t < tmax else None
  n_vis = t + 1 if wr is not None else tmax
  j1 = chunk if chunk < n_vis else (n_vis - 1) // 32 * 32
  _Boost(q, kn, ck, t, rel, scale, sorted({j1} | ({wr} if wr is not None else set())))
  ck0, cv0 = ck.clone(), cv.clone()
  nat = _Native()
  outs = []
  for dt in (torch.int64, torch.int64, torch.int32):
    outs.append(nat.decode_attn_fwd(q, kn, vn, ck, cv, torch.tensor(t, device='cuda', dtype=dt),
                                    rel, scale))
  assert all(torch.equal(_Bits(o), _Bits(outs[0])) for o in outs), '%s: not reproducible' % what
  rows = torch.arange(tmax, device='cuda') != (wr if wr is not None else -1)
  assert torch.equal(_Bits(ck[:, rows]), _Bits(ck0[:, rows])), '%s: k rows changed' % what
  assert torch.equal(_Bits(cv[:, rows]), _Bits(cv0[:, rows])), '%s: v rows changed' % what
  if wr is not None:
    assert torch.equal(_Bits(ck[:, wr]), _Bits(kn)) and torch.equal(_Bits(cv[:, wr]), _Bits(vn)), (
        '%s: row t is not k_new / v_new' % what)
  res = _Result()
  for sl in _DecodeSlabs(q, kn, vn, ck0, cv0, outs[0], t, rel, scale, chunk):
    _CheckSlab(res, sl, scale, chunk, n_split, what)
  return res.Finish(what)


# ------------------------------------------------------------------ flat beam ----
def _BeamSlabs(q, kn, vn, ck0, cv0, y, slot0, vis, qpos, kpos, rel, scale, controls=True):
  """Oracle pieces of `flat_beam_attn_fwd` per slab of batch rows. q / y [B, K, H, D],
  kn / vn [B, K, Hk, D], ck0 / cv0 the caches before the call, vis [B, K, W] int32."""
  bsz, kk, h, _ = q.shape
  n, hk = ck0.shape[1], ck0.shape[2]
  g = h // hk
  npair = kk * g
  dev = q.device
  live = min(max(slot0 + kk, 0), n)
  words = vis.shape[-1]
  j = torch.arange(n, device=dev)
  raw = A.unpack_visibility(vis, 32 * words)                        # [B, K, 32W]
  seen = raw[..., :n] & (j < live)
  fresh = [(slot0 + k, k) for k in range(kk) if 0 <= slot0 + k < n]
  relw = 2 * n - 1

  def Pairs(t, b):   # [b, K, H, ...] → [b, Hk, K·G, ...]
    rest = t.shape[3:]
    return t.reshape(b, kk, hk, g, *rest).transpose(1, 2).reshape(b, hk, npair, *rest)

  def Bias(qp, b0, b1):
    if rel is None:
      return None
    idx = (qp[b0:b1].long().unsqueeze(-1) - kpos[b0:b1].long().unsqueeze(1) + n - 1)
    idx = idx.clamp(0, relw - 1)                                        # [b, K, N]
    return Pairs(rel.double()[:, idx].permute(1, 2, 0, 3), b1 - b0)    # [b, Hk, K·G, N]

  def Vis(m, b):     # [b, K, N] → [b, 1, K·G, N]
    return m.unsqueeze(2).expand(b, kk, g, n).reshape(b, 1, npair, n)

  rows = max(1, _ELEMS // (n * hk * _D))
  for b0 in range(0, bsz, rows):
    b1 = min(bsz, b0 + rows)
    nb = b1 - b0
    qg = Pairs(q[b0:b1].double(), nb)
    kc, vc = ck0[b0:b1].double(), cv0[b0:b1].double()
    for r, k in fresh:
      kc[:, r] = kn[b0:b1, k].double()
      vc[:, r] = vn[b0:b1, k].double()
    bias = Bias(qpos, b0, b1)
    sb = seen[b0:b1]
    ctl = {}
    if controls:
      def Word(c, b0=b0, b1=b1, sb=sb, nb=nb):
        if n < 32:
          return None
        r = torch.arange(31, n, 32, device=dev)
        nxt = r + 32
        src = raw[b0:b1][..., nxt.clamp(max=32 * words - 1)] & (nxt < 32 * words)
        m2 = sb.clone()
        m2[..., r] = src & (r < live)
        return None if torch.equal(m2, sb) else dict(c, vis=Vis(m2, nb))
      ctl['bit 32w+31 from word w+1'] = Word
      if fresh:
        def Stale(c, b0=b0, b1=b1, qg=qg, bias=bias, sb=sb):
          r = fresh[-1][0]
          if not bool(sb[..., r].any()):
            return None
          x = c['x'].clone()
          x[..., r] = _RowX(qg, ck0[b0:b1, r].double(), scale,
                            None if bias is None else bias[..., r])
          v = c['v'].clone()
          v[:, r] = cv0[b0:b1, r].double()
          return dict(c, x=x, v=v)
        ctl['last fresh row from the cache'] = Stale
      if rel is not None and kk > 1:
        def Qpos(c, b0=b0, b1=b1, bias=bias, sb=sb, nb=nb):
          b2 = Bias(torch.roll(qpos, -1, 1), b0, b1)
          if not _Moves(b2 - bias, Vis(sb, nb)):
            return None
          return dict(c, x=scale * c['s'] + b2)
        ctl['qpos of hypothesis k+1'] = Qpos

      def Tile(c, sb=sb, nb=nb):
        if not bool(sb.any()):
          return None
        first = torch.where(sb, j, n).amin(-1, keepdim=True) // 32     # [b, K, 1]
        return dict(c, vis=Vis(sb & ((j // 32) != first), nb))
      ctl['first visible tile skipped'] = Tile
    yield dict(qg=qg, kc=kc, vc=vc, bias=bias, vis=Vis(sb, nb), y=Pairs(y[b0:b1], nb),
               controls=ctl)


def _AncestorMask(gen, b, kk, n, slot0, prompt):
  """The masks a flat beam search builds: `prompt` visible rows, then one row per earlier
  step (each hypothesis inherits a random parent's path) and its own row."""
  width = max(n, slot0 + kk)
  mask = torch.zeros(b, kk, width, dtype=torch.bool)
  mask[:, :, :prompt] = True
  for s0 in range(prompt, slot0 - kk + 1, kk):
    mask[:, torch.arange(kk), s0 + torch.arange(kk)] = True
    parent = torch.randint(0, kk, (b, kk), generator=gen)
    mask = mask.gather(1, parent.unsqueeze(-1).expand(b, kk, width))
  if slot0 >= 0:
    mask[:, torch.arange(kk), slot0 + torch.arange(kk)] = True
  return mask[..., :n]


def _BeamMask(gen, kind, b, kk, n, slot0, chunk, edges):
  """bool [b, K, N] masks. kind: 'ancestor' (64-row prompt), 'random' (30 % and the own
  row) or 'onesplit' (half the live rows of split 1, or of split 0 with one split). With
  `edges`: hypothesis 0 sees no row (K ≥ 2), hypothesis 1 only itself (K ≥ 3), and every
  row ≥ slot0 + K is set (the kernel must ignore them)."""
  live = min(max(slot0 + kk, 0), n)
  if kind == 'ancestor':
    mask = _AncestorMask(gen, b, kk, n, slot0, min(max(slot0, 0), 64))
  elif kind == 'random':
    mask = torch.rand(b, kk, n, generator=gen) < 0.3
    own = slot0 + torch.arange(kk)
    ok = own < n
    mask[:, torch.arange(kk)[ok], own[ok]] = True
  else:
    lo = chunk if chunk < live else 0
    hi = min(lo + chunk, live)
    mask = torch.zeros(b, kk, n, dtype=torch.bool)
    mask[..., lo:hi] = torch.rand(b, kk, hi - lo, generator=gen) < 0.5
  if edges:
    if kk >= 2:
      mask[:, 0] = False
    if kk >= 3:
      mask[:, 1] = False
      if 0 <= slot0 + 1 < n:
        mask[:, 1, slot0 + 1] = True
    mask[..., max(slot0 + kk, 0):] = True
  return mask


def _BeamSlot0(where, n, kk, chunk):
  on = chunk if chunk + kk <= n else n - kk
  return {'zero': 0, 'straddle': max(0, on - max(1, kk // 2)), 'on': on, 'end': n - kk,
          'past': n - kk + 2}[where]


def _RunBeam(seed, bsz, kk, n, h, hk, where, kind, mode, edges):
  what = 'beam B=%d K=%d N=%d H=%d Hk=%d slot0=%s %s %s' % (bsz, kk, n, h, hk, where, kind, mode)
  gen = _Gen(seed)
  cgen = torch.Generator().manual_seed(seed)
  qs, scale, rk = _MODES[mode]
  nat = _Native()
  chunk = nat.flat_beam_attn_chunk(bsz, kk, h, hk, n)
  n_split = (n + chunk - 1) // chunk
  slot0 = _BeamSlot0(where, n, kk, chunk)
  q = _Rnd(gen, bsz, kk, h, _D, scale=qs)
  kn, vn = _Rnd(gen, bsz, kk, hk, _D), _Rnd(gen, bsz, kk, hk, _D)
  ck, cv = _Rnd(gen, bsz, n, hk, _D), _Rnd(gen, bsz, n, hk, _D)
  rel = _Rel(gen, h, 2 * n - 1, rk)
  vis = A.pack_visibility(_BeamMask(cgen, kind, bsz, kk, n, slot0, chunk, edges))
  if edges and n % 32:
    vis[..., -1] |= -(1 << (n % 32))                   # bits past N in the last word
  vis = vis.cuda()
  if edges and mode == 'clamp':
    ends = torch.tensor([-(n // 2), 3 * n // 2, 0, n - 1])
    qpos = ends[torch.randint(0, 4, (bsz, kk), generator=cgen)].int()
    kpos = torch.randint(0, n, (bsz, n), generator=cgen).int()
    kpos[:, ::7] = 0
    kpos[:, 3::7] = n - 1
  elif edges:
    # With +30 runs, all hypotheses share one position, as in a real step: the fresh rows
    # then sit at index N − 1 for every hypothesis, in a +30 run, so none of them is
    # negligible. (The qpos control is then the identity and is not built.)
    qpos = torch.randint(0, n, (bsz, 1 if mode == 'half30' else kk), generator=cgen)
    qpos = qpos.expand(bsz, kk).int()
    kpos = torch.randint(0, n, (bsz, n), generator=cgen).int()
  else:
    qpos = (slot0 + torch.arange(kk)).int().repeat(bsz, 1)
    kpos = torch.arange(n).int().repeat(bsz, 1)
  for k in range(kk):     # a fresh row is its hypothesis's own token: it has the query's position
    if 0 <= slot0 + k < n:
      kpos[:, slot0 + k] = qpos[:, k]
  qpos, kpos = qpos.cuda(), kpos.cuda()
  ck0, cv0 = ck.clone(), cv.clone()
  outs = []
  for dt in (torch.int64, torch.int64, torch.int32):
    outs.append(nat.flat_beam_attn_fwd(q, kn, vn, ck, cv,
                                       torch.tensor(slot0, device='cuda', dtype=dt), vis, qpos,
                                       kpos, rel, scale))
  assert all(torch.equal(_Bits(o), _Bits(outs[0])) for o in outs), '%s: not reproducible' % what
  rows = torch.arange(n, device='cuda')
  new = (rows >= slot0) & (rows < slot0 + kk)
  assert torch.equal(_Bits(ck[:, ~new]), _Bits(ck0[:, ~new])), '%s: k rows changed' % what
  assert torch.equal(_Bits(cv[:, ~new]), _Bits(cv0[:, ~new])), '%s: v rows changed' % what
  k_in = torch.arange(kk, device='cuda')
  k_in = k_in[(slot0 + k_in) < n]
  assert torch.equal(_Bits(ck[:, new]), _Bits(kn[:, k_in])), '%s: fresh k rows' % what
  assert torch.equal(_Bits(cv[:, new]), _Bits(vn[:, k_in])), '%s: fresh v rows' % what
  res = _Result()
  for sl in _BeamSlabs(q, kn, vn, ck0, cv0, outs[0], slot0, vis, qpos, kpos, rel, scale):
    _CheckSlab(res, sl, scale, chunk, n_split, what)
  return res.Finish(what)


# ----------------------------------------------------------------------- cases ----
_SERVE_DECODE = [(b, tmax, hk, where) for b in (1, 8, 64) for tmax in (1024, 4096)
                 for hk in (16, 4, 1) for where in ('T-1', 'mid')]
_SERVE_BEAM = [(8, kk, hk) for kk in (4, 8) for hk in (16, 4, 1)] + [(1, 16, 16), (1, 16, 1)]

_SWEEP_G = (1, 2, 3, 5, 8, 16, 20, 32)
_SWEEP_T = (1, 31, 32, 33, 127, 128, 129, 4097)
_SWEEP_WHERE = ('0', '31', '32', 'chunk-1', 'chunk', 'chunk+1', 'T-1', 'T', '-1', '10T')
_DECODE_MODES = ('flat', 'peaky', 'scaled', 'rel30', 'norel')


def _DecodeSweep():
  """(B, T, H, Hk, where, mode): every T × t with G, Hk and the mode cycling, and every G at
  T = 4097, t = chunk."""
  cases = []
  i = 0
  for a, tmax in enumerate(_SWEEP_T):
    for c, where in enumerate(_SWEEP_WHERE):
      g = _SWEEP_G[(a + c) % len(_SWEEP_G)]
      hk = 1 + (a + c) % 2
      cases.append((2, tmax, g * hk, hk, where, _DECODE_MODES[i % len(_DECODE_MODES)]))
      i += 1
  for c, g in enumerate(_SWEEP_G):
    cases.append((2, 4097, g * 2, 2, 'chunk', _DECODE_MODES[c % len(_DECODE_MODES)]))
  return cases


_SWEEP_K = (1, 2, 3, 5, 16)
_SWEEP_SLOT = ('zero', 'straddle', 'on', 'end', 'past')
_SWEEP_KIND = ('random', 'ancestor', 'onesplit')
_BEAM_G = (1, 2, 3, 5, 8, 16, 20)
_BEAM_MODES = ('flat', 'scaled', 'half30', 'clamp', 'norel')


def _BeamSweep():
  """(B, K, N, H, Hk, where, kind, mode) over K × slot0 × mask kind at N = 1000, with G, Hk
  and the mode cycling, plus short buffers (one split)."""
  cases = []
  i = 0
  for a, kk in enumerate(_SWEEP_K):
    for b, where in enumerate(_SWEEP_SLOT):
      for c, kind in enumerate(_SWEEP_KIND):
        g = _BEAM_G[(a + b + c) % len(_BEAM_G)]
        hk = 1 + (b + c) % 2
        cases.append((2, kk, 1000, g * hk, hk, where, kind, _BEAM_MODES[i % len(_BEAM_MODES)]))
        i += 1
  for kk, n in ((1, 1), (3, 33), (5, 100), (16, 100)):
    for where in ('end', 'past'):
      cases.append((2, kk, n, 4, 2, where, 'random', 'flat'))
  return cases


def _SweepId(c):
  return '-'.join(str(x) for x in c)


@pytest.mark.gpu
@pytest.mark.parametrize('b,tmax,hk,where', _SERVE_DECODE,
                         ids=['B%d-T%d-Hk%d-%s' % c for c in _SERVE_DECODE])
def test_decode_serving_shapes(b, tmax, hk, where):
  _RunDecode(_SERVE_DECODE.index((b, tmax, hk, where)), b, tmax, 16, hk, where, 'flat')


@pytest.mark.gpu
@pytest.mark.parametrize('b,kk,hk', _SERVE_BEAM, ids=['B%d-K%d-Hk%d' % c for c in _SERVE_BEAM])
def test_flat_beam_serving_shapes(b, kk, hk):
  _RunBeam(100 + _SERVE_BEAM.index((b, kk, hk)), b, kk, 4096, 16, hk, 'end', 'ancestor',
           'flat', False)


@pytest.mark.gpu
def test_decode_edge_sweep():
  worst = 0.0
  for i, case in enumerate(_DecodeSweep()):
    worst = max(worst, _RunDecode(200 + i, *case)[0])
  print('decode edge sweep: worst err/bound %.4f' % worst)


@pytest.mark.gpu
def test_flat_beam_edge_sweep():
  worst = 0.0
  for i, case in enumerate(_BeamSweep()):
    worst = max(worst, _RunBeam(500 + i, *case, True)[0])
  print('flat beam edge sweep: worst err/bound %.4f' % worst)


def _Pow2(x):
  return 1 << (x - 1).bit_length()


@pytest.mark.gpu
def test_cases_reach_every_path():
  """Mirrors the hosts' dispatch: kG = min(G or K·G, 16) rounded up to a power of two, S from
  the device's chunk."""
  nat = _Native()
  seen = {'decode': set(), 'beam': set()}
  partial = {'decode': False, 'beam': False}
  for b, tmax, hk, _ in _SERVE_DECODE:
    seen['decode'].add((_Pow2(min(16 // hk, _MAXG)), (tmax + nat.decode_attn_chunk(
        b, 16, hk, tmax) - 1) // nat.decode_attn_chunk(b, 16, hk, tmax) > 1))
  for b, tmax, h, hk, _, _ in _DecodeSweep():
    g = h // hk
    chunk = nat.decode_attn_chunk(b, h, hk, tmax)
    seen['decode'].add((_Pow2(min(g, _MAXG)), (tmax + chunk - 1) // chunk > 1))
    partial['decode'] |= g > _MAXG and g % _MAXG != 0
  beams = [(b, kk, 4096, 16, hk) for b, kk, hk in _SERVE_BEAM]
  beams += [(b, kk, n, h, hk) for b, kk, n, h, hk, *_ in _BeamSweep()]
  for b, kk, n, h, hk in beams:
    pairs = kk * (h // hk)
    chunk = nat.flat_beam_attn_chunk(b, kk, h, hk, n)
    seen['beam'].add((_Pow2(min(pairs, _MAXG)), (n + chunk - 1) // chunk > 1))
    partial['beam'] |= pairs > _MAXG and pairs % _MAXG != 0
  for kern in ('decode', 'beam'):
    multi = {kg for kg, many in seen[kern] if many}
    assert multi == {1, 2, 4, 8, 16}, (kern, sorted(multi))
    assert any(not many for _, many in seen[kern]), '%s: no single-split case' % kern
    assert partial[kern], '%s: no case with a partial second query group' % kern


# ------------------------------------------------------------------- beam_topk ----
def _TopKOracle(lp, cum, active, k, eos):
  """The kernel's contract on the host: g = cum + lp in fp32; candidates are the non-EOS
  tokens of active rows with g > NEG, in (g desc, id asc) order; missing slots are (NEG, 0);
  best_in_hyp = max(NEG, max g)."""
  g = cum.float().cpu().unsqueeze(1) + lp.float().cpu()
  n, v = g.shape
  best = g.max(1).values.clamp_min(_NEG)
  cand = g.clone()
  cand[:, eos] = float('-inf')
  cand[~active.cpu()] = float('-inf')
  cand = torch.where(cand > _NEG, cand, torch.full_like(cand, float('-inf')))
  if v < k:
    cand = torch.cat([cand, torch.full((n, k - v), float('-inf'))], 1)
  order = torch.argsort(cand, dim=1, descending=True, stable=True)[:, :k]
  s = cand.gather(1, order)
  top_s = torch.where(s > _NEG, s, torch.full_like(s, _NEG))
  top_w = torch.where(top_s > _NEG / 2, order, torch.zeros_like(order))
  el = lp.float().cpu()[:, eos]
  return top_s, top_w, best, cum.float().cpu() + el, el


def _TopKInputs(gen, n, v, dtype, eos):
  """Log-probs with one row kind per row index mod 8: plain; exact ties at the top within
  one thread's slice (ids v0, v0 + 256, …); ties across threads (v0, v0 + 1, v0 + 2); EOS
  the best token; inactive; cum = −1e30 (how flat beam search seeds hypotheses 1…K−1); two
  finite scores; no finite score but EOS."""
  lp = torch.log_softmax(torch.randn(n, v, generator=gen) * 3, -1).to(dtype).float()
  cum = torch.randn(n, generator=gen) * 4
  active = torch.ones(n, dtype=torch.bool)
  top = lp.max(1).values
  v0 = (eos + 1 + v // 3) % v
  for r in range(n):
    kind = r % 8
    if kind == 1:
      lp[r, torch.arange(v0, v, 256)[:3]] = top[r]
    elif kind == 2:
      ids = torch.tensor([v0, (v0 + 1) % v, (v0 + 2) % v])
      lp[r, ids] = top[r]
    elif kind == 3:
      lp[r, eos] = top[r] + 1.0
    elif kind == 4:
      active[r] = False
    elif kind == 5:
      cum[r] = _NEG
    elif kind == 6:
      keep = lp[r, v0].clone(), lp[r, (v0 + 7) % v].clone()
      lp[r] = float('-inf')
      lp[r, v0], lp[r, (v0 + 7) % v] = keep
    elif kind == 7:
      el = lp[r, eos].clone()
      lp[r] = float('-inf')
      lp[r, eos] = el
  return lp.to(dtype), cum, active


_TOPK_CASES = ([(8 * k, k, 32000, dt, 2) for k in (1, 4, 5, 8, 9, 16)
                for dt in (torch.float32, torch.bfloat16)] +
               [(24, k, v, torch.float32 if (k + v) % 2 else torch.bfloat16, eos)
                for k in (1, 4, 5, 8, 9, 16) for v in (2, 200, 256, 257, 4099)
                for eos in (0, v - 1)])


def _TopKId(c):
  return 'n%d-K%d-V%d-%s-eos%d' % (c[0], c[1], c[2], str(c[3])[6:], c[4])


def _SameBits(a, b):
  a, b = a.cpu().contiguous(), b.cpu().contiguous()
  if a.dtype == torch.float32:
    a, b = a.view(torch.int32), b.view(torch.int32)
  return a.shape == b.shape and torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize('case', _TOPK_CASES, ids=[_TopKId(c) for c in _TOPK_CASES])
def test_beam_topk_matches_exact_oracle(case):
  n, k, v, dtype, eos = case
  lp, cum, active = _TopKInputs(torch.Generator().manual_seed(_TOPK_CASES.index(case)), n, v,
                                dtype, eos)
  got = _Native().beam_topk(lp.cuda(), cum.cuda(), active.cuda(), k, eos)
  want = _TopKOracle(lp, cum, active, k, eos)
  names = ('top_s', 'top_w', 'best_in_hyp', 'eos_glob', 'eos_local')
  for name, a, b in zip(names, got, want):
    assert _SameBits(a, b), '%s: %s differs' % (_TopKId(case), name)


# ------------------------------------------------------------------ CPU checks ----
def test_topk_ref_matches_exact_oracle():
  """`_TopKRef`, the CPU path of the beam step, against the kernel's contract, including
  rows with fewer than K candidates (padded with NEG, word 0). The beam step asks for at
  most V − 1 tokens per row."""
  for i, (n, k, v, dtype, eos) in enumerate(_TOPK_CASES[::3]):
    if k >= v:
      continue
    lp, cum, active = _TopKInputs(torch.Generator().manual_seed(i), n, v, dtype, eos)
    got = bs._TopKRef(lp, cum, active, k, eos)   # pylint: disable=protected-access
    want = _TopKOracle(lp, cum, active, k, eos)
    for a, b in zip(got, want):
      assert _SameBits(a, b), (n, k, v, dtype, eos)


def test_decode_ref_negative_t_sees_every_key():
  """For t outside [0, T) nothing is written and every key is visible, t = −1 included."""
  g = torch.Generator().manual_seed(0)
  b, tmax, h, hk = 2, 40, 4, 2
  q, kn, vn = (torch.randn(b, 1, x, 16, generator=g) for x in (h, hk, hk))
  ck, cv = torch.randn(b, tmax, hk, 16, generator=g), torch.randn(b, tmax, hk, 16, generator=g)
  outs = {}
  for t in (-1, tmax, 10 * tmax):
    k2, v2 = ck.clone(), cv.clone()
    outs[t] = A.decode_attention_ref(q, kn, vn, k2, v2, t)
    assert torch.equal(k2, ck) and torch.equal(v2, cv)
  assert torch.equal(outs[-1], outs[tmax]) and torch.equal(outs[-1], outs[10 * tmax])
  probs = torch.softmax(torch.einsum('bqhd,bkhd->bhqk', q, ck.repeat_interleave(h // hk, 2)), -1)
  want = torch.einsum('bhqk,bkhd->bqhd', probs, cv.repeat_interleave(h // hk, 2))
  torch.testing.assert_close(outs[-1], want, rtol=1e-6, atol=1e-6)


def _Truncate(v):
  """fp32 → bf16 by dropping the low 16 bits."""
  return (v.float().view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)


def _Fp32Decode(q, kc, vc, t, rel, scale, round_logits=False, round_p=False):
  """fp32 decode attention over caches that already hold row t, with optional bf16
  roundings of the logits or of the unnormalised weights before P·V. q [B, H, D]."""
  bsz, h, _ = q.shape
  tmax, hk = kc.shape[1], kc.shape[2]
  j = torch.arange(tmax)
  kk = kc.float().repeat_interleave(h // hk, 2)
  vv = vc.float().repeat_interleave(h // hk, 2)
  x = torch.einsum('bhd,bjhd->bhj', q.float(), kk) * scale
  if rel is not None:
    x = x + rel[:, (t - j + tmax - 1).clamp(0, 2 * tmax - 2)]
  if round_logits:
    x = x.bfloat16().float()
  x = x.masked_fill(~(j <= t if 0 <= t < tmax else j >= 0), float('-inf'))
  p = torch.exp(x - x.amax(-1, keepdim=True))
  l = p.sum(-1, keepdim=True)
  if round_p:
    p = p.bfloat16().float()
  return torch.einsum('bhj,bjhd->bhd', p, vv) / l


def _CheckDecodeCpu(y, q, kn, vn, ck0, cv0, t, rel, scale, chunk, controls=True, what=''):
  tmax = ck0.shape[1]
  n_split = (tmax + chunk - 1) // chunk
  res = _Result()
  for sl in _DecodeSlabs(q, kn, vn, ck0, cv0, y, t, rel, scale, chunk, controls):
    _CheckSlab(res, sl, scale, chunk, n_split, what)
  return res.Finish(what)


@pytest.mark.parametrize('mode', ['flat', 'peaky', 'rel30'])
@pytest.mark.parametrize('where', ['T-1', 'mid', '-1'])
def test_decode_bound_and_controls_on_cpu(where, mode):
  """The bound, the controls and the rounding check with `decode_attention_ref` rounded to
  bf16 in the kernel's place, at B = 4, T = 300, H = 32, Hk = 4 and a chunk of 128. A
  truncating pack and logits rounded to bf16 fail; whether bf16 P is rejected is printed."""
  bsz, tmax, h, hk, chunk = 4, 300, 32, 4, 128
  gen = _Gen(7, 'cpu')
  qs, scale, rk = _MODES[mode]
  t = _DecodeT(where, tmax, chunk)
  q = _Rnd(gen, bsz, h, _D, scale=qs)
  kn, vn = _Rnd(gen, bsz, hk, _D), _Rnd(gen, bsz, hk, _D)
  ck, cv = _Rnd(gen, bsz, tmax, hk, _D), _Rnd(gen, bsz, tmax, hk, _D)
  rel = _Rel(gen, h, 2 * tmax - 1, rk)
  wr = t if 0 <= t < tmax else None
  n_vis = t + 1 if wr is not None else tmax
  _Boost(q, kn, ck, t, rel, scale,
         sorted({chunk if chunk < n_vis else (n_vis - 1) // 32 * 32} |
                ({wr} if wr is not None else set())))
  kf, vf = ck.float(), cv.float()
  y32 = A.decode_attention_ref(q.float().unsqueeze(1), kn.float().unsqueeze(1),
                               vn.float().unsqueeze(1), kf, vf, t, rel, scale)[:, 0]
  args = (q, kn, vn, ck, cv, t, rel, scale, chunk)
  _CheckDecodeCpu(y32.bfloat16(), *args, what='decode_attention_ref')
  with pytest.raises(AssertionError, match='outside the bound|not rounded to nearest'):
    _CheckDecodeCpu(_Truncate(y32), *args, controls=False, what='truncated pack')
  if mode == 'peaky':
    y = _Fp32Decode(q, kf, vf, t, rel, scale, round_logits=True).bfloat16()
    with pytest.raises(AssertionError, match='outside the bound'):
      _CheckDecodeCpu(y, *args, controls=False, what='bf16 logits')
  y = _Fp32Decode(q, kf, vf, t, rel, scale, round_p=True).bfloat16()
  try:
    _CheckDecodeCpu(y, *args, controls=False, what='bf16 P')
    print('bf16 P (%s, t=%s): accepted by the bound' % (mode, where))
  except AssertionError as e:
    print('bf16 P (%s, t=%s): rejected: %s' % (mode, where, str(e).splitlines()[0]))


@pytest.mark.parametrize('kind', ['ancestor', 'random', 'onesplit'])
def test_flat_beam_bound_and_controls_on_cpu(kind):
  """The same with `flat_beam_attention_ref` rounded to bf16, at B = 2, K = 4, N = 300,
  H = 16, Hk = 4, a chunk of 128, the edge masks and slot0 straddling the chunk boundary."""
  bsz, kk, n, h, hk, chunk = 2, 4, 300, 16, 4, 128
  gen = _Gen(11, 'cpu')
  cgen = torch.Generator().manual_seed(11)
  q = _Rnd(gen, bsz, kk, h, _D, scale=0.1)
  kn, vn = _Rnd(gen, bsz, kk, hk, _D), _Rnd(gen, bsz, kk, hk, _D)
  ck, cv = _Rnd(gen, bsz, n, hk, _D), _Rnd(gen, bsz, n, hk, _D)
  rel = torch.randn(h, 2 * n - 1, generator=gen)
  slot0 = chunk - 2
  vis = A.pack_visibility(_BeamMask(cgen, kind, bsz, kk, n, slot0, chunk, True))
  qpos = torch.randint(0, n, (bsz, kk), generator=cgen).int()
  kpos = torch.randint(0, n, (bsz, n), generator=cgen).int()
  y32 = A.flat_beam_attention_ref(q.float(), kn.float(), vn.float(), ck.float(), cv.float(),
                                  slot0, vis, qpos, kpos, rel, 1.0)
  n_split = (n + chunk - 1) // chunk

  def Check(y, controls=True, what='flat_beam_attention_ref'):
    res = _Result()
    for sl in _BeamSlabs(q, kn, vn, ck, cv, y, slot0, vis, qpos, kpos, rel, 1.0, controls):
      _CheckSlab(res, sl, 1.0, chunk, n_split, what)
    return res.Finish(what)
  Check(y32.bfloat16())
  with pytest.raises(AssertionError, match='outside the bound|not rounded to nearest'):
    Check(_Truncate(y32), False, 'truncated pack')
