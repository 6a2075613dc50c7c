"""The fused MoE expert layer (parallel/symm.py: `MoeExchange.Apply` and `_MoeFn`) end to end,
forward and backward, against a float64 oracle of the top-2 MoE FFN, at the benchmark's shape.

Contract. For tokens x [T = G·S, M] (bf16), fp32 logits [G, S, E], expert weights wi [E, M, H]
and wo [E, H, M] (bf16), a capacity C and the legacy or renorm gate mode, `Apply` returns

    y[t] = Σ_k gate_k[t] · (relu(x[t]·wi[e_k]) · wo[e_k]),   aux = GShard's load-balancing loss,

with GShard top-2 gating: softmax, the first choice, a second choice that excludes it, the
padded tokens routed nowhere, an exclusive position scan per group with first-choice priority,
then the capacity. Legacy mode normalises the two gates before the capacity mask (+1e-9),
renorm mode after it. Backward returns dx, dlogits, dwi and dwo of any loss of (y, aux).

The oracle (`_Gates64`, `_Oracle`) is that formula in float64 torch, with float64 autograd
for the gradients. It never calls the repository's gating functions on the GPU path: they
compute in fp32 (`logits.float()`). A CPU test checks it once against
`gshard_layers.Top2GatingOnLogits` and `FeedForwardNetworksApplyGating` in fp32: the routing
(the dense dispatch tensor) exactly, y, aux and every gradient to fp32 tolerance.

Routing. The gate kernel ranks experts with fp32 `__expf`; the oracle with float64. Where two
probabilities nearly tie they may rank differently, and one swapped token moves the positions
of every later token of its group. So the kernel's (i1, i2) of a token is accepted when
p64[i1] is within τ of the float64 best probability and p64[i2] within τ of the second best,
τ = 2^-20: 16 ulps of a probability near 1, above the few ulps the kernel's `__expf`
(2 + 1.16·|Δ| ulp for the logit gap Δ, which is near 0 wherever the ranking is in doubt), its
E-term sum and its reciprocal can put on p. At most 0.1 % of the tokens may differ from the
float64 ranking. The oracle then takes those indices and recomputes positions and keep with
its own integer scan; they must equal the kernel's `pos` and `keep` exactly. Every value
comparison below runs on this shared routing.

Stage checks, through the exchange's own buffers. `bufs.xe`, `bufs.yc`, `ex.dye` and `ex.dxc`
are filled with a bf16 NaN before `Apply`, so a row never written fails. Each stage is compared
with float64 computed from the kernel's own inputs to that stage (the GEMM outputs h and dh are
recorded as the exchange makes them):

    xe     bitwise x[token] or 0 at row (e, g·C + c)
    h      relu(xe·wi): the GEMM bound of tests/test_gemm_float64_gpu.py (its `_Check`), and
           bit-identical to a second `gemm(xe, wi, act=RELU)`
    yc     h·wo within the GEMM bound at the combine-layout row (e·G + g)·C + c of every slot;
           the row-pointer table must point exactly there
    y      Σ_k gate·yc (float64, from yc and the Python gates) within 2·(½ ulp + 3u·Σ|gate·yc|)
    dgate  ⟨yc, dy⟩ within 1e-5·Σ|yc·dy|; exactly 0 for dropped choices
    dye    bitwise bf16(gate·dy)
    dh     (dye·woᵀ) masked by h > 0: GEMM bound, and exactly 0 where h ≤ 0
    dwo    hᵀ·dye, dwi xeᵀ·dh, dxc dh·wiᵀ at the combine-layout rows: GEMM bound
    dx     the gather of dxc within 2·(½ ulp + 2u·Σ|dxc|)

End to end, against pure float64 (no intermediate rounding). With u₈ = 2^-8, the unit
roundoff of a bf16 round to nearest, and every bound a constant times u₈ times the same
computation evaluated on absolute values:

    y       3u₈·(Σ_k g_k·(|h|·|wo|)_k + |y|) + Σ_k δg_k·(|h|·|wo|)_k
            three roundings on the path: h, yc, y. δg_k = 2^-20·g_k + Σ_e |∂g_k/∂l_e|·δl_e
            is the fp32 gate error: 16 ulps of the gate math plus the logits' own error δl
            (0 when the logits are the input, the router GEMM's fp32 bound in the layer test).
    dx      4u₈·(A_dx + |dx|): dye, dh, dxc, dx. A_dx = Σ_k gather(((g_k + δg_k)·|dy|·|wo|ᵀ)
            ⊙ mask · |wi|ᵀ), where the mask keeps every element whose sign the kernel's fp32
            accumulation could see differently from float64 (h + 2·n·u′·|xe|·|wi| > 0).
    dwo     3u₈·(|h|ᵀ·|dye| + |dwo|): h, dye, dwo.
    dwi     3u₈·(|xe|ᵀ·|dh| + |dwi|): dye, dh, dwi; a ReLU mask that flips at h ≈ 0 moves an
            element by one term of the sum, far inside it.
    dlogits Σ_k |∂g_k/∂l|·(Σ_m |yc − yc64|_k,m·|dy_m| + M·u·Σ_m |yc|·|dy|): dgate reads the
            kernel's yc, whose own error the yc stage bounds. The abs-value evaluation
            3u₈·Σ_m (|h|·|wo|)·|dy| would be valid too, but at M = 2048, H = 8192 it is ~3000x
            the dot product itself and could not see a wrong gate gradient.
            + 2^-16·p_e·(gp_e + Σ_j p_j·gp_j), gp = Σ_k |∂g_k/∂p|·|dgate_k| + coef·|∂aux/∂p|:
            the fp32 backward through the softmax p, whose terms cancel where the two gates
            are normalised, so its rounding is bounded by the terms, not by the result.
    aux     2^-16·|aux|: fp32 torch math on exact logits.

The bf16 stand-in — the float64 oracle rounded to bf16 at the kernel's rounding points, with
fp32 gates — must sit well inside every bound (the CPU test), and five mutated oracles built
from the same float64 pieces must each put some element above its bound: the last capacity
slot of each expert dropped; group 0's combine rows taken from group 1; the other mode's gates
(renorm in legacy mode); the first choice's dgate used for both choices; and the second
choice's dgate dropped for tokens whose first choice overflowed. The GPU test asserts the
controls in the two benchmark cases; the CPU test with the stand-in at a small shape.

Cases, all at ep = 1 through `MoeExchange(None, E, device)`, seeded, with the model's weight
init Uniform(√(3/M)) and Uniform(√(3/H)) and logits x·gw with gw ~ N(0, 1/M) as in `MoELayer`:

    bench          G 8, S 1024, M 2048, H 8192, E 8,  C 256, legacy    MoELm8E's MoE layer
    bench_skewed   as bench, +2 on experts 1 and 4: both choices overflow
    renorm_padded  G 3, S 1000, M 1024, H 2048, E 16, C 128, renorm, random padded spans and
                   a fully padded last group; S not a multiple of 256
    many_experts   G 2, S 4096, M 512,  H 1024, E 32, C 256, renorm: the gate kernel's
                   > 48 KiB shared-memory path
    ragged         G 5, S 77,   M 328,  H 264,  E 2,  C 20,  legacy: M not a multiple of the
                   256-column lane stride, ragged GEMM N and K, heavy overflow
    smallest       G 1, S 8,    M 64,   H 72,   E 4,  C 4,   renorm

`MoELayer` itself runs at the benchmark's dims in bf16 with the aux-loss coefficient 0.01; its
out, dx (with the router's contribution) and dgw are compared with the oracle, and the test
shows that the fused exchange served the layer. Buffer lifetime: two layers interleaved
(forward A, forward B, backward B, backward A) and one layer under `RematerializeFn` give
gradients bitwise equal to a plain run, and a backward whose layer buffers a later forward
has overwritten raises.

Measured on an H100 80GB HBM3 (700 W limit, 1980 MHz max SM clock), seeded so these repeat.
The kernels' choices matched the float64 ranking on every token of every case. Worst
err/bound per case and check:

                   h     yc    y     dgate dh    dwo   dwi   dxc   dx
    bench          0.484 0.406 0.500 0.001 0.484 0.489 0.490 0.425 0.500
    bench_skewed   0.483 0.405 0.500 0.001 0.482 0.494 0.495 0.420 0.500
    renorm_padded  0.490 0.484 0.500 0.002 0.491 0.499 0.499 0.486 0.500
    many_experts   0.495 0.494 0.500 0.002 0.496 0.498 0.498 0.493 0.500
    ragged         0.496 0.498 0.500 0.002 0.495 0.499 0.499 0.498 0.000
    smallest       0.497 0.498 0.499 0.003 0.497 0.500 0.500 0.498 0.500

                   y     dx    dwo   dwi   dlogits aux
    bench          0.043 0.001 0.084 0.032 0.092   0.001
    bench_skewed   0.047 0.002 0.136 0.055 0.121   0.006
    renorm_padded  0.063 0.002 0.203 0.011 0.123   0.001
    many_experts   0.094 0.005 0.146 0.010 0.168   0.005
    ragged         0.165 0.008 0.211 0.020 0.290   0.010
    smallest       0.132 0.018 0.410 0.148 0.158   0.007
    MoELayer       0.046 0.002 0.085 0.044 (dgw 0.003) 0.001

The stage ratios sit at ½: the final bf16 rounding, as in the GEMM test; ragged's dx is exact
because with two experts and heavy overflow no token keeps both choices. The end-to-end ratios
are far below 1 because the abs-value evaluations assume every rounding error aligns. The
bf16 stand-in on the CPU stays below 0.4 on every output. The whole module takes ~25 s on the
H100, of which the benchmark-sized cases take ~3 s each.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from lingvo_b200.core import gshard_layers
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap

import test_gemm_float64_gpu as gemm64
import test_moe_routing_gpu as routing

_U8 = 2.0**-8             # bf16 unit roundoff
_TAU = 2.0**-20           # routing tolerance on a float64 probability
_GATE_ULPS = 2.0**-20     # relative error of the fp32 gate math
_FP32_REL = 2.0**-16      # fp32 torch math on exact inputs (aux, softmax backward)
_AUX_COEF = 0.01          # MoELmTemplate.AUX_LOSS_COEF

# name, G, S, M, H, E, capacity factor, legacy, padded, skewed
CASES = [
    ('bench', 8, 1024, 2048, 8192, 8, 2.0, True, False, False),
    ('bench_skewed', 8, 1024, 2048, 8192, 8, 2.0, True, False, True),
    ('renorm_padded', 3, 1000, 1024, 2048, 16, 2.0, False, True, False),
    ('many_experts', 2, 4096, 512, 1024, 32, 2.0, False, False, False),
    ('ragged', 5, 77, 328, 264, 2, 0.5, True, False, False),
    ('smallest', 1, 8, 64, 72, 4, 2.0, False, False, False),
]
_CONTROL_CASES = ('bench', 'bench_skewed')


# ------------------------------------------------------------------ the oracle ----
def _Rank64(logits64, nonpad):
  """Float64 top-2 ranking: (i1, i2) [G, S]; a padded token's second choice repeats its first."""
  p = torch.softmax(logits64, -1)
  i1 = p.argmax(-1)
  i2 = p.scatter(-1, i1[..., None], -1.0).argmax(-1)
  return i1, torch.where(nonpad > 0, i2, i1)


def _Scan(i1, i2, nonpad, e, c):
  """GShard's exclusive position scan with first-choice priority, then capacity:
  → pos [2, G, S] (0 where dropped), keep [2, G, S] bool."""
  live = (nonpad > 0).long()[..., None]
  oh1 = F.one_hot(i1, e) * live
  pos1 = torch.cumsum(oh1, 1) - oh1
  keep1 = oh1 * (pos1 < c)
  count1 = keep1.sum(1, keepdim=True)
  oh2 = F.one_hot(i2, e) * live
  pos2 = torch.cumsum(oh2, 1) - oh2 + count1
  keep2 = oh2 * (pos2 < c)
  pos = torch.stack([(pos1 * keep1).sum(-1), (pos2 * keep2).sum(-1)])
  keep = torch.stack([keep1.sum(-1), keep2.sum(-1)]) > 0
  return pos, keep


def _Gates64(logits, i1, i2, nonpad, keep, legacy):
  """The two combine gates [2, G, S] and the aux loss, in the dtype of `logits`."""
  return _GatesOfProbs(torch.softmax(logits, -1), i1, i2, nonpad, keep, legacy)


def _GatesOfProbs(raw, i1, i2, nonpad, keep, legacy):
  e = raw.shape[-1]
  g1 = raw.gather(-1, i1[..., None])[..., 0] * nonpad
  g2 = raw.gather(-1, i2[..., None])[..., 0] * nonpad
  if legacy:
    den = g1 + g2 + 1e-9
    g1, g2 = g1 / den, g2 / den
  g1 = g1 * keep[0].to(g1.dtype)
  g2 = g2 * keep[1].to(g2.dtype)
  if not legacy:
    den = g1 + g2
    den = torch.where(den > 0, den, torch.ones_like(den))
    g1, g2 = g1 / den, g2 / den
  oh1 = F.one_hot(i1, e).to(raw.dtype) * nonpad[..., None]
  proxy = raw * nonpad[..., None]
  dden = 1.0 if legacy else nonpad.mean(1)[:, None] + 1e-6
  aux = ((proxy.mean(1) / dden) * (oh1.mean(1) / dden)).mean() * (e * e)
  return torch.stack([g1, g2]), aux


def _GateBackwardAbs(p, i1, i2, nonpad, keep, legacy, dgate_abs):
  """The backward of the gates g_k = a_k / den to the probabilities p, evaluated on absolute
  values without letting the numerator and denominator terms cancel."""
  e = p.shape[-1]
  oh = [F.one_hot(i, e).to(p.dtype) * nonpad[..., None] for i in (i1, i2)]
  a = [p.gather(-1, i[..., None])[..., 0] * nonpad for i in (i1, i2)]
  kf = [k.to(p.dtype) for k in keep]
  if legacy:
    den = a[0] + a[1] + 1e-9
    dmask = oh[0] + oh[1]
  else:
    a = [a[k] * kf[k] for k in range(2)]
    den = a[0] + a[1]
    den = torch.where(den > 0, den, torch.ones_like(den))
    dmask = oh[0] * kf[0][..., None] + oh[1] * kf[1][..., None]
  gp = torch.zeros_like(p)
  for k in range(2):
    gp = gp + (kf[k] * dgate_abs[k])[..., None] * (
        oh[k] / den[..., None] + (a[k] / den**2)[..., None] * dmask)
  return gp


def _Slots(index, pos, keep, e, c):
  """Flat slot [2, T] of every choice in an [E, G, C] buffer, and the token [E·G·C] of every
  slot (-1 where empty)."""
  _, g, s = index.shape
  gi = torch.arange(g, device=index.device).view(1, g, 1)
  slot = ((index.long() * g + gi) * c + pos.long()).reshape(2, -1)
  kf = keep.reshape(2, -1)
  token = torch.full((e * g * c,), -1, dtype=torch.long, device=index.device)
  tok = torch.arange(g * s, device=index.device).expand(2, -1)
  token[slot[kf]] = tok[kf]
  assert int((token >= 0).sum()) == int(kf.sum()), 'two kept choices share a slot'
  return slot, token


def _Dispatch(x, token, e):
  rows = x[token.clamp_min(0)] * (token >= 0).to(x.dtype)[:, None]
  return rows.view(e, -1, x.shape[-1])


def _Combine(rows, gate, slot):
  """Σ_k gate_k · rows[slot_k]: rows [E·G·C, M], gate and slot [2, T]."""
  return (gate[..., None] * rows[slot]).sum(0)


def _Oracle(x, logits, wi, wo, dy, nonpad, index, legacy, c, dlogit_err=None):
  """Float64 forward and backward of the MoE FFN with routing (i1, i2) = index, the abs-value
  evaluations the bounds need, and the pieces the controls mutate."""
  d = torch.float64
  e = logits.shape[-1]
  g_, s_ = logits.shape[:2]
  x64 = x.detach().to(d).requires_grad_()
  l64 = logits.detach().to(d).requires_grad_()
  wi64 = wi.detach().to(d).requires_grad_()
  wo64 = wo.detach().to(d).requires_grad_()
  dy64 = dy.detach().to(d)
  np64 = nonpad.to(d)
  i1, i2 = index[0].long(), index[1].long()
  pos, keep = _Scan(i1, i2, np64, e, c)
  slot, token = _Slots(index, pos, keep, e, c)
  gates, aux = _Gates64(l64, i1, i2, np64, keep, legacy)
  gl = gates.detach().reshape(2, -1).requires_grad_()
  xe = _Dispatch(x64, token, e)
  pre = torch.bmm(xe, wi64)
  h = torch.relu(pre)
  yc = torch.bmm(h, wo64)
  rows = yc.reshape(-1, yc.shape[-1])
  y = _Combine(rows, gl, slot)
  (y * dy64).sum().backward()
  dgate = (gl.grad * keep.reshape(2, -1)).reshape(2, g_, s_)
  dlogits, = torch.autograd.grad((gates, aux), l64, (dgate, torch.tensor(_AUX_COEF, dtype=d,
                                                                          device=l64.device)),
                                 retain_graph=True)
  jac = [torch.autograd.grad(gates[k].sum(), l64, retain_graph=True)[0].abs() for k in range(2)]
  # fp32 autograd rounds the unfused terms of the backward through the gate division and the
  # softmax, and those cancel where the gates are normalised: bound it by the terms.
  probs = torch.softmax(l64.detach(), -1).requires_grad_()
  _, paux = _GatesOfProbs(probs, i1, i2, np64, keep, legacy)
  gp = _AUX_COEF * torch.autograd.grad(paux, probs, retain_graph=True)[0].abs()
  gp = gp + _GateBackwardAbs(probs.detach(), i1, i2, np64, keep, legacy, dgate.abs())
  p = probs.detach()
  softmax_bwd_abs = p * (gp + (p * gp).sum(-1, keepdim=True))
  o = NestedMap(pos=pos, keep=keep, slot=slot, token=token, gates=gates.detach(),
                aux=aux.detach(), y=y.detach(), dx=x64.grad, dwi=wi64.grad, dwo=wo64.grad,
                dlogits=dlogits, dgate=dgate, xe=xe.detach(), h=h.detach(), yc=yc.detach(),
                l64=l64, gates_graph=gates, aux_graph=aux, e=e, c=c, g=g_, legacy=legacy,
                i1=i1, i2=i2, nonpad=np64, jac=jac)
  with torch.no_grad():
    # Abs-value evaluations.
    dl = 0.0 if dlogit_err is None else dlogit_err
    dg = (_GATE_ULPS * gates.detach() + torch.stack([(j * dl).sum(-1) for j in jac]))
    dg = dg.reshape(2, -1)
    g2 = gates.detach().reshape(2, -1)
    hw = torch.bmm(h.detach(), wo64.detach().abs()).reshape(-1, yc.shape[-1])   # |h|·|wo|
    o.a_y = (g2[..., None] * hw[slot]).sum(0)
    o.e_y = (dg[..., None] * hw[slot]).sum(0)
    n = math.ceil(x.shape[-1] / 16) + 16
    p_h = torch.bmm(xe.detach().abs(), wi64.detach().abs())
    mask = (pre.detach() + 2 * n * gemm64._U_ACC * p_h) > 0
    del p_h
    dye_abs = _Dispatch(((g2 + dg)[..., None] * dy64.abs()[None]).reshape(-1, dy.shape[-1]),
                        _ChoiceRows(token, slot, keep), e)
    dh_abs = torch.bmm(dye_abs, wo64.detach().abs().transpose(1, 2)) * mask
    dxc_abs = torch.bmm(dh_abs, wi64.detach().abs().transpose(1, 2)).reshape(-1, x.shape[-1])
    kept = keep.reshape(2, -1).to(d)
    o.a_dx = _Combine(dxc_abs, kept, slot)
    o.a_dwo = torch.bmm(h.detach().transpose(1, 2), dye_abs)
    o.a_dwi = torch.bmm(xe.detach().abs().transpose(1, 2), dh_abs)
    o.softmax_bwd_abs = softmax_bwd_abs
  return o


@torch.no_grad()
def _DLogitsBound(o, yc, dy):
  """Sets the dlogits bound from the yc the kernels computed (checked against its own bound
  as a stage): dgate_k is off by at most Σ_m |yc − yc64|·|dy| plus its fp32 dot error."""
  m = dy.shape[-1]
  g_, s_ = o.gates.shape[1:]
  rows = yc.reshape(-1, m).double()
  ref = o.yc.reshape(-1, m)
  dy64 = dy.double().abs()
  kept = o.keep.reshape(2, -1).double()
  terms = []
  for k in range(2):
    r, r64 = rows[o.slot[k]], ref[o.slot[k]]
    err = ((r - r64).abs() * dy64).sum(-1) + m * gemm64._U * (r.abs() * dy64).sum(-1)
    terms.append(o.jac[k] * (err * kept[k]).reshape(g_, s_)[..., None])
  o.b_dlogits = terms[0] + terms[1] + _FP32_REL * o.softmax_bwd_abs


def _ChoiceRows(token, slot, keep):
  """The row of the flat [2·T] (choice, token) table that fills each slot, -1 where empty."""
  t = slot.shape[1]
  src = torch.full_like(token, -1)
  kf = keep.reshape(2, -1)
  ids = torch.arange(2 * t, device=slot.device).view(2, t)
  src[slot[kf]] = ids[kf]
  return src


# ---------------------------------------------------------------------- bounds ----
def _Ratio(err, bound):
  return torch.where(err == 0, torch.zeros_like(err), err / bound)


def _Bounds(o):
  """name → (reference, bound as a function of the reference value)."""
  return {
      'y': (o.y, lambda r: 3 * _U8 * (o.a_y + r.abs()) + o.e_y),
      'dx': (o.dx, lambda r: 4 * _U8 * (o.a_dx + r.abs())),
      'dwo': (o.dwo, lambda r: 3 * _U8 * (o.a_dwo + r.abs())),
      'dwi': (o.dwi, lambda r: 3 * _U8 * (o.a_dwi + r.abs())),
      'dlogits': (o.dlogits, lambda r: o.b_dlogits),
      'aux': (o.aux, lambda r: _FP32_REL * r.abs()),
  }


@torch.no_grad()
def _EndToEnd(o, got, what, names=None):
  """Asserts the end-to-end bounds of `names` (all); returns the worst err/bound of each."""
  res = {}
  for name, (ref, bound) in _Bounds(o).items():
    if names is not None and name not in names:
      continue
    v = got[name].detach().to(torch.float64).reshape(ref.shape)
    assert bool(torch.isfinite(v).all()), '%s %s: non-finite' % (what, name)
    r = _Ratio((v - ref).abs(), bound(ref))
    worst = float(r.max())
    assert worst <= 1.0, '%s %s: %d elements outside the bound, worst err/bound %g' % (
        what, name, int((r > 1).sum()), worst)
    res[name] = worst
  return res


@torch.no_grad()
def _Mutations(o):
  """(name, output, mutated float64 reference) of the five controls."""
  e, g, c, m = o.e, o.g, o.c, o.y.shape[-1]
  rows = o.yc.reshape(e, g, c, m)
  g2 = o.gates.reshape(2, -1)
  last = rows.clone()
  last[:, :, c - 1] = 0
  neighbour = rows.clone()
  neighbour[:, 0] = rows[:, 1 % g]
  with torch.enable_grad():
    other, _ = _Gates64(o.l64.detach(), o.i1, o.i2, o.nonpad, o.keep, not o.legacy)

  def DLogits(dgate):
    with torch.enable_grad():
      return torch.autograd.grad((o.gates_graph, o.aux_graph), o.l64,
                                 (dgate, torch.tensor(_AUX_COEF, dtype=dgate.dtype,
                                                      device=dgate.device)),
                                 retain_graph=True)[0]
  overflow1 = (o.nonpad > 0) & ~o.keep[0] & o.keep[1]
  second_dropped = o.dgate.clone()
  second_dropped[1][overflow1] = 0
  out = [
      ('last capacity slot dropped', 'y', _Combine(last.reshape(-1, m), g2, o.slot)),
      ('group 0 combined from group 1', 'y', _Combine(neighbour.reshape(-1, m), g2, o.slot)),
      ('the other mode\'s gates', 'y', _Combine(o.yc.reshape(-1, m), other.reshape(2, -1),
                                                o.slot)),
      ('first dgate for both choices', 'dlogits',
       DLogits(torch.stack([o.dgate[0], o.dgate[0]]))),
  ]
  # In renorm mode the surviving gate of such a token is identically 1, so its dgate reaches
  # no output and that defect would be harmless; without such tokens it has nothing to hit.
  if o.legacy and bool(overflow1.any()):
    out.append(('second dgate dropped after a first overflow', 'dlogits',
                DLogits(second_dropped)))
  return out


@torch.no_grad()
def _AssertControlsFail(o, got, what):
  bounds = _Bounds(o)
  missed = []
  checked = _Mutations(o)
  for name, out, ref in checked:
    v = got[out].detach().to(torch.float64).reshape(ref.shape)
    if not bool(((v - ref).abs() > bounds[out][1](ref)).any()):
      missed.append(name)
  assert not missed, '%s: the bounds do not reject: %s' % (what, ', '.join(missed))
  return len(checked)


# ------------------------------------------------------------ the bf16 stand-in ----
def _Bf(t):
  return t.to(torch.bfloat16).to(torch.float64)


def _StandIn(x, logits, wi, wo, dy, nonpad, index, legacy, c):
  """The exchange's arithmetic in float64, rounded to bf16 where the kernels round and with
  the gates in fp32 as `Apply` computes them."""
  d = torch.float64
  e = logits.shape[-1]
  i1, i2 = index[0].long(), index[1].long()
  pos, keep = _Scan(i1, i2, nonpad, e, c)
  slot, token = _Slots(index, pos, keep, e, c)
  l32 = logits.detach().float().requires_grad_()
  gates, aux = _Gates64(l32, i1, i2, nonpad.float(), keep, legacy)
  g32 = gates.detach().reshape(2, -1).to(d)
  x64, wi64, wo64, dy64 = (t.to(d) for t in (x, wi, wo, dy))
  xe = _Dispatch(x64, token, e)
  h = _Bf(torch.relu(torch.bmm(xe, wi64)))
  yc = _Bf(torch.bmm(h, wo64))
  rows = yc.reshape(-1, yc.shape[-1])
  y = _Bf(_Combine(rows, g32, slot))
  dgate = (rows[slot] * dy64[None]).sum(-1).float() * keep.reshape(2, -1)
  dlogits, = torch.autograd.grad((gates, aux), l32, (dgate.view_as(gates),
                                                     torch.tensor(_AUX_COEF)))
  src = _ChoiceRows(token, slot, keep)
  dye = _Bf(_Dispatch((g32[..., None] * dy64[None]).reshape(-1, dy.shape[-1]), src, e))
  dh = _Bf(torch.bmm(dye, wo64.transpose(1, 2)) * (h > 0))
  dwo = _Bf(torch.bmm(h.transpose(1, 2), dye))
  dwi = _Bf(torch.bmm(xe.transpose(1, 2), dh))
  dxc = _Bf(torch.bmm(dh, wi64.transpose(1, 2))).reshape(-1, x.shape[-1])
  dx = _Bf(_Combine(dxc, keep.reshape(2, -1).to(d), slot))
  return NestedMap(y=y, aux=aux.detach(), dx=dx, dlogits=dlogits, dwi=dwi, dwo=dwo, yc=yc)


# ---------------------------------------------------------------------- inputs ----
def _Inputs(g, s, m, h, e, skewed, padded, device, seed):
  gen = torch.Generator(device=device).manual_seed(seed)
  x = torch.randn(g * s, m, device=device, generator=gen).to(torch.bfloat16)
  gw = torch.randn(m, e, device=device, generator=gen, dtype=torch.float64) * m**-0.5
  logits = (x.double() @ gw).view(g, s, e)
  if skewed:
    logits[..., 1 % e] += 2.0
    logits[..., e // 2] += 2.0
  wi = ((torch.rand(e, m, h, device=device, generator=gen) * 2 - 1) * math.sqrt(3 / m))
  wo = ((torch.rand(e, h, m, device=device, generator=gen) * 2 - 1) * math.sqrt(3 / h))
  dy = torch.randn(g * s, m, device=device, generator=gen).to(torch.bfloat16)
  pad = routing._Paddings(g, s, seed + 1).to(device) if padded else None
  return NestedMap(x=x, logits=logits.float(), wi=wi.to(torch.bfloat16),
                   wo=wo.to(torch.bfloat16), dy=dy, pad=pad)


def _NonPad(inp):
  g, s = inp.logits.shape[:2]
  if inp.pad is None:
    return torch.ones(g, s, device=inp.logits.device)
  return 1.0 - inp.pad


# ------------------------------------------------------------------------ CPU ----
@pytest.mark.parametrize('legacy', [True, False], ids=['legacy', 'renorm'])
def test_oracle_matches_gshard_gating_and_dense_ffn(legacy):
  """The float64 oracle against the repository's dense fp32 formulation, with padding and
  both choices overflowing: the same dispatch exactly, and y, aux and the gradients of
  y·dy + coef·aux to fp32 tolerance."""
  g, s, m, h, e, c = 3, 40, 64, 72, 4, 8
  logits, pad = routing._Logits(g, s, e, 5), routing._Paddings(g, s, 6)
  gen = torch.Generator().manual_seed(7)
  x = torch.randn(g * s, m, generator=gen).bfloat16()
  wi = (torch.randn(e, m, h, generator=gen) * 0.1).bfloat16()
  wo = (torch.randn(e, h, m, generator=gen) * 0.1).bfloat16()
  dy = torch.randn(g * s, m, generator=gen).bfloat16()
  nonpad = 1.0 - pad
  i1, i2 = _Rank64(logits.double(), nonpad)
  o = _Oracle(x, logits, wi, wo, dy, nonpad, torch.stack([i1, i2]), legacy, c)
  assert 0 < int(o.keep[0].sum()) < int(nonpad.sum())      # some first choices dropped
  assert 0 < int(o.keep[1].sum()) < int(nonpad.sum())      # and some second choices

  l32 = logits.clone().requires_grad_()
  x32, wi32, wo32 = (t.float().requires_grad_() for t in (x, wi, wo))
  aux, combine, dispatch = gshard_layers.Top2GatingOnLogits(
      None, pad, l32, 1, e, c, torch.float32, False, 'all', 0.0, legacy, None)
  dense = torch.zeros(g, s, e, c)
  ei, gi, ci = torch.nonzero(o.token.view(e, g, c) >= 0, as_tuple=True)
  dense[gi, o.token.view(e, g, c)[ei, gi, ci] - gi * s, ei, ci] = 1.0
  assert torch.equal(dense, dispatch)
  xg = x32.view(g, s, m)
  y, aux = gshard_layers.FeedForwardNetworksApplyGating(
      NestedMap(combine_tensor=combine, dispatch_tensor=dispatch, aux_loss=aux), xg, xg,
      wi32, wo32, 1, g)
  ((y.reshape(g * s, m) * dy.float()).sum() + _AUX_COEF * aux).backward()
  for name, got, want in (('y', y.reshape(g * s, m), o.y), ('aux', aux, o.aux),
                          ('dx', x32.grad, o.dx), ('dlogits', l32.grad, o.dlogits),
                          ('dwi', wi32.grad, o.dwi), ('dwo', wo32.grad, o.dwo)):
    torch.testing.assert_close(got.double(), want, rtol=1e-5, atol=1e-5, msg=name)


@pytest.mark.parametrize('legacy', [True, False], ids=['legacy', 'renorm'])
def test_bounds_pass_the_bf16_stand_in_and_reject_the_controls(legacy):
  """The end-to-end bounds with the bf16-rounded float64 stand-in for the kernels: it passes
  well inside them, and each of the five mutated oracles puts an element above a bound."""
  g, s, m, h, e = 3, 64, 64, 72, 4
  c = gshard_layers.ExpertCapacity(s, e, 0, 0.5)
  inp = _Inputs(g, s, m, h, e, True, True, 'cpu', 11)
  nonpad = _NonPad(inp)
  index = torch.stack(_Rank64(inp.logits.double(), nonpad))
  o = _Oracle(inp.x, inp.logits, inp.wi, inp.wo, inp.dy, nonpad, index, legacy, c)
  assert bool(((o.nonpad > 0) & ~o.keep[0] & o.keep[1]).any())
  assert bool((o.token.view(e, g, c)[:, :, c - 1] >= 0).any())
  got = _StandIn(inp.x, inp.logits, inp.wi, inp.wo, inp.dy, nonpad, index, legacy, c)
  _DLogitsBound(o, got.yc, inp.dy)
  res = _EndToEnd(o, got, 'stand-in')
  print('stand-in worst err/bound', {k: round(v, 3) for k, v in res.items()})
  assert max(res.values()) < 0.5
  assert _AssertControlsFail(o, got, 'stand-in') == (5 if legacy else 4)


# ------------------------------------------------------------------------ GPU ----
@pytest.fixture
def local_exchanges():
  """`symm.LocalExchange` keeps one exchange per (E, device) and refuses a new geometry: give
  this module's layers their own and put the others back afterwards."""
  from lingvo_b200.parallel import symm
  saved = dict(symm._LOCAL)
  symm._LOCAL.clear()
  yield symm._LOCAL
  symm._LOCAL.clear()
  symm._LOCAL.update(saved)


class _Spy:
  """Records the exchange's GEMM outputs and its `_MoeFn` inputs, and the gate gradient."""

  def __init__(self, monkeypatch):
    from lingvo_b200.ops import gemm
    from lingvo_b200.parallel import symm
    self.gemms, self.calls = [], []
    real_gemm, real_apply = gemm.gemm, symm._MoeFn.apply

    def Gemm(*args, **kw):
      out = real_gemm(*args, **kw)
      self.gemms.append(out)
      return out

    def Apply(x2d, gate, *rest):
      rec = NestedMap(gate=gate.detach(), g=rest[4], bufs=rest[3])
      if gate.requires_grad:
        gate.register_hook(lambda d: rec.update(dgate=d.detach().clone()))
      self.calls.append(rec)
      return real_apply(x2d, gate, *rest)
    monkeypatch.setattr(gemm, 'gemm', Gemm)
    monkeypatch.setattr(symm._MoeFn, 'apply', staticmethod(Apply))


def _Sentinel(*ts):
  for t in ts:
    t.view(torch.int16).fill_(routing._SENTINEL)


@torch.no_grad()
def _CheckRouting(index, pos, keep, logits, nonpad, c, what):
  """The kernel's choices against float64: → how many tokens the float64 ranking orders
  differently. pos and keep must be what the oracle's scan makes of the kernel's choices."""
  p = torch.softmax(logits.double(), -1)
  top = p.topk(2, -1).values
  i1, i2 = index[0].long(), index[1].long()
  live = nonpad > 0
  ok1 = (p.gather(-1, i1[..., None])[..., 0] - top[..., 0]).abs() <= _TAU
  ok2 = torch.where(live, ((p.gather(-1, i2[..., None])[..., 0] - top[..., 1]).abs() <= _TAU)
                    & (i1 != i2), i2 == i1)
  assert bool((ok1 & ok2).all()), '%s: %d tokens routed outside τ' % (
      what, int((~(ok1 & ok2)).sum()))
  r1, r2 = _Rank64(logits.double(), nonpad)
  differ = int(((r1 != i1) | (r2 != i2)).sum())
  assert differ <= max(1, i1.numel() // 1000), '%s: %d tokens ranked differently' % (what, differ)
  want_pos, want_keep = _Scan(i1, i2, nonpad, logits.shape[-1], c)
  routing._AssertEqual(what + ' keep', keep, want_keep)
  routing._AssertEqual(what + ' pos', pos.long(), want_pos)
  return differ


@torch.no_grad()
def _WithinUlp(got, ref, p, n, what):
  """bf16 `got` within 2·(½ ulp + n·u·P) of the float64 `ref`."""
  bound = gemm64._Bound(ref, got.double(), n * gemm64._U * p)
  r = _Ratio((got.double() - ref).abs(), bound)
  assert bool(torch.isfinite(got).all()), '%s: non-finite' % what
  assert float(r.max()) <= 1.0, '%s: worst err/bound %g' % (what, float(r.max()))
  return float(r.max())


def _StageChecks(ex, rec, spy, inp, o, x, e, c):
  """The stage table of the module docstring; returns the worst ratio per stage."""
  from lingvo_b200.ops import gemm as G
  bufs, gate = rec.bufs, rec.gate
  g_, s_ = inp.logits.shape[:2]
  m = x.shape[-1]
  wi, wo, dy = inp.wi, inp.wo, inp.dy
  token = o.token.view(e, g_, c).cpu().int()
  choice = torch.full_like(token, -1)
  src = _ChoiceRows(o.token, o.slot, o.keep).view(e, g_, c).cpu()
  choice[src >= 0] = (src[src >= 0] // (g_ * s_)).int()
  res = {}
  routing._AssertRowsBitwise('xe', bufs.xe.view(e, g_, c, m), routing._ExpectedRows(x, token))
  assert len(spy.gemms) == 6, len(spy.gemms)
  h, _, dh, dwo, dwi, _ = spy.gemms
  assert torch.equal(gemm64._Bits(h), gemm64._Bits(G.gemm(bufs.xe, wi, True, False, act='RELU')))
  res['h'] = gemm64._Check(h, bufs.xe, wi, True, False, act=1, what='h')[0]
  rows = torch.arange(e * g_ * c, device=x.device).view(e, g_ * c)
  assert torch.equal(bufs.row_ptrs_yc, bufs.yc.data_ptr() + rows * (m * 2)), 'row table'
  res['yc'] = gemm64._Check(bufs.yc, h, wo, True, False, what='yc')[0]
  yc = bufs.yc.reshape(-1, m).double()
  gv = gate.double()
  res['y'] = _WithinUlp(rec.y, _Combine(yc, gv, o.slot), _Combine(yc.abs(), gv.abs(), o.slot),
                        3, 'y')
  dots = (yc[o.slot] * dy.double()[None]).sum(-1)
  pdots = (yc[o.slot] * dy.double()[None]).abs().sum(-1)
  dgate = rec.dgate.double()
  assert bool((dgate[gate == 0] == 0).all()), 'dgate of a dropped choice'
  err = torch.where(gate != 0, (dgate - dots).abs(), torch.zeros_like(dots))
  res['dgate'] = float(_Ratio(err, 1e-5 * pdots).max())
  assert res['dgate'] <= 1.0, 'dgate: worst err/bound %g' % res['dgate']
  routing._AssertRowsBitwise('dye', ex.dye.view(e, g_, c, m),
                             routing._ExpectedRows(dy, token, choice, gate))
  res['dh'] = gemm64._Check(dh, ex.dye, wo, True, True, aux=h, aux_mode=G.AUX_RELU_MASK,
                            what='dh')[0]
  res['dwo'] = gemm64._Check(dwo, h, ex.dye, False, False, what='dwo')[0]
  res['dwi'] = gemm64._Check(dwi, bufs.xe, dh, False, False, what='dwi')[0]
  res['dxc'] = gemm64._Check(ex.dxc, dh, wi, True, True, what='dxc')[0]
  dxc = ex.dxc.reshape(-1, m).double()
  kept = o.keep.reshape(2, -1).double()
  res['dx'] = _WithinUlp(x.grad, _Combine(dxc, kept, o.slot), _Combine(dxc.abs(), kept, o.slot),
                         2, 'dx')
  return res


def _Leaves(inp):
  return NestedMap({k: inp[k].clone().requires_grad_() for k in ('x', 'logits', 'wi', 'wo')})


def _RunExchange(ex, key, inp, c, legacy):
  r = _Leaves(inp)
  r.y, r.aux = ex.Apply(key, r.x, r.logits, inp.pad, c, legacy, r.wi, r.wo)
  return r


def _Backward(r, dy):
  ((r.y.float() * dy.float()).sum() + _AUX_COEF * r.aux).backward()
  return NestedMap(y=r.y.detach(), aux=r.aux.detach(), dx=r.x.grad, dlogits=r.logits.grad,
                   dwi=r.wi.grad, dwo=r.wo.grad)


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[cs[0] for cs in CASES])
def test_exchange_against_float64(case, monkeypatch):
  from lingvo_b200.parallel import symm
  name, g, s, m, h, e, factor, legacy, padded, skewed = case
  dev = torch.device('cuda', torch.cuda.current_device())
  c = gshard_layers.ExpertCapacity(s, e, 0, factor)
  inp = _Inputs(g, s, m, h, e, skewed, padded, dev, 1000 + g * s + e)
  ex = symm.MoeExchange(None, e, dev)
  bufs = ex._Bufs(name, g, s, c, m)
  _Sentinel(bufs.xe, bufs.yc, ex.dye, ex.dxc)
  spy = _Spy(monkeypatch)
  r = _RunExchange(ex, name, inp, c, legacy)
  got = _Backward(r, inp.dy)
  monkeypatch.undo()
  rec = spy.calls[0]
  rec.y = got.y
  nonpad = _NonPad(inp)
  differ = _CheckRouting(rec.g.index, rec.g.pos, rec.g.keep, inp.logits, nonpad, c, name)
  o = _Oracle(inp.x, inp.logits, inp.wi, inp.wo, inp.dy, nonpad, rec.g.index, legacy, c)
  x = r.x
  stages = _StageChecks(ex, rec, spy, inp, o, x, e, c)
  _DLogitsBound(o, bufs.yc, inp.dy)
  ends = _EndToEnd(o, got, name)
  if name in _CONTROL_CASES:
    n = _AssertControlsFail(o, got, name)
    # Only the skewed case is sure to overflow first choices whose second choice is kept.
    assert name != 'bench_skewed' or n == 5, n
  print('%s: %d tokens ranked differently from float64' % (name, differ))
  print('%s stages: %s' % (name, ' '.join('%s %.3f' % kv for kv in stages.items())))
  print('%s end to end: %s' % (name, ' '.join('%s %.3f' % kv for kv in ends.items())))


# ------------------------------------------------------------- buffer lifetime ----
_LIFE = (2, 256, 256, 512, 8, 2.0)     # G, S, M, H, E, capacity factor


def _LifeInputs(seed):
  g, s, m, h, e, _ = _LIFE
  return _Inputs(g, s, m, h, e, False, False, torch.device('cuda'), seed)


def _AssertBitwise(a, b, what):
  for k in ('y', 'aux', 'dx', 'dlogits', 'dwi', 'dwo'):
    assert torch.equal(a[k].view(-1).view(torch.int16 if a[k].dtype == torch.bfloat16 else
                                          torch.int32),
                       b[k].view(-1).view(torch.int16 if b[k].dtype == torch.bfloat16 else
                                          torch.int32)), '%s: %s differs' % (what, k)


@pytest.mark.gpu
def test_two_layers_interleaved_match_running_each_alone():
  """Forward A, forward B, backward B, backward A: the layers share the dye / dxc scratch."""
  from lingvo_b200.parallel import symm
  g, s, m, h, e, factor = _LIFE
  c = gshard_layers.ExpertCapacity(s, e, 0, factor)
  ex = symm.MoeExchange(None, e, torch.device('cuda'))
  a, b = _LifeInputs(1), _LifeInputs(2)
  alone_a = _Backward(_RunExchange(ex, 'A', a, c, True), a.dy)
  alone_b = _Backward(_RunExchange(ex, 'B', b, c, True), b.dy)
  ra = _RunExchange(ex, 'A', a, c, True)
  rb = _RunExchange(ex, 'B', b, c, True)
  got_b = _Backward(rb, b.dy)
  got_a = _Backward(ra, a.dy)
  _AssertBitwise(got_a, alone_a, 'layer A')
  _AssertBitwise(got_b, alone_b, 'layer B')


@pytest.mark.gpu
def test_rematerialized_layer_matches_the_plain_run():
  """Under `RematerializeFn` backward re-runs the dispatch first; the gradients must not
  change, and the buffer-generation guard must not fire."""
  from lingvo_b200.parallel import symm
  g, s, m, h, e, factor = _LIFE
  c = gshard_layers.ExpertCapacity(s, e, 0, factor)
  ex = symm.MoeExchange(None, e, torch.device('cuda'))
  a = _LifeInputs(3)
  plain = _Backward(_RunExchange(ex, 'A', a, c, True), a.dy)
  r = _Leaves(a)

  def Fn(x, logits, wi, wo):
    return ex.Apply('A', x, logits, None, c, True, wi, wo)
  r.y, r.aux = py_utils.RematerializeFn(Fn, r.x, r.logits, r.wi, r.wo)
  _AssertBitwise(_Backward(r, a.dy), plain, 'remat')


@pytest.mark.gpu
def test_backward_after_a_second_forward_of_the_layer_raises():
  """A second forward of the same layer refills its xe / yc; the first forward's backward
  would read them, so it must refuse instead of returning wrong gradients."""
  from lingvo_b200.parallel import symm
  g, s, m, h, e, factor = _LIFE
  c = gshard_layers.ExpertCapacity(s, e, 0, factor)
  ex = symm.MoeExchange(None, e, torch.device('cuda'))
  a, b = _LifeInputs(4), _LifeInputs(5)
  first = _RunExchange(ex, 'A', a, c, True)
  second = _RunExchange(ex, 'A', b, c, True)
  with pytest.raises(RuntimeError, match='ran forward again'):
    _Backward(first, a.dy)
  assert bool(torch.isfinite(_Backward(second, b.dy).dx.float()).all())


# ---------------------------------------------------------------- the MoE layer ----
def _Layer(g, m, h, e):
  from lingvo_b200.core import gshard_builder
  b = gshard_builder.MoEBuilder.Params().Set(
      model_dim=m, moe_hidden_dim=h, e_dim=e, c_dim=0, capacity_factor=2.0, num_groups=g,
      num_devices=1, moe_activation='RELU', second_expert_policy='all',
      gating_logits_dtype=torch.float32, mask_dtype=torch.float32,
      legacy_mtf_behavior=True).Instantiate()
  return b.MoE('moe').Instantiate()


@pytest.mark.gpu
def test_moe_layer_against_float64(local_exchanges, monkeypatch):
  """`MoELayer` in bf16 at the benchmark's dims: out, dx (the exchange's and the router's
  gradient, summed by the router kernel) and dgw against the oracle, with the router's fp32
  logits error δl measured against float64 and carried into the gate-error terms."""
  from lingvo_b200.ops import gate as gate_ops
  g, s, m, h, e = 8, 1024, 2048, 8192, 8
  dev = torch.device('cuda', torch.cuda.current_device())
  torch.manual_seed(21)
  layer = _Layer(g, m, h, e).to(dev)
  gen = torch.Generator(device=dev).manual_seed(22)
  x = torch.randn(g, s, m, device=dev, generator=gen).to(torch.bfloat16).requires_grad_()
  dy = torch.randn(g * s, m, device=dev, generator=gen).to(torch.bfloat16)
  seg = torch.ones(g, s, dtype=torch.int32, device=dev)
  spy = _Spy(monkeypatch)
  out, aux = layer.FProp(layer.theta, x, seg)
  ((out.reshape(g * s, m).float() * dy.float()).sum() + _AUX_COEF * aux).backward()
  monkeypatch.undo()
  ex = local_exchanges[(e, dev.index)]
  assert id(layer) in ex._layers and len(spy.calls) == 1, 'the fused exchange did not run'
  rec = spy.calls[0]
  gw = layer.vars.gw
  wi, wo = layer.vars.wi.detach().to(torch.bfloat16), layer.vars.wo.detach().to(torch.bfloat16)
  x2 = x.detach().reshape(g * s, m)
  l64 = (x2.double() @ gw.detach().double()).view(g, s, e)
  with torch.no_grad():
    lk = gate_ops.gate_logits(x.detach(), gw.detach()).double().view(g, s, e)
  dl = 2 * (lk - l64).abs() + gemm64._U * l64.abs()
  nonpad = torch.ones(g, s, device=dev)
  c = rec.g.capacity
  _CheckRouting(rec.g.index, rec.g.pos, rec.g.keep, lk.float(), nonpad, c, 'layer')
  o = _Oracle(x2, l64, wi, wo, dy, nonpad, rec.g.index, True, c, dlogit_err=dl)
  _DLogitsBound(o, rec.bufs.yc, dy)
  res = _EndToEnd(o, NestedMap(y=out.reshape(g * s, m), aux=aux, dwi=layer.vars.wi.grad,
                               dwo=layer.vars.wo.grad), 'layer', ('y', 'aux', 'dwi', 'dwo'))
  with torch.no_grad():
    gw64 = gw.detach().double()
    dlf = o.dlogits.reshape(g * s, e)
    bdl = o.b_dlogits.reshape(g * s, e)
    dx64 = o.dx + dlf @ gw64.t()
    bound = (4 * _U8 * (o.a_dx + o.dx.abs()) + bdl @ gw64.abs().t() +
             e * gemm64._U * dlf.abs() @ gw64.abs().t() + _U8 * dx64.abs())
    r = _Ratio((x.grad.reshape(g * s, m).double() - dx64).abs(), bound)
    res['dx'] = float(r.max())
    assert res['dx'] <= 1.0, 'layer dx: worst err/bound %g' % res['dx']
    x64 = x2.double()
    dgw64 = x64.t() @ dlf
    bound = x64.abs().t() @ bdl + g * s * gemm64._U * (x64.abs().t() @ dlf.abs())
    r = _Ratio((gw.grad.double() - dgw64).abs(), bound)
    res['dgw'] = float(r.max())
    assert res['dgw'] <= 1.0, 'layer dgw: worst err/bound %g' % res['dgw']
  print('layer end to end: %s' % ' '.join('%s %.3f' % kv for kv in res.items()))
