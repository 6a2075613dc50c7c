"""The wgmma GEMM (ops/csrc/gemm_wgmma.cu) against a float64 oracle at every GEMM site of the
MoELm8E training step, through the linear-layer wrappers, and at the edges of its tiling.

Contract checked here, for bf16 operands A [G, M, K], B [G, N, K] (either may be stored
MN-major), an fp32 bias [G, N], a bf16 aux [G, M, N] and an fp32 row scale [G, M]:

    y = bf16( ((S + bias) → ReLU → ReLU-mask(aux) or + aux) · rs ),   S = Σ_k A·B

with every step optional, in that order. Rows may be redirected through a row-pointer table;
a null entry leaves its destination untouched. The output is bit-identical from call to call.

The oracle computes S in float64 from the bf16 inputs (every bf16 product is exact in
float64, so S is exact to ~K·2^-53), applies the epilogue in the kernel's order, and computes
P = Σ|A·B| with a second float64 matmul. Both run in row slabs of at most 2^23 elements, so
the oracle adds about a GB of device memory.

Where the kernel rounds, and the bound that follows. Per element

    |y − ref| ≤ C·(½·ulp_bf16(max(|ref|, |y|)) + E),   C = 2,
    E = (n·u′·P + 3u·(|S| + |bias| + |aux|))·|rs|,

with u = 2^-24, u′ = 2^-23 (room for a truncating tensor-core adder) and n = ⌈K/16⌉ + 16: one
fp32 accumulator add per k16 wgmma plus an allowance for the adds inside the instruction.
|aux| counts only where aux is added. NVIDIA does not document Hopper's internal bf16
accumulation precision, so n and u′ are a model, not a fact; the measured worst err/bound
below shows how much room it leaves. The 3u term covers the fp32 bias add, residual add and
row-scale product; the ½ ulp is the final bf16 rounding.

Parts of the output are exact, because aux and the ReLU act on exact comparisons:
  * in ReLU-mask mode, y = 0 exactly wherever aux ≤ 0, including −0.0 and exact zeros;
  * with act = ReLU, y = 0 exactly wherever S + bias < −C·(n·u′·P + 3u·(|S| + |bias|)).

The per-element bound is one ulp wide, so it cannot see a defect of at most one ulp, such
as truncating instead of rounding in the bf16 pack. A rounding check catches that: under
round-to-nearest and an fp32 accumulator, an error above ⅝·ulp_bf16(|ref|) needs the fp32
error to reach ⅛ ulp of the result, which happens only where S nearly cancels. So at most
1 % of the elements of a GEMM with at least 2^14 outputs may exceed ⅝ ulp. With `gemm_ref`
standing in for the kernel, a truncating pack puts ~38 % of the elements there while its
worst err/bound stays below 1. A bias read as bf16, or a bf16 rounding before the bias add,
fails the bound itself wherever the bias cancels S.

Every site's comparison must also reject five mutated oracles built from the same float64
pieces: the last k-block (the K mod 64 tail for ragged K) dropped or counted twice, the bias
taken from column n + 1, the row scale from row m + 1 and the aux operand from row m + 1.
Each must put some element above the bound. A CPU test runs the same bound, controls and
rounding check with `gemm_ref` rounded to bf16 standing in for the kernel, and shows that
the three sub-ulp defects above fail.

Sites are the rows of `INVENTORY` in tools/gpu_gemm_bench.py, imported so the two lists
cannot drift, with their operand majors and epilogues; four benchmark-sized cases per store
path add a bias and a row scale to each operand-major pair. An edge sweep covers
G ∈ {1, 3}, M ∈ {1, 8, 127, 128, 129, 200}, N ∈ {8, 64, 72, 128, 136, 264},
K ∈ {8, 16, 56, 64, 72, 136}, all four operand majors (an MN-major A needs M % 8 == 0) and
the four epilogue kinds through the TMA store and the row-pointer path. Together they reach
all 16 kernel instantiations (tile width 128 / 256 × 4 majors × 2 store paths).

Measured on an H100 80GB HBM3 (700 W limit, 1980 MHz max SM clock); the inputs are seeded,
so these repeat exactly. Worst err/bound per site, and the share of elements above ⅝ ulp:

    qkv_fwd         0.480  2.3e-4        ffn_dwi         0.380  1.1e-3
    qkv_dgrad       0.423  7.8e-4        moe_wi_fwd      0.480  1.1e-4
    qkv_wgrad       0.380  1.1e-3        moe_wo_fwd      0.380  1.1e-3
    attn_out_fwd    0.487  2.8e-4        moe_dh          0.480  0.9e-4
    attn_out_dgrad  0.480  2.3e-4        moe_dx          0.380  1.1e-3
    attn_out_wgrad  0.379  1.1e-3        moe_dwo         0.485  2.3e-4
    ffn_wi_fwd      0.480  1.1e-4        moe_dwi         0.486  2.3e-4
    ffn_wo_fwd      0.429  1.3e-3        lm_logits       0.480  2.3e-4
    ffn_dh          0.480  0.9e-4        lm_dx           0.149  4.6e-3
    ffn_dx          0.380  1.1e-3        lm_dw           0.380  1.1e-3
    ffn_dwo         0.380  1.1e-3
    bias + row scale cases  ≤ 0.490  ≤ 2.8e-4
    wrapper stages          ≤ 0.498  ≤ 1.1e-3

Every ratio is below ½: the error is the final bf16 rounding, and the accumulation term of
the model is never needed. At lm_dx (K = 32000) n·u′·P dominates the bound, which is ~3x
looser there than the measured error. The share above ⅝ ulp grows with K; at K = 32000 it is
half the 1 % limit. The whole module takes ~30 s on the H100.
"""
import importlib.util
import math
import os

import pytest
import torch

from lingvo_b200 import ops
from lingvo_b200.ops import gemm as G

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _Inventory():
  spec = importlib.util.spec_from_file_location(
      'gpu_gemm_bench', os.path.join(_ROOT, 'tools', 'gpu_gemm_bench.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod.INVENTORY


INVENTORY = _Inventory()

_U = 2.0**-24
_U_ACC = 2.0**-23          # u′: a truncating tensor-core adder
_C = 2.0
_BLOCK_K = 64              # kBlockM / kBlockK / BN tiling of the kernel
_BLOCK_M = 128
_SLAB = 2**23              # oracle elements per slab
_ROUND_ULPS = 0.625        # the rounding check's threshold ...
_ROUND_FRAC = 0.01         # ... and the share of elements allowed above it
_ROUND_MIN = 2**14         # outputs needed for the rounding check
_SENTINEL = 0x7f99         # a NaN bit pattern marking untouched redirected rows

# The four bias + row-scale cases per store path: one per operand-major pair, each with the
# epilogue the step uses at that pair (G, M, N, K of the attention output projection).
_BIAS_CASES = [
    ('bias_relu', 1, 8192, 2048, 2048, True, False, 'relu'),
    ('bias_residual', 1, 8192, 2048, 2048, True, True, 'residual'),
    ('bias_relu_mask', 1, 8192, 2048, 2048, False, True, 'relu_mask'),
    ('bias_plain', 1, 8192, 2048, 2048, False, False, None),
]

_SWEEP_G = (1, 3)
_SWEEP_M = (1, 8, 127, 128, 129, 200)
_SWEEP_N = (8, 64, 72, 128, 136, 264)
_SWEEP_K = (8, 16, 56, 64, 72, 136)
_MAJORS = [(True, True), (True, False), (False, True), (False, False)]
_EPIS = [None, 'relu', 'residual', 'relu_mask']


def _Ulp(t):
  """One bf16 ulp at |t| (float64), floored at the smallest normal."""
  a = t.abs().clamp_min(2.0**-126)
  return torch.exp2(torch.floor(torch.log2(a)) - 7)


def _Bits(t):
  return t.detach().contiguous().view(torch.int16)


# ------------------------------------------------------------------ the oracle ----
def _Epilogue(s, p, n, bias, act, aux, aux_mode, rs):
  """Float64 epilogue in the kernel's order, with E of the module docstring. Returns
  (ref, E, pre-activation value, its fp32 error bound without the row scale)."""
  v = s if bias is None else s + bias
  mag = s.abs() if bias is None else s.abs() + bias.abs()
  e_pre = n * _U_ACC * p + 3 * _U * mag
  e = e_pre
  pre = v
  if act == 1:
    v = v.clamp_min(0.0)
  if aux_mode == G.AUX_RELU_MASK:
    v = torch.where(aux > 0, v, torch.zeros((), dtype=v.dtype, device=v.device))
  elif aux_mode == G.AUX_ADD:
    v = v + aux
    e = e + 3 * _U * aux.abs()
  if rs is not None:
    v = v * rs
    e = e * rs.abs()
  return v, e, pre, e_pre


def _Bound(ref, y, e):
  return _C * (0.5 * _Ulp(torch.maximum(ref.abs(), y.abs())) + e)


@torch.no_grad()
def _Check(y, a, b, ak, bk, bias=None, act=0, aux=None, aux_mode=0, rs=None, valid=None,
           controls=False, what=''):
  """Asserts the bound, the exact zeros and the rounding check of the module docstring for
  the bf16 result y of the GEMM of a, b (2-D or 3-D, `gemm`'s layouts) with that epilogue.
  `valid` [G, M] selects the rows to check. With `controls`, also asserts that each mutated
  oracle puts some element above the bound. Returns the worst err/bound and the share of
  elements above the rounding check's threshold."""
  a3 = a if a.dim() == 3 else a.unsqueeze(0)
  b3 = b if b.dim() == 3 else b.unsqueeze(0)
  y3 = y if y.dim() == 3 else y.unsqueeze(0)
  assert y3.dtype == torch.bfloat16, what
  ng, m, nn = y3.shape
  k = a3.shape[2] if ak else a3.shape[1]
  n = math.ceil(k / 16) + 16
  k0 = (k - 1) // _BLOCK_K * _BLOCK_K           # first column of the last k-block
  aux3 = None if aux is None else aux.reshape(ng, m, nn)
  bias2 = None if bias is None else bias.reshape(ng, nn)
  rs2 = None if rs is None else rs.reshape(ng, m)
  valid2 = None if valid is None else valid.reshape(ng, m)
  rows = max(1, min(m, _SLAB // max(nn, k)))
  worst = 0.0
  over, total = 0, 0
  caught = {}
  if controls:
    caught['k-block dropped'] = caught['k-block twice'] = False
    if bias is not None:
      caught['bias from column n + 1'] = False
    if rs is not None:
      caught['row scale from row m + 1'] = False
    if aux is not None and aux_mode != 0:
      caught['aux from row m + 1'] = False
  for g in range(ng):
    bm = (b3[g] if bk else b3[g].t()).double()         # [N, K]
    bma = bm.abs()
    bml = bm[:, k0:]
    bg = None if bias2 is None else bias2[g].double()
    for m0 in range(0, m, rows):
      m1 = min(m, m0 + rows)
      am = (a3[g, m0:m1] if ak else a3[g, :, m0:m1].t()).double()   # [rows, K]
      s = am @ bm.t()
      p = am.abs() @ bma.t()
      yy = y3[g, m0:m1].double()
      x = None if aux3 is None else aux3[g, m0:m1].double()
      r = None if rs2 is None else rs2[g, m0:m1].double()[:, None]
      ref, e, pre, e_pre = _Epilogue(s, p, n, bg, act, x, aux_mode, r)
      err = (yy - ref).abs()
      bound = _Bound(ref, yy, e)
      sel = None if valid2 is None else valid2[g, m0:m1]
      def Pick(t):
        return t if sel is None else t[sel]
      yv, errv, boundv = Pick(yy), Pick(err), Pick(bound)
      assert bool(torch.isfinite(yv).all()), '%s: non-finite output' % what
      bad = errv > boundv
      assert not bool(bad.any()), (
          '%s: %d elements outside the bound, worst err/bound %g (g=%d, rows %d..%d)' % (
              what, int(bad.sum()), float((errv / boundv)[bad].max()), g, m0, m1))
      if errv.numel():
        worst = max(worst, float((errv / boundv).max()))
      if aux_mode == G.AUX_RELU_MASK:
        z = Pick(x <= 0)
        assert bool((yv[z] == 0).all()), '%s: nonzero output where aux <= 0' % what
      if act == 1:
        z = Pick(pre < -_C * e_pre)
        assert bool((yv[z] == 0).all()), '%s: nonzero output below the ReLU' % what
      over += int((errv > _ROUND_ULPS * _Ulp(Pick(ref))).sum())
      total += errv.numel()
      if not controls:
        continue
      def Caught(name, **kw):
        args = dict(s=s, bias=bg, aux=x, rs=r)
        args.update(kw)
        ref2, e2, _, _ = _Epilogue(args['s'], p, n, args['bias'], act, args['aux'], aux_mode,
                                   args['rs'])
        if bool(Pick((yy - ref2).abs() > _Bound(ref2, yy, e2)).any()):
          caught[name] = True
      last = am[:, k0:] @ bml.t()
      Caught('k-block dropped', s=s - last)
      Caught('k-block twice', s=s + last)
      nxt = (torch.arange(m0, m1, device=y.device) + 1) % m
      if bg is not None:
        Caught('bias from column n + 1', bias=torch.roll(bg, -1))
      if r is not None:
        Caught('row scale from row m + 1', rs=rs2[g, nxt].double()[:, None])
      if x is not None and aux_mode != 0:
        Caught('aux from row m + 1', aux=aux3[g, nxt].double())
  if total >= _ROUND_MIN:
    assert over <= _ROUND_FRAC * total, (
        '%s: %d of %d elements above %g ulp: not rounded to nearest from fp32' % (
            what, over, total, _ROUND_ULPS))
  missed = [k for k, v in caught.items() if not v]
  assert not missed, '%s: the bound does not reject: %s' % (what, ', '.join(missed))
  return worst, over / max(total, 1)


@torch.no_grad()
def _CheckSum(db, dy, what):
  """fp32 db = Σ_rows dy against a float64 sum: |Δ| ≤ R·u·Σ|dy| for R summed rows."""
  assert db.dtype == torch.float32, what
  ref = dy.double().sum(-2)
  bound = dy.shape[-2] * _U * dy.double().abs().sum(-2)
  err = (db.double() - ref).abs()
  assert not bool((err > bound).any()), '%s: worst excess %g' % (what, float((err - bound).max()))


# ------------------------------------------------------------------- the kernel ----
def _Rnd(gen, *shape, scale=1.0):
  return (torch.randn(*shape, device=gen.device, generator=gen) * scale).to(torch.bfloat16)


def _Inputs(gen, ng, m, n, k, ak, bk, epi, with_bias):
  """Operands and epilogue arguments of one case; `epi` as in INVENTORY."""
  a = _Rnd(gen, ng, m, k) if ak else _Rnd(gen, ng, k, m)
  b = _Rnd(gen, ng, n, k) if bk else _Rnd(gen, ng, k, n)
  kw = {}
  if epi == 'relu':
    kw['act'] = 1
  elif epi == 'residual':
    kw.update(aux=_Rnd(gen, ng, m, n, scale=math.sqrt(k)), aux_mode=G.AUX_ADD)
  elif epi == 'relu_mask':
    aux = _Rnd(gen, ng, m, n)
    flat = aux.view(-1)
    flat[::7] = 0.0
    flat[3::11] = -0.0
    kw.update(aux=aux, aux_mode=G.AUX_RELU_MASK)
  elif epi == 'row_scale':
    kw['row_scale'] = torch.rand(ng, m, device=gen.device, generator=gen)
  if with_bias:
    kw['bias'] = torch.randn(ng, n, device=gen.device, generator=gen) * math.sqrt(k)
    kw['row_scale'] = 0.25 + 1.75 * torch.rand(ng, m, device=gen.device, generator=gen)
  return a, b, kw


def _RowTable(gen, ng, m, n):
  """A permuted destination table over a [G·M, N] buffer; every fifth row is null."""
  perm = torch.randperm(ng * m, device=gen.device, generator=gen)
  valid = torch.arange(ng * m, device=gen.device) % 5 != 3
  return perm, valid


def _Run(a, b, ak, bk, kw, table=None):
  """Runs the kernel. With a row table, returns the output gathered from the redirected
  rows and the raw destination buffer."""
  if table is None:
    return G.gemm(a, b, ak, bk, **kw), None
  perm, valid = table
  ng, m = a.shape[0], (a.shape[1] if ak else a.shape[2])
  n = b.shape[1] if bk else b.shape[2]
  dest = torch.empty(ng * m, n, device=a.device, dtype=torch.bfloat16)
  dest.view(torch.int16).fill_(_SENTINEL)
  ptrs = torch.where(valid, dest.data_ptr() + perm * (n * 2), 0).to(torch.int64)
  G.gemm(a, b, ak, bk, row_ptrs=ptrs, **kw)
  return dest[perm].view(ng, m, n), dest


def _RunAndCheck(gen, name, ng, m, n, k, ak, bk, epi, redirect, with_bias, controls):
  a, b, kw = _Inputs(gen, ng, m, n, k, ak, bk, epi, with_bias)
  table = _RowTable(gen, ng, m, n) if redirect else None
  y, dest = _Run(a, b, ak, bk, kw, table)
  y2, dest2 = _Run(a, b, ak, bk, kw, table)
  if redirect:
    perm, valid = table
    assert torch.equal(_Bits(dest), _Bits(dest2)), '%s: not reproducible' % name
    untouched = _Bits(dest[perm[~valid]])
    assert bool((untouched == _SENTINEL).all()), '%s: a null row was written' % name
  else:
    assert torch.equal(_Bits(y), _Bits(y2)), '%s: not reproducible' % name
  return _Check(y, a, b, ak, bk, bias=kw.get('bias'), act=kw.get('act', 0), aux=kw.get('aux'),
                aux_mode=kw.get('aux_mode', 0), rs=kw.get('row_scale'),
                valid=None if table is None else table[1], controls=controls, what=name)


def _Report(what, res):
  print('%s: worst err/bound %.4f, share above %g ulp %.1e' % (what, res[0], _ROUND_ULPS, res[1]))


def _Gen(seed):
  return torch.Generator(device='cuda').manual_seed(seed)


# --------------------------------------------------------------------- the sites ----
@pytest.mark.gpu
@pytest.mark.parametrize('site', INVENTORY, ids=[s[0] for s in INVENTORY])
def test_step_gemm_sites(site):
  name, ng, m, n, k, ak, bk, epi = site
  _Report(name, _RunAndCheck(_Gen(INVENTORY.index(site)), name, ng, m, n, k, ak, bk, epi,
                             epi == 'row_ptrs', False, True))


@pytest.mark.gpu
@pytest.mark.parametrize('redirect', [False, True], ids=['tma_store', 'row_ptrs'])
@pytest.mark.parametrize('case', _BIAS_CASES, ids=[c[0] for c in _BIAS_CASES])
def test_bias_and_row_scale(case, redirect):
  name, ng, m, n, k, ak, bk, epi = case
  what = '%s_%s' % (name, 'row_ptrs' if redirect else 'tma_store')
  _Report(what, _RunAndCheck(_Gen(100 + _BIAS_CASES.index(case)), what, ng, m, n, k, ak, bk,
                             epi, redirect, True, True))


def _SweepShapes(ak):
  """(G, M, N, K) of the edge sweep: every M × N × K at G = 1, and a cyclic K at G = 3."""
  for ng in _SWEEP_G:
    for i, m in enumerate(_SWEEP_M):
      if not ak and m % 8:
        continue
      for j, n in enumerate(_SWEEP_N):
        ks = _SWEEP_K if ng == 1 else (_SWEEP_K[(i + j) % len(_SWEEP_K)],)
        for k in ks:
          yield ng, m, n, k


@pytest.mark.gpu
@pytest.mark.parametrize('redirect', [False, True], ids=['tma_store', 'row_ptrs'])
@pytest.mark.parametrize('epi', _EPIS, ids=['plain', 'relu', 'residual', 'relu_mask'])
@pytest.mark.parametrize('ak,bk', _MAJORS, ids=['KK', 'KMN', 'MNK', 'MNMN'])
def test_edge_sweep(ak, bk, epi, redirect):
  gen = _Gen(7)
  for i, (ng, m, n, k) in enumerate(_SweepShapes(ak)):
    _RunAndCheck(gen, 'G=%d M=%d N=%d K=%d' % (ng, m, n, k), ng, m, n, k, ak, bk, epi,
                 redirect, i % 2 == 1, False)


def _Bn256(ng, m, n, sms):
  """UseBn256 of gemm_wgmma.cu: the tile width the kernel picks."""
  if n <= 128:
    return False
  mt = ng * ((m + _BLOCK_M - 1) // _BLOCK_M)
  t256, t128 = mt * ((n + 255) // 256), mt * ((n + 127) // 128)
  w256, w128 = 2 * ((t256 + sms - 1) // sms), (t128 + sms - 1) // sms
  return w128 * 10 > w256 * 9


@pytest.mark.gpu
def test_cases_reach_every_instantiation():
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  seen = set()
  def Add(ng, m, n, ak, bk, redirect):
    seen.add((256 if _Bn256(ng, m, n, sms) else 128, ak, bk, not redirect))
  for _, ng, m, n, _, ak, bk, epi in INVENTORY:
    Add(ng, m, n, ak, bk, epi == 'row_ptrs')
  for _, ng, m, n, _, ak, bk, _ in _BIAS_CASES:
    for redirect in (False, True):
      Add(ng, m, n, ak, bk, redirect)
  for ak, bk in _MAJORS:
    for ng, m, n, _ in _SweepShapes(ak):
      for redirect in (False, True):
        Add(ng, m, n, ak, bk, redirect)
  want = {(bn, ak, bk, t) for bn in (128, 256) for ak, bk in _MAJORS for t in (True, False)}
  assert seen == want, sorted(want - seen)


# -------------------------------------------------------- the linear-layer wrappers ----
_T, _D, _H, _E = 8192, 2048, 8192, 8     # tokens, model dim, FFN dim, experts


def _Checked(*args, **kw):
  _Report(kw['what'], _Check(*args, **kw))


def _Same(got, want, what):
  assert torch.equal(_Bits(got), _Bits(want)), '%s: differs from the recomputed GEMM' % what


@pytest.mark.gpu
def test_linear_bias_relu():
  gen = _Gen(200)
  x = _Rnd(gen, _T, _D).requires_grad_()
  w = _Rnd(gen, _D, _H, scale=_D**-0.5).requires_grad_()
  bias = torch.randn(_H, device='cuda', generator=gen).requires_grad_()
  dy = _Rnd(gen, _T, _H)
  y = G.linear(x, w, bias, act='RELU')
  y.backward(dy)
  _Same(y, G.gemm(x, w, True, False, bias=bias, act=1), 'y')
  _Checked(y, x, w, True, False, bias=bias, act=1, what='linear y')
  dym = torch.where(y > 0, dy, torch.zeros((), dtype=dy.dtype, device=dy.device))
  _Same(x.grad, G.gemm(dym, w, True, True), 'dx')
  _Checked(x.grad, dym, w, True, True, what='linear dx')
  _Same(w.grad, G.gemm(x, dym, False, False), 'dw')
  _Checked(w.grad, x, dym, False, False, what='linear dw')
  _CheckSum(bias.grad, dym, 'linear db')


@pytest.mark.gpu
def test_linear_t_bias():
  gen = _Gen(201)
  x = _Rnd(gen, _T, _D).requires_grad_()
  w = _Rnd(gen, _D, _D, scale=_D**-0.5).requires_grad_()     # [N, K]
  bias = torch.randn(_D, device='cuda', generator=gen).requires_grad_()
  dy = _Rnd(gen, _T, _D)
  y = G.linear_t(x, w, bias)
  y.backward(dy)
  _Same(y, G.gemm(x, w, True, True, bias=bias), 'y')
  _Checked(y, x, w, True, True, bias=bias, what='linear_t y')
  _Same(x.grad, G.gemm(dy, w, True, False), 'dx')
  _Checked(x.grad, dy, w, True, False, what='linear_t dx')
  _Same(w.grad, G.gemm(dy, x, False, False), 'dw')
  _Checked(w.grad, dy, x, False, False, what='linear_t dw')
  _CheckSum(bias.grad, dy, 'linear_t db')


@pytest.mark.gpu
@pytest.mark.parametrize('act', ['NONE', 'RELU'])
def test_grouped_linear_bias(act):
  gen = _Gen(202)
  c = 2048                                                  # expert capacity
  x = _Rnd(gen, _E, c, _D).requires_grad_()
  w = _Rnd(gen, _E, _D, _H, scale=_D**-0.5).requires_grad_()
  bias = torch.randn(_E, _H, device='cuda', generator=gen).requires_grad_()
  dy = _Rnd(gen, _E, c, _H)
  y = G.grouped_linear(x, w, bias, act=act)
  y.backward(dy)
  a = G.ACT_IDS[act]
  _Same(y, G.gemm(x, w, True, False, bias=bias, act=a), 'y')
  _Checked(y, x, w, True, False, bias=bias, act=a, what='grouped y')
  dym = dy if a == 0 else torch.where(y > 0, dy, torch.zeros((), dtype=dy.dtype,
                                                              device=dy.device))
  _Same(x.grad, G.gemm(dym, w, True, True), 'dx')
  _Checked(x.grad, dym, w, True, True, what='grouped dx')
  _Same(w.grad, G.gemm(x, dym, False, False), 'dw')
  _Checked(w.grad, x, dym, False, False, what='grouped dw')
  _CheckSum(bias.grad, dym, 'grouped db')


@pytest.mark.gpu
def test_ffn_relu_residual():
  gen = _Gen(203)
  x = _Rnd(gen, _T, _D).requires_grad_()
  wi = _Rnd(gen, _D, _H, scale=_D**-0.5).requires_grad_()
  wo = _Rnd(gen, _H, _D, scale=_H**-0.5).requires_grad_()
  dy = _Rnd(gen, _T, _D)
  y = G.ffn_relu(x, wi, wo, residual=x)
  fn = y.grad_fn
  while type(fn).__name__ != '_FfnReluFnBackward':
    fn = fn.next_functions[0][0]
  h = fn.saved_tensors[3]
  y.backward(dy)
  _Same(h, G.gemm(x, wi, True, False, act=1), 'h')
  _Checked(h, x, wi, True, False, act=1, what='ffn h')
  _Same(y, G.gemm(h, wo, True, False, aux=x.detach(), aux_mode=G.AUX_ADD), 'y')
  _Checked(y, h, wo, True, False, aux=x.detach(), aux_mode=G.AUX_ADD, what='ffn y')
  dh = G.gemm(dy, wo, True, True, aux=h, aux_mode=G.AUX_RELU_MASK)
  _Checked(dh, dy, wo, True, True, aux=h, aux_mode=G.AUX_RELU_MASK, what='ffn dh')
  _Same(wo.grad, G.gemm(h, dy, False, False), 'dwo')
  _Checked(wo.grad, h, dy, False, False, what='ffn dwo')
  _Same(wi.grad, G.gemm(x, dh, False, False), 'dwi')
  _Checked(wi.grad, x, dh, False, False, what='ffn dwi')
  # dx = bf16(dh·wiᵀ) + dy, the residual's gradient added in bf16 by autograd.
  dxg = G.gemm(dh, wi, True, True)
  _Checked(dxg, dh, wi, True, True, what='ffn dx (GEMM)')
  _Same(x.grad, dxg + dy, 'dx')
  exact = dxg.double() + dy.double()
  got = x.grad.double()
  half = 0.5 * _Ulp(torch.maximum(exact.abs(), got.abs()))
  assert not bool(((got - exact).abs() > half).any()), 'ffn dx: residual add not rounded'


# --------------------------------------------------------------- argument checks ----
@pytest.mark.gpu
def test_aux_sizes_and_empty_k_are_refused_without_launching():
  """aux must have out's sizes: the aux tensor map takes them from out, so a smaller aux
  would be read past its end. K = 0 is refused by name."""
  gen = _Gen(300)
  m, n, k = 256, 256, 128
  a = _Rnd(gen, m, k)
  b = _Rnd(gen, n, k)
  a3 = _Rnd(gen, 3, m, k)
  b3 = _Rnd(gen, 3, n, k)
  wide = _Rnd(gen, m, n + 64)
  out = torch.empty(m, n + 64, device='cuda', dtype=torch.bfloat16)[:, :n]
  nat = ops.native()
  launches = nat.launch_count()
  for mode in (G.AUX_ADD, G.AUX_RELU_MASK):
    with pytest.raises(RuntimeError, match='aux must have'):
      G.gemm(a, b, True, True, aux=_Rnd(gen, m - 8, n), aux_mode=mode)     # fewer rows
    with pytest.raises(RuntimeError, match='aux must have'):
      G.gemm(a3, b3, True, True, aux=_Rnd(gen, m, n), aux_mode=mode)      # 2-D with G = 3
    with pytest.raises(RuntimeError, match='aux must have'):
      G.gemm(a, b, True, True, aux=wide[:, 64:64 + n - 8], aux_mode=mode,  # narrower view
             out=out)
  for ak in (True, False):
    for bk in (True, False):
      a0 = torch.empty((m, 0) if ak else (0, m), device='cuda', dtype=torch.bfloat16)
      b0 = torch.empty((n, 0) if bk else (0, n), device='cuda', dtype=torch.bfloat16)
      with pytest.raises(RuntimeError, match='K = 0'):
        G.gemm(a0, b0, ak, bk)
  assert nat.launch_count() == launches


# ----------------------------------------------------------------- the bound on CPU ----
def _Truncate(v):
  """fp32 → bf16 by dropping the low 16 bits."""
  return (v.float().view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)


@pytest.mark.parametrize('ng,m,n,k', [(1, 256, 264, 136), (2, 129, 136, 72), (3, 128, 72, 200)])
def test_bound_and_controls_on_cpu(ng, m, n, k):
  """The bound, the controls and the rounding check with `gemm_ref` rounded to bf16 in the
  kernel's place. The three sub-ulp defects of the module docstring fail the rounding check,
  or the bound itself where the bias cancels S."""
  gen = torch.Generator().manual_seed(ng * 1000 + k)
  for ak, bk in _MAJORS:
    for epi in _EPIS:
      a, b, kw = _Inputs(gen, ng, m, n, k, ak, bk, epi, True)
      y = G.gemm_ref(a, b, ak, bk, **kw)
      _Check(y, a, b, ak, bk, bias=kw['bias'], act=kw.get('act', 0), aux=kw.get('aux'),
             aux_mode=kw.get('aux_mode', 0), rs=kw['row_scale'], controls=True,
             what='gemm_ref')
  a, b, kw = _Inputs(gen, ng, m, n, k, True, False, None, True)
  bias = kw['bias']
  args = dict(bias=bias, rs=kw['row_scale'])
  v = G.gemm_ref(a, b, True, False, bias=bias, row_scale=kw['row_scale'], out_fp32=True)
  defects = {
      'truncated pack': _Truncate(v),
      'bias read as bf16': G.gemm_ref(a, b, True, False, bias=bias.bfloat16().float(),
                                      row_scale=kw['row_scale']),
      'rounded before the bias add': (
          (G.gemm_ref(a, b, True, False).float() + bias.reshape(ng, 1, n)) *
          kw['row_scale'].reshape(ng, m, 1)).bfloat16(),
  }
  for name, y in defects.items():
    with pytest.raises(AssertionError, match='outside the bound|not rounded to nearest'):
      _Check(y, a, b, True, False, what=name, **args)
