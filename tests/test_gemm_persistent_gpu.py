"""Persistent wgmma GEMM: tile scheduling, every epilogue, and run-to-run determinism."""
import pytest
import torch

from lingvo_b200.ops import gemm as G

pytestmark = pytest.mark.gpu


def _mk(shape, scale=1.0, seed=0):
  g = torch.Generator(device='cuda').manual_seed(seed)
  return (torch.randn(shape, device='cuda', generator=g) * scale).to(torch.bfloat16)


def _operands(g, m, n, k, ak, bk, seed=0):
  a = _mk((g, m, k) if ak else (g, k, m), seed=seed)
  b = _mk((g, n, k) if bk else (g, k, n), seed=seed + 1)
  return a, b


def _close(y, ref):
  y, ref = y.float(), ref.float()
  err = (y - ref).abs().max().item()
  den = ref.abs().max().item() + 1e-6
  assert err / den < 2e-2, (err, den)


# On a 132-SM H100: 1600 tiles of 128 x 256 (many per CTA); 133 tiles of 128 x 256, for
# which 266 tiles of 128 x 128 are chosen; 72 ragged tiles with a ragged K; and G = 8
# groups of 33 tiles, so each CTA's second tile lies in another group.
_SHAPES = [(1, 4096, 12800, 256), (1, 2432, 1792, 192), (1, 904, 2184, 200), (8, 328, 2808, 136)]
_G, _M, _N, _K = _SHAPES[-1]


@pytest.mark.parametrize('ak,bk', [(True, True), (True, False), (False, True), (False, False)])
@pytest.mark.parametrize('g,m,n,k', _SHAPES)
def test_layouts_and_schedules(g, m, n, k, ak, bk):
  a, b = _operands(g, m, n, k, ak, bk)
  _close(G.gemm(a, b, ak, bk), G.gemm_ref(a, b, ak, bk, out_fp32=True))


@pytest.mark.parametrize('ak,bk', [(True, True), (True, False), (False, True), (False, False)])
@pytest.mark.parametrize('act', [0, 1])
def test_bias_and_activations(act, ak, bk):
  g, m, n, k = _G, _M, _N, _K
  a, b = _operands(g, m, n, k, ak, bk, seed=3)
  bias = torch.randn(g, n, device='cuda')
  y = G.gemm(a, b, ak, bk, bias=bias, act=act)
  _close(y, G.gemm_ref(a, b, ak, bk, bias=bias, act=act, out_fp32=True))


def test_aux_and_row_scale():
  g, m, n, k = _G, _M, _N, _K
  a, b = _operands(g, m, n, k, True, True, seed=5)
  aux = _mk((g, m, n), seed=7)
  for mode in (G.AUX_RELU_MASK, G.AUX_ADD):
    y = G.gemm(a, b, True, True, aux=aux, aux_mode=mode)
    _close(y, G.gemm_ref(a, b, True, True, aux=aux, aux_mode=mode, out_fp32=True))
  rs = torch.rand(g, m, device='cuda')
  a2, b2 = _operands(g, m, n, k, False, False, seed=9)
  y = G.gemm(a2, b2, False, False, row_scale=rs)
  _close(y, G.gemm_ref(a2, b2, False, False, row_scale=rs, out_fp32=True))


def test_row_ptrs_with_null_rows():
  g, m, n, k = _G, _M, _N, _K
  a, b = _operands(g, m, n, k, True, False, seed=11)
  dst = torch.zeros(g * m, n, device='cuda', dtype=torch.bfloat16)
  perm = torch.randperm(g * m, device='cuda')
  ptrs = dst.data_ptr() + perm * (n * 2)
  keep = torch.arange(g * m, device='cuda') % 5 != 3
  ptrs = torch.where(keep, ptrs, torch.zeros_like(ptrs)).to(torch.int64)
  G.gemm(a, b, True, False, act=1, row_ptrs=ptrs)
  ref = G.gemm_ref(a, b, True, False, act=1, out_fp32=True).reshape(g * m, n)
  expect = torch.zeros(g * m, n, device='cuda')
  expect[perm[keep]] = ref[keep]
  _close(dst, expect)
  # null rows are skipped: their destination rows stay untouched
  assert not dst[perm[~keep]].any()


def test_repeat_and_graph_bitwise():
  g, m, n, k = 1, 2432, 1792, 512
  a, b = _operands(g, m, n, k, False, True, seed=13)
  aux = _mk((g, m, n), seed=14)
  y0 = G.gemm(a, b, False, True, aux=aux, aux_mode=G.AUX_ADD)
  y1 = G.gemm(a, b, False, True, aux=aux, aux_mode=G.AUX_ADD)
  assert torch.equal(y0, y1)
  out = torch.empty_like(y0)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    G.gemm(a, b, False, True, aux=aux, aux_mode=G.AUX_ADD, out=out)
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    G.gemm(a, b, False, True, aux=aux, aux_mode=G.AUX_ADD, out=out)
  out.zero_()
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(out, y0)
