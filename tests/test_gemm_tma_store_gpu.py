"""TMA-store epilogue of the wgmma GEMM: bitwise equal to the general (row-pointer) epilogue.

A plain bf16 output leaves through TMA bulk stores; redirected rows route the same GEMM
through the general st.global epilogue, whose per-element arithmetic is the same. So the
two must agree bit for bit, for every fused epilogue, ragged edge, group layout and output
stride.
"""
import pytest
import torch

from lingvo_b200.ops import gemm as G

pytestmark = pytest.mark.gpu


def _mk(shape, seed):
  g = torch.Generator(device='cuda').manual_seed(seed)
  return torch.randn(shape, device='cuda', generator=g).to(torch.bfloat16)


def _operands(g, m, n, k, ak, bk, seed=0):
  a = _mk((g, m, k) if ak else (g, k, m), seed)
  b = _mk((g, n, k) if bk else (g, k, n), seed + 1)
  return a, b


def _general(a, b, ak, bk, **kw):
  """Same GEMM through the general epilogue, forced by an identity row-pointer table."""
  g, m = (a.shape[0], a.shape[1] if ak else a.shape[2])
  n = b.shape[1] if bk else b.shape[2]
  out = torch.empty(g, m, n, device='cuda', dtype=torch.bfloat16)
  rows = torch.arange(g * m, device='cuda', dtype=torch.int64)
  G.gemm(a, b, ak, bk, row_ptrs=out.data_ptr() + rows * (n * 2), **kw)
  return out


# (G, M, N, K) on a 132-SM H100: an odd number of M-tiles with ragged M and N (776 =
# 6 * 128 + 8 rows, so the last tile's second warpgroup has no rows; 840 columns in 128-wide
# tiles); ragged M inside groups (200 rows per group, 3 groups); K = 2048 with 128-wide
# tiles and the benchmark's K = 2048 and K = 8192 with 256-wide tiles; a ragged K with a
# partial last 64-column slice.
_SHAPES = [(1, 776, 840, 256), (3, 200, 640, 256), (1, 1024, 2048, 2048), (1, 2048, 2048, 2048),
           (1, 2048, 2048, 8192), (2, 328, 2808, 136)]

_EPILOGUES = {
    'plain': {},
    'relu': dict(act=1),
    'bias_relu': dict(act=1, bias=True),
    'residual': dict(aux_mode=G.AUX_ADD),
    'relu_mask': dict(aux_mode=G.AUX_RELU_MASK),
    'row_scale': dict(row_scale=True),
    'bias_residual_row_scale': dict(aux_mode=G.AUX_ADD, bias=True, row_scale=True),
    'bias_relu_mask_row_scale': dict(aux_mode=G.AUX_RELU_MASK, bias=True, row_scale=True),
}


def _kwargs(spec, g, m, n, seed):
  kw = dict(spec)
  if kw.pop('bias', False):
    kw['bias'] = torch.randn(g, n, device='cuda')
  if kw.pop('row_scale', False):
    kw['row_scale'] = torch.rand(g, m, device='cuda')
  if kw.get('aux_mode'):
    kw['aux'] = _mk((g, m, n), seed)
  return kw


@pytest.mark.parametrize('epi', list(_EPILOGUES))
@pytest.mark.parametrize('g,m,n,k', _SHAPES)
def test_tma_store_matches_row_pointer_epilogue(g, m, n, k, epi):
  ak, bk = (True, True) if epi in ('relu_mask', 'plain') else (True, False)
  a, b = _operands(g, m, n, k, ak, bk, seed=21)
  kw = _kwargs(_EPILOGUES[epi], g, m, n, seed=23)
  y = G.gemm(a, b, ak, bk, **kw)
  assert torch.equal(y, _general(a, b, ak, bk, **kw))
  ref = G.gemm_ref(a, b, ak, bk, out_fp32=True, **kw)
  err = (y.float() - ref).abs().max().item()
  assert err / (ref.abs().max().item() + 1e-6) < 2e-2


def test_wgrad_majors_match_row_pointer_epilogue():
  a, b = _operands(4, 904, 1024, 512, False, False, seed=31)
  rs = torch.rand(4, 904, device='cuda')
  y = G.gemm(a, b, False, False, row_scale=rs)
  assert torch.equal(y, _general(a, b, False, False, row_scale=rs))


def test_row_strided_output_view():
  g, m, n, k = 2, 328, 840, 320
  a, b = _operands(g, m, n, k, True, False, seed=41)
  aux = _mk((g, m, n + 72), 43)[:, :, :n]
  big = torch.full((g, m, n + 72), 7.0, device='cuda', dtype=torch.bfloat16)
  out = big[:, :, :n]
  assert out.stride(1) > n
  G.gemm(a, b, True, False, aux=aux, aux_mode=G.AUX_ADD, out=out)
  dense = G.gemm(a, b, True, False, aux=aux.contiguous(), aux_mode=G.AUX_ADD)
  assert torch.equal(out, dense)
  assert bool((big[:, :, n:] == 7.0).all())   # the padding columns are not written


@pytest.mark.parametrize('mode', [G.AUX_ADD, G.AUX_RELU_MASK])
def test_repeat_and_graph_bitwise(mode):
  g, m, n, k = 1, 2432, 1792, 2048
  a, b = _operands(g, m, n, k, True, True, seed=51)
  aux = _mk((g, m, n), 53)
  y0 = G.gemm(a, b, True, True, aux=aux, aux_mode=mode)
  y1 = G.gemm(a, b, True, True, aux=aux, aux_mode=mode)
  assert torch.equal(y0, y1)
  out = torch.empty_like(y0)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    G.gemm(a, b, True, True, aux=aux, aux_mode=mode, out=out)
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    G.gemm(a, b, True, True, aux=aux, aux_mode=mode, out=out)
  out.zero_()
  graph.replay()
  torch.cuda.synchronize()
  assert torch.equal(out, y0)
