"""wgmma GEMM numerics vs a plain PyTorch fp32 reference."""
import pytest
import torch

from lingvo_b200 import ops
from lingvo_b200.ops import gemm as G

pytestmark = pytest.mark.gpu


def _mk(shape, scale=1.0, seed=0):
  g = torch.Generator(device='cuda').manual_seed(seed)
  return (torch.randn(shape, device='cuda', generator=g) * scale).to(torch.bfloat16)


def _check(y, ref, k):
  y, ref = y.float(), ref.float()
  tol = 2e-2 * (k ** 0.5) / 8 + 1e-2
  err = (y - ref).abs().max().item()
  den = ref.abs().max().item() + 1e-6
  assert err / den < 2e-2, (err, den, tol)


@pytest.mark.parametrize('ak,bk', [(True, True), (True, False), (False, True), (False, False)])
@pytest.mark.parametrize('m,n,k', [(128, 256, 64), (256, 512, 256), (384, 128, 192),
                                   (200, 328, 136), (1024, 2048, 1024)])
def test_layouts(ak, bk, m, n, k):
  a = _mk((m, k) if ak else (k, m), seed=1)
  b = _mk((n, k) if bk else (k, n), seed=2)
  y = G.gemm(a, b, ak, bk)
  _check(y, G.gemm_ref(a, b, ak, bk, out_fp32=True), k)


def test_grouped_and_bf16_epilogues():
  g, m, n, k = 8, 320, 512, 256
  a = _mk((g, m, k), seed=3)
  b = _mk((g, k, n), seed=4)
  bias = torch.randn(g, n, device='cuda')
  y = G.gemm(a, b, True, False, bias=bias, act='RELU')
  _check(y, G.gemm_ref(a, b, True, False, bias=bias, act=1, out_fp32=True), k)
  aux = _mk((g, m, n), seed=5)
  y = G.gemm(a, b, True, False, aux=aux, aux_mode=G.AUX_RELU_MASK)
  _check(y, G.gemm_ref(a, b, True, False, aux=aux, aux_mode=1, out_fp32=True), k)
  rs = torch.rand(g, m, device='cuda')
  y = G.gemm(a, b, True, False, row_scale=rs)
  assert y.dtype == torch.bfloat16
  _check(y, G.gemm_ref(a, b, True, False, row_scale=rs, out_fp32=True), k)


def test_unsupported_epilogues_are_rejected_without_launching():
  """Only NONE / RELU are fused, ReLU takes no aux operand, and the kernel reads the
  row-pointer table, so a host table is refused. The oracle refuses the same activations."""
  m, n, k = 256, 256, 128
  a = _mk((m, k), seed=9)
  b = _mk((k, n), seed=10)
  aux = _mk((m, n), seed=11)
  out = torch.empty(m, n, device='cuda', dtype=torch.bfloat16)
  host_ptrs = out.data_ptr() + torch.arange(m, dtype=torch.int64) * (n * 2)
  nat = ops.native()
  launches = nat.launch_count()
  with pytest.raises(KeyError):
    G.gemm(a, b, True, False, act='GELU')
  with pytest.raises(RuntimeError, match='act'):
    G.gemm(a, b, True, False, act=2)
  for mode in (G.AUX_ADD, G.AUX_RELU_MASK):
    with pytest.raises(RuntimeError, match='ReLU'):
      G.gemm(a, b, True, False, act=1, aux=aux, aux_mode=mode)
  with pytest.raises(RuntimeError, match='row_ptrs'):
    G.gemm(a, b, True, False, out=out, row_ptrs=host_ptrs)
  assert nat.launch_count() == launches
  ac, bc = a.cpu(), b.cpu()
  with pytest.raises(KeyError):
    G.gemm(ac, bc, True, False, act='GELU')
  with pytest.raises(KeyError):
    G.gemm_ref(ac, bc, True, False, act='GELU')
  with pytest.raises(ValueError):
    G.gemm_ref(ac, bc, True, False, act=2)


def test_linear_autograd():
  m, k, n = 512, 256, 384
  x = _mk((m, k), seed=6).requires_grad_()
  w = _mk((k, n), 0.05, seed=7).requires_grad_()
  b = torch.zeros(n, device='cuda', requires_grad=True)
  y = G.linear(x, w, b, act='RELU')
  dy = _mk((m, n), seed=8)
  y.backward(dy)
  xr = x.detach().float().requires_grad_()
  wr = w.detach().float().requires_grad_()
  br = b.detach().clone().requires_grad_()
  yr = torch.relu(xr @ wr + br)
  yr.backward(dy.float())
  _check(y, yr, k)
  _check(x.grad, xr.grad, n)
  _check(w.grad, wr.grad, m)
  _check(b.grad, br.grad, m)


def test_linear_and_ffn_residual_epilogue():
  """x + f(x) fused into the last GEMM's epilogue matches the unfused computation."""
  from lingvo_b200.ops import gemm as G
  torch.manual_seed(0)
  dev = torch.device('cuda')
  bf = torch.bfloat16
  x = torch.randn(512, 256, device=dev, dtype=bf, requires_grad=True)
  r = torch.randn(512, 128, device=dev, dtype=bf, requires_grad=True)
  w = (torch.randn(256, 128, device=dev) * 0.05).to(bf).requires_grad_()
  y = G.linear(x, w, residual=r)
  dy = torch.randn_like(y)
  y.backward(dy)
  ref = (x.float() @ w.float() + r.float())
  assert float((y.float() - ref).norm() / ref.norm()) < 1e-2
  assert float((r.grad.float() - dy.float()).abs().max()) == 0
  wi = (torch.randn(256, 512, device=dev) * 0.05).to(bf).requires_grad_()
  wo = (torch.randn(512, 256, device=dev) * 0.05).to(bf).requires_grad_()
  x2 = x.detach().clone().requires_grad_()
  y2 = G.ffn_relu(x2, wi, wo, residual=x2)
  ref2 = torch.relu(x2.float() @ wi.float()) @ wo.float() + x2.float()
  assert float((y2.float() - ref2.detach()).norm() / ref2.norm()) < 1e-2
  dy2 = torch.randn_like(y2)
  y2.backward(dy2)
  xr = x2.detach().float().requires_grad_()
  (torch.relu(xr @ wi.float()) @ wo.float() + xr).backward(dy2.float())
  assert float((x2.grad.float() - xr.grad).norm() / xr.grad.norm()) < 2e-2
