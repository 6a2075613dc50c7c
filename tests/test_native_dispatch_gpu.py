"""Every dispatcher refuses CUDA inputs when the native extension is missing.

`ops.use_cuda_kernels` is the one gate between a fused kernel and its reference: for CUDA
tensors it raises when `_C.so` did not load. Each case below simulates a failed load and calls
one dispatcher on bf16 CUDA inputs of a shape its kernel serves. It must raise rather than run
the fp32 reference or the eager optimizer on the GPU, and nothing of ours may launch.
"""

import pytest
import torch

from lingvo_b200 import ops
from lingvo_b200.core import optimizer
from lingvo_b200.core import py_utils
from lingvo_b200.ops import attention
from lingvo_b200.ops import beam_search
from lingvo_b200.ops import gate

pytestmark = pytest.mark.gpu


def _Bf16(*shape):
  return torch.randn(*shape, device='cuda').bfloat16()


def _FlashAttention():
  q = _Bf16(1, 128, 2, 128)
  attention.flash_attention(q, q.clone(), q.clone())


def _DecodeAttention():
  q = _Bf16(1, 1, 2, 128)
  cache = _Bf16(1, 64, 2, 128)
  attention.decode_attention(q, q.clone(), q.clone(), cache, cache.clone(), 0)


def _FlatBeamAttention():
  q = _Bf16(1, 2, 2, 128)
  cache = _Bf16(1, 64, 2, 128)
  vis = torch.full((1, 2, 2), -1, dtype=torch.int32, device='cuda')
  qpos = torch.zeros(1, 2, dtype=torch.int32, device='cuda')
  kpos = torch.arange(64, dtype=torch.int32, device='cuda').unsqueeze(0)
  attention.flat_beam_attention(q, q.clone(), q.clone(), cache, cache.clone(), 0, vis, qpos,
                                kpos)


def _BeamSearchStep():
  num_beams, k, vocab = 2, 4, 64
  state = beam_search.init_state(num_beams, k, 4, 1, 'cuda')
  log_probs = torch.log_softmax(torch.randn(num_beams * k, vocab, device='cuda'), -1)
  beam_search.beam_search_step(log_probs.bfloat16(), None, state, 0, eos_id=2, beam_size=3.0,
                               num_hyps_per_beam=k)


def _GateSupported():
  gate.supported(_Bf16(2, 64, 256), torch.randn(256, 8, device='cuda'))


def _OptimizerStep(params):
  w = torch.nn.Parameter(torch.randn(256, 256, device='cuda'))
  w.var_name = 'w/var'
  opt = params.Set(name='opt').Instantiate()
  opt.Apply(0.1, [py_utils.VarGrad(w, torch.randn_like(w))])


def _AdafactorStep():
  _OptimizerStep(optimizer.XLAShardingAdafactor.Params())


def _AdamStep():
  _OptimizerStep(optimizer.Adam.Params())


@pytest.mark.parametrize('dispatch', [
    _FlashAttention, _DecodeAttention, _FlatBeamAttention, _BeamSearchStep, _GateSupported,
    _AdafactorStep, _AdamStep
], ids=lambda f: f.__name__.lstrip('_'))
def test_missing_extension_is_an_error(dispatch, monkeypatch):
  nat = ops.native()
  before = nat.launch_count()
  monkeypatch.setattr(ops, '_MOD', None)
  monkeypatch.setattr(ops, '_ERR', ImportError('simulated'))
  with pytest.raises(RuntimeError, match='native extension is not available'):
    dispatch()
  assert nat.launch_count() == before
