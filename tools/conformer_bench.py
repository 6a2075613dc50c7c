"""Conformer ASR encoder step (BASELINE config #4) on one GPU: device-timed train step of
`asr.librispeech.Librispeech960ConformerWpm`'s encoder on a synthetic static-shape batch,
plus the time of the fused LConv kernel path vs the plain-PyTorch composition.
Writes gpurun_out/conformer_bench.json."""
import json
import os
import sys
from unittest import mock

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from lingvo_b200.core.nested_map import NestedMap


def Time(fn, iters=10):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters


def main():
  dev = torch.device('cuda', 0)
  from lingvo_b200 import model_registry
  from lingvo_b200 import ops
  import lingvo_b200.models.asr.params.librispeech  # noqa: F401
  cfg = model_registry.GetParams('asr.librispeech.Librispeech960ConformerWpm', 'Train')
  ep = cfg.task.encoder
  ep.use_specaugment = False
  ep.dropout_prob = 0.0
  enc = ep.Instantiate()
  enc.to(dev)
  b, t = int(os.environ.get('LB_BATCH', '32')), 1600          # 16 s of 10 ms frames
  x = torch.randn(b, t, 80, 1, device=dev)
  pad = torch.zeros(b, t, device=dev)
  batch = NestedMap(src_inputs=x, paddings=pad)
  params = [v for v in enc.vars.Flatten() if v.requires_grad]
  nat = ops.native()

  def step():
    out = enc.FPropDefaultTheta(batch)
    loss = out.encoded.float().square().mean()
    grads = torch.autograd.grad(loss, params, allow_unused=True)
    return grads

  l0 = nat.launch_count()
  ms = Time(step)
  launches = (nat.launch_count() - l0) / 13
  frames = b * t
  out = {'model': 'asr.librispeech.Librispeech960ConformerWpm (encoder fwd+bwd)',
         'batch': b, 'frames_per_utt': t, 'ms_per_step': ms,
         'frames_per_s': frames / (ms / 1e3), 'own_kernel_launches_per_step': launches,
         'encoder_params_m': sum(p.numel() for p in params) / 1e6}
  # LConv module alone: fused kernel path vs PyTorch composition
  from lingvo_b200.core import conformer_layer
  lp = conformer_layer.LConvLayer.CommonParams(input_dim=512, kernel_size=32)
  lp.name = 'lconv'
  lp.fprop_dtype = torch.bfloat16
  lc = lp.Instantiate()
  lc.to(dev)
  h = torch.randn(b, t // 4, 512, device=dev, dtype=torch.bfloat16, requires_grad=True)
  hp = torch.zeros(b, t // 4, device=dev)

  def lconv():
    y, _ = lc.FPropDefaultTheta(h, hp)
    torch.autograd.grad(y.float().sum(), [h] + [v for v in lc.vars.Flatten() if v.requires_grad],
                        allow_unused=True)
  out['lconv_fused_ms'] = Time(lconv)
  from lingvo_b200.ops import conv as conv_ops
  with mock.patch.object(conv_ops, 'glu_dwconv1d_supported', lambda *a: False):
    out['lconv_unfused_ms'] = Time(lconv)
  os.makedirs('gpurun_out', exist_ok=True)
  json.dump(out, open('gpurun_out/conformer_bench.json', 'w'), indent=1)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
