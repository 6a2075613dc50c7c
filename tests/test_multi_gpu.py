"""Multi-GPU checks (need ≥ 2 GPUs; launched under torchrun on one node)."""

import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _Run(script, nproc, port, *args):
  cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node',
         str(nproc), '--master-addr', '127.0.0.1', '--master-port', str(port),
         os.path.join(ROOT, script), *args]
  env = dict(os.environ, PYTHONPATH=ROOT)
  r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
  return r.returncode, r.stdout + r.stderr


def _NeedGpus(n):
  if torch.cuda.device_count() < n:
    pytest.skip('needs %d GPUs' % n)


def test_fused_ep_dp_matches_nccl_baseline():
  """Fused peer-memory MoE exchange + all-reduce give the same losses as NCCL mode."""
  _NeedGpus(2)
  rc, out = _Run('tools/mgpu_check.py', 2, 29621)
  assert rc == 0 and 'MGPU_OK' in out, out[-3000:]


def test_product_trainer_two_gpus_identical_replicas_resume_and_gradients():
  """`runners.Trainer` under torchrun: replicated weights identical across ranks after 10
  steps, sharded checkpoint + resume, and per-variable gradients fused ≈ NCCL baseline."""
  _NeedGpus(2)
  rc, out = _Run('tools/trainer_mgpu_check.py', 2, 29623)
  assert rc == 0 and 'TRAINER_MGPU_OK' in out, out[-4000:]


def test_tensor_parallel_model_matches_single_gpu():
  """DenseBuilder UniTransformer with heads / FFN hidden sharded over 2 GPUs (NCCL f/g +
  local wgmma GEMMs): loss, gathered gradients and 8 Adam steps ≈ the unsharded model."""
  _NeedGpus(2)
  rc, out = _Run('tools/tp_model_check.py', 2, 29624)
  assert rc == 0 and 'TP_MODEL_OK' in out, out[-4000:]
