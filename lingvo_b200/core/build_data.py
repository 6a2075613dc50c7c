"""Build information (ref `lingvo/core/build_data.py`)."""
import platform

import torch

from lingvo_b200.core import hyperparams


def BuildData():
  """Params recording the toolchain this binary runs with."""
  p = hyperparams.Params()
  p.Define('torch_version', torch.__version__, 'PyTorch version.')
  p.Define('cuda_version', str(torch.version.cuda), 'CUDA runtime version.')
  p.Define('python_version', platform.python_version(), 'Python version.')
  p.Define('target_arch', 'sm_90a', 'GPU architecture the native kernels are built for.')
  return p
