"""In-tree build of the native extension `lingvo_b200/ops/_C.so`.

`python -m lingvo_b200.ops.build` cross-compiles every `csrc/*.cu|*.cpp` for
sm_90a (`-gencode arch=compute_90a,code=sm_90a -lineinfo`) with nvcc / g++
and links against the installed libtorch. Object files are cached under
`csrc/_obj/` and rebuilt when the source (or any header) is newer. The `.so`
stays in-tree so it travels with the repo snapshot to GPU boxes.
"""

from __future__ import annotations

import concurrent.futures
import glob
import os
import shutil
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(CSRC, '_obj')
TARGET = os.path.join(HERE, '_C.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')

ARCH_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a']


def _TorchPaths():
  from torch.utils import cpp_extension
  inc = cpp_extension.include_paths(device_type='cuda') if 'device_type' in (
      cpp_extension.include_paths.__code__.co_varnames) else (
          cpp_extension.include_paths(cuda=True))
  lib = cpp_extension.library_paths(device_type='cuda') if 'device_type' in (
      cpp_extension.library_paths.__code__.co_varnames) else (
          cpp_extension.library_paths(cuda=True))
  return inc, lib


def _Newest(paths):
  return max(os.path.getmtime(p) for p in paths) if paths else 0.0


def _Compile(src, obj, inc, verbose):
  common = ['-O3', '-std=c++17', '-DTORCH_EXTENSION_NAME=_C',
            '-D_GLIBCXX_USE_CXX11_ABI=1', '-DTORCH_API_INCLUDE_EXTENSION_H']
  incs = [f'-I{p}' for p in inc] + [f'-I{sysconfig.get_paths()["include"]}',
                                    f'-I{CSRC}']
  if src.endswith('.cu'):
    cmd = [NVCC, *ARCH_FLAGS, '-lineinfo', '--expt-relaxed-constexpr',
           '--expt-extended-lambda', '-Xcompiler', '-fPIC', '-Xptxas', '-v',
           '-D__CUDA_NO_HALF_OPERATORS__', '-D__CUDA_NO_HALF_CONVERSIONS__',
           '-D__CUDA_NO_BFLOAT16_CONVERSIONS__', '-D__CUDA_NO_HALF2_OPERATORS__',
           *common, *incs, '-c', src, '-o', obj]
  else:
    cmd = ['g++', '-fPIC', '-fvisibility=hidden', *common, *incs,
           '-isystem', '/usr/local/cuda/include', '-c', src, '-o', obj]
  r = subprocess.run(cmd, capture_output=True, text=True)
  log = r.stdout + r.stderr
  with open(obj + '.log', 'w') as f:
    f.write(' '.join(cmd) + '\n' + log)
  if r.returncode != 0:
    raise RuntimeError('compile failed: %s\n%s' % (src, log[-6000:]))
  if verbose:
    print('[build] compiled', os.path.basename(src))
  return obj


def Build(force: bool = False, verbose: bool = True) -> str:
  os.makedirs(OBJ, exist_ok=True)
  srcs = sorted(glob.glob(os.path.join(CSRC, '*.cu')) +
                glob.glob(os.path.join(CSRC, '*.cpp')))
  headers = glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(
      os.path.join(CSRC, '*.h'))
  hdr_time = _Newest(headers + [os.path.abspath(__file__)])
  inc, lib = _TorchPaths()
  jobs = []
  objs = []
  for src in srcs:
    obj = os.path.join(OBJ, os.path.basename(src) + '.o')
    objs.append(obj)
    stale = force or not os.path.exists(obj) or os.path.getmtime(obj) < max(
        os.path.getmtime(src), hdr_time)
    if stale:
      jobs.append((src, obj))
  if jobs:
    workers = min(len(jobs), max(1, (os.cpu_count() or 2)))
    with concurrent.futures.ThreadPoolExecutor(workers) as ex:
      futs = [ex.submit(_Compile, s, o, inc, verbose) for s, o in jobs]
      for f in futs:
        f.result()
  if jobs or not os.path.exists(TARGET) or os.path.getmtime(TARGET) < _Newest(objs):
    libs = ['-lc10', '-ltorch', '-ltorch_cpu', '-ltorch_python', '-lc10_cuda',
            '-ltorch_cuda', '-lcudart']
    cmd = ['g++', '-shared', '-o', TARGET + '.tmp', *objs,
           *[f'-L{p}' for p in lib], *[f'-Wl,-rpath,{p}' for p in lib],
           '-L/usr/local/cuda/lib64', *libs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
      raise RuntimeError('link failed:\n' + r.stdout + r.stderr)
    os.replace(TARGET + '.tmp', TARGET)
    if verbose:
      print('[build] linked', TARGET)
  return TARGET


HOST_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc_host')
HOST_TARGET = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_H.so')


def BuildHost(force: bool = False, verbose: bool = True) -> str:
  """Builds the torch-free host library `_H.so` (records / batching / tokenizers /
  packing) with g++ + pybind11."""
  import pybind11  # pylint: disable=g-import-not-at-top
  srcs = sorted(glob.glob(os.path.join(HOST_SRC, '*.cpp')))
  deps = srcs + glob.glob(os.path.join(HOST_SRC, '*.h')) + [os.path.abspath(__file__)]
  if (not force and os.path.exists(HOST_TARGET) and
      os.path.getmtime(HOST_TARGET) >= _Newest(deps)):
    return HOST_TARGET
  os.makedirs(OBJ, exist_ok=True)
  incs = ['-I' + pybind11.get_include(), '-I' + sysconfig.get_paths()['include'],
          '-I' + HOST_SRC]

  def _One(src):
    obj = os.path.join(OBJ, 'host_' + os.path.basename(src) + '.o')
    cmd = ['g++', '-O2', '-std=c++17', '-fPIC', '-fvisibility=hidden', '-pthread',
           *incs, '-c', src, '-o', obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
      raise RuntimeError('compile failed: %s\n%s' % (src, (r.stdout + r.stderr)[-6000:]))
    if verbose:
      print('[build] compiled', os.path.basename(src))
    return obj

  with concurrent.futures.ThreadPoolExecutor(len(srcs)) as ex:
    objs = list(ex.map(_One, srcs))
  cmd = ['g++', '-shared', '-pthread', '-o', HOST_TARGET + '.tmp', *objs, '-lz']
  r = subprocess.run(cmd, capture_output=True, text=True)
  if r.returncode != 0:
    raise RuntimeError('link failed:\n' + r.stdout + r.stderr)
  os.replace(HOST_TARGET + '.tmp', HOST_TARGET)
  if verbose:
    print('[build] linked', HOST_TARGET)
  return HOST_TARGET


if __name__ == '__main__':
  Build(force='--force' in sys.argv)
  BuildHost(force='--force' in sys.argv)
