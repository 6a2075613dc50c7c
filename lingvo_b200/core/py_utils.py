"""Framework utility belt on top of PyTorch.

Covers the "must-port" subset of reference `lingvo/core/py_utils.py`
(SURVEY §2.2): shape asserts (:388-575), `WeightInit` family (:1085-1232) and
initializer math (:2209-2313), `WeightParams` (:1250), `CreateVariable` with
name-hashed seeds (:1555, :1882-2085), global step (:2549-2688), gradient
helpers (:3084-3500), metric averaging (:3641-3689), variational noise
(:3738), step seeds + deterministic dropout (:3880-4064), padding helpers
(:4282-4696), Retry (:4696), remat (:5005), xent helpers (:5183-5299),
AuxLossContext (:6572), trainable-var filters (:6610), BlockDiagonalMatmul
(:6645), processed-checkpoint bookkeeping (:6759), Timer (:6890).

Design differences (H100/PyTorch-first): variables are `torch.nn.Parameter`s
created directly on the cluster's current device; gradients come from autograd
(`torch.autograd.grad`), initializers are a method-name → function table, and
thread-local *context stacks* are tiny `_Stack` objects.
"""

from __future__ import annotations

import contextlib
import functools
import hashlib
import logging
import math
import os
import random as _pyrandom
import re
import threading
import time
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from lingvo_b200.core import hyperparams
from lingvo_b200.core import py_utils_flags as flags
from lingvo_b200.core.nested_map import NestedMap

# Re-exported names (reference `py_utils` re-exports these).
NestedMap = NestedMap  # pylint: disable=self-assigning-variable
use_tpu = flags.use_tpu
use_gpu = flags.use_gpu

Params = hyperparams.Params
InstantiableParams = hyperparams.InstantiableParams


# ----------------------------------------------------------------------------
# Thread-local context stacks
# ----------------------------------------------------------------------------
class _Stack(threading.local):
  """A thread-local stack used for dynamic-scope configuration."""

  def __init__(self):
    super().__init__()
    self.items: List[Any] = []

  @contextlib.contextmanager
  def Push(self, item):
    self.items.append(item)
    try:
      yield item
    finally:
      self.items.pop()

  def Top(self, default=None):
    return self.items[-1] if self.items else default


# ----------------------------------------------------------------------------
# Shape / value assertions
# ----------------------------------------------------------------------------
def GetShape(tensor, ndims: Optional[int] = None) -> List[int]:
  shape = list(tensor.shape)
  return shape if ndims is None else shape[:ndims]


def GetRank(tensor) -> int:
  return tensor.dim()


def GetSize(tensor) -> int:
  return tensor.numel()


def HasRank(tensor, expected_rank: int):
  if flags.enable_asserts():
    assert tensor.dim() == expected_rank, (
        'Ranks did not match, got %d, expected %d' % (tensor.dim(),
                                                      expected_rank))
  return tensor


def HasAtLeastRank(tensor, expected_rank: int):
  if flags.enable_asserts():
    assert tensor.dim() >= expected_rank, (
        'Rank of tensor %d did not exceed the expected value %d.' %
        (tensor.dim(), expected_rank))
  return tensor


def HasShape(tensor, expected_shape: Sequence[int], ndims: Optional[int] = None):
  """Checks `tensor.shape[:ndims]` against `expected_shape`; -1 = wildcard."""
  if flags.enable_asserts():
    got = list(tensor.shape) if ndims is None else list(tensor.shape[:ndims])
    exp = list(expected_shape)
    if isinstance(expected_shape, torch.Tensor):
      exp = [int(x) for x in expected_shape.tolist()]
    assert len(got) == len(exp) and all(
        e == -1 or int(e) == g for g, e in zip(got, exp)), (
            'Tensor shape %s does not match expected %s' % (got, exp))
  return tensor


def assert_shape_match(lhs, rhs, msg=''):
  lhs, rhs = list(lhs), list(rhs)
  assert len(lhs) == len(rhs) and all(
      a == b or a == -1 or b == -1 for a, b in zip(lhs, rhs)), (
          'Shape mismatch %s vs %s %s' % (lhs, rhs, msg))


def assert_same_dim0(tensors, msg=''):
  d0 = {t.shape[0] for t in tensors}
  assert len(d0) <= 1, 'dim0 mismatch %s %s' % (sorted(d0), msg)


def assert_equal(a, b, msg=''):
  if flags.enable_asserts():
    ok = bool(torch.all(torch.as_tensor(a) == torch.as_tensor(b)))
    assert ok, 'assert_equal failed: %s vs %s %s' % (a, b, msg)


def assert_between(x, lo, hi, msg=''):
  if flags.enable_asserts():
    x = torch.as_tensor(x)
    assert bool(torch.all(x >= lo)) and bool(torch.all(x < hi)), msg


def assert_even_divide(denorm, num):
  assert num % denorm == 0, '%s does not evenly divide %s' % (denorm, num)
  return num // denorm


def CheckNumerics(inp, message=None):
  """Raises if `inp` holds NaN/Inf (only when enable_check_numerics)."""
  if not flags.enable_check_numerics():
    return inp
  def chk(t):
    if isinstance(t, torch.Tensor) and t.is_floating_point():
      if not bool(torch.isfinite(t).all()):
        raise FloatingPointError(message or 'CheckNumerics failed')
    return t
  if isinstance(inp, (list, tuple)):
    return type(inp)(chk(t) for t in inp)
  return chk(inp)


def Debug(tensor, message='', enabled=True, summarize=100):
  if enabled and flags.print_debug_tensors():
    logging.info('%s: %s', message, tensor.flatten()[:summarize])
  return tensor


# ----------------------------------------------------------------------------
# Devices
# ----------------------------------------------------------------------------
_DEVICE_STACK = _Stack()


def CurrentDevice() -> torch.device:
  top = _DEVICE_STACK.Top()
  if top is not None:
    return top
  if torch.cuda.is_available() and flags.use_gpu():
    return torch.device('cuda', torch.cuda.current_device())
  return torch.device('cpu')


def DeviceScope(device):
  return _DEVICE_STACK.Push(torch.device(device))


# ----------------------------------------------------------------------------
# Weight init
# ----------------------------------------------------------------------------
class WeightInit:
  """Factory of frozen init-spec Params {method, scale, seed, custom_v_init}."""

  @staticmethod
  def _Spec(method, scale, seed, custom_v_init=None):
    p = hyperparams.Params()
    p.Define('method', method, 'Initialization method.')
    p.Define('scale', scale, 'Initialization scale.')
    p.Define('seed', seed, 'Random seed used to generate initial values.')
    p.Define('custom_v_init', custom_v_init, 'Callable(shape, dtype, gen).')
    p.Freeze()
    return p


def _AddInitMethod(py_name: str, method: str, default_scale=1.0, seeded=True):
  if seeded:
    def make(scale=default_scale, seed=None):
      return WeightInit._Spec(method, scale, seed)
  else:
    def make(scale=default_scale):
      return WeightInit._Spec(method, scale, 0)
  make.__name__ = py_name
  make.__doc__ = 'WeightInit spec for method %r.' % method
  setattr(WeightInit, py_name, staticmethod(make))


for _py, _m in [
    ('Gaussian', 'gaussian'), ('Uniform', 'uniform'),
    ('UniformPositive', 'uniform_positive'), ('Xavier', 'xavier'),
    ('GeoMeanXavier', 'geo_mean_xavier'),
    ('TruncatedGaussian', 'truncated_gaussian'),
    ('GaussianSqrtDim', 'gaussian_sqrt_dim'),
    ('GaussianSqrtFanIn', 'gaussian_sqrt_fanin'),
    ('GaussianSqrtFanOut', 'gaussian_sqrt_fanout'),
    ('GaussianSqrtFanAvg', 'gaussian_sqrt_fanavg'),
    ('UniformSqrtDim', 'uniform_sqrt_dim'),
    ('UniformUnitScaling', 'uniform_unit_scaling'),
    ('UniformUnitScalingFanAvg', 'uniform_unit_scaling_fan_avg'),
    ('TruncatedGaussianSqrtDim', 'truncated_gaussian_sqrt_dim'),
    ('TruncatedGaussianSqrtFanIn', 'truncated_gaussian_sqrt_fanin'),
    ('TruncatedGaussianSqrtFanOut', 'truncated_gaussian_sqrt_fanout'),
    ('KaimingUniformFanInRelu', 'kaiming_uniform_fanin_relu'),
    ('ScaledDeltaOrthogonal', 'delta_orthogonal'),
]:
  _AddInitMethod(_py, _m)
_AddInitMethod('Category', 'category', default_scale=2)
_AddInitMethod('KaimingUniformFanInLeakyRelu',
               'kaiming_uniform_fanin_leakyrelu', default_scale=math.sqrt(5.))
_AddInitMethod('Constant', 'constant', seeded=False)


def _XavierWithFixup(scale=1.0, depth=1.0, layers_per_residual_block=1.0,
                     seed=None):
  scale = scale * math.pow(depth, -1.0 / (2 * layers_per_residual_block))
  return WeightInit._Spec('xavier', scale, seed)


WeightInit.XavierWithFixupParams = staticmethod(_XavierWithFixup)
WeightInit.CustomVarInit = staticmethod(
    lambda fn: WeightInit._Spec('custom', 1.0, None, fn))
WeightInit.CustomConstantVarInit = staticmethod(
    lambda fn: WeightInit._Spec('custom_constant', 1.0, None, fn))

_DEFAULT_XAVIER_SCALE = 1.000001


def DefaultParamInit():
  return WeightInit.Xavier(_DEFAULT_XAVIER_SCALE)


def IsDefaultParamInit(p) -> bool:
  return (p.method == 'xavier' and p.seed is None and
          abs(p.scale - _DEFAULT_XAVIER_SCALE) < 1e-7)


def WeightParams(shape, init=None, dtype=None, collections=None,
                 device_mesh=None, tensor_split_dims_mapping=None):
  """Spec of a variable to create (reference :1250)."""
  p = hyperparams.Params()
  p.Define('dtype', dtype if dtype is not None else torch.float32,
           'The weight data type.')
  p.Define('shape', list(shape), 'The weight shape.')
  p.Define('init', init if init is not None else DefaultParamInit(),
           'Initialization method.')
  p.Define('collections', collections,
           'Variable collections this weight belongs to.')
  p.Define('device_mesh', device_mesh,
           'np.ndarray of device ids describing the mesh topology.')
  p.Define('tensor_split_dims_mapping', tensor_split_dims_mapping,
           'Per-dim mesh axis (or -1) the weight is split on.')
  p.Define('init_shard', None,
           '(dim, index, count): `shape` is one of `count` equal shards along '
           '`dim` of the logical variable; init draws the *logical* tensor '
           '(so values match the unsharded model) and keeps shard `index`.')
  return p


# Stacked ("combined") layers put leading dims on every variable; fan-in/out
# computations must skip them (reference :1631-1690).
_VAR_SHAPE_PREFIX = _Stack()
_SKIP_LP_COLLECTION = '__lingvo_skip_lp_regularization'


def VariableShapePrefixContext(shape_prefix: int):
  assert shape_prefix > 0
  return _VAR_SHAPE_PREFIX.Push(int(shape_prefix))


def GetVariableShapePrefixes() -> List[int]:
  return list(_VAR_SHAPE_PREFIX.items)


def GetFanInFanOut(shape, prefix_dims_to_skip=0):
  if not shape:
    return None, None
  shape = list(shape)[prefix_dims_to_skip:]
  if len(shape) < 1:
    return 1, 1
  if len(shape) == 1:
    return shape[0], shape[0]
  receptive = 1
  for s in shape[:-2]:
    receptive *= s
  return shape[-2] * receptive, shape[-1] * receptive


def GenerateSeedFromName(name: str) -> int:
  """md5(name) mod (2^31 - 1) (reference :1555-1566)."""
  md5 = hashlib.md5(name.encode('utf-8'))
  return int(int(md5.hexdigest(), 16) % (2**31 - 1))


def _TruncNormal(shape, gen, std=1.0):
  out = torch.empty(shape, dtype=torch.float32)
  torch.nn.init.trunc_normal_(out, mean=0.0, std=1.0, a=-2.0, b=2.0,
                              generator=gen)
  return out * std


def _DeltaOrthogonal(shape, gen, scale):
  # Orthogonal matrix placed at the spatial centre of a conv kernel.
  if len(shape) < 3:
    raise ValueError('delta_orthogonal needs a conv kernel shape')
  cin, cout = shape[-2], shape[-1]
  a = torch.randn((max(cin, cout), max(cin, cout)), generator=gen)
  q, r = torch.linalg.qr(a)
  q = q * torch.sign(torch.diagonal(r))
  w = torch.zeros(shape, dtype=torch.float32)
  centre = tuple(s // 2 for s in shape[:-2])
  w[centre] = q[:cin, :cout] * scale
  return w


def InitialValue(shape, init, dtype=torch.float32, seed: Optional[int] = None,
                 prefix_dims: int = 0) -> torch.Tensor:
  """Evaluates an init spec to a CPU tensor (reference :2209-2313)."""
  method, scale = init.method, init.scale
  shape = [int(s) for s in shape]
  gen = torch.Generator(device='cpu')
  gen.manual_seed(int(seed) if seed is not None else
                  _pyrandom.randrange(2**31 - 1))
  dim0 = shape[prefix_dims] if len(shape) > prefix_dims else 1
  fan_in, fan_out = GetFanInFanOut(shape, prefix_dims)
  fan_in = fan_in or 1
  fan_out = fan_out or 1

  def unif(lo, hi):
    return torch.rand(shape, generator=gen) * (hi - lo) + lo

  def normal(std):
    return torch.randn(shape, generator=gen) * std

  if method == 'custom':
    v = init.custom_v_init(shape, dtype, gen)
  elif method == 'custom_constant':
    v = torch.as_tensor(init.custom_v_init).reshape(shape)
  elif method == 'constant':
    if isinstance(scale, (list, tuple, np.ndarray, torch.Tensor)):
      v = torch.as_tensor(np.asarray(scale, dtype=np.float64)).reshape(shape)
    else:
      v = torch.full(shape, float(scale) if not isinstance(scale, bool)
                     else float(scale))
  elif method == 'gaussian':
    v = normal(scale)
  elif method == 'uniform':
    v = unif(-scale, scale)
  elif method == 'uniform_positive':
    v = unif(0.0, scale)
  elif method == 'category':
    v = torch.floor(unif(0.0, scale))
  elif method == 'xavier':
    lim = scale * math.sqrt(6.0 / (fan_in + fan_out))
    v = unif(-lim, lim)
  elif method == 'geo_mean_xavier':
    lim = scale * math.sqrt(3.0 / math.sqrt(fan_in * fan_out))
    v = unif(-lim, lim)
  elif method == 'truncated_gaussian':
    v = _TruncNormal(shape, gen, scale)
  elif method == 'gaussian_sqrt_dim':
    v = normal(scale / math.sqrt(dim0))
  elif method == 'gaussian_sqrt_fanin':
    v = normal(scale / math.sqrt(fan_in))
  elif method == 'gaussian_sqrt_fanout':
    v = normal(scale / math.sqrt(fan_out))
  elif method == 'gaussian_sqrt_fanavg':
    v = normal(scale * math.sqrt(2.0 / (fan_in + fan_out)))
  elif method == 'uniform_sqrt_dim':
    lim = scale / math.sqrt(dim0)
    v = unif(-lim, lim)
  elif method == 'uniform_unit_scaling':
    lim = scale * math.sqrt(3.0) / math.sqrt(dim0)
    v = unif(-lim, lim)
  elif method == 'uniform_unit_scaling_fan_avg':
    lim = math.sqrt(3.0 * scale / max(1.0, (fan_in + fan_out) / 2.0))
    v = unif(-lim, lim)
  elif method == 'truncated_gaussian_sqrt_dim':
    v = _TruncNormal(shape, gen, scale / math.sqrt(dim0))
  elif method == 'truncated_gaussian_sqrt_fanin':
    v = _TruncNormal(shape, gen, scale / math.sqrt(fan_in))
  elif method == 'truncated_gaussian_sqrt_fanout':
    v = _TruncNormal(shape, gen, scale / math.sqrt(fan_out))
  elif method == 'kaiming_uniform_fanin_relu':
    lim = scale * math.sqrt(6.0 / fan_in)
    v = unif(-lim, lim)
  elif method == 'kaiming_uniform_fanin_leakyrelu':
    lim = math.sqrt(6.0 / ((1 + scale**2) * fan_in))
    v = unif(-lim, lim)
  elif method == 'delta_orthogonal':
    v = _DeltaOrthogonal(shape, gen, scale)
  else:
    raise ValueError('init_type %s not supported.' % method)
  if dtype.is_floating_point or dtype.is_complex:
    return v.to(dtype)
  return v.to(torch.float32).to(dtype)


# Variable-name scope (maps layer nesting to checkpoint keys).
_VAR_SCOPE = _Stack()
_VAR_DTYPE_OVERRIDES = _Stack()   # list of (regex, dtype)
_VAR_RENAME_RULES = _Stack()      # list of (regex, fmt)
_STUB_VARIABLES = _Stack()        # truthy → create meta/zeros vars (models_test)
_ALL_VARS: 'Dict[str, torch.nn.Parameter]' = {}


@contextlib.contextmanager
def VariableScope(names: Sequence[str]):
  """Pushes scope components (a list so layers may push 0, 1 or many)."""
  with _VAR_SCOPE.Push(list(names)):
    yield


def CurrentVariableScope() -> str:
  parts: List[str] = []
  for names in _VAR_SCOPE.items:
    parts.extend(n for n in names if n)
  return '/'.join(parts)


def VariableListDtypeRegexScope(regex_dtype_list):
  return _VAR_DTYPE_OVERRIDES.Push(list(regex_dtype_list))


def VariableRenameScope(renames):
  return _VAR_RENAME_RULES.Push(list(renames))


def StubVariablesScope(mode: str = 'zeros'):
  """`zeros` → vars are 0-strided expanded zeros; `meta` → meta tensors."""
  return _STUB_VARIABLES.Push(mode)


def _RenamedVarName(name: str) -> str:
  for rules in _VAR_RENAME_RULES.items:
    for regex, fmt in rules:
      m = re.match(regex, name)
      if m:
        return fmt % m.groups()
  return name


def CreateVariable(name: str, params, trainable: bool = True,
                   default_seed: Optional[int] = None,
                   device: Optional[torch.device] = None):
  """Creates a `torch.nn.Parameter` according to WeightParams `params`.

  The checkpoint key is `<scope>/<name>/var` (SURVEY A.2). With a
  `default_seed` (layer `random_seed`) and no per-init seed the stream seed is
  `GenerateSeedFromName(key)` so init is reproducible across shardings.
  """
  p = params.Copy()
  shape = list(p.shape)
  prefixes = GetVariableShapePrefixes()
  full_shape = prefixes + shape
  scope = CurrentVariableScope()
  key = _RenamedVarName((scope + '/' if scope else '') + name) + '/var'
  dtype = p.dtype
  for rules in _VAR_DTYPE_OVERRIDES.items:
    for regex, dt in rules:
      if re.match(regex, key):
        dtype = dt
  seed = p.init.seed
  if p.init.method != 'constant' and seed is None and default_seed is not None:
    seed = GenerateSeedFromName(key)
  device = device or CurrentDevice()
  stub = _STUB_VARIABLES.Top()
  if stub == 'meta':
    value = torch.empty(full_shape, dtype=dtype, device='meta')
  elif stub == 'zeros':
    value = torch.zeros((), dtype=dtype).expand(full_shape)
  elif p.init_shard is not None:
    sdim, sidx, scount = p.init_shard
    sdim += len(prefixes)
    logical = list(full_shape)
    logical[sdim] *= scount
    value = InitialValue(logical, p.init, dtype, seed,
                         prefix_dims=len(prefixes)).narrow(
                             sdim, sidx * full_shape[sdim],
                             full_shape[sdim]).contiguous().to(device)
  else:
    value = InitialValue(full_shape, p.init, dtype, seed,
                         prefix_dims=len(prefixes)).to(device)
  var = torch.nn.Parameter(value, requires_grad=bool(trainable) and
                           (dtype.is_floating_point or dtype.is_complex))
  var.var_name = key
  var.collections = list(p.collections or [])
  var.device_mesh = p.device_mesh
  var.tensor_split_dims_mapping = p.tensor_split_dims_mapping
  var.trainable = bool(trainable)
  return var


def AttachComputeCopies(root_layer, dtype=torch.bfloat16) -> int:
  """Mixed precision: persistent low-precision *compute copies* of weights.

  Every trainable fp32 variable of a layer whose `fprop_dtype` is `dtype`
  gets `var.compute` (a leaf tensor in `dtype`) which `theta` returns instead
  of casting the master weight every step. Gradients are taken w.r.t. the
  copy (bf16), optimizers update the fp32 master and refresh the copy — the
  fused kernels (`ops/optim`) write it in the same pass as the update.
  """
  n = 0
  for _, layer in root_layer.Walk():
    if layer.fprop_dtype != dtype:
      continue
    for name, var in layer._private_vars.items():  # pylint: disable=protected-access
      if var.dtype == torch.float32 and var.requires_grad and (
          getattr(var, 'compute', None) is None):
        var.compute = var.data.to(dtype).requires_grad_(True)
        layer.SetThetaOverride(name, var.compute)
        n += 1
  return n


def RefreshComputeCopies(variables) -> None:
  with torch.no_grad():
    for v in variables:
      c = getattr(v, 'compute', None)
      if c is not None:
        c.data.copy_(v.data)


def SkipLpRegularization(var) -> bool:
  return _SKIP_LP_COLLECTION in getattr(var, 'collections', [])


# ----------------------------------------------------------------------------
# Global step
# ----------------------------------------------------------------------------
class _GlobalStepState(threading.local):

  def __init__(self):
    super().__init__()
    self.stack: List[Any] = []


_GS = _GlobalStepState()
_PROCESS_GLOBAL_STEP = [0]


def GetGlobalStep():
  """Current global step (python int, or tensor inside a context)."""
  if _GS.stack:
    return _GS.stack[-1]
  return _PROCESS_GLOBAL_STEP[0]


def SetGlobalStep(value: int):
  _PROCESS_GLOBAL_STEP[0] = int(value)


@contextlib.contextmanager
def GlobalStepContext(global_step):
  _GS.stack.append(global_step)
  try:
    yield
  finally:
    _GS.stack.pop()


def GetOrCreateGlobalStepVar():
  return GetGlobalStep()


# ----------------------------------------------------------------------------
# Step seeds and deterministic dropout (SURVEY A.5)
# ----------------------------------------------------------------------------
class _StepSeedState(threading.local):

  def __init__(self):
    super().__init__()
    self.step_seed = 0
    self.increments: List[int] = []
    self.global_step_override: List[Any] = []


_SEED = _StepSeedState()


def ResetStepSeed(seed: int = 0):
  _SEED.step_seed = int(seed)


def GetStepSeed() -> int:
  return _SEED.step_seed


@contextlib.contextmanager
def StepSeedIncrementContext(step: int):
  """Pipelines advance the step seed by `num_stages` per draw."""
  assert step > 0
  _SEED.increments.append(int(step))
  try:
    yield
  finally:
    _SEED.increments.pop()


def GetIncStepSeed() -> int:
  s = _SEED.step_seed
  inc = 1
  for i in _SEED.increments:
    inc *= i
  _SEED.step_seed = s + inc
  return s


@contextlib.contextmanager
def StepSeedGlobalStepOverride(value):
  """GPipe swaps global_step for a per-micro-batch id (gpipe.py:65-98)."""
  _SEED.global_step_override.append(value)
  try:
    yield
  finally:
    _SEED.global_step_override.pop()


def GenerateStepSeedPair(p, op_seed: Optional[int] = None) -> Tuple[int, int]:
  """`[global_step, step_seed++] (+random_seed) (+op_seed)`."""
  gs = (_SEED.global_step_override[-1] if _SEED.global_step_override
        else GetGlobalStep())
  gs = int(gs) if not isinstance(gs, torch.Tensor) else int(gs.item())
  a, b = gs, GetIncStepSeed()
  rs = getattr(p, 'random_seed', None) if p is not None else None
  if rs is not None:
    a += int(rs)
    b += int(rs)
  if op_seed is not None:
    a += int(op_seed)
    b += int(op_seed)
  return a, b


def GenerateSeed() -> int:
  return _pyrandom.randrange(2**31 - 1)


def _PhiloxUniform(shape, seed_pair, device, dtype=torch.float32):
  """Stateless uniform[0,1) keyed by the seed pair (same on every device)."""
  a, b = int(seed_pair[0]) & 0x7fffffff, int(seed_pair[1]) & 0x7fffffff
  gen = torch.Generator(device=device)
  gen.manual_seed((a << 31) ^ b ^ 0x5DEECE66D)
  return torch.rand(shape, generator=gen, device=device, dtype=dtype)


def DeterministicDropout(x, keep_prob, seeds, noise_shape=None, name=None):
  """floor(keep_prob + U(seed)) * x / keep_prob (reference :3978-4021)."""
  if isinstance(keep_prob, (int, float)) and keep_prob == 1.0:
    return x
  shape = list(noise_shape) if noise_shape is not None else list(x.shape)
  u = _PhiloxUniform(shape, seeds, x.device)
  keep = torch.floor(keep_prob + u).to(x.dtype)
  return x * keep / keep_prob


def DeterministicVN(params, seeds, noise_shape, mean=0.0, std=1.0, device=None):
  a, b = int(seeds[0]) & 0x7fffffff, int(seeds[1]) & 0x7fffffff
  device = device or CurrentDevice()
  gen = torch.Generator(device=device)
  gen.manual_seed((a << 31) ^ b ^ 0x2545F491)
  return torch.randn(list(noise_shape), generator=gen, device=device) * std + mean


# ----------------------------------------------------------------------------
# Variational noise
# ----------------------------------------------------------------------------
def VariationalNoiseParams(scale, global_vn=False, per_step_vn=False, seed=None,
                           deterministic=None, start_step=0):
  p = hyperparams.Params()
  p.Define('scale', scale, 'Std of the variational noise to apply.')
  p.Define('global_vn', global_vn, 'Adds global (per-weight) noise.')
  p.Define('per_step_vn', per_step_vn, 'Adds per-timestep noise.')
  p.Define('seed', seed, 'Random seed for the noise.')
  p.Define('deterministic', deterministic, 'Use step-seed keyed noise.')
  p.Define('start_step', start_step, 'Step after which noise is applied.')
  return p


DefaultVN = lambda: VariationalNoiseParams(scale=None)  # pylint: disable=invalid-name


def AddVN(p, x, per_step=False):
  """Adds variational noise to `x` per layer params `p.vn` (reference :3738)."""
  vn = p.vn
  if vn is None or vn.scale is None:
    return x
  if per_step != bool(vn.per_step_vn) and not (not per_step and vn.global_vn):
    return x
  if per_step and not vn.per_step_vn:
    return x
  if (not per_step) and not vn.global_vn:
    return x
  if getattr(p, 'is_inference', False):
    return x
  step = GetGlobalStep()
  step = int(step) if not isinstance(step, torch.Tensor) else int(step.item())
  if step < (vn.start_step or 0):
    return x
  if vn.deterministic:
    noise = DeterministicVN(p, GenerateStepSeedPair(p, vn.seed), x.shape,
                            device=x.device)
  else:
    gen = None
    if vn.seed is not None:
      gen = torch.Generator(device=x.device)
      gen.manual_seed(int(vn.seed))
    noise = torch.randn(x.shape, generator=gen, device=x.device)
  return x + (vn.scale * noise).to(x.dtype)


# ----------------------------------------------------------------------------
# Gradients
# ----------------------------------------------------------------------------
class VarGrad:
  """(var, grad[, scale]) triple; iterable like a tuple."""

  __slots__ = ('var', 'grad', 'scale')

  def __init__(self, var, grad, scale=None):
    self.var, self.grad, self.scale = var, grad, scale

  def __iter__(self):
    yield self.var
    yield self.grad
    if self.scale is not None:
      yield self.scale

  def __getitem__(self, i):
    return list(self)[i]

  def __repr__(self):
    return 'VarGrad(%s, %s)' % (getattr(self.var, 'var_name', self.var),
                                None if self.grad is None else
                                tuple(self.grad.shape))


def ComputeGradients(loss, vmap: NestedMap, skip_zero_gradients=None,
                     skip_none_gradients=True, retain_graph=False,
                     use_bf16_gradients_ar=False, **unused) -> NestedMap:
  """d loss / d vmap via autograd → NestedMap of VarGrad (reference :3123)."""
  assert isinstance(vmap, NestedMap)
  flat = [(k, v) for k, v in vmap.FlattenItems()
          if isinstance(v, torch.Tensor) and v.requires_grad]
  # Mixed precision: differentiate w.r.t. the bf16 compute copy when present.
  grads = torch.autograd.grad(
      loss, [getattr(v, 'compute', None) if getattr(v, 'compute', None)
             is not None else v for _, v in flat],
      retain_graph=retain_graph, allow_unused=True)
  out = NestedMap()
  for (k, v), g in zip(flat, grads):
    if g is None:
      if skip_none_gradients:
        continue
      g = torch.zeros_like(v)
    out.Set(k, VarGrad(v, g))
  if skip_zero_gradients:
    out = SkipZeroGradients(out, skip_zero_gradients)
  return out


def SkipZeroGradients(var_grads: NestedMap, mode: str) -> NestedMap:
  """`variable`: rescale by #replicas with non-zero grad — single process ⇒ id."""
  return var_grads


def _Leaves(var_grads) -> List[VarGrad]:
  if isinstance(var_grads, NestedMap):
    return [vg for vg in var_grads.Flatten() if isinstance(vg, VarGrad)]
  return list(var_grads)


def SumSquared(tensors) -> torch.Tensor:
  tensors = [t for t in tensors if t is not None]
  if not tensors:
    return torch.zeros(())
  if tensors[0].is_cuda and len(tensors) > 1:
    norms = torch._foreach_norm(tensors, 2, dtype=torch.float32)
    return torch.stack(norms).square().sum()
  return sum((t.float().square().sum() for t in tensors))


def ApplyGradMultiplier(vs_gs: NestedMap, grad_scale=None) -> NestedMap:
  def scale(vg):
    s = grad_scale if grad_scale is not None else vg.scale
    if s is None or vg.grad is None:
      return VarGrad(vg.var, vg.grad)
    return VarGrad(vg.var, vg.grad * torch.as_tensor(s, device=vg.grad.device,
                                                     dtype=vg.grad.dtype))
  return vs_gs.Transform(lambda vg: scale(vg) if isinstance(vg, VarGrad) else vg)


def HasNanOrInfGradient(var_grads) -> torch.Tensor:
  leaves = [vg.grad for vg in _Leaves(var_grads) if vg.grad is not None]
  if not leaves:
    return torch.zeros((), dtype=torch.bool)
  bad = torch.stack([(~torch.isfinite(g)).any() for g in leaves]).any()
  return bad


def ApplyGradNormClipping(vs_gs: NestedMap, norm=1.0) -> NestedMap:
  def clip(vg):
    if not isinstance(vg, VarGrad) or vg.grad is None:
      return vg
    n = vg.grad.float().norm()
    return VarGrad(vg.var, vg.grad * (norm / torch.clamp(n, min=norm)).to(
        vg.grad.dtype))
  return vs_gs.Transform(clip)


def AdjustGradientsWithLpLoss(var_grads: NestedMap, lp_regularizer_weight,
                              p=2.0) -> Tuple[torch.Tensor, NestedMap]:
  """Adds d(Lp)/dw to each grad; returns (lp_loss, new var_grads) (:3440)."""
  assert p in (1.0, 2.0)
  leaves = [vg for vg in _Leaves(var_grads)
            if not SkipLpRegularization(vg.var)]
  if not leaves:
    return torch.zeros(()), var_grads
  if p == 2.0:
    lp_loss = 0.5 * lp_regularizer_weight * SumSquared(
        [vg.var.detach() for vg in leaves])
  else:
    lp_loss = lp_regularizer_weight * sum(
        vg.var.detach().abs().sum() for vg in leaves)

  def adj(vg):
    if not isinstance(vg, VarGrad) or SkipLpRegularization(vg.var):
      return vg
    v = vg.var.detach().to(vg.grad.dtype)
    delta = v if p == 2.0 else torch.sign(v)
    return VarGrad(vg.var, vg.grad + lp_regularizer_weight * delta)

  return lp_loss, var_grads.Transform(adj)


def SplitRecursively(x, num_splits: int, axis: int = -1):
  if isinstance(x, torch.Tensor):
    return list(torch.chunk(x, num_splits, dim=axis))
  if isinstance(x, list):
    parts = [SplitRecursively(e, num_splits, axis) for e in x]
    return [[p[i] for p in parts] for i in range(num_splits)]
  if isinstance(x, NestedMap):
    out = [NestedMap() for _ in range(num_splits)]
    for k, v in x.items():
      for i, piece in enumerate(SplitRecursively(v, num_splits, axis)):
        out[i][k] = piece
    return out
  raise TypeError('Unexpected type for SplitRecursively: %s' % type(x))


def ConcatRecursively(splits, axis: int = -1):
  first = splits[0]
  if isinstance(first, torch.Tensor):
    return torch.cat(splits, dim=axis)
  if isinstance(first, list):
    return [ConcatRecursively([s[i] for s in splits], axis)
            for i in range(len(first))]
  if isinstance(first, NestedMap):
    out = NestedMap()
    for k in first:
      out[k] = ConcatRecursively([s[k] for s in splits], axis)
    return out
  raise TypeError('Unexpected type for ConcatRecursively: %s' % type(first))


# ----------------------------------------------------------------------------
# Metrics helpers
# ----------------------------------------------------------------------------
def WeightedAvg(values, weights, sum_reduction_fn=torch.sum):
  values = torch.as_tensor(values)
  weights = torch.as_tensor(weights).to(values.dtype)
  total_weight = sum_reduction_fn(weights)
  denom = torch.where(total_weight == 0, torch.ones_like(total_weight),
                      total_weight)
  avg = sum_reduction_fn(values * weights) / denom
  return avg, total_weight


def WeightedAvgOfMetrics(metrics: List[Dict[str, Tuple[Any, Any]]]):
  """Weighted average of a list of {name: (value, weight)} dicts (:3641)."""
  keys = list(metrics[0].keys())
  out = {}
  for k in keys:
    vals = torch.stack([torch.as_tensor(m[k][0], dtype=torch.float32).reshape(())
                        if not isinstance(m[k][0], torch.Tensor)
                        else m[k][0].float().reshape(()) for m in metrics])
    wts = torch.stack([torch.as_tensor(m[k][1], dtype=torch.float32).reshape(())
                       if not isinstance(m[k][1], torch.Tensor)
                       else m[k][1].float().reshape(()).to(vals.device)
                       for m in metrics])
    out[k] = WeightedAvg(vals, wts)
  return out


def ConcatPerExampleTensors(per_example: List[Dict[str, torch.Tensor]]):
  keys = list(per_example[0].keys())
  return {k: torch.cat([pe[k] for pe in per_example], dim=0) for k in keys}


def CombineMetrics(loss_metric_weight_pairs):
  """Combines [(metrics_dict, weight)] by weighted sum of values (:3689)."""
  all_keys = set(k for m, _ in loss_metric_weight_pairs for k in m)
  for m, _ in loss_metric_weight_pairs:
    if set(m) != all_keys:
      raise ValueError('Found mismatched metric keys: %s vs %s' %
                       (sorted(all_keys), sorted(m)))
  out = {}
  for k in all_keys:
    count = None
    vals, wts = [], []
    for m, w in loss_metric_weight_pairs:
      v, c = m[k]
      if count is None:
        count = c
      vals.append(v * w)
      wts.append(w)
    out[k] = (sum(vals) / max(sum(wts), 1e-8) if k != 'loss' else sum(vals),
              count)
  return out


# ----------------------------------------------------------------------------
# Padding / sequence helpers
# ----------------------------------------------------------------------------
def FPropDtype(params):
  """`fprop_dtype` if set, else `dtype` (ref `py_utils.FPropDtype`)."""
  return params.fprop_dtype if params.fprop_dtype is not None else params.dtype


def Softmax(logits, axis=-1, extra_logit=None, name=None):
  """Softmax with an optional constant extra logit in the denominator
  (ref `py_utils.py` Softmax)."""
  del name
  if extra_logit is None:
    return torch.softmax(logits, axis)
  mx = torch.clamp(logits.max(axis, keepdim=True).values.detach(), min=float(extra_logit))
  e = torch.exp(logits - mx)
  return e / (e.sum(axis, keepdim=True) + torch.exp(extra_logit - mx))


def ApplyPadding(padding, x, padded=None, use_select=True, ensure_shape=True):
  """Zeros (or substitutes `padded`) where padding==1; broadcasts trailing."""
  padding = padding.to(x.device)
  while padding.dim() < x.dim():
    padding = padding.unsqueeze(-1)
  if use_select:
    mask = padding > 0.5 if padding.dtype != torch.bool else padding
    if padded is None:
      return torch.where(mask, torch.zeros((), dtype=x.dtype, device=x.device), x)
    return torch.where(mask, padded, x)
  pad = padding.to(x.dtype)
  if padded is None:
    return x * (1.0 - pad)
  return x * (1.0 - pad) + padded * pad


def LengthsFromPaddings(paddings, dtype=torch.int32):
  """Length = index of last non-pad + 1 per row of `[B, T]` paddings."""
  mask = (1.0 - paddings.float())
  t = paddings.shape[1]
  idx = torch.arange(1, t + 1, device=paddings.device, dtype=torch.float32)
  return (mask * idx).amax(dim=1).to(dtype)


LengthsFromBitMask = lambda mask: LengthsFromPaddings(1.0 - mask.float())  # pylint: disable=invalid-name


def PaddingsFromLengths(lengths, maxlen=None, dtype=torch.float32):
  lengths = torch.as_tensor(lengths)
  maxlen = int(maxlen if maxlen is not None else int(lengths.max().item()))
  rng = torch.arange(maxlen, device=lengths.device)
  return (rng.unsqueeze(0) >= lengths.unsqueeze(1)).to(dtype)


SequencePaddings = PaddingsFromLengths


def TrimTrailingPaddings(inputs, paddings):
  """Trims trailing all-padding time steps of `[B, T, ...]` inputs."""
  max_len = max(int(LengthsFromPaddings(paddings).max().item()), 1)
  return inputs[:, :max_len], paddings[:, :max_len]


def ReversePaddedSequence(inputs, paddings):
  """Reverses the non-pad prefix of time-major `[T, B, ...]` inputs."""
  t = inputs.shape[0]
  pad = paddings.reshape(t, -1)
  lens = (1.0 - pad.float()).sum(0).long()  # [B]
  idx = torch.arange(t, device=inputs.device).unsqueeze(1)  # [T,1]
  src = torch.where(idx < lens.unsqueeze(0), lens.unsqueeze(0) - 1 - idx, idx)
  gather_idx = src.reshape([t, -1] + [1] * (inputs.dim() - 2)).expand_as(inputs)
  return torch.gather(inputs, 0, gather_idx)


def ConcatenatePaddedSequences(input0, input1, padding0, padding1, seq_dim=1):
  """Concats batch-major padded sequences removing the gap (:4558)."""
  assert seq_dim == 1
  b, t0 = padding0.shape
  t1 = padding1.shape[1]
  len0 = (1.0 - padding0.float()).sum(1).long()
  len1 = (1.0 - padding1.float()).sum(1).long()
  total = t0 + t1
  out = torch.zeros((b, total) + tuple(input0.shape[2:]), dtype=input0.dtype,
                    device=input0.device)
  out[:, :t0] = ApplyPadding(padding0, input0)
  pos = torch.arange(total, device=input0.device).unsqueeze(0)
  rel = pos - len0.unsqueeze(1)
  valid = (rel >= 0) & (rel < len1.unsqueeze(1))
  relc = rel.clamp(0, t1 - 1)
  g = relc.reshape([b, total] + [1] * (input1.dim() - 2)).expand(
      (b, total) + tuple(input1.shape[2:]))
  moved = torch.gather(input1, 1, g)
  v = valid.reshape([b, total] + [1] * (input1.dim() - 2))
  out = torch.where(v, moved, out)
  new_pad = (pos >= (len0 + len1).unsqueeze(1)).to(padding0.dtype)
  return out, new_pad


def ShiftLeft(tensor, shift_size, pad_val=0, axis=1):
  """Shifts along `axis` to the left, padding the tail."""
  t = tensor.shape[axis]
  body = tensor.narrow(axis, shift_size, t - shift_size)
  pad_shape = list(tensor.shape)
  pad_shape[axis] = shift_size
  pad = torch.full(pad_shape, pad_val, dtype=tensor.dtype, device=tensor.device)
  return torch.cat([body, pad], dim=axis)


def PadOrTrimTo(x, shape, pad_val=0, pad_after_contents=True):
  """Pads/trims every dim of x to `shape`."""
  shape = list(shape)
  assert x.dim() == len(shape)
  slices = tuple(slice(0, min(s, d)) if pad_after_contents
                 else slice(max(0, d - s), d)
                 for s, d in zip(shape, x.shape))
  x = x[slices]
  pads = []
  for s, d in reversed(list(zip(shape, x.shape))):
    extra = s - d
    pads.extend([0, extra] if pad_after_contents else [extra, 0])
  if any(pads):
    x = F.pad(x, pads, value=pad_val)
  return x


def PadSequenceDimension(x, length, pad_val, shape=None, axis=1):
  cur = x.shape[axis]
  if cur >= length:
    return x
  pad_shape = list(x.shape)
  pad_shape[axis] = length - cur
  return torch.cat([x, torch.full(pad_shape, pad_val, dtype=x.dtype,
                                  device=x.device)], dim=axis)


def PadBatchDimension(x, batch_size, pad_val):
  return PadSequenceDimension(x, batch_size, pad_val, axis=0)


def RepeatDim(tensor, multiple, axis):
  return torch.repeat_interleave(tensor, multiple, dim=axis)


def SequencesToDebugStrings(ids, lens, summarize=5):
  return [str(row[:int(l)].tolist()) for row, l in zip(ids, lens)]


def StackTensorsRecursively(values):
  """Stacks a list of NestedMaps into one NestedMap of stacked tensors."""
  flat = [v.Flatten() for v in values]
  stacked = [torch.stack([f[i] for f in flat]) for i in range(len(flat[0]))]
  return values[0].Pack(stacked)


def CumSum(x, axis=0, exclusive=False):
  c = torch.cumsum(x, dim=axis)
  return c - x if exclusive else c


def Matmul(x, y):
  return torch.matmul(x, y)


def ProjectLastDim(inputs, weight, input_dim=None, output_dim=None):
  return torch.matmul(inputs, weight)


def Top2GatingPlaceholder():  # kept for API discoverability
  raise NotImplementedError('see lingvo_b200.core.gshard_layers')


def BlockDiagonalMatmul(inputs, w, input_num_blocks):
  """inputs [..., D] split into blocks, each multiplied by w[b] (:6645)."""
  shp = list(inputs.shape)
  x = inputs.reshape(shp[:-1] + [input_num_blocks, shp[-1] // input_num_blocks])
  y = torch.einsum('...bi,bio->...bo', x, w)
  return y.reshape(shp[:-1] + [-1])


def BlockDiagonalProjectLastDim(inputs, weight, input_dim, output_dim,
                                num_blocks=None):
  return BlockDiagonalMatmul(inputs, weight, weight.shape[0])


# ----------------------------------------------------------------------------
# Losses
# ----------------------------------------------------------------------------
def SoftmaxCrossEntropyFocalLoss(logits, label_ids=None, label_probs=None,
                                 alpha=None, gamma=None, stop_gradient_on_focal_loss_coefficient=False):
  """Focal softmax xent (reference :5183)."""
  log_probs = F.log_softmax(logits.float(), dim=-1)
  if label_probs is None:
    label_probs = F.one_hot(label_ids.long(), logits.shape[-1]).float()
  loss = -(label_probs * log_probs).sum(-1)
  if gamma is not None and gamma != 0:
    probs = log_probs.exp()
    coef = torch.pow(1.0 - probs, gamma)
    if stop_gradient_on_focal_loss_coefficient:
      coef = coef.detach()
    loss = -(label_probs * coef * log_probs).sum(-1)
  if alpha is not None:
    a = torch.as_tensor(alpha, dtype=loss.dtype, device=loss.device)
    loss = loss * (label_probs * a).sum(-1)
  return loss


def SigmoidCrossEntropyFocalLoss(logits, labels, alpha=None, gamma=None):
  logits = logits.float()
  labels = labels.float()
  loss = F.binary_cross_entropy_with_logits(logits, labels, reduction='none')
  if gamma is not None and gamma != 0:
    p = torch.sigmoid(logits)
    pt = labels * p + (1 - labels) * (1 - p)
    loss = loss * torch.pow(1.0 - pt, gamma)
  if alpha is not None:
    loss = loss * (labels * alpha + (1 - labels) * (1 - alpha))
  return loss


# ----------------------------------------------------------------------------
# Aux loss context
# ----------------------------------------------------------------------------
class AuxLossContext:
  """Collects auxiliary losses (e.g. MoE load balancing) (reference :6572)."""

  _stack = _Stack()

  def __init__(self, reentrant=False):
    self.aux_losses: List[torch.Tensor] = []
    self._reentrant = reentrant
    self._cm = None

  @classmethod
  def Current(cls):
    return cls._stack.Top()

  def AddLoss(self, loss):
    self.aux_losses.append(loss)

  def __enter__(self):
    if not self._reentrant:
      assert not AuxLossContext._stack.items, 'no re-entry'
    self._cm = AuxLossContext._stack.Push(self)
    self._cm.__enter__()
    return self

  def __exit__(self, *args):
    self._cm.__exit__(*args)


# ----------------------------------------------------------------------------
# Variable filters
# ----------------------------------------------------------------------------
def GetTrainableVariables(scope, bprop_variable_filter,
                          bprop_variable_exclusion, vmap: NestedMap) -> NestedMap:
  """Filters `vmap` by include/exclude regexes on var names (:6610)."""
  pos = re.compile(bprop_variable_filter) if bprop_variable_filter else None
  neg = re.compile(bprop_variable_exclusion) if bprop_variable_exclusion else None

  def keep(v):
    name = getattr(v, 'var_name', '')
    if not getattr(v, 'trainable', getattr(v, 'requires_grad', False)):
      return False
    if pos and not pos.search(name):
      logging.info('%s: disabled by bprop_variable_filter: %s', scope, name)
      return False
    if neg and neg.search(name):
      logging.info('%s: disabled by bprop_variable_exclusion: %s', scope, name)
      return False
    return True

  return vmap.Filter(keep)


# ----------------------------------------------------------------------------
# Rematerialisation
# ----------------------------------------------------------------------------
def RematerializeFn(fn: Callable, *xs):
  """Runs `fn(*xs)` discarding activations; recomputed in backward (:5005).

  Step-seed state is captured so dropout masks match in the recompute.
  """
  from torch.utils.checkpoint import checkpoint
  seed0 = GetStepSeed()
  end_seed = [None]

  def wrapped(*args):
    ResetStepSeed(seed0)
    out = fn(*args)
    end_seed[0] = GetStepSeed()
    return out

  out = checkpoint(wrapped, *xs, use_reentrant=False,
                   preserve_rng_state=True)
  if end_seed[0] is not None:
    ResetStepSeed(end_seed[0])
  return out


# ----------------------------------------------------------------------------
# Retry / Timer / misc
# ----------------------------------------------------------------------------
def Retry(initial_delay_sec=1.0, delay_growth_factor=1.5, delay_growth_fuzz=0.1,
          max_delay_sec=60, retry_value=Exception, max_retries=None):
  """Exponential-backoff retry decorator (reference core/retry.py:27-70)."""
  def deco(fn):
    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
      delay = initial_delay_sec
      tries = 0
      while True:
        try:
          return fn(*args, **kwargs)
        except retry_value as e:  # pylint: disable=broad-except
          tries += 1
          if max_retries is not None and tries > max_retries:
            raise
          logging.warning('Retry %d of %s after %.2fs: %r', tries,
                          fn.__name__, delay, e)
          time.sleep(delay)
          fuzz = 1.0 + _pyrandom.uniform(-delay_growth_fuzz, delay_growth_fuzz)
          delay = min(delay * delay_growth_factor * fuzz, max_delay_sec)
    return wrapper
  return deco


class Timer:
  """Wall-clock context timer (reference :6890)."""

  def __init__(self):
    self._start = None
    self._stop = None

  def __enter__(self):
    self.Start()
    return self

  def __exit__(self, *args):
    self.Stop()

  def Start(self):
    self._start = time.time()
    self._stop = None

  def Stop(self):
    self._stop = time.time()

  @property
  def duration(self):
    end = self._stop if self._stop is not None else time.time()
    return end - self._start


class CudaTimer:
  """Device-side timer using CUDA events on the current stream."""

  def __init__(self):
    self._a = torch.cuda.Event(enable_timing=True)
    self._b = torch.cuda.Event(enable_timing=True)

  def __enter__(self):
    self._a.record()
    return self

  def __exit__(self, *args):
    self._b.record()

  @property
  def duration_ms(self):
    self._b.synchronize()
    return self._a.elapsed_time(self._b)


def UpdateProcessedCheckpoints(run_dir: str, ckpt_path: str) -> None:
  """Appends to `<run_dir>/processed_ckpts.txt` (reference :6759-6784)."""
  with open(os.path.join(run_dir, 'processed_ckpts.txt'), 'a') as f:
    f.write(ckpt_path + '\n')


def GetProcessedCheckpoints(run_dir: str) -> List[str]:
  path = os.path.join(run_dir, 'processed_ckpts.txt')
  if not os.path.exists(path):
    return []
  with open(path) as f:
    return [l.strip() for l in f if l.strip()]


def Flatten(x):
  if isinstance(x, NestedMap):
    return x.Flatten()
  if isinstance(x, dict):
    return NestedMap(x).Flatten()
  if isinstance(x, (list, tuple)):
    out = []
    for e in x:
      out.extend(Flatten(e))
    return out
  return [x]


def Transform(fn, *v):
  first = v[0]
  if isinstance(first, NestedMap):
    flat = [x.Flatten() for x in v]
    return first.Pack([fn(*args) for args in zip(*flat)])
  if isinstance(first, (list, tuple)):
    return type(first)(Transform(fn, *args) for args in zip(*v))
  return fn(*v)


def ToStaticShape(shape):
  return [int(s) for s in shape]


def Zeros(shape, dtype=torch.float32, device=None):
  return torch.zeros(list(shape), dtype=dtype, device=device or CurrentDevice())


def MaybeCast(x, dtype):
  if isinstance(x, torch.Tensor) and x.is_floating_point() and x.dtype != dtype:
    return x.to(dtype)
  return x


def CastFloats(nmap: NestedMap, dtype) -> NestedMap:
  return nmap.Transform(lambda x: MaybeCast(x, dtype))


def ReadFileLines(file_path: str) -> List[str]:
  with open(file_path) as f:
    return f.readlines()


def MultiTaskProjection(weights, biases, inputs, tasks, einsum_order='select_and_multiply'):
  """Projection whose weights (and bias) are picked per example — or per time step — by a
  task id (reference :6950).

  weights `[num_tasks, in, out]`, biases `[num_tasks, out]` or None, inputs `[B, in]` or
  `[B, T, in]`; tasks: int ids of shape `[]`, `[B]` or `[B, T]` (missing dims broadcast), or
  one-hot/float task weights with a trailing `num_tasks` axis.
    * 'select_and_multiply': gather the task's matrix, then multiply — moves `in·out` weights
      per example, the right order when there are few examples per task;
    * 'multiply_and_select': project with every task's matrix in one batched GEMM and then
      pick — more FLOPs, but one large tensor-core GEMM with no gathered weight copies.
  """
  if einsum_order not in ('select_and_multiply', 'multiply_and_select'):
    raise ValueError('Unknown einsum_order: %s' % einsum_order)
  num_tasks = weights.shape[0]
  squeeze_time = inputs.dim() == 2
  x = inputs.unsqueeze(1) if squeeze_time else inputs          # [B, T, in]
  b, t = x.shape[0], x.shape[1]
  if tasks.is_floating_point() and tasks.dim() >= 1 and tasks.shape[-1] == num_tasks:
    sel = tasks.to(x.dtype)                                     # soft / one-hot selection
    while sel.dim() < 3:
      sel = sel.unsqueeze(-2) if sel.dim() == 2 else sel.unsqueeze(0)
    sel = sel.expand(b, t, num_tasks)
    out = torch.einsum('bti,kio,btk->bto', x, weights, sel)
    if biases is not None:
      out = out + torch.einsum('btk,ko->bto', sel, biases)
    return out.squeeze(1) if squeeze_time else out
  ids = tasks.long()
  if ids.dim() == 0:
    ids = ids.reshape(1, 1).expand(b, t)
  elif ids.dim() == 1:
    ids = ids.reshape(b, 1).expand(b, t)
  else:
    assert not squeeze_time, 'per-time-step tasks need inputs with a time dimension'
    assert tuple(ids.shape) == (b, t), (ids.shape, (b, t))
  if einsum_order == 'select_and_multiply':
    out = torch.einsum('bti,btio->bto', x, weights[ids])
  else:
    allp = torch.einsum('bti,kio->btko', x, weights)
    out = allp.gather(2, ids.reshape(b, t, 1, 1).expand(b, t, 1, allp.shape[-1])).squeeze(2)
  if biases is not None:
    out = out + biases[ids]
  return out.squeeze(1) if squeeze_time else out


# =========================================================================================
# Tensor / structure helpers of the reference's py_utils used across tasks (the
# framework-agnostic ones; TF-session / TPU-rewrite helpers have no counterpart here).
# =========================================================================================
def IsEagerMode() -> bool:
  """This runtime always executes eagerly (CUDA graphs replay eager captures)."""
  return True


def IsTpuTraining(p=None) -> bool:
  del p
  return False


def Log(value, prefix, **kwargs):
  """Logs the given tensors (host sync: debugging only) and returns `value`."""
  parts = ['%s=%s' % (k, v.tolist() if isinstance(v, torch.Tensor) and v.numel() <= 16 else v)
           for k, v in kwargs.items()]
  logging.info('%s: %s', prefix, ', '.join(parts))
  return value


def LogMultiLines(label, lines):
  if isinstance(lines, str):
    lines = lines.split('\n')
  for line in lines:
    logging.info('%s: %s', label, line)


def Assert(condition, data, *args, **kwargs):
  del args, kwargs
  ok = bool(condition.all()) if isinstance(condition, torch.Tensor) else bool(condition)
  if not ok:
    raise AssertionError('Assertion failed: %s' % (data,))
  return True


def with_dependencies(dependencies, output_tensor):   # pylint: disable=invalid-name
  """Eager execution already ran `dependencies`; kept so ported code reads the same."""
  del dependencies
  return output_tensor


def _AssertCmp(op, name, x, y, summarize=None, message=None):
  del summarize
  xt, yt = torch.as_tensor(x), torch.as_tensor(y)
  if not bool(op(xt, yt).all()):
    raise AssertionError(message or 'assert_%s failed: %s vs %s' % (name, xt, yt))
  return True


def assert_greater(x, y, *args, **kwargs):   # pylint: disable=invalid-name
  return _AssertCmp(torch.gt, 'greater', x, y, *args, **kwargs)


def assert_greater_equal(x, y, *args, **kwargs):   # pylint: disable=invalid-name
  return _AssertCmp(torch.ge, 'greater_equal', x, y, *args, **kwargs)


def assert_less(x, y, *args, **kwargs):   # pylint: disable=invalid-name
  return _AssertCmp(torch.lt, 'less', x, y, *args, **kwargs)


def assert_less_equal(x, y, *args, **kwargs):   # pylint: disable=invalid-name
  return _AssertCmp(torch.le, 'less_equal', x, y, *args, **kwargs)


def clip_by_value(t, clip_value_min, clip_value_max, name=None):   # pylint: disable=invalid-name
  del name
  lo = clip_value_min if isinstance(clip_value_min, torch.Tensor) else torch.as_tensor(
      clip_value_min, dtype=t.dtype, device=t.device)
  hi = clip_value_max if isinstance(clip_value_max, torch.Tensor) else torch.as_tensor(
      clip_value_max, dtype=t.dtype, device=t.device)
  return torch.maximum(torch.minimum(t, hi.to(t.dtype)), lo.to(t.dtype))


def HasSameShape(x, ref):
  return HasShape(x, GetShape(ref))


def IsCompatible(lhs, rhs) -> bool:
  """True if the two (nested) structures have the same nesting and keys."""
  def Sig(x):
    if isinstance(x, dict):
      return ('d', tuple((k, Sig(v)) for k, v in sorted(x.items())))
    if isinstance(x, (list, tuple)):
      return ('l', tuple(Sig(v) for v in x))
    return 'x'
  return Sig(lhs) == Sig(rhs)


def AssertIsCompatible(lhs, rhs):
  if not IsCompatible(lhs, rhs):
    raise ValueError('Structures are not compatible:\n%s\nvs\n%s' % (lhs, rhs))


def AssertIdShape(expected_ids_shape_pattern, ids_shape, *args):
  """Checks `ids_shape` against a pattern (None entries are wildcards) and that every
  further shape in `args` equals `ids_shape`."""
  ids_shape = list(ids_shape)
  assert len(expected_ids_shape_pattern) == len(ids_shape), (expected_ids_shape_pattern,
                                                             ids_shape)
  for want, got in zip(expected_ids_shape_pattern, ids_shape):
    if want is not None and int(want) != int(got):
      raise AssertionError('ids shape %s does not match %s' % (ids_shape,
                                                              expected_ids_shape_pattern))
  for other in args:
    if list(other) != ids_shape:
      raise AssertionError('shape %s != ids shape %s' % (list(other), ids_shape))
  return True


def CheckShapes(shapes):
  """Asserts that `shapes` is a tuple of fully defined shapes (gpipe FPropMeta contract)."""
  assert isinstance(shapes, tuple), str(shapes)
  for s in shapes:
    if s is None:
      continue
    dims = list(getattr(s, 'ToTensorShape', lambda: s)()) if not isinstance(
        s, (list, tuple)) else list(s)
    assert all(d is not None for d in dims), '%s is not fully defined' % (s,)


def Chunked(values):
  """[a, b, c, d] → [(a, b), (c, d)]."""
  return list(zip(values[::2], values[1::2]))


def ToUniqueList(nmap):
  """Flattened `nmap` without duplicate objects (first occurrence wins)."""
  seen, out = set(), []
  for v in nmap.Flatten():
    if id(v) not in seen:
      seen.add(id(v))
      out.append(v)
  return out


def MergeDictsWithValueCheck(dict1, dict2):
  """Merges two dicts; a key present in both must map to the *same object*."""
  for key in set(dict1) & set(dict2):
    if dict1[key] is not dict2[key]:
      raise RuntimeError('The same key %s corresponds to different values in the '
                         'dictionaries: %s vs %s.' % (key, dict1[key], dict2[key]))
  return {**dict1, **dict2}


class ReadOnlyAttrDictView:
  """Read-only attribute / item view of a dict; used to hand layers' children out."""

  def __init__(self, backing):
    object.__setattr__(self, '_backing', backing)

  def __getattr__(self, name):
    try:
      return self._backing[name]
    except KeyError:
      raise AttributeError(name) from None

  def __getitem__(self, name):
    return self._backing[name]

  def __len__(self):
    return len(self._backing)

  def __iter__(self):
    return iter(self._backing)

  def __contains__(self, name):
    return name in self._backing

  def __setattr__(self, name, value):
    raise AttributeError('Dictionary is read-only.')

  def __setitem__(self, name, value):
    raise AttributeError('Dictionary is read-only.')

  def keys(self):   # pylint: disable=invalid-name
    return self._backing.keys()

  def items(self):   # pylint: disable=invalid-name
    return self._backing.items()


def SanitizeScopeKey(key: str) -> str:
  if key.startswith('_'):
    key = key[1:]
  return key.replace('[', '_').replace(']', '')


def ShardedFilePatternToGlob(file_pattern: str) -> str:
  """`path@shards` → `path-?????-of-000NN` (`@*` → `-of-*`)."""
  if ',' in file_pattern:
    raise ValueError('ShardedFilePatternToGlob does not support multiple file patterns.')
  if '@' not in file_pattern:
    return file_pattern
  path, shards = file_pattern.split('@')
  if shards == '*':
    return '%s-?????-of-*' % path
  return '%s-?????-of-%05d' % (path, int(shards))


_RECORD_FORMAT_RE = re.compile(r'(^[A-Za-z_]+):(.*)')


def RecordFormatFromFilePattern(file_pattern: str):
  """`tfrecord:/path/x*` → ('tfrecord', '/path/x*'); no prefix → ('sstable', pattern)."""
  m = _RECORD_FORMAT_RE.match(file_pattern)
  if m is None:
    return 'sstable', file_pattern
  return m.groups()


def GenerateSeedFromId(obj_id) -> int:
  md5 = hashlib.md5()
  md5.update(np.int64(obj_id).tobytes())
  return int(int(md5.hexdigest(), 16) % (2**31 - 1))


def AppendDims(x, ndims: int):
  return x.reshape(list(x.shape) + [1] * int(ndims))


def ExpandTo(x, target_rank: int):
  """Appends unit dims until `x` has rank `target_rank`."""
  if x is None:
    return None
  return x.reshape(list(x.shape) + [1] * (int(target_rank) - x.dim()))


def ExpandAndPadOrTrimTo(x, target_shape, pad_val=0):
  """Makes `x` broadcast-compatible with `target_shape`: expand to its rank, then pad / trim
  every non-unit dim to the target size."""
  if x is None:
    return None
  target_shape = [int(d) for d in target_shape]
  x = ExpandTo(x, len(target_shape))
  masked = [1 if x.shape[i] == 1 else target_shape[i] for i in range(x.dim())]
  return PadOrTrimTo(x, masked, pad_val).reshape(masked)


def PadSequenceTo(xs, padding, length: int, pad_val):
  """Pads `[B, T, …]` tensor(s) with `pad_val` and `padding [B, T]` with 1 to `length`."""
  many = isinstance(xs, (list, tuple))
  res = []
  for x in (xs if many else [xs]):
    assert tuple(x.shape[:2]) == tuple(padding.shape), (x.shape, padding.shape)
    res.append(PadSequenceDimension(x, length, pad_val))
  padding = PadSequenceDimension(padding, length, 1)
  return (tuple(res), padding) if many else (res[0], padding)


def CausalSelfAttenPadding(seqlen: int, dtype=torch.float32, device=None):
  """`[T, T]` padding with 1 where key index > query index (the future)."""
  r = torch.arange(seqlen, device=device)
  return (r.unsqueeze(-1) < r.unsqueeze(0)).to(dtype)


def ArgMax(inputs):
  return inputs.argmax(-1)


def TopK(x_in, k: int):
  """(values, indices) of the top-k entries of the last dim."""
  return torch.topk(x_in, k, dim=-1)


def DivideNoNan(x, y):
  """x / y with 0 where y == 0 (any float dtype, bf16 included)."""
  zero = y == 0
  safe = torch.where(zero, torch.ones_like(y), y)
  return torch.where(zero, torch.zeros((), dtype=x.dtype, device=x.device), x / safe)


def ReduceRms(x):
  """Root mean square (fp32 accumulation)."""
  if x.dim() == 0:
    return x
  return torch.sqrt(x.float().square().mean()).to(x.dtype if x.is_floating_point()
                                                   else torch.float32)


def SumAbs(tensor_list):
  ts = [t for t in tensor_list if t is not None]
  if not ts:
    return torch.zeros(())
  return torch.stack([t.float().abs().sum() for t in ts]).sum()


def HasNanOrInf(x):
  """0-d bool tensor: any element of `x` (tensor or list / NestedMap of tensors) is not finite."""
  ts = x.Flatten() if isinstance(x, NestedMap) else (list(x) if isinstance(x, (list, tuple))
                                                     else [x])
  ts = [t for t in ts if isinstance(t, torch.Tensor) and t.is_floating_point()]
  if not ts:
    return torch.zeros((), dtype=torch.bool)
  return torch.stack([~torch.isfinite(t).all() for t in ts]).any()


def MaybeSoftCapLogits(x, cap: float = 0.0):
  return x if cap <= 0.0 else cap * torch.tanh(x / cap)


def PiecewiseConstant(x_in, boundaries, values, vdtype=torch.float32):
  """values[k] where k = number of boundaries ≤ x_in (device-side, no sync)."""
  assert len(values) == len(boundaries) + 1 and sorted(boundaries) == list(boundaries)
  x = torch.as_tensor(x_in, dtype=torch.float32)
  bs = torch.tensor(list(boundaries), dtype=torch.float32, device=x.device)
  vs = torch.tensor(list(values), dtype=vdtype, device=x.device)
  return vs[(x >= bs).sum()] if bs.numel() else vs[0]


def GatherTensorValuesBySeqIndices(tensor, class_indices, keepdims=False):
  """ret[b, t] = tensor[b, t, class_indices[b, t]]."""
  assert tensor.dim() == 3 and class_indices.dim() == 2
  assert tuple(tensor.shape[:2]) == tuple(class_indices.shape)
  ret = tensor.gather(-1, class_indices.long().unsqueeze(-1))
  return ret if keepdims else ret.squeeze(-1)


def GetSoftmaxProbsBySeqIndices(logits, indices, keepdims=False):
  return GatherTensorValuesBySeqIndices(torch.softmax(logits.float(), -1), indices, keepdims)


def CreateIdsAndLabels(ids, paddings, sos_id=1, eos_id=2, trim=False):
  """Decoder targets from raw ids `[B, T]`: `ids` with sos prepended, `labels` with eos
  appended, `paddings`, `weights` — one longer than the input unless `trim`."""
  ids = torch.where(paddings == 0, ids, torch.full_like(ids, eos_id))
  targets = NestedMap()
  targets.ids = F.pad(ids, (1, 0), value=sos_id)
  targets.labels = F.pad(ids, (0, 1), value=eos_id)
  targets.paddings = F.pad(paddings, (1, 0))
  targets.weights = 1.0 - targets.paddings
  if trim:
    targets = targets.Transform(lambda v: v[:, :-1])
  return targets


def MergeDuplicateIds(ids, paddings, extra_tensors=None):
  """Collapses runs of equal consecutive ids (CTC-style): `[4,4,5,6,6,5,0,0]` with paddings
  `[0,0,0,0,0,0,1,1]` → ids `[4,5,6,5,0,0,0,0]`, paddings `[0,0,0,0,1,1,1,1]`. Tensors in
  `extra_tensors` (`[B, T, …]`) are compacted with the same selection."""
  assert bool((ids >= 0).all())
  b, t = ids.shape
  prev = F.pad(ids, (1, 0), value=-1)[:, :-1]
  keep = ((ids != prev) & (paddings == 0)).to(torch.int64)
  descend = keep * torch.arange(t, 0, -1, device=ids.device)
  order = torch.argsort(descend, dim=1, descending=True, stable=True)
  n = keep.sum(-1, keepdim=True)
  seq_mask = (torch.arange(t, device=ids.device).unsqueeze(0) < n)
  ret_paddings = 1.0 - seq_mask.to(paddings.dtype)
  ret_ids = ids.gather(1, order) * seq_mask.to(ids.dtype)
  ret_tensors = NestedMap()
  for key, tensor in (extra_tensors or {}).items():
    idx = order.reshape(b, t, *([1] * (tensor.dim() - 2))).expand_as(tensor)
    ret_tensors[key] = tensor.gather(1, idx) * ExpandTo(seq_mask, tensor.dim()).to(tensor.dtype)
  return ret_ids, ret_paddings, ret_tensors


def MixByWeight(inputs, weights, seed=None):
  """Calls ONE of the callables `inputs`, chosen with probability ∝ `weights`; returns
  (its result, one-hot of the chosen source). Unchosen streams are not advanced."""
  w = torch.as_tensor(weights, dtype=torch.float32)
  assert w.shape == (len(inputs),) and float(w.min()) >= 0.0
  gen = None
  if seed is not None:
    gen = torch.Generator().manual_seed(int(seed))
  r = torch.rand((), generator=gen) * w.sum()
  idx = int(torch.searchsorted(torch.cumsum(w, 0), r, right=True).clamp(max=len(inputs) - 1))
  return inputs[idx](), F.one_hot(torch.tensor(idx), len(inputs)).float()


def MaskGradients(var_grad, grad_mask):
  """`grad_mask`: variable name → mask; returns var_grads with `mask * gradient`."""
  def ApplyMask(entry):
    var, grad = entry
    name = getattr(var, 'var_name', getattr(var, 'name', None))
    return VarGrad(var, grad * grad_mask[name])
  return var_grad.Transform(ApplyMask)


def SkipNoneGradients(var_grads):
  """Drops (var, None) pairs."""
  return var_grads.Filter(lambda vg: vg.grad is not None) if isinstance(
      var_grads, NestedMap) else [vg for vg in var_grads if vg.grad is not None]


def ConvertNoneGradientToZeros(xs, dxs):
  """None gradients become zeros shaped like their `xs` entry."""
  return xs.Pack([torch.zeros_like(x) if dx is None else dx
                  for x, dx in zip(xs.Flatten(), dxs.Flatten() if isinstance(
                      dxs, NestedMap) else dxs)])


def ComputeNceAndAuc(probs, targets, mask):
  """Normalised cross entropy and PR-curve AUC of per-token confidence scores
  (`probs`, `targets ∈ {0,1}`, `mask`, all `[B, T]`)."""
  probs, targets, mask = probs.float(), targets.float(), mask.float()

  def LogClip(t):
    return torch.log(t.clamp(1e-8, 1.0))

  bce = -targets * LogClip(probs) - (1 - targets) * LogClip(1 - probs)
  num_tokens = mask.sum()
  wcr = (targets * mask).sum() / num_tokens
  entropy = -wcr * LogClip(wcr) - (1 - wcr) * LogClip(1 - wcr)
  nce = (entropy - (bce * mask).sum() / num_tokens) / entropy
  # PR AUC by the trapezoid rule over 200 thresholds (what tf.metrics.auc does)
  sel = mask > 0
  p, y = probs[sel], targets[sel]
  th = torch.linspace(0.0, 1.0, 200, device=p.device).unsqueeze(1)
  pred = (p.unsqueeze(0) > th).float()
  tp = (pred * y).sum(1)
  fp = (pred * (1 - y)).sum(1)
  fn = ((1 - pred) * y).sum(1)
  precision = (tp + 1e-7) / (tp + fp + 1e-7)
  recall = (tp + 1e-7) / (tp + fn + 1e-7)
  auc = torch.trapz(precision.flip(0), recall.flip(0)).abs()
  return nce, auc


class UniformSampler:
  """Reservoir sampler keeping a uniform sample of `num_samples` items of a stream."""

  def __init__(self, num_samples, seed=None):
    assert num_samples > 0
    self._num_samples = num_samples
    self._num_seen_items = 0
    self._samples = []
    self._rng = np.random.RandomState(seed)

  def Add(self, item):
    self._num_seen_items += 1
    if len(self._samples) < self._num_samples:
      self._samples.append(item)
      return
    index = self._rng.randint(0, self._num_seen_items)
    if index < self._num_samples:
      self._samples[index] = item

  @property
  def samples(self):
    return self._samples


_SAMPLE_STEP_STACK = []


@contextlib.contextmanager
def SampleStep(step):
  """Context naming the current decode step (`with py_utils.SampleStep(t): …`)."""
  _SAMPLE_STEP_STACK.append(step)
  try:
    yield step
  finally:
    _SAMPLE_STEP_STACK.pop()


# -- task call scopes (which task is calling into shared layers) ---------------------
_TASK_CALL_SCOPE = []


@contextlib.contextmanager
def TaskCallScope(task):
  _TASK_CALL_SCOPE.append(task)
  try:
    yield
  finally:
    _TASK_CALL_SCOPE.pop()


def GetTaskCallScope():
  return _TASK_CALL_SCOPE[-1] if _TASK_CALL_SCOPE else None


def TaskCallScopeName(task):
  return getattr(getattr(task, 'params', None), 'name', None) or str(task)


# -- params helpers -----------------------------------------------------------------------
def UpdateDtype(params, dtype):
  """Sets `dtype` on `params` and every nested layer params that has the field."""
  def Visit(p):
    if isinstance(p, hyperparams.Params):
      if 'dtype' in p and 'cls' in p:
        p.dtype = dtype
      for _, v in p.IterParams():
        Visit(v)
    elif isinstance(p, (list, tuple)):
      for v in p:
        Visit(v)
    elif isinstance(p, dict):
      for v in p.values():
        Visit(v)
  Visit(params)
  return params


def UpdateFpropDtype(params, fprop_dtype):
  """Sets `fprop_dtype` on `params` and every nested layer params."""
  def Visit(p):
    if isinstance(p, hyperparams.Params):
      if 'fprop_dtype' in p:
        p.fprop_dtype = fprop_dtype
      for _, v in p.IterParams():
        Visit(v)
    elif isinstance(p, (list, tuple)):
      for v in p:
        Visit(v)
    elif isinstance(p, dict):
      for v in p.values():
        Visit(v)
  Visit(params)
  return params


def GetVariableName(name: str) -> str:
  """Full variable name under the current variable scope (as CreateVariable would use)."""
  scope = CurrentVariableScope()
  return (scope + '/' if scope else '') + name


# -- functional control flow (host loops: every iteration launches device work) -------------
def ForLoop(body, start, limit, delta, loop_state):
  """state = body(i, state) for i in range(start, limit, delta)."""
  state = loop_state
  for i in range(int(start), int(limit), int(delta)):
    state = body(i, state)
  return state


def WhileLoop(cond, body, loop_state):
  """while cond(state): state = body(state) — `cond` may return a 0-d tensor (host sync)."""
  state = loop_state
  while bool(cond(state)):
    state = body(state)
  return state


def If(cond, inputs, then_branch, else_branch):
  return then_branch(inputs) if bool(cond) else else_branch(inputs)


def Pack(tmpl, values):
  """Packs the flat list `values` into the structure of `tmpl`."""
  return tmpl.Pack(list(values))


# -- RNN initial-state policy (ref py_utils.py:1014-1080) --------------------------------------
class RNNCellStateInit:
  """Params describing how a cell's initial state is drawn."""

  @staticmethod
  def _Params(method, seed):
    p = hyperparams.Params()
    p.Define('method', method, 'One of zeros, random_normal.')
    p.Define('seed', seed, 'Random seed of random_normal.')
    p.Freeze()
    return p

  @staticmethod
  def Zeros():
    return RNNCellStateInit._Params('zeros', None)

  @staticmethod
  def RandomNormal(seed=None):
    return RNNCellStateInit._Params('random_normal', seed)


def DefaultRNNCellStateInit():
  return RNNCellStateInit.Zeros()


def InitRNNCellState(shape, init=None, dtype=None, name=None, is_eval=False, device=None):
  """Initial state tensor of `shape`: zeros, or N(0,1) in training for `random_normal`
  (seeded from (name, init.seed) when either is given so replicas agree)."""
  init = init or DefaultRNNCellStateInit()
  dtype = dtype or torch.float32
  shape = [int(d) for d in shape]
  if init.method == 'zeros' or (init.method == 'random_normal' and is_eval):
    return torch.zeros(shape, dtype=dtype, device=device)
  if init.method != 'random_normal':
    raise ValueError('Initialization method (%s) not supported.' % init.method)
  gen = None
  if init.seed is not None or name is not None:
    seed = GenerateSeedFromName(name or 'rnn_state') ^ int(init.seed or 0)
    gen = torch.Generator().manual_seed(seed % (2**31 - 1))
  return torch.randn(shape, generator=gen, dtype=torch.float32).to(device=device, dtype=dtype)


# -- functions with hand-written gradients (ref py_utils.py:5560-6110: Function / CallDefun) ------
def _PackLike(tmpl, flat):
  """Inverse of Flatten for NestedMap / dict / list / tuple / leaf templates."""
  it = iter(flat)

  def Build(t):
    if isinstance(t, NestedMap):
      return t.Pack([next(it) for _ in t.Flatten()])
    if isinstance(t, dict):
      return {k: Build(t[k]) for k in sorted(t)}
    if isinstance(t, (list, tuple)):
      return type(t)(Build(e) for e in t)
    return next(it)

  return Build(tmpl)


def CallDefun(fwd, args=None, bak=None, bak_as_function=False, device=None):
  """ys = fwd(args); with `bak`, the backward pass calls `bak(xs, ys, dys) -> dxs` instead of
  differentiating `fwd` (which then runs without building an autograd graph).

  `args` / results are arbitrary nested structures of tensors. The forward activations are
  not kept: `bak` sees the saved inputs and outputs only — the memory contract the reference's
  Defun gives (it is what `recurrent` and reversible layers are built on).
  """
  del bak_as_function, device
  if bak is None:
    return fwd(args) if args is not None else fwd()
  flat_in = Flatten(args)
  is_t = [isinstance(x, torch.Tensor) for x in flat_in]
  holder = {}

  class _Fn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, *tensors):
      it = iter(tensors)
      xs = _PackLike(args, [next(it) if t else x for t, x in zip(is_t, flat_in)])
      with torch.no_grad():
        ys = fwd(xs)
      flat_out = Flatten(ys)
      holder['tmpl'] = ys
      ctx.n_in = len(tensors)
      ctx.save_for_backward(*tensors, *[y for y in flat_out if isinstance(y, torch.Tensor)])
      ctx.out_is_t = [isinstance(y, torch.Tensor) for y in flat_out]
      ctx.out_consts = [None if isinstance(y, torch.Tensor) else y for y in flat_out]
      nondiff = [y for y in flat_out if isinstance(y, torch.Tensor)
                 and not y.is_floating_point()]
      ctx.mark_non_differentiable(*nondiff)
      return tuple(y for y in flat_out if isinstance(y, torch.Tensor))

    @staticmethod
    def backward(ctx, *grads):
      saved = ctx.saved_tensors
      ins, outs = saved[:ctx.n_in], saved[ctx.n_in:]
      it = iter(ins)
      xs = _PackLike(args, [next(it) if t else x for t, x in zip(is_t, flat_in)])
      oi, gi = iter(outs), iter(grads)
      flat_y, flat_dy = [], []
      for t, c in zip(ctx.out_is_t, ctx.out_consts):
        if t:
          y, g = next(oi), next(gi)
          flat_y.append(y)
          flat_dy.append(torch.zeros_like(y) if g is None else g)
        else:
          flat_y.append(c)
          flat_dy.append(None)
      ys = _PackLike(holder['tmpl'], flat_y)
      dys = _PackLike(holder['tmpl'], flat_dy)
      with torch.no_grad():
        dxs = bak(xs, ys, dys)
      flat_dx = Flatten(dxs)
      assert len(flat_dx) == len(flat_in), 'bak must return one gradient per input leaf'
      res = []
      for t, x, dx in zip(is_t, flat_in, flat_dx):
        if t:
          res.append(dx if (isinstance(dx, torch.Tensor) and x.is_floating_point()) else None)
      return tuple(res)

  outs = _Fn.apply(*[x for x, t in zip(flat_in, is_t) if t])
  oi = iter(outs)
  flat_out = [next(oi) if isinstance(y, torch.Tensor) else y
              for y in Flatten(holder['tmpl'])]
  return _PackLike(holder['tmpl'], flat_out)


def Function(fwd_sig=None, bak=None, bak_as_function=False, device=None):
  """Decorator form: `@Function(bak=Grad) def Fwd(xs): …` → a callable using `Grad` backward."""
  del fwd_sig

  def Decorate(fwd):
    @functools.wraps(fwd)
    def Call(args=None):
      return CallDefun(fwd, args, bak=bak, bak_as_function=bak_as_function, device=device)
    Call.func = fwd
    return Call

  return Decorate


DefinedFunction = Function


def ComputeGradientsSimple(loss_or_activations, all_vars, grad_aggregation_method=None,
                           colocate_gradients_with_ops=None, gate_gradients=None,
                           activations_grad=None):
  """Plain autograd of a loss (or of activations seeded with `activations_grad`) w.r.t. a
  flat list of variables; unused variables get None."""
  del grad_aggregation_method, colocate_gradients_with_ops, gate_gradients
  return list(torch.autograd.grad(loss_or_activations, list(all_vars),
                                  grad_outputs=activations_grad, allow_unused=True,
                                  retain_graph=True))


@contextlib.contextmanager
def GradientTape(*args, **kwargs):
  """Autograd records eagerly; the context exists so reference-shaped code runs unchanged."""
  del args, kwargs
  with torch.enable_grad():
    yield None


def CurrentGradientTape():
  return None


def DisableVN():
  return VariationalNoiseParams(1.0, False, False)


def FindDataType(var_name):
  """dtype of the first VariableListDtypeRegexScope rule matching `var_name`, else None."""
  for rules in _VAR_DTYPE_OVERRIDES.items:
    for regex, dtype in rules:
      if re.match(regex, var_name):
        return dtype
  return None


def Save(value, filename_prefix, **kwargs):
  """Debug helper: writes every tensor in kwargs to `<prefix>.<step>.<name>.npy`."""
  step = int(GetGlobalStep())
  for name, t in sorted(kwargs.items()):
    arr = t.detach().float().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    np.save('%s.%08d.%s.npy' % (filename_prefix, step, name), arr)
  return value


def ReadVariable(var):
  return var.detach() if isinstance(var, torch.Tensor) else var


def SetShapes(dst_nmap, src_nmap):
  """Checks that both structures carry tensors of the same shapes (shapes are always static
  here, so there is nothing to set)."""
  AssertIsCompatible(src_nmap, dst_nmap)
  for d, s in zip(dst_nmap.Flatten(), src_nmap.Flatten()):
    assert tuple(d.shape) == tuple(s.shape), (d.shape, s.shape)


@contextlib.contextmanager
def RemoveAssertContext(remove=True):
  """Disables the py_utils shape / value asserts inside the context."""
  if not remove:
    yield
    return
  prev = flags.enable_asserts
  flags.enable_asserts = lambda: False
  try:
    yield
  finally:
    flags.enable_asserts = prev


@contextlib.contextmanager
def outside_all_rewrites():   # pylint: disable=invalid-name
  yield


@contextlib.contextmanager
def tpu_host(func=None):   # pylint: disable=invalid-name
  yield func


def RunOnTpuHost(func, *args, **kwargs):
  return func(*args, **kwargs)


def RetryOnTransientTfError(*args, **kwargs):
  """Retry decorator for transient IO / collective errors."""
  kwargs.setdefault('retry_value', (OSError, RuntimeError))
  return Retry(*args, **kwargs)


def OverrideVarsFromCheckpoint(all_vars, checkpoint_path, variable_loading_rules,
                               var_ignore_rules, **unused):
  """Loads the variables of `all_vars` matched by `variable_loading_rules` ([(regex, fmt)])
  and not by `var_ignore_rules` from the bundle at `checkpoint_path` (ref :5200-5330)."""
  from lingvo_b200.core import saver as saver_lib
  from lingvo_b200.utils import tensor_bundle
  if os.path.isdir(checkpoint_path):
    checkpoint_path = saver_lib.LatestCheckpoint(checkpoint_path)
  reader = tensor_bundle.BundleReader(checkpoint_path)
  keys = set(reader.Keys())
  loaded = []
  with torch.no_grad():
    for v in all_vars:
      name = v.var_name[:-len('/var')] if v.var_name.endswith('/var') else v.var_name
      if any(re.match(r, name) for r in var_ignore_rules):
        continue
      for regex, fmt in variable_loading_rules:
        m = re.match(regex, name)
        if not m:
          continue
        src = fmt % m.groups() if m.groups() else fmt
        hit = [c for c in (src, src + '/var') if c in keys]
        if not hit:
          raise KeyError('%s → %s not found in %s' % (name, src, checkpoint_path))
        v.data.copy_(saver_lib.FromNumpy(reader.Read(hit[0])).to(v.device, v.dtype))
        loaded.append(name)
        break
  reader.Close()
  return loaded


def OverrideVarsFromCheckpoints(all_vars, ckpts_loading_rules, **unused):
  """`ckpts_loading_rules`: {ckpt_path: ([(regex, fmt)], [ignore_regex])}; a variable may be
  claimed by one checkpoint only."""
  claimed = {}
  for ckpt, (rules, ignore) in ckpts_loading_rules.items():
    for name in OverrideVarsFromCheckpoint(all_vars, ckpt, rules, ignore):
      if name in claimed:
        raise ValueError('Variable %s is overridden by both %s and %s' % (name, claimed[name],
                                                                         ckpt))
      claimed[name] = ckpt
  return claimed
