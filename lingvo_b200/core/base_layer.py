"""`BaseLayer`: the unit of composition (config → layer → FProp(theta, …)).

Contract: reference `lingvo/core/base_layer.py` — common params (:224-285),
`CopyBaseParams` (:288-320), child management (:974-1046), `CreateVariable`
(:823-874), `theta`/`vars` (:645-694), accumulators (:40-98, :755-817),
post-step hooks (:1129-1152), `GetDescendant` (:531), `FPropMeta` (:447).

PyTorch-first design notes
  * Variables are `torch.nn.Parameter`s; `theta` is a NestedMap of *tensors*
    with the same structure (EMA-swapped in eval, cast to `fprop_dtype`), so
    every layer is functional in its weights: `layer.FProp(theta, x)`. That is
    what remat, GPipe stages, stacked-variable repeat layers and fused
    flat-buffer optimizers (`parallel/dp.py` swaps in bf16 views) rely on.
  * Variable creation is *deferred*: `CreateVariable` only records a spec;
    the outermost constructor materialises all variables depth-first under the
    proper name scopes, so checkpoint keys are `<layer path>/<var>/var`.
  * No TF graph: the metaclass keeps a thread-local construction stack only
    to find parents and to forbid child creation outside `__init__`.
"""

from __future__ import annotations

import contextlib
import re
import threading
from typing import Any, Callable, Dict, List, Optional

import torch

from lingvo_b200.core import cluster_factory
from lingvo_b200.core import hyperparams
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap


class _Construction(threading.local):

  def __init__(self):
    super().__init__()
    self.stack: List['BaseLayer'] = []


_BUILD = _Construction()


class Accumulator:
  """Layer-associated running state threaded through scans/pipelines.

  Reference :40-98. Values are plain tensors; `Disable/Enable` nest.
  """

  def __init__(self):
    self._disable_count = 0
    self._value = None

  @property
  def is_disabled(self):
    return self._disable_count > 0

  def Disable(self):
    self._disable_count += 1

  def Enable(self):
    assert self._disable_count > 0, 'Unbalanced Accumulator Enable/Disable'
    self._disable_count -= 1

  def DefaultValue(self):
    raise NotImplementedError('DefaultValue must be implemented')

  def GetValue(self):
    if self.is_disabled or self._value is None:
      return self.DefaultValue()
    return self._value

  def Update(self, new_value):
    if not self.is_disabled:
      self._value = new_value

  def SetValue(self, new_value):
    self._value = new_value

  def Reset(self):
    if not self.is_disabled:
      self._value = None


class BaseLayerMeta(type):
  """Wraps construction: tracks the layer stack and instantiates variables."""

  def __call__(cls, *args, **kwargs):
    layer = cls.__new__(cls, *args, **kwargs)
    _BUILD.stack.append(layer)
    try:
      layer.__init__(*args, **kwargs)
      layer._disable_create_child = True  # pylint: disable=protected-access
      if len(_BUILD.stack) == 1:
        if cluster_factory.Current().params.immediately_instantiate_variables:
          layer.InstantiateVariables()
        layer._VerifyChildren()  # pylint: disable=protected-access
    finally:
      _BUILD.stack.pop()
    return layer


def initializer(func):  # pylint: disable=invalid-name
  """Legacy decorator kept for source compatibility; a no-op here."""
  return func


def DefaultVN():
  return py_utils.DefaultVN()


def RecursiveFindLayerParams(params):
  """Yields every layer Params nested inside `params`."""
  found = []

  def visit(p):
    if isinstance(p, hyperparams.Params):
      if isinstance(p, hyperparams.InstantiableParams) and isinstance(
          p.cls, type) and issubclass(p.cls, BaseLayer):
        found.append(p)
      for _, v in p.IterParams():
        visit(v)
    elif isinstance(p, (list, tuple)):
      for v in p:
        visit(v)
    elif isinstance(p, dict):
      for v in p.values():
        visit(v)

  visit(params)
  return found


class BaseLayer(metaclass=BaseLayerMeta):
  """Base class of every layer, task and model."""

  # Subclasses may map child name → list of scope components (e.g. [] hoists
  # the child to the parent's scope: SingleTaskModel {'_task': []}).
  _child_variable_scope_override: Dict[str, List[str]] = {}

  @classmethod
  def Params(cls):
    p = hyperparams.InstantiableParams(cls)
    p.Define('inference_driver_name', cls.__name__ + 'Inference',
             'Name of the inference driver for this layer.')
    p.Define('name', '', 'Name of this layer object, must be a valid id.')
    p.Define('dtype', torch.float32, 'Datatype of the variables.')
    p.Define('fprop_dtype', None,
             'Activations datatype; None ⇒ same as dtype. bf16 is the H100 '
             'tensor-core path.')
    p.Define('random_seed', None,
             'Layer-local random seed. None ⇒ non-deterministic init; set ⇒ '
             'per-variable seed = hash(var name).')
    p.Define('vn', DefaultVN(), 'Variational-noise params.')
    p.Define('params_init', py_utils.DefaultParamInit(),
             'How trainable params are initialised.')
    p.Define('is_inference', None, 'True if in inference mode.')
    p.Define('skip_lp_regularization', None,
             'Exclude this layer (and children) from Lp regularization.')
    p.Define('device_mesh', None,
             'np.ndarray of device ids: the mesh for SPMD sharding.')
    p.Define('weight_split_dims_mapping', None,
             'Default mesh-axis mapping for weights.')
    p.Define('activation_split_dims_mapping', None,
             'Default mesh-axis mapping for activations.')
    return p

  @staticmethod
  def CopyBaseParams(from_params, to_params):
    """Parent → child inheritance of unset base params (reference :288)."""
    assert issubclass(from_params.cls, BaseLayer)
    assert issubclass(to_params.cls, BaseLayer)
    if to_params.dtype == torch.float32:
      to_params.dtype = from_params.dtype
    if from_params.fprop_dtype is not None and to_params.fprop_dtype is None:
      to_params.fprop_dtype = from_params.fprop_dtype
    if to_params.random_seed is None:
      to_params.random_seed = from_params.random_seed
    if to_params.is_inference is None:
      to_params.is_inference = from_params.is_inference
    if to_params.skip_lp_regularization is None:
      to_params.skip_lp_regularization = from_params.skip_lp_regularization
    if to_params.device_mesh is None and 'device_mesh' in from_params:
      to_params.device_mesh = from_params.device_mesh
    # Only propagate init if the child is still at the default.
    if py_utils.IsDefaultParamInit(to_params.params_init):
      to_params.params_init = from_params.params_init.Copy()
    if to_params.vn is None or to_params.vn.scale is None:
      if from_params.vn is not None and from_params.vn.scale is not None:
        to_params.vn = from_params.vn.Copy()
    return to_params

  # ----------------------------------------------------------- construction --
  def __init__(self, params):
    assert params.name, (
        'Layer params for %s must have a "name"' % self.__class__.__name__)
    if not re.match(r'^[A-Za-z0-9_][A-Za-z0-9_.\-]*$', params.name):
      raise ValueError('Invalid layer name %r' % params.name)
    self._parent = _BUILD.stack[-2] if len(_BUILD.stack) > 1 else None
    self._params = params.Copy()
    self._params.Freeze()
    self._path = params.name
    self._private_children = NestedMap()
    self._private_vars = NestedMap()
    self._private_var_specs: List = []
    self._private_theta_override: Dict[str, torch.Tensor] = {}
    self._private_accumulators: Dict[str, Accumulator] = {}
    self._private_fns: Dict[str, Callable] = {}
    self._extra_theta = NestedMap()
    self._disable_create_child = False
    self._variables_instantiated = False
    self._child_scopes: Dict[str, List[str]] = {}
    self._ema_shadow: Dict[str, torch.Tensor] = {}

  # -------------------------------------------------------------- accessors --
  @property
  def params(self):
    return self._params

  p = params

  @property
  def cluster(self):
    return cluster_factory.Current()

  @property
  def do_eval(self) -> bool:
    return self.cluster.do_eval

  @property
  def parent(self):
    return self._parent

  @property
  def path(self) -> str:
    return self._path

  @property
  def layer_type(self) -> str:
    return type(self).__name__

  @property
  def children(self) -> NestedMap:
    return self._private_children

  @property
  def fprop_dtype(self):
    p = self.params
    return p.fprop_dtype if p.fprop_dtype is not None else p.dtype

  def __getattr__(self, name):
    # Only reached when normal lookup fails: resolve children, then mimic the
    # reference's error text.
    d = self.__dict__
    ch = d.get('_private_children')
    if ch is not None and name in ch:
      return ch[name]
    raise AttributeError('%s is not a sub-layer of %s (%s).' %
                         (name, d.get('_path', '?'), type(self).__name__))

  def GetDescendant(self, path: str):
    """`a.b[2].c` → the descendant layer (reference :531)."""
    sub = self
    if path:
      for seg in path.split('.'):
        m = re.match(r'^(\w+)((?:\[\d+\])*)$', seg)
        if not m:
          raise KeyError('Invalid path: %s' % path)
        sub = sub.children[m.group(1)]
        for i in re.findall(r'\[(\d+)\]', m.group(2)):
          sub = sub[int(i)]
    return sub

  # --------------------------------------------------------------- children --
  def _CheckCanCreate(self, what):
    if self._disable_create_child:
      raise ValueError('%s may only be called from __init__ (layer %s).' %
                       (what, self.path))

  def _PrepareChildParams(self, name, params):
    p = self.CopyBaseParams(self.params, params.Copy())
    if not p.name:
      p.name = name
    return p

  def _SetChildPath(self, child, key):
    child._path = self._path + '.' + key  # pylint: disable=protected-access
    child._parent = self  # pylint: disable=protected-access

  def CreateChild(self, name: str, params):
    """Creates sub-layer `name` from `params` (reference :974)."""
    self._CheckCanCreate('CreateChild')
    if hasattr(type(self), name):
      raise AttributeError('Child name %s collides with an attribute' % name)
    p = self._PrepareChildParams(name, params)
    child = p.Instantiate()
    self._SetChildPath(child, name)
    self._private_children[name] = child
    self._FixPaths(child)

  def CreateChildren(self, name: str, params, child_scopes=None):
    """Creates a (nested) list / dict of sub-layers (reference :1003)."""
    self._CheckCanCreate('CreateChildren')
    uid = [0]

    def build(node, key):
      if isinstance(node, (list, tuple)):
        return [build(x, '%s[%d]' % (key, i)) for i, x in enumerate(node)]
      if isinstance(node, dict):
        return NestedMap({k: build(v, '%s.%s' % (key, k))
                          for k, v in node.items()})
      p = self.CopyBaseParams(self.params, node.Copy())
      if not p.name:
        p.name = '%s_%d' % (name, uid[0])
      uid[0] += 1
      child = p.Instantiate()
      self._SetChildPath(child, key)
      self._FixPaths(child)
      return child

    self._private_children[name] = build(params, name)

  def AddChild(self, name: str, child):
    """Adopts an already-built layer (reference :1039)."""
    assert isinstance(child, BaseLayer)
    self._SetChildPath(child, name)
    self._private_children[name] = child
    self._FixPaths(child)

  def AddChildren(self, name: str, children):
    for i, c in enumerate(children):
      self._SetChildPath(c, '%s[%d]' % (name, i))
      self._FixPaths(c)
    self._private_children[name] = list(children)

  def _FixPaths(self, layer):
    """Re-roots descendant paths after a child's own path is assigned."""
    def fix(node, key):
      if isinstance(node, BaseLayer):
        node._path = key  # pylint: disable=protected-access
        for k, v in node._private_children.items():  # pylint: disable=protected-access
          fix(v, key + '.' + k)
      elif isinstance(node, list):
        for i, v in enumerate(node):
          fix(v, '%s[%d]' % (key, i))
      elif isinstance(node, dict):
        for k, v in node.items():
          fix(v, key + '.' + k)
    for k, v in layer._private_children.items():  # pylint: disable=protected-access
      fix(v, layer._path + '.' + k)  # pylint: disable=protected-access

  def _VerifyChildren(self):
    """Every BaseLayer attribute must be registered as a child (:1109)."""
    def walk(layer):
      registered = set(id(c) for c in layer._private_children.Flatten())  # pylint: disable=protected-access
      for k, v in layer.__dict__.items():
        if k in ('_parent',) or k.startswith('_private'):
          continue
        if isinstance(v, BaseLayer) and id(v) not in registered:
          raise ValueError('%s.%s is a BaseLayer but not a registered child' %
                           (layer.path, k))
      for c in layer._private_children.Flatten():  # pylint: disable=protected-access
        if isinstance(c, BaseLayer):
          walk(c)
    walk(self)

  # -------------------------------------------------------------- variables --
  def CreateVariable(self, name: str, var_params, trainable: bool = True,
                     **kwargs):
    """Declares variable `name` (materialised by InstantiateVariables)."""
    if self._variables_instantiated and not kwargs.pop('_late', False):
      raise ValueError('CreateVariable after variables were instantiated: '
                       '%s.%s' % (self.path, name))
    if any(n == name for n, _, _ in self._private_var_specs):
      raise AttributeError('Variable %s is already defined in %s' %
                           (name, self.path))
    if self.params.skip_lp_regularization:
      var_params = var_params.Copy()
      var_params.collections = list(var_params.collections or []) + [
          py_utils._SKIP_LP_COLLECTION]  # pylint: disable=protected-access
    if var_params.device_mesh is None and self.params.device_mesh is not None:
      var_params = var_params.Copy()
      var_params.device_mesh = self.params.device_mesh
    self._private_var_specs.append((name, var_params, trainable))

  def _CreateLayerVariables(self):
    """Subclass hook: call self.CreateVariable(...) here."""

  def _ChildScope(self, child_key: str, child: 'BaseLayer') -> List[str]:
    if child_key in self._child_variable_scope_override:
      return list(self._child_variable_scope_override[child_key])
    if child_key in self._child_scopes:
      return list(self._child_scopes[child_key])
    return [child.params.name]

  def InstantiateVariables(self):
    """Materialises own + descendants' variables under proper scopes."""
    if self._variables_instantiated:
      return
    if self._parent is None or not _ScopeIsManaged():
      ctx = py_utils.VariableScope([self.params.name])
    else:
      ctx = contextlib.nullcontext()
    with ctx, _ManagedScope():
      self._InstantiateSelfAndChildren()

  def _InstantiateSelfAndChildren(self):
    self._CreateLayerVariables()
    self._variables_instantiated = True
    for name, wp, trainable in self._private_var_specs:
      var = py_utils.CreateVariable(name, wp, trainable=trainable,
                                    default_seed=self.params.random_seed)
      self._private_vars[name] = var
    self._CreateChildrenVariables()

  def _CreateChildrenVariables(self):
    """Default: each child under its own name scope. Layers that stack vars
    (RepeatLayer) override this to push shape-prefix contexts."""
    for key, node in self._private_children.items():
      self._InstantiateNode(key, node)

  def _InstantiateNode(self, key, node):
    if isinstance(node, BaseLayer):
      if node._variables_instantiated:  # pylint: disable=protected-access
        return
      with py_utils.VariableScope(self._ChildScope(key, node)):
        node._InstantiateSelfAndChildren()  # pylint: disable=protected-access
    elif isinstance(node, list):
      for v in node:
        self._InstantiateNode(key, v)
    elif isinstance(node, dict):
      for v in node.values():
        self._InstantiateNode(key, v)

  @property
  def vars(self) -> NestedMap:
    """NestedMap of Parameters (own + children), reference :696."""
    ret = self._private_children.Transform(
        lambda c: c.vars if isinstance(c, BaseLayer) else c)
    for k, v in self._private_vars.items():
      ret[k] = v
    return ret

  def _OwnThetaValue(self, name: str, var):
    override = self._private_theta_override.get(name)
    value = override if override is not None else var
    if self.do_eval and name in self._ema_shadow:
      value = self._ema_shadow[name]
    fd = self.fprop_dtype
    if value.is_floating_point() and value.dtype != fd:
      value = value.to(fd)
    if (self.params.vn is not None and self.params.vn.global_vn and
        not self.do_eval):
      value = py_utils.AddVN(self.params, value)
    return value

  @property
  def theta(self) -> NestedMap:
    """NestedMap of weight *values* aligned with `vars` (reference :645)."""
    ret = self._private_children.Transform(
        lambda c: c.theta if isinstance(c, BaseLayer) else c)
    for k, v in self._private_vars.items():
      ret[k] = self._OwnThetaValue(k, v)
    for k, v in self._extra_theta.items():
      ret[k] = v
    return ret

  def AddExtraTheta(self, theta_name: str, theta_value):
    self._extra_theta[theta_name] = theta_value

  @contextlib.contextmanager
  def TransformVarsTempContext(self, fn: Callable[[torch.Tensor], torch.Tensor]):
    """Temporarily views every own var through `fn` (reference :636)."""
    saved = dict(self._private_theta_override)
    try:
      for k, v in self._private_vars.items():
        self._private_theta_override[k] = fn(v)
      yield
    finally:
      self._private_theta_override = saved

  def SetThetaOverride(self, name: str, tensor):
    """Points theta.<name> at an external buffer (flat bf16 replica etc.)."""
    if tensor is None:
      self._private_theta_override.pop(name, None)
    else:
      self._private_theta_override[name] = tensor

  def SetEmaShadow(self, name: str, tensor):
    if tensor is None:
      self._ema_shadow.pop(name, None)
    else:
      self._ema_shadow[name] = tensor

  def Walk(self):
    """Yields (path, layer) for self and every descendant, depth-first."""
    yield self.path, self
    for c in self._private_children.Flatten():
      if isinstance(c, BaseLayer):
        yield from c.Walk()

  def to(self, device=None, dtype=None):  # pylint: disable=invalid-name
    """Moves all variables in place (Parameters keep identity)."""
    for _, layer in self.Walk():
      for k, v in layer._private_vars.items():  # pylint: disable=protected-access
        with torch.no_grad():
          new = v.data.to(device=device,
                          dtype=dtype if (dtype is not None and
                                          v.is_floating_point()) else None)
        v.data = new
      for acc in layer._private_accumulators.values():  # pylint: disable=protected-access
        if isinstance(acc._value, torch.Tensor):  # pylint: disable=protected-access
          acc._value = acc._value.to(device)  # pylint: disable=protected-access
    return self

  def Device(self) -> torch.device:
    """Device of this layer's (or its descendants') first variable."""
    for _, layer in self.Walk():
      for v in layer._private_vars.values():  # pylint: disable=protected-access
        return v.device
    return py_utils.CurrentDevice()

  def cuda(self, index=None):  # pylint: disable=invalid-name
    return self.to(torch.device('cuda', index if index is not None
                                else torch.cuda.current_device()))

  # ------------------------------------------------------------------- fprop --
  def FProp(self, theta, *args, **kwargs):
    """Forward propagation; `theta` holds this layer's + children's weights."""
    del theta, args, kwargs
    raise NotImplementedError('Abstract method of %s' % self)

  def FPropDefaultTheta(self, *args, **kwargs):
    return self.FProp(self.theta, *args, **kwargs)

  def __call__(self, *args, **kwargs):
    return self.FPropDefaultTheta(*args, **kwargs)

  @classmethod
  def FPropMeta(cls, params, *args, **kwargs):
    """Returns NestedMap(flops=…, out_shapes=(…)) (reference :447)."""
    raise NotImplementedError('FPropMeta of %s' % cls)

  # ------------------------------------------------------------ accumulators --
  def RegisterAccumulator(self, name: str, acc: Accumulator):
    if name in self._private_accumulators:
      raise AttributeError('Accumulator %s already registered' % name)
    self._private_accumulators[name] = acc

  @property
  def accumulators(self) -> NestedMap:
    ret = self._private_children.Transform(
        lambda c: c.accumulators if isinstance(c, BaseLayer) else c)
    for k, acc in self._private_accumulators.items():
      ret[k] = acc
    return ret

  def GetAccumulatorValues(self) -> NestedMap:
    return self.accumulators.Transform(lambda a: a.GetValue())

  def SetAccumulatorValues(self, new_values_nmap: NestedMap):
    accs = self.accumulators.Flatten()
    vals = new_values_nmap.Flatten()
    assert len(accs) == len(vals)
    for a, v in zip(accs, vals):
      a.SetValue(v)

  # ------------------------------------------------------------------ hooks --
  def PostTrainingStepUpdate(self):
    """Returns nothing; children hooks are invoked (reference :1129)."""
    for c in self._private_children.Flatten():
      if isinstance(c, BaseLayer):
        c.PostTrainingStepUpdate()

  def PostEmaUpdate(self):
    for c in self._private_children.Flatten():
      if isinstance(c, BaseLayer):
        c.PostEmaUpdate()

  def AddFunction(self, name: str, fn: Callable, replace: bool = False):
    if not replace and name in self._private_fns:
      raise AttributeError('Function "%s" is already defined on layer "%s"' %
                           (name, self.params.name))
    self._private_fns[name] = fn

  @property
  def fns(self):
    """Read-only view (index or attribute access) of the layer's local functions (ref
    :705)."""
    return py_utils.ReadOnlyAttrDictView(self._private_fns)

  @property
  def ema(self):
    """The EMA shadow map of the task / model this layer belongs to, if any (ref :587)."""
    root = self
    while root.parent is not None:
      root = root.parent
      if getattr(root, '_ema_map', None):
        return root._ema_map   # pylint: disable=protected-access
    return getattr(root, '_ema_map', None)

  def _GetSelfVariablesDict(self):
    return {v.var_name: v for v in self._private_vars.values()}

  def GetVariablesDict(self, visited=None):
    """{variable name: Parameter} of this layer and all its children; shared layers are
    visited once (ref :322)."""
    if visited is None:
      visited = set()
    elif id(self) in visited:
      return {}
    visited.add(id(self))
    res = self._GetSelfVariablesDict()
    for child in self._private_children.Flatten():
      if isinstance(child, BaseLayer):
        res = py_utils.MergeDictsWithValueCheck(res, child.GetVariablesDict(visited))
    return res

  def GetVariableSymbolicShape(self, var_name):
    """Shapes are static here: the symbolic shape of a variable is its shape."""
    return list(self._private_vars[var_name].shape)

  def AddVN(self, value, per_step=False):
    return py_utils.AddVN(self.params, value, per_step)

  def AddGlobalVN(self, theta):
    """Global (per-weight) variational noise on a theta that bypassed `self.theta` — e.g.
    values restored from a checkpoint or produced by another layer (ref :937). `self.theta`
    itself already carries the noise."""
    if self.do_eval:
      return theta
    out = theta.copy() if hasattr(theta, 'copy') else theta
    for name, child in self._private_children.items():
      if name not in theta:
        continue
      if isinstance(child, BaseLayer):
        out[name] = child.AddGlobalVN(theta[name])
      elif isinstance(child, (list, tuple)):
        out[name] = [c.AddGlobalVN(t) if isinstance(c, BaseLayer) else t
                     for c, t in zip(child, theta[name])]
    vn = self.params.vn
    if vn is not None and vn.global_vn:
      for name in self._private_vars:
        if name in theta and isinstance(theta[name], torch.Tensor) and \
            theta[name].is_floating_point():
          out[name] = py_utils.AddVN(self.params, theta[name])
    return out

  def _CastToFPropDtype(self, value):
    def cast(x):
      if isinstance(x, torch.Tensor) and x.is_floating_point() and (
          x.dtype != self.fprop_dtype):
        return x.to(self.fprop_dtype)
      return x
    if isinstance(value, NestedMap):
      return value.Transform(cast)
    if isinstance(value, (list, tuple)):
      return type(value)(cast(v) for v in value)
    return cast(value)

  def __repr__(self):
    return '<%s %s>' % (type(self).__name__, self.__dict__.get('_path', '?'))


class _ScopeFlag(threading.local):

  def __init__(self):
    super().__init__()
    self.depth = 0


_SCOPE_FLAG = _ScopeFlag()


def _ScopeIsManaged() -> bool:
  return _SCOPE_FLAG.depth > 0


@contextlib.contextmanager
def _ManagedScope():
  _SCOPE_FLAG.depth += 1
  try:
    yield
  finally:
    _SCOPE_FLAG.depth -= 1


def IsLayerParams(x) -> bool:
  return (isinstance(x, hyperparams.InstantiableParams) and
          isinstance(x.cls, type) and issubclass(x.cls, BaseLayer))
