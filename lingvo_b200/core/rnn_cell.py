"""RNN cells (ref `lingvo/core/rnn_cell.py`).

Cell contract (ref :37-211): `zero_state(theta, batch_size)` → state NestedMap;
`FProp(theta, state0, inputs)` → `(state1, extras)` with
`inputs = NestedMap(act=[tensor, …], padding=[B, 1])`; `GetOutput(state)`.
Padded batch rows carry their previous state forward.

H100 design: every cell splits its step into
  * `ProjectInput(theta, acts [T, B, D])` — the input half of the gate GEMM,
    hoisted out of the time loop and run ONCE for the whole sequence on the
    tensor cores, and
  * `_Step(theta, state0, xw_t, padding)` — the recurrent half (`h·W_h` +
    pointwise gates), the only work left inside the loop.
`FProp` (single step, reference semantics) composes the two.
Variable names/shapes follow the reference (`wm [in+out, 4·hidden]`, `b`,
`w_proj`) so checkpoints line up.
"""

from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from lingvo_b200.core import base_layer
from lingvo_b200.core import py_utils
from lingvo_b200.core import quant_utils
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.core.py_utils import WeightInit
from lingvo_b200.core.py_utils import WeightParams


def _ZoneOut(prev_v, cur_v, padding_v, zo_prob, is_eval, random_uniform=None):
  """Zoneout + padding carry-over (ref :100-140)."""
  if zo_prob > 0.0:
    if is_eval:
      cur_v = zo_prob * prev_v + (1.0 - zo_prob) * cur_v
    else:
      ru = random_uniform if random_uniform is not None else torch.rand_like(cur_v)
      cur_v = torch.where(ru < zo_prob, prev_v, cur_v)
  if padding_v is None:
    return cur_v
  return torch.where(padding_v > 0, prev_v, cur_v)


class RNNCell(quant_utils.QuantizableLayer):
  """Base cell (ref :37)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('inputs_arity', 1, 'Number of tensors in inputs.act.')
    p.Define('num_input_nodes', 0, 'Total input width.')
    p.Define('num_output_nodes', 0, 'Output (m) width.')
    p.Define('reset_cell_state', False, 'Reset state where inputs.reset_mask == 0.')
    p.Define('zo_prob', 0.0, 'Zoneout probability.')
    p.Define('zero_state_init_params', py_utils.DefaultRNNCellStateInit(),
             'How zero_state draws the initial state (py_utils.RNNCellStateInit).')
    return p

  def _InitState(self, shape, name):
    p = self.params
    return py_utils.InitRNNCellState(
        shape, init=p.zero_state_init_params, dtype=py_utils.FPropDtype(p),
        name='%s/%s' % (self.path, name), is_eval=self.do_eval, device=self.Device())

  def _Act(self, inputs):
    act = inputs.act
    if isinstance(act, (list, tuple)):
      return act[0] if len(act) == 1 else torch.cat(list(act), -1)
    return act

  def _ResetState(self, state, inputs):
    """Packed inputs: zero the state at segment starts (reset_mask == 0)."""
    if self.params.reset_cell_state and inputs.get('reset_mask') is not None:
      return state.Transform(lambda x: x * inputs.reset_mask.to(x.dtype))
    return state

  def zero_state(self, theta, batch_size):
    raise NotImplementedError

  def GetOutput(self, state):
    raise NotImplementedError

  @property
  def output_size(self):
    """Width of `GetOutput(state)`."""
    return self.params.num_output_nodes

  @staticmethod
  def LayerNorm(x, scale=None, bias=None, epsilon=1e-6):
    """Mean/variance normalisation over the last axis, `(1 + scale)`-gained (the cells'
    layer-norm convention)."""
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    y = (x - mean) * torch.rsqrt(var + epsilon)
    if scale is not None:
      y = y * (1.0 + scale)
    if bias is not None:
      y = y + bias
    return y

  def batch_size(self, inputs):
    return self._Act(inputs).shape[0]

  # -- hoisting protocol --------------------------------------------------------
  def ProjectInput(self, theta, acts):
    """Input half of the step for a whole sequence `[T, B, D]` → `[T, B, G]`."""
    raise NotImplementedError

  def _Step(self, theta, state0, xw, padding, inputs=None):
    raise NotImplementedError

  def FProp(self, theta, state0, inputs):
    state0 = self._ResetState(state0, inputs)
    xw = self.ProjectInput(theta, self._Act(inputs).unsqueeze(0))[0]
    state1 = self._Step(theta, state0, xw, inputs.get('padding'), inputs)
    return state1, NestedMap()


class LSTMCellSimple(RNNCell):
  """LSTM; gates ordered (i_i, i_g, f_g, o_g) along `wm`'s columns (ref :213)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_hidden_nodes', 0, 'Cell width when a projection is used.')
    p.Define('cell_value_cap', 10.0, 'Clip |c| (None: no clip).')
    p.Define('forget_gate_bias', 0.0, 'Added to the forget gate.')
    p.Define('output_nonlinearity', True, 'm = o·tanh(c) (else o·c).')
    p.Define('enable_lstm_bias', True, 'Use the bias vector.')
    p.Define('couple_input_forget_gates', False, 'i = 1 − f (3 gates).')
    p.Define('apply_pruning', False, 'Kept for parity.')
    p.Define('apply_pruning_to_projection', False, 'Kept for parity.')
    p.Define('gradient_pruning', False, 'Kept for parity.')
    p.Define('bias_init', WeightInit.Constant(0.0), 'Bias initialiser.')
    p.Define('pruning_hparams_dict', None, 'Kept for parity.')
    p.Define('no_wm_if_compress', False, 'Kept for parity.')
    p.Define('deterministic', False, 'Kept for parity (seeded zoneout).')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.num_input_nodes > 0 and p.num_output_nodes > 0

  @property
  def hidden_size(self):
    return self.params.num_hidden_nodes or self.params.num_output_nodes

  @property
  def num_gates(self):
    return 3 if self.params.couple_input_forget_gates else 4

  def _CreateLayerVariables(self):
    p = self.params
    coll = [self.__class__.__name__ + '_vars']
    self.CreateVariable('wm', WeightParams(
        [p.num_input_nodes + p.num_output_nodes, self.num_gates * self.hidden_size],
        p.params_init, p.dtype, coll))
    if p.num_hidden_nodes:
      self.CreateVariable('w_proj', WeightParams(
          [p.num_hidden_nodes, p.num_output_nodes], p.params_init, p.dtype, coll))
    if p.enable_lstm_bias:
      self.CreateVariable('b', WeightParams(
          [self.num_gates * self.hidden_size], p.bias_init, p.dtype, coll))

  def zero_state(self, theta, batch_size):
    p = self.params
    return NestedMap(m=self._InitState([batch_size, p.num_output_nodes], 'zero_m'),
                     c=self._InitState([batch_size, self.hidden_size], 'zero_c'))

  def GetOutput(self, state):
    return state.m

  def _Bias(self, theta):
    p = self.params
    if not p.enable_lstm_bias:
      return None
    b = theta.b
    if p.forget_gate_bias != 0.0:
      h = self.hidden_size
      adj = torch.zeros_like(b)
      f_idx = 1 if p.couple_input_forget_gates else 2
      adj[f_idx * h:(f_idx + 1) * h] = p.forget_gate_bias
      b = b + adj
    return b

  def ProjectInput(self, theta, acts):
    p = self.params
    w_x = theta.wm[:p.num_input_nodes].to(acts.dtype)
    xw = torch.matmul(acts, w_x)
    b = self._Bias(theta)
    return xw + b.to(xw.dtype) if b is not None else xw

  def _Normalize(self, theta, gates):
    return gates

  def _ProcessNewC(self, theta, new_c):
    return new_c

  def _Step(self, theta, state0, xw, padding, inputs=None):
    p = self.params
    w_h = theta.wm[p.num_input_nodes:].to(xw.dtype)
    gates = xw + torch.matmul(state0.m.to(xw.dtype), w_h)
    gates = self._Normalize(theta, gates)
    if p.couple_input_forget_gates:
      i_i, f_g, o_g = gates.chunk(3, -1)
      f = torch.sigmoid(f_g)
      new_c = f * state0.c + (1.0 - f) * torch.tanh(i_i)
    else:
      i_i, i_g, f_g, o_g = gates.chunk(4, -1)
      new_c = torch.sigmoid(f_g) * state0.c + torch.sigmoid(i_g) * torch.tanh(i_i)
    new_c = self._ProcessNewC(theta, new_c)
    if p.cell_value_cap is not None:
      new_c = new_c.clamp(-p.cell_value_cap, p.cell_value_cap)
    new_m = torch.sigmoid(o_g) * (torch.tanh(new_c) if p.output_nonlinearity else new_c)
    if p.num_hidden_nodes:
      new_m = torch.matmul(new_m, theta.w_proj.to(new_m.dtype))
    new_c = _ZoneOut(state0.c, new_c, padding, p.zo_prob, self.do_eval)
    new_m = _ZoneOut(state0.m, new_m, padding, p.zo_prob, self.do_eval)
    return NestedMap(m=new_m, c=new_c)


class LSTMCellGrouped(RNNCell):
  """`num_groups` independent LSTMs over feature slices + optional shuffle (ref :735)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_hidden_nodes', 0, 'Total hidden nodes (0: == output).')
    p.Define('num_groups', 1, 'Number of groups.')
    p.Define('num_shuffle_shards', 1, 'Shuffle shards applied to the output.')
    p.Define('child_lstm_tpl', LSTMCellSimple.Params(), 'Per-group cell.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    g = p.num_groups
    assert p.num_input_nodes % g == 0 and p.num_output_nodes % g == 0
    kids = []
    for i in range(g):
      kids.append(p.child_lstm_tpl.Copy().Set(
          name='group_%d' % i, num_input_nodes=p.num_input_nodes // g,
          num_output_nodes=p.num_output_nodes // g,
          num_hidden_nodes=(p.num_hidden_nodes // g) if p.num_hidden_nodes else 0,
          reset_cell_state=p.reset_cell_state))
    self.CreateChildren('groups', kids)

  def zero_state(self, theta, batch_size):
    st = [c.zero_state(theta.groups[i], batch_size) for i, c in enumerate(self.groups)]
    return NestedMap(m=torch.cat([s.m for s in st], -1), c=torch.cat([s.c for s in st], -1))

  def GetOutput(self, state):
    return state.m

  def FProp(self, theta, state0, inputs):
    p = self.params
    g = p.num_groups
    acts = self._Act(inputs).chunk(g, -1)
    ms, cs = state0.m.chunk(g, -1), state0.c.chunk(g, -1)
    out_m, out_c = [], []
    for i, cell in enumerate(self.groups):
      sub_in = NestedMap(act=[acts[i]], padding=inputs.get('padding'))
      if inputs.get('reset_mask') is not None:
        sub_in.reset_mask = inputs.reset_mask
      s1, _ = cell.FProp(theta.groups[i], NestedMap(m=ms[i], c=cs[i]), sub_in)
      out_m.append(s1.m)
      out_c.append(s1.c)
    m = torch.cat(out_m, -1)
    if p.num_shuffle_shards > 1:
      b = m.shape[0]
      m = m.reshape(b, p.num_shuffle_shards, -1).transpose(1, 2).reshape(b, -1)
    return NestedMap(m=m, c=torch.cat(out_c, -1)), NestedMap()


class LayerNormalizedLSTMCellSimple(LSTMCellSimple):
  """LN on each gate pre-activation and on the new cell (ref :1283)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('layer_norm_epsilon', 1e-8, 'LN epsilon.')
    return p

  def _CreateLayerVariables(self):
    super()._CreateLayerVariables()
    p = self.params
    self.CreateVariable('ln_scale', WeightParams(
        [self.num_gates * self.hidden_size], WeightInit.Constant(1.0), p.dtype))

  def _LN(self, x, eps):
    xf = x.float()
    mean = xf.mean(-1, keepdim=True)
    var = ((xf - mean) ** 2).mean(-1, keepdim=True)
    return ((xf - mean) * torch.rsqrt(var + eps)).to(x.dtype)

  def ProjectInput(self, theta, acts):
    p = self.params
    return torch.matmul(acts, theta.wm[:p.num_input_nodes].to(acts.dtype))

  def _Normalize(self, theta, gates):
    p = self.params
    h = self.hidden_size
    n = self.num_gates
    g = self._LN(gates.reshape(*gates.shape[:-1], n, h), p.layer_norm_epsilon)
    g = g.reshape(*gates.shape) * theta.ln_scale.to(gates.dtype)
    b = self._Bias(theta)
    return g + b.to(g.dtype) if b is not None else g

  def _ProcessNewC(self, theta, new_c):
    return self._LN(new_c, self.params.layer_norm_epsilon)


class WeightNormalizedLSTMCellSimple(LSTMCellSimple):
  """`wm` columns are re-normalised: w·g/‖w‖ (ref :1377)."""

  def _CreateLayerVariables(self):
    super()._CreateLayerVariables()
    p = self.params
    self.CreateVariable('wn_scale', WeightParams(
        [self.num_gates * self.hidden_size], WeightInit.Constant(0.0), p.dtype))

  def _Wm(self, theta):
    w = theta.wm
    return F.normalize(w.float(), dim=0).to(w.dtype) * (1.0 + theta.wn_scale)

  def ProjectInput(self, theta, acts):
    p = self.params
    xw = torch.matmul(acts, self._Wm(theta)[:p.num_input_nodes].to(acts.dtype))
    b = self._Bias(theta)
    return xw + b.to(xw.dtype) if b is not None else xw

  def _Step(self, theta, state0, xw, padding, inputs=None):
    th = theta.copy() if hasattr(theta, 'copy') else theta
    th = NestedMap(th)
    th.wm = self._Wm(theta)
    return super()._Step(th, state0, xw, padding, inputs)


class NormalizedLSTMCellSimple(LSTMCellSimple):
  """LSTM whose gate pre-activations each go through a configurable normalisation layer
  (`norm_layer_tpl`, children `norm_i_i / norm_i_g / norm_f_g / norm_o_g`) (ref :1438).
  Requires `enable_lstm_bias=False` and `forget_gate_bias=0` (the norm layers own the
  affine terms)."""

  _GATES = ('i_i', 'i_g', 'f_g', 'o_g')

  @classmethod
  def Params(cls):
    from lingvo_b200.core import layers   # pylint: disable=g-import-not-at-top
    p = super().Params()
    p.Define('norm_layer_tpl', layers.LayerNorm.Params().Set(epsilon=1e-8),
             'The normalization layer params.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.forget_gate_bias == 0.0
    assert not p.enable_lstm_bias
    for gate in self._GATES:
      self.CreateChild('norm_' + gate, p.norm_layer_tpl.Copy().Set(
          name='norm_' + gate, input_dim=self.hidden_size))

  def _Normalize(self, theta, gates):
    p = self.params
    parts = list(gates.chunk(self.num_gates, -1))
    names = ('i_i', 'f_g', 'o_g') if p.couple_input_forget_gates else self._GATES
    out = [self.children['norm_' + n].FProp(theta['norm_' + n], x)
           for n, x in zip(names, parts)]
    return torch.cat(out, -1)


class LayerNormalizedLSTMCell(RNNCell):
  """The original (deprecated in the reference) layer-normalised LSTM (ref :1010): LN on each
  of the four gate pre-activations with scale `1 + ln_scale` and bias, both packed in one
  vector `b` of size 8·H = [4 gate biases | 4 LN scales]; optional clipping-cap schedule for
  the cell value."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('cell_value_cap', 10.0, 'Cell values are capped to ±cap (python number).')
    p.Define('forget_gate_bias', 0.0, 'Bias to apply to the forget gate.')
    p.Define('output_nonlinearity', True, 'm = o·tanh(c) (else o·c).')
    p.Define('layer_norm_epsilon', 1e-8, 'Tiny value to guard rsqrt.')
    p.Define('cc_schedule', None, 'Clipping cap schedule (overrides cell_value_cap).')
    p.Define('use_fused_layernorm', False, 'Kept for parity: one fused LN expression is used '
             'either way.')
    p.Define('pruning_hparams_dict', None, 'Kept for parity.')
    p.Define('apply_pruning', False, 'Multiply wm by a (non-trainable) `mask` variable.')
    p.Define('no_wm_if_compress', False, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    if not isinstance(p.cell_value_cap, (int, float)):
      raise ValueError('Cell value cap must be of type int or float!')
    assert p.num_input_nodes > 0 and p.num_output_nodes > 0
    if p.cc_schedule is not None:
      self.CreateChild('cc_schedule', p.cc_schedule)
    self.TrackQWeight('wm', shape=[p.num_input_nodes + p.num_output_nodes,
                                   4 * p.num_output_nodes], feature_axis=-1)

  @property
  def output_size(self):
    return self.params.num_output_nodes

  hidden_size = output_size

  def _CreateLayerVariables(self):
    p = self.params
    shape = [p.num_input_nodes + p.num_output_nodes, 4 * p.num_output_nodes]
    self.CreateVariable('wm', WeightParams(shape, p.params_init, p.dtype))
    if p.apply_pruning:
      self.CreateVariable('mask', WeightParams(shape, WeightInit.Constant(1.0), p.dtype),
                          trainable=False)
      self.CreateVariable('threshold', WeightParams([], WeightInit.Constant(0.0), p.dtype),
                          trainable=False)
    self.CreateVariable('b', WeightParams([8 * p.num_output_nodes], WeightInit.Constant(0.0),
                                          p.dtype))

  def zero_state(self, theta, batch_size):
    p = self.params
    dev, dt = self.Device(), py_utils.FPropDtype(p)
    return NestedMap(m=torch.zeros(batch_size, p.num_output_nodes, device=dev, dtype=dt),
                     c=torch.zeros(batch_size, p.num_output_nodes, device=dev, dtype=dt))

  def GetOutput(self, state):
    return state.m

  def _ResetState(self, state, inputs):
    if inputs.get('reset_mask') is not None:
      return state.Transform(lambda x: x * inputs.reset_mask.to(x.dtype))
    return state

  def _Wm(self, theta):
    w = theta.wm
    if self.params.apply_pruning:
      w = self.QWeight(w * theta.mask)
    return w

  def ProjectInput(self, theta, acts):
    p = self.params
    return torch.matmul(acts, self._Wm(theta)[:p.num_input_nodes].to(acts.dtype))

  def _Step(self, theta, state0, xw, padding, inputs=None):
    p = self.params
    h = p.num_output_nodes
    gates = xw + torch.matmul(state0.m.to(xw.dtype), self._Wm(theta)[p.num_input_nodes:].to(
        xw.dtype))
    g = gates.float().reshape(-1, 4, h)
    mean = g.mean(-1, keepdim=True)
    var = (g - mean).square().mean(-1, keepdim=True)
    bias = theta.b[:4 * h].float().reshape(4, h)
    scale = theta.b[4 * h:].float().reshape(4, h) + 1.0
    g = ((g - mean) * torch.rsqrt(var + p.layer_norm_epsilon) * scale + bias).to(xw.dtype)
    i_i, i_g, f_g, o_g = g.unbind(1)
    if p.forget_gate_bias != 0.0:
      f_g = f_g + p.forget_gate_bias
    new_c = torch.sigmoid(f_g) * state0.c + torch.sigmoid(i_g) * torch.tanh(i_i)
    if p.cc_schedule is not None:
      cap = self.cc_schedule.GetState(theta.cc_schedule).to(device=new_c.device,
                                                            dtype=new_c.dtype)
      new_c = torch.maximum(torch.minimum(new_c, cap), -cap)
    else:
      new_c = new_c.clamp(-p.cell_value_cap, p.cell_value_cap)
    new_m = torch.sigmoid(o_g) * (torch.tanh(new_c) if p.output_nonlinearity else new_c)
    new_c = _ZoneOut(state0.c, new_c, padding, p.zo_prob, self.do_eval)
    new_m = _ZoneOut(state0.m, new_m, padding, p.zo_prob, self.do_eval)
    return NestedMap(m=new_m, c=new_c)


class LayerNormalizedLSTMCellLean(RNNCell):
  """Lean LN-LSTM: LN per gate (4 separate scale/bias pairs) + LN on c (ref :1495)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_hidden_nodes', 0, 'Cell width when projecting.')
    p.Define('output_nonlinearity', True, 'm = o·tanh(c).')
    p.Define('layer_norm_epsilon', 1e-8, 'LN epsilon.')
    p.Define('cell_value_cap', 10.0, 'Clip |c|.')
    p.Define('enable_ln_on_c', True, 'LN on the new cell before the output gate.')
    p.Define('use_ln_bias', True, 'LN biases.')
    p.Define('enable_lstm_bias', False, 'Kept for parity.')
    p.Define('forget_gate_bias', 0.0, 'Kept for parity.')
    return p

  @property
  def hidden_size(self):
    return self.params.num_hidden_nodes or self.params.num_output_nodes

  def _CreateLayerVariables(self):
    p = self.params
    h = self.hidden_size
    self.CreateVariable('wm', WeightParams(
        [p.num_input_nodes + p.num_output_nodes, 4 * h], p.params_init, p.dtype))
    if p.num_hidden_nodes:
      self.CreateVariable('w_proj', WeightParams(
          [p.num_hidden_nodes, p.num_output_nodes], p.params_init, p.dtype))
    names = ['i_i', 'i_g', 'f_g', 'o_g'] + (['c'] if p.enable_ln_on_c else [])
    for n in names:
      self.CreateVariable('ln_scale_' + n, WeightParams([h], WeightInit.Constant(1.0), p.dtype))
      if p.use_ln_bias:
        self.CreateVariable('bias_' + n, WeightParams([h], WeightInit.Constant(0.0), p.dtype))

  def zero_state(self, theta, batch_size):
    p = self.params
    dev, dt = self.Device(), py_utils.FPropDtype(p)
    return NestedMap(m=torch.zeros(batch_size, p.num_output_nodes, device=dev, dtype=dt),
                     c=torch.zeros(batch_size, self.hidden_size, device=dev, dtype=dt))

  def GetOutput(self, state):
    return state.m

  def ProjectInput(self, theta, acts):
    return torch.matmul(acts, theta.wm[:self.params.num_input_nodes].to(acts.dtype))

  def _LN(self, theta, x, name):
    p = self.params
    xf = x.float()
    mean = xf.mean(-1, keepdim=True)
    var = ((xf - mean) ** 2).mean(-1, keepdim=True)
    y = (xf - mean) * torch.rsqrt(var + p.layer_norm_epsilon) * theta['ln_scale_' + name].float()
    if p.use_ln_bias:
      y = y + theta['bias_' + name].float()
    return y.to(x.dtype)

  def _Step(self, theta, state0, xw, padding, inputs=None):
    p = self.params
    gates = xw + torch.matmul(state0.m.to(xw.dtype),
                              theta.wm[p.num_input_nodes:].to(xw.dtype))
    i_i, i_g, f_g, o_g = gates.chunk(4, -1)
    i_i = torch.tanh(self._LN(theta, i_i, 'i_i'))
    i_g = torch.sigmoid(self._LN(theta, i_g, 'i_g'))
    f_g = torch.sigmoid(self._LN(theta, f_g, 'f_g'))
    o_g = torch.sigmoid(self._LN(theta, o_g, 'o_g'))
    new_c = f_g * state0.c + i_g * i_i
    if p.cell_value_cap is not None:
      new_c = new_c.clamp(-p.cell_value_cap, p.cell_value_cap)
    c_out = self._LN(theta, new_c, 'c') if p.enable_ln_on_c else new_c
    new_m = o_g * (torch.tanh(c_out) if p.output_nonlinearity else c_out)
    if p.num_hidden_nodes:
      new_m = torch.matmul(new_m, theta.w_proj.to(new_m.dtype))
    new_c = _ZoneOut(state0.c, new_c, padding, p.zo_prob, self.do_eval)
    new_m = _ZoneOut(state0.m, new_m, padding, p.zo_prob, self.do_eval)
    return NestedMap(m=new_m, c=new_c)


class DoubleProjectionLSTMCell(LayerNormalizedLSTMCellLean):
  """Projects the input down before the gates and the output after (ref :1838)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_input_hidden_nodes', 0, 'Width of the input projection.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    if p.num_input_hidden_nodes:
      self.CreateVariable('w_input_proj', WeightParams(
          [p.num_input_nodes, p.num_input_hidden_nodes], p.params_init, p.dtype))
    real_in = p.num_input_nodes
    p_in = p.num_input_hidden_nodes or real_in
    self._proj_in = p_in
    h = self.hidden_size
    self.CreateVariable('wm', WeightParams(
        [p_in + p.num_output_nodes, 4 * h], p.params_init, p.dtype))
    if p.num_hidden_nodes:
      self.CreateVariable('w_proj', WeightParams(
          [p.num_hidden_nodes, p.num_output_nodes], p.params_init, p.dtype))
    names = ['i_i', 'i_g', 'f_g', 'o_g'] + (['c'] if p.enable_ln_on_c else [])
    for n in names:
      self.CreateVariable('ln_scale_' + n, WeightParams([h], WeightInit.Constant(1.0), p.dtype))
      if p.use_ln_bias:
        self.CreateVariable('bias_' + n, WeightParams([h], WeightInit.Constant(0.0), p.dtype))

  def ProjectInput(self, theta, acts):
    p = self.params
    if p.num_input_hidden_nodes:
      acts = torch.matmul(acts, theta.w_input_proj.to(acts.dtype))
    return torch.matmul(acts, theta.wm[:self._proj_in].to(acts.dtype))

  def _Step(self, theta, state0, xw, padding, inputs=None):
    p = self.params
    gates_w = theta.wm[self._proj_in:]   # recurrent rows follow the projected-input rows
    gates = xw + torch.matmul(state0.m.to(xw.dtype), gates_w.to(xw.dtype))
    i_i, i_g, f_g, o_g = gates.chunk(4, -1)
    i_i = torch.tanh(self._LN(theta, i_i, 'i_i'))
    i_g = torch.sigmoid(self._LN(theta, i_g, 'i_g'))
    f_g = torch.sigmoid(self._LN(theta, f_g, 'f_g'))
    o_g = torch.sigmoid(self._LN(theta, o_g, 'o_g'))
    new_c = f_g * state0.c + i_g * i_i
    if p.cell_value_cap is not None:
      new_c = new_c.clamp(-p.cell_value_cap, p.cell_value_cap)
    c_out = self._LN(theta, new_c, 'c') if p.enable_ln_on_c else new_c
    new_m = o_g * (torch.tanh(c_out) if p.output_nonlinearity else c_out)
    if p.num_hidden_nodes:
      new_m = torch.matmul(new_m, theta.w_proj.to(new_m.dtype))
    new_c = _ZoneOut(state0.c, new_c, padding, p.zo_prob, self.do_eval)
    new_m = _ZoneOut(state0.m, new_m, padding, p.zo_prob, self.do_eval)
    return NestedMap(m=new_m, c=new_c)


class QuantizedLSTMCell(LSTMCellSimple):
  """LSTM whose cell state is clipped/fake-quantised to ±cc (ref :900)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('cc_schedule', None, 'Clipping-cap schedule layer params.')
    p.enable_lstm_bias = False
    p.cell_value_cap = None
    return p

  def __init__(self, params):
    super().__init__(params)
    if self.params.cc_schedule is not None:
      self.CreateChild('cc_schedule', self.params.cc_schedule)

  def _ProcessNewC(self, theta, new_c):
    if self.params.cc_schedule is not None:
      return self.cc_schedule.ApplyClipping(theta.cc_schedule, new_c)
    return new_c


class ConvLSTMCell(RNNCell):
  """Convolutional LSTM over `[B, H, W, C]` states (ref :2015)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('inputs_shape', [None, None, None, None], '[B, H, W, Cin].')
    p.Define('cell_shape', [None, None, None, None], '[B, H, W, Cout].')
    p.Define('filter_shape', [3, 3], 'Conv kernel.')
    p.Define('cell_value_cap', 10.0, 'Clip |c|.')
    p.Define('output_nonlinearity', True, 'm = o·tanh(c).')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    cin, cout = p.inputs_shape[3], p.cell_shape[3]
    self.CreateVariable('wm', WeightParams(
        list(p.filter_shape) + [cin + cout, 4 * cout], p.params_init, p.dtype))
    self.CreateVariable('b', WeightParams([4 * cout], WeightInit.Constant(0.0), p.dtype))

  def zero_state(self, theta, batch_size):
    p = self.params
    shape = [batch_size] + list(p.cell_shape[1:])
    dev, dt = self.Device(), py_utils.FPropDtype(p)
    return NestedMap(m=torch.zeros(shape, device=dev, dtype=dt),
                     c=torch.zeros(shape, device=dev, dtype=dt))

  def GetOutput(self, state):
    return state.m

  def FProp(self, theta, state0, inputs):
    p = self.params
    x = torch.cat([self._Act(inputs), state0.m], -1).permute(0, 3, 1, 2)   # NCHW
    w = theta.wm.permute(3, 2, 0, 1).to(x.dtype)
    kh, kw = p.filter_shape
    g = F.conv2d(x, w, theta.b.to(x.dtype), padding=(kh // 2, kw // 2)).permute(0, 2, 3, 1)
    i_i, i_g, f_g, o_g = g.chunk(4, -1)
    new_c = torch.sigmoid(f_g) * state0.c + torch.sigmoid(i_g) * torch.tanh(i_i)
    if p.cell_value_cap is not None:
      new_c = new_c.clamp(-p.cell_value_cap, p.cell_value_cap)
    new_m = torch.sigmoid(o_g) * (torch.tanh(new_c) if p.output_nonlinearity else new_c)
    pad = inputs.get('padding')
    if pad is not None:
      pad = pad.reshape(-1, 1, 1, 1)
    new_c = _ZoneOut(state0.c, new_c, pad, p.zo_prob, self.do_eval)
    new_m = _ZoneOut(state0.m, new_m, pad, p.zo_prob, self.do_eval)
    return NestedMap(m=new_m, c=new_c), NestedMap()


class SRUCell(RNNCell):
  """Simple Recurrent Unit: all matmuls depend only on the input, the recurrence
  is element-wise (ref :2174) — the whole GEMM is hoisted."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_hidden_nodes', 0, 'Cell width when projecting.')
    p.Define('cell_value_cap', 10.0, 'Clip |c|.')
    p.Define('couple_input_forget_gates', True, 'i = 1 − f.')
    p.Define('apply_layer_norm', False, 'LN on the pre-activations.')
    p.Define('layer_norm_epsilon', 1e-8, 'LN eps.')
    p.Define('bias_init', WeightInit.Constant(0.0), 'Bias init.')
    p.Define('pointwise_peephole', False, 'c-dependent peepholes on f and r.')
    p.Define('apply_pruning', False, 'Kept for parity.')
    p.Define('apply_pruning_to_projection', False, 'Kept for parity.')
    p.Define('gradient_pruning', False, 'Kept for parity.')
    return p

  @property
  def hidden_size(self):
    return self.params.num_hidden_nodes or self.params.num_output_nodes

  @property
  def num_gates(self):
    return 4 if self.params.couple_input_forget_gates else 5

  def _CreateLayerVariables(self):
    p = self.params
    h, n = self.hidden_size, self.num_gates
    self.CreateVariable('wm', WeightParams([p.num_input_nodes, n * h], p.params_init, p.dtype))
    self.CreateVariable('b', WeightParams([n * h], p.bias_init, p.dtype))
    if p.num_hidden_nodes:
      self.CreateVariable('w_proj', WeightParams(
          [p.num_hidden_nodes, p.num_output_nodes], p.params_init, p.dtype))
    if p.pointwise_peephole:
      self.CreateVariable('f_peephole', WeightParams([h], p.params_init, p.dtype))
      self.CreateVariable('r_peephole', WeightParams([h], p.params_init, p.dtype))
    if p.apply_layer_norm:
      for g in ['x', 'resized', 'f', 'r'] + ([] if p.couple_input_forget_gates else ['i']):
        self.CreateVariable('ln_scale_' + g, WeightParams([h], WeightInit.Constant(1.0), p.dtype))

  def zero_state(self, theta, batch_size):
    p = self.params
    dev, dt = self.Device(), py_utils.FPropDtype(p)
    return NestedMap(m=torch.zeros(batch_size, p.num_output_nodes, device=dev, dtype=dt),
                     c=torch.zeros(batch_size, self.hidden_size, device=dev, dtype=dt))

  def GetOutput(self, state):
    return state.m

  def ProjectInput(self, theta, acts):
    return torch.matmul(acts, theta.wm.to(acts.dtype)) + theta.b.to(acts.dtype)

  def _LN(self, theta, x, name):
    p = self.params
    if not p.apply_layer_norm:
      return x
    xf = x.float()
    mean = xf.mean(-1, keepdim=True)
    var = ((xf - mean) ** 2).mean(-1, keepdim=True)
    return ((xf - mean) * torch.rsqrt(var + p.layer_norm_epsilon) *
            theta['ln_scale_' + name].float()).to(x.dtype)

  def _Step(self, theta, state0, xw, padding, inputs=None):
    p = self.params
    parts = xw.chunk(self.num_gates, -1)
    if p.couple_input_forget_gates:
      x_g, resized, f_g, r_g = parts
      i_g = None
    else:
      x_g, resized, i_g, f_g, r_g = parts
    x_g = self._LN(theta, x_g, 'x')
    resized = self._LN(theta, resized, 'resized')
    f_g = self._LN(theta, f_g, 'f')
    r_g = self._LN(theta, r_g, 'r')
    if p.pointwise_peephole:
      f_g = f_g + theta.f_peephole.to(f_g.dtype) * state0.c
      r_g = r_g + theta.r_peephole.to(r_g.dtype) * state0.c
    f = torch.sigmoid(f_g)
    if i_g is None:
      new_c = f * state0.c + (1.0 - f) * x_g
    else:
      new_c = f * state0.c + torch.sigmoid(self._LN(theta, i_g, 'i')) * x_g
    if p.cell_value_cap is not None:
      new_c = new_c.clamp(-p.cell_value_cap, p.cell_value_cap)
    r = torch.sigmoid(r_g)
    new_m = r * torch.tanh(new_c) + (1.0 - r) * resized
    if p.num_hidden_nodes:
      new_m = torch.matmul(new_m, theta.w_proj.to(new_m.dtype))
    new_c = _ZoneOut(state0.c, new_c, padding, p.zo_prob, self.do_eval)
    new_m = _ZoneOut(state0.m, new_m, padding, p.zo_prob, self.do_eval)
    return NestedMap(m=new_m, c=new_c)


class QRNNPoolingCell(RNNCell):
  """Pooling half of a quasi-RNN; inputs.act already holds the gates (ref :2554)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('cell_value_cap', 10.0, 'Clip |c|.')
    p.Define('pooling_formula', 'INVALID', 'f | fo | ifo | quasi_ifo.')
    return p

  def __init__(self, params):
    super().__init__(params)
    assert self.params.pooling_formula in ('f', 'fo', 'ifo', 'quasi_ifo')

  def zero_state(self, theta, batch_size):
    p = self.params
    dev, dt = self.Device(), py_utils.FPropDtype(p)
    z = torch.zeros(batch_size, p.num_output_nodes, device=dev, dtype=dt)
    return NestedMap(m=z, c=z.clone())

  def GetOutput(self, state):
    return state.m

  def FProp(self, theta, state0, inputs):
    p = self.params
    act = self._Act(inputs)
    f = p.pooling_formula
    if f in ('ifo', 'quasi_ifo'):
      z, i_g, f_g, o_g = act.chunk(4, -1)
      z = torch.tanh(z)
      f_s = torch.sigmoid(f_g)
      i_s = (1.0 - f_s) if f == 'quasi_ifo' else torch.sigmoid(i_g)
      new_c = f_s * state0.c + i_s * z
      new_m = torch.sigmoid(o_g) * new_c
    elif f == 'fo':
      z, f_g, o_g = act.chunk(3, -1)
      f_s = torch.sigmoid(f_g)
      new_c = f_s * state0.c + (1.0 - f_s) * torch.tanh(z)
      new_m = torch.sigmoid(o_g) * new_c
    else:
      z, f_g = act.chunk(2, -1)
      f_s = torch.sigmoid(f_g)
      new_c = f_s * state0.c + (1.0 - f_s) * torch.tanh(z)
      new_m = new_c
    if p.cell_value_cap is not None:
      new_c = new_c.clamp(-p.cell_value_cap, p.cell_value_cap)
    pad = inputs.get('padding')
    new_c = _ZoneOut(state0.c, new_c, pad, p.zo_prob, self.do_eval)
    new_m = _ZoneOut(state0.m, new_m, pad, p.zo_prob, self.do_eval)
    return NestedMap(m=new_m, c=new_c), NestedMap()


class GRUCell(RNNCell):
  """GRU with optional LN and output projection (ref :2683).

  Variables: `w_n, w_u, w_r` each `[in+out, hidden]` (candidate / update /
  reset), `b_n, b_u, b_r`.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_hidden_nodes', 0, 'Hidden width (0: == output).')
    p.Define('cell_value_cap', 10.0, 'Clip the new state.')
    p.Define('enable_gru_bias', False, 'Use biases.')
    p.Define('bias_init', WeightInit.Constant(0.0), 'Bias init.')
    p.Define('apply_layer_norm', True, 'LN on gate pre-activations.')
    p.Define('layer_norm_epsilon', 1e-8, 'LN eps.')
    return p

  @property
  def hidden_size(self):
    return self.params.num_hidden_nodes or self.params.num_output_nodes

  def _CreateLayerVariables(self):
    p = self.params
    h = self.hidden_size
    io = p.num_input_nodes + p.num_output_nodes
    self.CreateVariable('w_n', WeightParams([io, h], p.params_init, p.dtype))
    self.CreateVariable('w_u', WeightParams([io, h], p.params_init, p.dtype))
    self.CreateVariable('w_r', WeightParams([io, p.num_output_nodes], p.params_init, p.dtype))
    if p.num_hidden_nodes:
      self.CreateVariable('w_proj', WeightParams(
          [p.num_hidden_nodes, p.num_output_nodes], p.params_init, p.dtype))
    if p.enable_gru_bias:
      self.CreateVariable('b_n', WeightParams([h], p.bias_init, p.dtype))
      self.CreateVariable('b_u', WeightParams([h], p.bias_init, p.dtype))
      self.CreateVariable('b_r', WeightParams([p.num_output_nodes], p.bias_init, p.dtype))
    if p.apply_layer_norm:
      for n, d in (('n', h), ('u', h), ('r', p.num_output_nodes)):
        self.CreateVariable('ln_scale_' + n, WeightParams([d], WeightInit.Constant(1.0), p.dtype))

  def zero_state(self, theta, batch_size):
    p = self.params
    dev, dt = self.Device(), py_utils.FPropDtype(p)
    return NestedMap(m=torch.zeros(batch_size, p.num_output_nodes, device=dev, dtype=dt),
                     c=torch.zeros(batch_size, self.hidden_size, device=dev, dtype=dt))

  def GetOutput(self, state):
    return state.m

  def _Gate(self, theta, name, x):
    p = self.params
    y = torch.matmul(x, theta['w_' + name].to(x.dtype))
    if p.apply_layer_norm:
      yf = y.float()
      mean = yf.mean(-1, keepdim=True)
      var = ((yf - mean) ** 2).mean(-1, keepdim=True)
      y = ((yf - mean) * torch.rsqrt(var + p.layer_norm_epsilon) *
           theta['ln_scale_' + name].float()).to(y.dtype)
    if p.enable_gru_bias:
      y = y + theta['b_' + name].to(y.dtype)
    return y

  def FProp(self, theta, state0, inputs):
    p = self.params
    state0 = self._ResetState(state0, inputs)
    x = self._Act(inputs)
    xm = torch.cat([x, state0.m.to(x.dtype)], -1)
    r = torch.sigmoid(self._Gate(theta, 'r', xm))
    u = torch.sigmoid(self._Gate(theta, 'u', xm))
    n = torch.tanh(self._Gate(theta, 'n', torch.cat([x, r * state0.m.to(x.dtype)], -1)))
    new_c = u * state0.c + (1.0 - u) * n
    if p.cell_value_cap is not None:
      new_c = new_c.clamp(-p.cell_value_cap, p.cell_value_cap)
    new_m = torch.matmul(new_c, theta.w_proj.to(new_c.dtype)) if p.num_hidden_nodes else new_c
    pad = inputs.get('padding')
    new_c = _ZoneOut(state0.c, new_c, pad, p.zo_prob, self.do_eval)
    new_m = _ZoneOut(state0.m, new_m, pad, p.zo_prob, self.do_eval)
    return NestedMap(m=new_m, c=new_c), NestedMap()


class EmbeddingAugmentedLayerNormalizedLSTMCellSimple(LayerNormalizedLSTMCellSimple):
  """LN-LSTM whose input is augmented with an embedding of the current (and previous) token
  ids (ref :1715): `inputs.ids [B]` go through a `StatefulEmbeddingStep` and the result is
  added to the activations (`inject_emb_method='add'`), or — for 'concat' — added into the
  last `emb_dim` columns of the activations, which the caller must have left as zeros.
  State gains `emb` (the embedding step's state: position + previous ids)."""

  @classmethod
  def Params(cls):
    from lingvo_b200.core.steps import embedding_steps   # pylint: disable=g-import-not-at-top
    p = super().Params()
    p.Define('emb', embedding_steps.StatefulEmbeddingStep.Params(),
             'Inject this embedding into the input to the cell.')
    p.Define('inject_emb_method', 'add', "How to inject the embedding: 'add' or 'concat'.")
    p.name = 'embedding_augmented_lstm'
    return p

  def __init__(self, params):
    from lingvo_b200.core.steps import embedding_steps   # pylint: disable=g-import-not-at-top
    super().__init__(params)
    p = self.params
    assert issubclass(p.emb.cls, embedding_steps.StatefulEmbeddingStep), (
        'Only StatefulEmbeddingStep is supported for p.emb')
    assert p.inject_emb_method in ('add', 'concat'), p.inject_emb_method
    self.CreateChild('emb', p.emb)

  def zero_state(self, theta, batch_size):
    state0 = super().zero_state(theta, batch_size)
    state0.emb = self.emb.ZeroState(theta.emb, None, batch_size)
    return state0

  def FProp(self, theta, state0, inputs):
    p = self.params
    emb_out, emb_state1 = self.emb.FProp(theta.emb, None, NestedMap(inputs=[inputs.ids]), None,
                                         state0.emb)
    embedding = emb_out.output
    act = self._Act(inputs)
    if p.inject_emb_method == 'concat':
      emb_dim = embedding.shape[-1]
      # "concatenation" by addition into the zero-padded tail of the activations
      embedding = F.pad(embedding, (p.num_input_nodes - emb_dim, 0))
    inner = NestedMap(inputs)
    inner.act = [act + embedding.to(act.dtype)]
    lstm_state0 = NestedMap(m=state0.m, c=state0.c)
    state1, extras = super().FProp(theta, lstm_state0, inner)
    state1.emb = emb_state1
    return state1, extras
