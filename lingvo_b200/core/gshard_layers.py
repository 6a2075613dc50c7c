"""GShard layers: gating, MoE dispatch/combine, helpers.

Reference `lingvo/core/gshard_layers.py`:
  * `Top2GatingOnLogits` (:1932-2364) — reproduced verbatim in *math* as the
    dense `GSEC` oracle (`Top2GatingOnLogits`), and re-designed as an
    **index-based** gate (`Top2GatingIndices`) that returns
    `(expert, slot, gate) × 2` per token — the routing the fused sm_90a gate +
    dispatch kernel (`moe_gate_dispatch`, run by `parallel.symm.MoeExchange`)
    produces. `Top2Gates` computes the differentiable gate values and aux loss
    of a given routing for both. Both implement: softmax over E, top-1,
    second-expert policy (`all` / `sampling` (Gumbel) / `random` threshold),
    exclusive cumsum positions with first-choice priority (:2230, :2294),
    capacity rounding ↑4 (:2062-2076), renorm before/after capacity
    (`legacy_mtf_behavior`), aux loss `mean(density_1·density_1_proxy)·E²`
    (:2250-2255).
  * `ComputeGating` (:2840-2964), `FeedForwardNetworksApplyGating`
    (:2992-3163) — dense einsum oracle `GSEC,GSM->EGCM` … `GSEC,GECM->GSM`.
  * `MoEApplyIndexed` — the H100 path: permute-scatter dispatch, grouped
    wgmma expert GEMMs, gated 2-row gather combine; with expert parallelism
    the scatter/gather cross NVLink (`lingvo_b200.parallel.ep`).
  * `HashGatingOnLogits` (:2367), `TokenShufflingOnlogits` (:2496),
    sentence/task-level gating (:3359, :3450), `ReshapeInputLayer` (:1614),
    `StateLayer` (:1186-1430), `CausalDepthwiseConv1DLayer`, `VarLayer`.
"""

from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

from lingvo_b200 import ops
from lingvo_b200.core import activations
from lingvo_b200.core import base_layer
from lingvo_b200.core import gshard_utils
from lingvo_b200.core import py_utils
from lingvo_b200.core import summary_utils
from lingvo_b200.core.nested_map import NestedMap

Split = gshard_utils.Split
MeshSplit = gshard_utils.MeshSplit
WeightParams = py_utils.WeightParams
WeightInit = py_utils.WeightInit


def EinsumWithModelDim(equation, x, y, model_dim_reshape_segments=None,
                       name=None):
  """Einsum where `M` may have been reshaped to [segments, M/segments]."""
  if model_dim_reshape_segments is None:
    return torch.einsum(equation, x, y)
  if isinstance(model_dim_reshape_segments, int):
    model_dim_reshape_segments = [model_dim_reshape_segments]
  letters = 'NOPQR'[:len(model_dim_reshape_segments)]
  return torch.einsum(equation.replace('M', letters + 'M'), x, y)


def ExpertCapacity(group_size: int, experts_dim: int, expert_capacity_dim: int,
                   capacity_factor: Optional[float]) -> int:
  """C = max(c_dim, ⌊S·cf/E⌋ rounded ↑ to a multiple of 4) (:2062-2076)."""
  if capacity_factor is not None and capacity_factor > 0:
    auto = int((group_size * capacity_factor) / experts_dim)
    if auto == 0:
      auto = 4
    if expert_capacity_dim < auto:
      expert_capacity_dim = auto
      while expert_capacity_dim % 4:
        expert_capacity_dim += 1
  return expert_capacity_dim


def _Gumbel(shape, device, dtype, seeds=None):
  gen = None
  if seeds is not None:
    gen = torch.Generator(device=device)
    gen.manual_seed(((int(seeds[0]) & 0x7fffffff) << 31) ^ int(seeds[1]))
  u = torch.rand(shape, device=device, dtype=torch.float32, generator=gen)
  u = u.clamp_min(1e-20)
  return (-torch.log(-torch.log(u))).to(dtype)


def Top2GatingOnLogits(inputs, paddings, logits, num_devices, experts_dim,
                       expert_capacity_dim, fprop_dtype, use_xla_sharding=True,
                       second_expert_policy='all', second_expert_threshold=0.0,
                       legacy_mtf_behavior=True, capacity_factor=None,
                       importance=None, mask_dtype=None,
                       expert_padding_idx=None, seeds=None):
  """Dense oracle: returns (aux_loss, combine_tensor GSEC, dispatch GSEC)."""
  del inputs, num_devices, use_xla_sharding
  if mask_dtype is None:
    mask_dtype = fprop_dtype
  if expert_padding_idx:
    very_neg = torch.finfo(logits.dtype).max * -0.7
    m = torch.zeros_like(logits, dtype=torch.bool)
    m[..., list(expert_padding_idx)] = True
    logits = torch.where(m, torch.full_like(logits, very_neg), logits)
  raw_gates = torch.softmax(logits, dim=-1).to(fprop_dtype)
  expert_capacity_dim = ExpertCapacity(int(logits.shape[1]), experts_dim,
                                       expert_capacity_dim, capacity_factor)
  summary_utils.scalar('expert_capacity', expert_capacity_dim)

  index_1 = raw_gates.argmax(dim=-1)
  mask_1 = F.one_hot(index_1, experts_dim).to(mask_dtype)
  density_1_proxy = raw_gates
  if importance is not None:
    one = (importance == 1.0)
    mask_1 = mask_1 * one.unsqueeze(-1).to(mask_1.dtype)
    density_1_proxy = density_1_proxy * one.unsqueeze(-1).to(raw_gates.dtype)
  else:
    importance = torch.ones_like(mask_1[..., 0])
    if paddings is not None:
      nonpad = 1.0 - paddings.to(mask_1.dtype)
      mask_1 = mask_1 * nonpad.unsqueeze(-1)
      density_1_proxy = density_1_proxy * nonpad.unsqueeze(-1).to(raw_gates.dtype)
      importance = nonpad
  gate_1 = (raw_gates * mask_1.to(raw_gates.dtype)).sum(-1)
  gates_without_top_1 = raw_gates * (1.0 - mask_1.to(raw_gates.dtype))
  if second_expert_policy == 'sampling':
    noise = _Gumbel(logits.shape, logits.device, logits.dtype, seeds)
    very_neg = torch.finfo(logits.dtype).max * -0.7
    upd = torch.where(mask_1 > 0, torch.full_like(logits, very_neg), logits)
    index_2 = (upd + noise).argmax(dim=-1)
  else:
    index_2 = gates_without_top_1.argmax(dim=-1)
  mask_2 = F.one_hot(index_2, experts_dim).to(mask_dtype)
  if paddings is not None:
    mask_2 = mask_2 * (importance > 0).unsqueeze(-1).to(mask_2.dtype)
  gate_2 = (gates_without_top_1 * mask_2.to(raw_gates.dtype)).sum(-1)
  if legacy_mtf_behavior:
    denom = gate_1 + gate_2 + 1e-9
    gate_1 = gate_1 / denom
    gate_2 = gate_2 / denom

  position_in_expert_1 = torch.cumsum(mask_1, dim=-2) - mask_1
  capacity = float(expert_capacity_dim)
  if legacy_mtf_behavior:
    density_denom = 1.0
  else:
    density_denom = importance.to(fprop_dtype).mean(dim=1)[:, None] + 1e-6
  density_1 = mask_1.to(fprop_dtype).mean(dim=-2) / density_denom
  density_1_proxy = density_1_proxy.mean(dim=-2) / density_denom
  aux_loss = (density_1_proxy * density_1).mean() * (experts_dim * experts_dim)

  def over_capacity(mask, pos, name):
    ge = ((mask * pos) >= capacity).float().sum()
    summary_utils.scalar(name, ge)
    summary_utils.scalar(name + '_ratio', ge / torch.clamp(mask.float().sum(),
                                                           min=1.0))
  over_capacity(mask_1, position_in_expert_1, 'over_capacity_1')
  mask_1 = mask_1 * (position_in_expert_1 < capacity).to(mask_1.dtype)
  position_in_expert_1 = (position_in_expert_1 * mask_1).sum(-1)
  mask_1_count = mask_1.sum(dim=-2)
  mask_1_flat = mask_1.sum(dim=-1)

  if second_expert_policy == 'random':
    gen = None
    if seeds is not None:
      gen = torch.Generator(device=logits.device)
      gen.manual_seed(((int(seeds[0]) & 0x7fffffff) << 31) ^ int(seeds[1]) ^ 7)
    u = torch.rand(gate_2.shape, device=gate_2.device, generator=gen).to(
        gate_2.dtype)
    sampled_2 = u < (gate_2 / max(second_expert_threshold, 1e-9))
    gate_2 = gate_2 * sampled_2.to(gate_2.dtype)
    mask_2 = mask_2 * sampled_2.unsqueeze(-1).to(mask_2.dtype)
  elif second_expert_policy not in ('all', 'sampling'):
    raise ValueError(second_expert_policy)

  position_in_expert_2 = (torch.cumsum(mask_2, dim=-2) - mask_2 +
                          mask_1_count.unsqueeze(-2))
  over_capacity(mask_2, position_in_expert_2, 'over_capacity_2')
  mask_2 = mask_2 * (position_in_expert_2 < capacity).to(mask_2.dtype)
  position_in_expert_2 = (position_in_expert_2 * mask_2).sum(-1)
  mask_2_flat = mask_2.sum(dim=-1)
  gate_1 = gate_1 * mask_1_flat.to(gate_1.dtype)
  gate_2 = gate_2 * mask_2_flat.to(gate_2.dtype)
  if not legacy_mtf_behavior:
    denom = gate_1 + gate_2
    denom = torch.where(denom > 0, denom, torch.ones_like(denom))
    gate_1 = gate_1 / denom
    gate_2 = gate_2 / denom

  def part(gate, mask_flat, index, pos):
    b = F.one_hot(pos.long(), expert_capacity_dim).to(fprop_dtype)
    a = (gate * mask_flat.to(fprop_dtype)).unsqueeze(-1) * F.one_hot(
        index, experts_dim).to(fprop_dtype)
    return torch.einsum('...GSE,...GSC->...GSEC', a, b)

  combine_tensor = (part(gate_1, mask_1_flat, index_1, position_in_expert_1) +
                    part(gate_2, mask_2_flat, index_2, position_in_expert_2))
  dispatch_tensor = (combine_tensor != 0).to(fprop_dtype)
  return aux_loss, combine_tensor, dispatch_tensor


def _Top2GatesBeforeCapacity(logits, paddings, index, legacy_mtf_behavior):
  """→ (gate_1, gate_2, aux_loss) of the chosen experts `index`, before capacity.

  As if read from the softmax with the top-1 entry removed, `gate_2` is 0 where
  the second choice repeats the first (padding, or underflow to 0)."""
  e = logits.shape[-1]
  raw = torch.softmax(logits.float(), dim=-1)
  nonpad = None if paddings is None else (1.0 - paddings.float())
  index_1, index_2 = index[0].long(), index[1].long()
  oh1 = F.one_hot(index_1, e).float()
  gate_1 = torch.gather(raw, -1, index_1.unsqueeze(-1)).squeeze(-1)
  gate_2 = torch.gather(raw, -1, index_2.unsqueeze(-1)).squeeze(-1)
  live_2 = index_2 != index_1
  proxy = raw
  if nonpad is not None:
    oh1 = oh1 * nonpad.unsqueeze(-1)
    proxy = raw * nonpad.unsqueeze(-1)
    gate_1 = gate_1 * nonpad
    live_2 = live_2 & (nonpad > 0)
  gate_2 = gate_2 * live_2
  if legacy_mtf_behavior:
    denom = gate_1 + gate_2 + 1e-9
    gate_1, gate_2 = gate_1 / denom, gate_2 / denom
  density_denom = 1.0 if legacy_mtf_behavior else (
      (nonpad if nonpad is not None else torch.ones_like(gate_1)).mean(1)[:, None]
      + 1e-6)
  density_1 = oh1.mean(dim=1) / density_denom
  aux_loss = ((proxy.mean(dim=1) / density_denom) * density_1).mean() * (e * e)
  return gate_1, gate_2, aux_loss


def _Top2GatesAfterCapacity(gate_1, gate_2, keep, legacy_mtf_behavior):
  """Zeroes the gates of dropped choices; without `legacy_mtf_behavior` the kept
  pair is then renormalised to sum to 1. → gate `[2, G, S]`."""
  gate_1 = gate_1 * keep[0].float()
  gate_2 = gate_2 * keep[1].float()
  if not legacy_mtf_behavior:
    denom = gate_1 + gate_2
    denom = torch.where(denom > 0, denom, torch.ones_like(denom))
    gate_1, gate_2 = gate_1 / denom, gate_2 / denom
  return torch.stack([gate_1, gate_2])


def Top2Gates(logits, paddings, index, keep, legacy_mtf_behavior):
  """Top-2 gate values and aux loss of a routing, differentiable w.r.t. logits.

  index `[2, G, S]` holds the chosen experts, keep `[2, G, S]` is true (or 1)
  where the choice was dispatched. → (gate `[2, G, S]` fp32, aux_loss)."""
  gate_1, gate_2, aux_loss = _Top2GatesBeforeCapacity(logits, paddings, index,
                                                      legacy_mtf_behavior)
  return (_Top2GatesAfterCapacity(gate_1, gate_2, keep, legacy_mtf_behavior),
          aux_loss)


def Top2GatingIndices(logits, paddings, experts_dim, expert_capacity_dim,
                      fprop_dtype=torch.float32, second_expert_policy='all',
                      second_expert_threshold=0.0, legacy_mtf_behavior=True,
                      capacity_factor=None, seeds=None, use_kernel=True):
  """Index-form top-2 gate.

  Args: logits `[G, S, E]` (fp32 recommended), paddings `[G, S]` or None.
  Returns NestedMap:
    index `[2, G, S]` int32 expert ids, pos `[2, G, S]` int32 slot in expert,
    gate `[2, G, S]` fp32 combine weights (0 ⇒ dropped / not dispatched; the
    gate is differentiable w.r.t. logits), aux_loss (scalar), capacity (int).
  Semantically identical to `Top2GatingOnLogits` (tested bit-for-bit on the
  resulting combine tensor).
  """
  g, s, e = logits.shape
  assert e == experts_dim
  cap = ExpertCapacity(s, experts_dim, expert_capacity_dim, capacity_factor)
  raw = torch.softmax(logits.float(), dim=-1)
  nonpad = None if paddings is None else (1.0 - paddings.float())
  index_1 = raw.argmax(-1)
  oh1 = F.one_hot(index_1, e).float()
  if nonpad is not None:
    oh1 = oh1 * nonpad.unsqueeze(-1)
  if second_expert_policy == 'sampling':
    noise = _Gumbel(logits.shape, logits.device, torch.float32, seeds)
    very_neg = torch.finfo(torch.float32).max * -0.7
    upd = torch.where(oh1 > 0, torch.full_like(raw, very_neg), logits.float())
    index_2 = (upd + noise).argmax(-1)
  else:
    # A padded token keeps its top-1 entry, so its second choice repeats it.
    index_2 = (raw * (1.0 - oh1)).argmax(-1)
  oh2 = F.one_hot(index_2, e).float()
  if nonpad is not None:
    oh2 = oh2 * (nonpad > 0).float().unsqueeze(-1)
  index = torch.stack([index_1, index_2])
  # `random` samples on gate_2 after the legacy renormalisation, before capacity.
  gate_1, gate_2, aux_loss = _Top2GatesBeforeCapacity(logits, paddings, index,
                                                      legacy_mtf_behavior)
  pos1_all = torch.cumsum(oh1, dim=1) - oh1
  keep1 = oh1 * (pos1_all < cap).float()
  pos1 = (pos1_all * keep1).sum(-1)
  count1 = keep1.sum(dim=1)
  if second_expert_policy == 'random':
    gen = None
    if seeds is not None:
      gen = torch.Generator(device=logits.device)
      gen.manual_seed(((int(seeds[0]) & 0x7fffffff) << 31) ^ int(seeds[1]) ^ 7)
    u = torch.rand(gate_2.shape, device=gate_2.device, generator=gen)
    sampled = (u < gate_2 / max(second_expert_threshold, 1e-9)).float()
    oh2 = oh2 * sampled.unsqueeze(-1)
  pos2_all = torch.cumsum(oh2, dim=1) - oh2 + count1.unsqueeze(1)
  keep2 = oh2 * (pos2_all < cap).float()
  pos2 = (pos2_all * keep2).sum(-1)
  gate = _Top2GatesAfterCapacity(gate_1, gate_2,
                                 (keep1.sum(-1), keep2.sum(-1)),
                                 legacy_mtf_behavior)
  with torch.no_grad():
    over1 = (oh1.sum() - keep1.sum())
    over2 = (oh2.sum() - keep2.sum())
  summary_utils.scalar('expert_capacity', cap)
  summary_utils.scalar('over_capacity_1', over1)
  summary_utils.scalar('over_capacity_2', over2)
  return NestedMap(
      index=index.to(torch.int32),
      pos=torch.stack([pos1, pos2]).to(torch.int32),
      gate=gate, aux_loss=aux_loss, capacity=cap)


def CombineTensorFromIndices(gating: NestedMap, experts_dim: int):
  """Index form → dense `GSEC` combine tensor (for tests / oracle parity)."""
  out = 0
  for k in range(2):
    a = gating.gate[k].unsqueeze(-1) * F.one_hot(
        gating.index[k].long(), experts_dim).float()
    b = F.one_hot(gating.pos[k].long(), gating.capacity).float()
    out = out + torch.einsum('GSE,GSC->GSEC', a, b)
  return out


def HashGatingOnLogits(inputs, expert_id, paddings, num_devices, experts_dim,
                       expert_capacity_dim, fprop_dtype, use_xla_sharding=True,
                       capacity_factor=None, mask_dtype=None):
  """Token-id hash routing, top-1 with capacity (reference :2367)."""
  del num_devices, use_xla_sharding
  mask_dtype = mask_dtype or fprop_dtype
  cap = ExpertCapacity(int(expert_id.shape[1]), experts_dim,
                       expert_capacity_dim, capacity_factor)
  mask = F.one_hot(expert_id.long(), experts_dim).to(mask_dtype)
  if paddings is not None:
    mask = mask * (1.0 - paddings.to(mask_dtype)).unsqueeze(-1)
  pos = torch.cumsum(mask, dim=-2) - mask
  mask = mask * (pos < cap).to(mask_dtype)
  pos = (pos * mask).sum(-1)
  flat = mask.sum(-1)
  b = F.one_hot(pos.long(), cap).to(fprop_dtype)
  a = flat.to(fprop_dtype).unsqueeze(-1) * F.one_hot(
      expert_id.long(), experts_dim).to(fprop_dtype)
  combine = torch.einsum('...GSE,...GSC->...GSEC', a, b)
  dispatch = (combine != 0).to(fprop_dtype)
  return torch.zeros((), device=combine.device), combine, dispatch


def TokenShufflingOnlogits(inputs, logits, experts_dim, fprop_dtype,
                           use_xla_sharding=True, mask_dtype=None,
                           capacity_factor=1.0):
  """Expert-choice routing: every expert takes its top-C tokens (:2496).

  Returns (aux_loss, combine `GECS`-equivalent packed as GSEC, dispatch GSEC).
  """
  del inputs, use_xla_sharding, mask_dtype
  g, s, e = logits.shape
  cap = max(int(s * capacity_factor / e), 1)
  probs = torch.softmax(logits.float(), dim=-1)       # over experts
  top = probs.transpose(1, 2).topk(cap, dim=-1)       # [G, E, C] over tokens
  combine = torch.zeros(g, s, e, cap, device=logits.device, dtype=fprop_dtype)
  gi = torch.arange(g, device=logits.device)[:, None, None].expand(g, e, cap)
  ei = torch.arange(e, device=logits.device)[None, :, None].expand(g, e, cap)
  ci = torch.arange(cap, device=logits.device)[None, None, :].expand(g, e, cap)
  combine[gi, top.indices, ei, ci] = top.values.to(fprop_dtype)
  dispatch = (combine != 0).to(fprop_dtype)
  return torch.zeros((), device=logits.device), combine, dispatch


def SentenceTop2Gating(w, sentence_embeddings, paddings, **kwargs):
  """Sentence-level routing: all tokens of a sentence share experts (:3359)."""
  logits = torch.einsum('GM,ME->GE', sentence_embeddings.float(), w.float())
  return logits


def ComputeGating(w, inputs, paddings, num_devices, experts_dim,
                  expert_capacity_dim, local_dispatch, fprop_dtype,
                  gating_func='top_2', use_xla_sharding=True,
                  second_expert_policy='all', second_expert_threshold=0.0,
                  legacy_mtf_behavior=True, capacity_factor=None,
                  model_dim_reshape_segments=None, mask_dtype=None,
                  gating_logits_dtype=None, expert_id=None,
                  expert_padding_idx=None, seeds=None):
  """Dense gating → NestedMap(combine_tensor, dispatch_tensor, aux_loss)."""
  orig = inputs
  if not local_dispatch:
    inputs = inputs.reshape(1, inputs.shape[0] * inputs.shape[1], -1)
    if paddings is not None:
      paddings = paddings.reshape(1, -1)
  ldt = gating_logits_dtype or fprop_dtype
  logits = EinsumWithModelDim('GSM,ME->GSE', inputs.to(ldt), w.to(ldt),
                              model_dim_reshape_segments)
  if gating_func == 'token_shuffle':
    aux, comb, disp = TokenShufflingOnlogits(inputs, logits, experts_dim,
                                             fprop_dtype)
  elif gating_func == 'top_2':
    aux, comb, disp = Top2GatingOnLogits(
        inputs, paddings, logits, num_devices, experts_dim,
        expert_capacity_dim, fprop_dtype, use_xla_sharding,
        second_expert_policy, second_expert_threshold, legacy_mtf_behavior,
        capacity_factor, None, mask_dtype, expert_padding_idx, seeds=seeds)
  elif gating_func == 'hashing':
    aux, comb, disp = HashGatingOnLogits(
        inputs, expert_id, paddings, num_devices, experts_dim,
        expert_capacity_dim, fprop_dtype, use_xla_sharding, capacity_factor,
        mask_dtype)
  else:
    raise ValueError('Gating function: %s not supported yet!' % gating_func)
  if not local_dispatch:
    disp = disp.reshape(list(orig.shape[:2]) + list(disp.shape[2:]))
    comb = comb.reshape(list(orig.shape[:2]) + list(comb.shape[2:]))
  return NestedMap(combine_tensor=comb, dispatch_tensor=disp, aux_loss=aux)


def FeedForwardNetworksApplyGating(gating, inputs, reshaped_inputs, wi_split,
                                   wo_split, num_devices, num_groups,
                                   bi_split=None, bo_split=None,
                                   dropout_rate=0.0, device_mesh=None,
                                   model_dim_reshape_segments=None,
                                   use_glu=False, gating_func='top_2',
                                   activation_name='RELU', **unused_splits):
  """Dense einsum oracle of MoE apply (reference :2992-3163).

  `wi_split` is `[E, M, H]` (or `[2, E, M, H]` for GLU), `wo_split` `[E, H, M]`.
  Returns (outputs `GSM`, aux_loss).
  """
  del num_devices, device_mesh
  act = activations.GetFn(activation_name)
  disp = gating.dispatch_tensor.to(reshaped_inputs.dtype)
  expert_inputs = torch.einsum('GSEC,GSM->EGCM', disp, reshaped_inputs)
  e, g, c, m = expert_inputs.shape
  x = expert_inputs.reshape(e, g * c, m)
  if use_glu:
    h = torch.einsum('EAM,KEMH->KEAH', x, wi_split.to(x.dtype))
    if bi_split is not None:
      h = h + bi_split.to(h.dtype)
    h = act(h[0]) * h[1]
  else:
    h = torch.einsum('EAM,EMH->EAH', x, wi_split.to(x.dtype))
    if bi_split is not None:
      h = h + bi_split.to(h.dtype)
    h = act(h)
  if dropout_rate:
    h = F.dropout(h, dropout_rate, training=True)
  out = torch.einsum('EAH,EHM->EAM', h, wo_split.to(h.dtype))
  if bo_split is not None:
    out = out + bo_split.to(out.dtype)
  out = out.reshape(e, g, c, m).transpose(0, 1)       # EGCM → GECM
  combined = torch.einsum('GSEC,GECM->GSM',
                          gating.combine_tensor.to(out.dtype), out)
  outputs = combined.reshape(inputs.shape)
  return outputs, gating.aux_loss


# --------------------------------------------------------------------------
# Index-based dispatch / combine. Under expert parallelism
# lingvo_b200.parallel.ep moves the dispatched rows between ranks; both sides
# use these slot conventions:
#   slot(e, g, c) = (e * G + g) * C + c   in a [E, G*C, M] buffer.
# --------------------------------------------------------------------------
def _Slots(gating: NestedMap, g: int, s: int):
  cap = gating.capacity
  gi = torch.arange(g, device=gating.index.device).reshape(1, g, 1)
  slot = (gating.index.long() * g + gi) * cap + gating.pos.long()   # [2,G,S]
  valid = gating.gate.detach() > 0
  return slot, valid


class _DispatchFn(torch.autograd.Function):
  """x[G*S, M] → buf[E*G*C, M] (rows of dropped tokens are zero)."""

  @staticmethod
  def forward(ctx, x, slot, valid, num_slots):
    buf = torch.zeros(num_slots, x.shape[-1], dtype=x.dtype, device=x.device)
    for k in range(2):
      tok = valid[k].nonzero(as_tuple=True)[0]
      buf.index_copy_(0, slot[k][tok], x.index_select(0, tok))
    ctx.save_for_backward(slot, valid)
    return buf

  @staticmethod
  def backward(ctx, dbuf):
    slot, valid = ctx.saved_tensors
    dx = None
    for k in range(2):
      part = dbuf.index_select(0, slot[k].clamp(0, dbuf.shape[0] - 1))
      part = part * valid[k].unsqueeze(-1).to(part.dtype)
      dx = part if dx is None else dx + part
    return dx, None, None, None


def MoEDispatchIndexed(x2d, gating: NestedMap, g: int, s: int, e: int):
  """tokens `[G*S, M]` → expert inputs `[E, G*C, M]`."""
  slot, valid = _Slots(gating, g, s)
  buf = _DispatchFn.apply(x2d, slot.reshape(2, -1), valid.reshape(2, -1),
                          e * g * gating.capacity)
  return buf.reshape(e, g * gating.capacity, x2d.shape[-1])


def MoECombineIndexed(expert_out, gating: NestedMap, g: int, s: int):
  """expert outputs `[E, G*C, M]` → tokens `[G*S, M]` (gated 2-row gather)."""
  slot, valid = _Slots(gating, g, s)
  flat = expert_out.reshape(-1, expert_out.shape[-1])
  out = 0
  for k in range(2):
    rows = flat.index_select(0, slot[k].reshape(-1).clamp(0, flat.shape[0] - 1))
    w = gating.gate[k].reshape(-1, 1).to(rows.dtype)
    out = out + rows * w
  return out


def MoEApplyIndexed(x, gating: NestedMap, wi, wo, activation_name='RELU',
                    bi=None, bo=None, use_glu=False, ep_engine=None):
  """Index-based MoE FFN: `x [G, S, M]` → `[G, S, M]`.

  `wi [E_local, M, H]`, `wo [E_local, H, M]`. With an `ep_engine`
  (`parallel.ep.ExpertParallel`) tokens travel to the ranks owning their
  experts and back; otherwise all experts are local.
  """
  from lingvo_b200.ops import gemm
  g, s, m = x.shape
  e = wi.shape[-3] if ep_engine is None else ep_engine.num_experts
  xin = MoEDispatchIndexed(x.reshape(g * s, m), gating, g, s, e)
  if ep_engine is not None:
    xin = ep_engine.ToExperts(xin)
    wi, wo = ep_engine.ScaleExpertGrad(wi), ep_engine.ScaleExpertGrad(wo)
  if use_glu:
    h0 = gemm.grouped_linear(xin, wi[0].to(xin.dtype))
    h1 = gemm.grouped_linear(xin, wi[1].to(xin.dtype))
    h = activations.GetFn(activation_name)(h0) * h1
  elif activation_name in ('RELU', 'NONE'):
    h = gemm.grouped_linear(xin, wi.to(xin.dtype), bi, act=activation_name)
  else:
    h = activations.GetFn(activation_name)(
        gemm.grouped_linear(xin, wi.to(xin.dtype), bi))
  out = gemm.grouped_linear(h, wo.to(h.dtype), bo)
  if ep_engine is not None:
    out = ep_engine.FromExperts(out)
  return MoECombineIndexed(out, gating, g, s).reshape(g, s, m)


# ------------------------------------------------------------------- layers --
class VarLayer(base_layer.BaseLayer):
  """Holds named weights; FProp returns them (reference `VarLayer`)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('weights', None, '[(name, WeightParams)].')
    p.Define('shared_var_collection_suffix', None, 'Kept for parity.')
    return p

  def _CreateLayerVariables(self):
    for k, wp in self.params.weights:
      self.CreateVariable(k, wp)

  def FProp(self, theta, *args, **kwargs):
    def cast(v):
      if v.is_floating_point() and v.dtype != self.fprop_dtype:
        return v.to(self.fprop_dtype)
      return v
    vals = [cast(theta[k]) for k, _ in self.params.weights]
    return vals[0] if len(vals) == 1 else tuple(vals)


class ShardedVarLayer(VarLayer):
  """VarLayer whose weights carry mesh-split annotations."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('cast_to_fprop_dtype', True, 'Cast weights to fprop_dtype.')
    return p


class ReshapeInputLayer(base_layer.BaseLayer):
  """`[B, L, M]` → `[G, S, M]` + paddings from segment ids (reference :1614)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_groups', None, 'Number of groups.')
    p.Define('num_devices', 1, 'Number of devices.')
    p.Define('model_dims', None, 'Model dims (list).')
    return p

  def FProp(self, theta, inputs, segment_id):
    p = self.params
    paddings = (segment_id == 0).to(inputs.dtype)
    b, l = inputs.shape[0], inputs.shape[1]
    g = p.num_groups or b
    if (b * l) % g:
      raise ValueError('tokens %d not divisible by num_groups %d' % (b * l, g))
    return (inputs.reshape(g, (b * l) // g, *inputs.shape[2:]),
            paddings.reshape(g, (b * l) // g))


class CausalDepthwiseConv1DLayer(base_layer.BaseLayer):
  """Causal depthwise conv over time on `[B, L, …, D]` (Primer/_LNConv)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('kernel_size', None, 'Kernel size.')
    p.Define('model_dims', None, 'Trailing (channel) dims.')
    p.Define('compatible_with_mtf_ckpt', False, 'Kept for parity.')
    p.Define('conv_vars_reshape', False, 'Kept for parity.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    dims = list(p.model_dims) if isinstance(p.model_dims, (list, tuple)) else [
        p.model_dims]
    for i in range(p.kernel_size):
      init = WeightInit.Constant(0.5 if i == 0 else 0.5 / p.kernel_size)
      self.CreateVariable('w_%d' % i, WeightParams(dims, init, p.dtype))

  def FProp(self, theta, inputs):
    p = self.params
    out = 0
    for i in range(p.kernel_size):
      shifted = inputs if i == 0 else F.pad(
          inputs, [0, 0] * (inputs.dim() - 2) + [i, 0])[:, :inputs.shape[1]]
      out = out + shifted * theta['w_%d' % i].to(inputs.dtype)
    return out


class StateLayer(base_layer.BaseLayer):
  """Per-layer decode state (KV caches) threaded through DecodeIds (:1186).

  `NewState(theta, shape)` allocates; `FProp` reads; `UpdateState(name, t, v)`
  writes at time `t`. State lives in a thread-local overlay keyed by layer
  path so the functional FProp signature is unchanged.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('shape', [None, None], 'batch, time, etc...')
    p.Define('use_xla_dynamic_update_slice', True, 'Kept for parity.')
    return p

  _STATE = py_utils._Stack()  # pylint: disable=protected-access

  @classmethod
  def StateContext(cls, state: NestedMap):
    return cls._STATE.Push(state)

  def NewState(self, shape, dtype=None, device=None):
    return torch.zeros(list(shape), dtype=dtype or self.fprop_dtype,
                       device=device or py_utils.CurrentDevice())

  def _Current(self):
    st = self._STATE.Top()
    assert st is not None, 'StateLayer used outside StateContext'
    return st

  def FProp(self, theta):
    return self._Current().Get(self.path.replace('[', '_').replace(']', ''))

  def UpdateState(self, value, t=None):
    st = self._Current()
    key = self.path.replace('[', '_').replace(']', '')
    if t is None:
      st.Set(key, value)
    else:
      cur = st.Get(key)
      cur[:, t] = value.to(cur.dtype)
    return value


class OverrideLayer(base_layer.BaseLayer):
  """Lets decoding override a value at a named key (reference OverrideLayer)."""

  _OVERRIDE = {}

  @classmethod
  def Set(cls, key, value):
    cls._OVERRIDE[key] = value

  @classmethod
  def Clear(cls):
    cls._OVERRIDE.clear()

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('key', None, 'Override key.')
    return p

  def FProp(self, theta, x):
    return self._OVERRIDE.get(self.params.key, x)


# ==================================================================================
# SPMD shifting-buffer / circular pipeline (reference :180-1185; SURVEY K15)
# ==================================================================================
class _RingShift(torch.autograd.Function):
  """Stage r hands its tensor to stage r+1 (and receives stage r-1's): the collective-
  permute of the shifting-buffer pipeline, as one batched NCCL/gloo P2P exchange. The
  backward pass is the reverse rotation."""

  @staticmethod
  def forward(ctx, x, group, direction):
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    ctx.group, ctx.direction = group, direction
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    dst = dist.get_global_rank(group, (rank + direction) % world) if group is not None else (
        (rank + direction) % world)
    src = dist.get_global_rank(group, (rank - direction) % world) if group is not None else (
        (rank - direction) % world)
    x = x.contiguous()
    out = torch.empty_like(x)
    ops = [dist.P2POp(dist.isend, x, dst, group), dist.P2POp(dist.irecv, out, src, group)]
    for req in dist.batch_isend_irecv(ops):
      req.wait()
    return out

  @staticmethod
  def backward(ctx, dy):
    return _RingShift.apply(dy, ctx.group, -ctx.direction), None, None


class LayerwiseShardablePipelinedLayer(base_layer.BaseLayer):
  """Pipelines `num_stages × circular_repeat` copies of `single_stage_body` over
  micro-batches with a *shifting buffer*: iteration t lets every stage work on the
  micro-batch that reached it, then the buffer moves one stage forward
  (`num_microbatches + num_stages·circular_repeat − 1` iterations in total).

  Two execution modes with identical math:

  * **local** (default): all stages live in this process; the shift is a roll of the
    stage buffer. Useful to test a pipelined model definition and as the oracle.
  * **rank-sharded** (`stage_group` passed to `AttachStageGroup`, world = `num_stages`):
    rank r builds only the bodies of stage r (layer r, r+S, r+2S, … under a circular
    schedule), so weights and optimizer state are partitioned 1/S; the shift is one
    batched P2P ring exchange per iteration (`_RingShift`, NVLink via NCCL), overlapping
    the next iteration's compute of the other stages. Autograd runs the reverse ring.

  `FProp(theta, inputs, *shared)`: `inputs` is `[batch, …]` (micro-batched here with
  `num_microbatches` / `microbatch_size`) or already `[num_microbatches, mb, …]`;
  `shared` tensors are passed unchanged to every stage (e.g. a causal mask). Per-batch
  side inputs with a leading batch dim (paddings, segment ids) travel through the buffer
  with the activations when given as a NestedMap of tensors.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_stages', 1, 'Number of pipeline stages.')
    p.Define('stage_parallel_body', None, 'Kept for parity (bodies are built per stage).')
    p.Define('single_stage_body', None, 'Layer params of one stage.')
    p.Define('num_microbatches', None, 'Split the batch into this many micro-batches.')
    p.Define('microbatch_size', None, 'Or: micro-batch size.')
    p.Define('shard_stages_1d', False, 'Kept for parity (see AttachStageGroup).')
    p.Define('pipeline_stage_mesh_dim', None, 'Kept for parity.')
    p.Define('per_stage_vars', True, 'Separate variables per stage (always true here).')
    p.Define('circular_repeat', 1, 'Circular pipeline: repeats of each stage.')
    p.Define('unroll', 'eval_only', 'Kept for parity (the loop is always explicit).')
    p.Define('aux_loss_microbatch_accumulation', 'mean', 'mean | sum.')
    return p

  def __init__(self, params, stage_group=None, stage_rank=None):
    super().__init__(params)
    p = self.params
    assert p.single_stage_body is not None or p.stage_parallel_body is not None
    body = p.single_stage_body or p.stage_parallel_body
    self._group = stage_group
    self._stage_rank = stage_rank
    self._num_layers = p.num_stages * p.circular_repeat
    owned = range(self._num_layers)
    if stage_rank is not None:
      owned = [k for k in owned if k % p.num_stages == stage_rank]
    self._owned = list(owned)
    for k in self._owned:
      self.CreateChild('body_%03d' % k, body.Copy().Set(name='body_%03d' % k))

  @classmethod
  def ForStageGroup(cls, params, group=None):
    """Rank-sharded instance: this process is stage `rank(group)` of `num_stages`."""
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    assert dist.is_initialized()
    world = dist.get_world_size(group)
    assert world == params.num_stages, (world, params.num_stages)
    return cls(params, stage_group=group, stage_rank=dist.get_rank(group))

  # ---------------------------------------------------------------- helpers --
  def _Microbatch(self, x):
    p = self.params
    if p.num_microbatches is None and p.microbatch_size is None:
      return x, False
    def split(t):
      if not isinstance(t, torch.Tensor) or t.dim() == 0:
        return t
      b = t.shape[0]
      nmb = p.num_microbatches or b // p.microbatch_size
      assert b % nmb == 0, (b, nmb)
      return t.reshape(nmb, b // nmb, *t.shape[1:])
    if isinstance(x, NestedMap):
      return x.Transform(split), True
    return split(x), True

  @staticmethod
  def _Lead(x):
    for t in (x.Flatten() if isinstance(x, NestedMap) else [x]):
      if isinstance(t, torch.Tensor):
        return t.shape[0]
    raise ValueError('no tensor input')

  @staticmethod
  def _Index(x, i):
    f = lambda t: t[i] if isinstance(t, torch.Tensor) and t.dim() > 0 else t
    return x.Transform(f) if isinstance(x, NestedMap) else f(x)

  def _RunBody(self, theta, k, x, shared):
    name = 'body_%03d' % k
    out = getattr(self, name).FProp(theta[name], x, *shared)
    return out

  # ------------------------------------------------------------------ FProp --
  def FProp(self, theta, inputs, *shared):
    p = self.params
    x, did_split = self._Microbatch(inputs)
    nmb = self._Lead(x)
    outs = (self._FPropLocal(theta, x, nmb, shared) if self._stage_rank is None
            else self._FPropSharded(theta, x, nmb, shared))
    def stack(items):
      if isinstance(items[0], NestedMap):
        flat = [it.Flatten() for it in items]
        return items[0].Pack([torch.stack([f[j] for f in flat])
                              if isinstance(flat[0][j], torch.Tensor) else flat[0][j]
                              for j in range(len(flat[0]))])
      return torch.stack(items)
    y = stack(outs)
    if did_split:
      merge = lambda t: t.reshape(-1, *t.shape[2:]) if isinstance(t, torch.Tensor) and t.dim() > 1 else t
      y = y.Transform(merge) if isinstance(y, NestedMap) else merge(y)
    return y

  def _FPropLocal(self, theta, x, nmb, shared):
    """All stages in-process. The buffer slot of stage s at iteration t holds micro-batch
    (t − s) mod …; with a circular schedule a micro-batch re-enters stage 0 after stage
    S−1 until it has visited all `num_layers` bodies."""
    p = self.params
    s_n, rep = p.num_stages, p.circular_repeat
    n_iter = nmb * rep + s_n - 1 if rep > 1 else nmb + s_n - 1
    if rep > 1:
      assert nmb >= s_n, 'circular pipeline needs num_microbatches >= num_stages'
    buf = [None] * s_n                 # (microbatch id, pass index, activation)
    outs = [None] * nmb
    feed = 0
    pending = []                       # micro-batches that wrapped around, FIFO
    for t in range(n_iter):
      # stage 0 intake: a wrapped micro-batch has priority once the first wave has entered
      new_buf = [None] * s_n
      if pending and (feed >= nmb or pending[0][3] <= t):
        mb, pas, act, _ = pending.pop(0)
        new_buf[0] = (mb, pas, act)
      elif feed < nmb:
        new_buf[0] = (feed, 0, self._Index(x, feed))
        feed += 1
      for s in range(1, s_n):
        new_buf[s] = buf[s - 1]
      results = [None] * s_n
      for s in range(s_n):
        if new_buf[s] is None:
          continue
        mb, pas, act = new_buf[s]
        results[s] = (mb, pas, self._RunBody(theta, pas * s_n + s, act, shared))
      # last stage output: finished, or wraps to stage 0 for the next pass
      last = results[s_n - 1]
      if last is not None:
        mb, pas, act = last
        if pas + 1 < rep:
          pending.append((mb, pas + 1, act, t + 1))
        else:
          outs[mb] = act
      buf = results
    assert all(o is not None for o in outs), 'pipeline schedule did not drain'
    return outs

  def _FPropSharded(self, theta, x, nmb, shared):
    """This rank is one stage. Iteration t: run my body on what sits in my slot, then the
    ring shift moves every slot one stage forward. Stage 0 injects fresh micro-batches,
    the last stage's results come back around to stage 0, which either re-injects them
    (circular) or records them; the final outputs are broadcast from stage 0."""
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    p = self.params
    s_n, rep, r = p.num_stages, p.circular_repeat, self._stage_rank
    if rep > 1:
      assert nmb >= s_n
    n_iter = (nmb * rep if rep > 1 else nmb) + s_n - 1
    template = self._Index(x, 0)
    is_map = isinstance(template, NestedMap)
    def zeros_like(v):
      f = lambda t: torch.zeros_like(t) if isinstance(t, torch.Tensor) else t
      return v.Transform(f) if is_map else f(v)
    def shift(v):
      f = lambda t: _RingShift.apply(t, self._group, 1) if isinstance(t, torch.Tensor) and (
          t.is_floating_point()) else t
      if not is_map:
        return f(v)
      # integer side inputs (segment ids …) ride along un-differentiated
      def g(t):
        if isinstance(t, torch.Tensor) and not t.is_floating_point():
          return _RingShift.apply(t.float(), self._group, 1).to(t.dtype)
        return f(t)
      return v.Transform(g)
    slot = zeros_like(template)        # what currently sits in my stage
    if torch.is_grad_enabled():
      # Every rank must record (and later replay, reversed) every ring exchange, also the
      # ones that only carry bubbles: make the bubble a leaf that requires grad.
      mk = lambda t: t.requires_grad_(True) if isinstance(t, torch.Tensor) and (
          t.is_floating_point()) else t
      slot = slot.Transform(mk) if is_map else mk(slot)
    outs = [None] * nmb
    # Deterministic schedule (identical on all ranks): which (mb, pass) is at stage s at t.
    sched = self._Schedule(nmb)
    # Every rank must replay *every* ring exchange in its backward pass, in the same
    # (reverse) order — also those whose payload this rank later overwrote or that only
    # carried a bubble. `alive` (always exactly 0) hangs every exchange onto the outputs.
    alive = None
    def touch(v):
      nonlocal alive
      for t_ in (v.Flatten() if is_map else [v]):
        if isinstance(t_, torch.Tensor) and t_.is_floating_point() and t_.requires_grad:
          z = t_.reshape(-1)[:1].sum() * 0
          alive = z if alive is None else alive + z
    for t in range(n_iter):
      cur = sched[t][r]
      if r == 0 and cur is not None and cur[1] == 0:
        slot = self._Index(x, cur[0])                     # fresh micro-batch enters
      if cur is not None:
        slot = self._RunBody(theta, cur[1] * s_n + r, slot, shared)
      arrived = shift(slot)                               # collective: every rank, every t
      touch(arrived)
      done = sched[t][s_n - 1]
      if r == 0 and done is not None and done[1] + 1 == rep:
        outs[done[0]] = arrived                           # finished micro-batch came round
      slot = arrived
    # everyone returns the outputs (stage 0 has them): broadcast, differentiable via shift
    root = dist.get_global_rank(self._group, 0) if self._group is not None else 0
    res = []
    def with_alive(v):
      if alive is None:
        return v
      f = lambda t: t + alive.to(t.dtype) if isinstance(t, torch.Tensor) and (
          t.is_floating_point()) else t
      return v.Transform(f) if is_map else f(v)
    for mb in range(nmb):
      o = with_alive(outs[mb] if r == 0 else zeros_like(template))
      f = lambda t: _Broadcast.apply(t, self._group, root) if isinstance(t, torch.Tensor) and (
          t.is_floating_point()) else t
      res.append(o.Transform(f) if is_map else f(o))
    return res

  def _Schedule(self, nmb):
    """sched[t][s] = (micro-batch, pass) processed by stage s at iteration t, or None —
    the same wave pattern as `_FPropLocal`, computed without touching data."""
    p = self.params
    s_n, rep = p.num_stages, p.circular_repeat
    n_iter = (nmb * rep if rep > 1 else nmb) + s_n - 1
    sched = [[None] * s_n for _ in range(n_iter)]
    buf = [None] * s_n
    feed = 0
    pending = []
    for t in range(n_iter):
      new_buf = [None] * s_n
      if pending and (feed >= nmb or pending[0][2] <= t):
        mb, pas, _ = pending.pop(0)
        new_buf[0] = (mb, pas)
      elif feed < nmb:
        new_buf[0] = (feed, 0)
        feed += 1
      for s in range(1, s_n):
        new_buf[s] = buf[s - 1]
      last = new_buf[s_n - 1]
      if last is not None and last[1] + 1 < rep:
        pending.append((last[0], last[1] + 1, t + 1))
      sched[t] = list(new_buf)
      buf = new_buf
    return sched


class _Broadcast(torch.autograd.Function):
  """Differentiable broadcast from `root`. Every rank then computes the same (replicated)
  loss from the same outputs, so the backward pass averages the identical incoming
  gradients back onto the root."""

  @staticmethod
  def forward(ctx, x, group, root):
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    ctx.group, ctx.root = group, root
    out = x.contiguous().clone()
    dist.broadcast(out, src=root, group=group)
    return out

  @staticmethod
  def backward(ctx, dy):
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    g = dy.contiguous().clone()
    dist.reduce(g, dst=ctx.root, group=ctx.group)
    if dist.get_rank() != ctx.root:
      g = torch.zeros_like(g)
    else:
      g = g / dist.get_world_size(ctx.group)
    return g, None, None


class MultiHeadAttentionStateLayer(base_layer.BaseLayer):
  """Key/value decode cache of one attention layer `[B, T, N, H]` written one time step at
  a time (reference `MultiHeadAttentionStateLayer`); thin typed wrapper over `StateLayer`
  that also supports beam re-ordering."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('shape', [None, None, None, None], 'batch, time, heads, dim_per_head.')
    p.Define('use_xla_dynamic_update_slice', True, 'Kept for parity.')
    return p

  def InitState(self, batch, max_len, device=None, dtype=None):
    p = self.params
    shape = [batch, max_len] + list(p.shape[2:])
    return torch.zeros(shape, dtype=dtype or self.fprop_dtype,
                       device=device or py_utils.CurrentDevice())

  def FProp(self, theta, state):
    return state

  def UpdateState(self, state, value, t):
    """value `[B, N, H]` (or `[B, 1, N, H]`) written at time `t`; returns the new state."""
    if value.dim() == state.dim():
      value = value[:, 0]
    out = state.clone()
    out[:, int(t)] = value.to(out.dtype)
    return out

  @staticmethod
  def Reorder(state, beam_parent):
    """Beam search: row b continues hypothesis `beam_parent[b]`."""
    return state.index_select(0, beam_parent.long())


class SharedEmbeddingSoftmaxLayer(base_layer.BaseLayer):
  """One `[V, M]` table used both as the input embedding (with optional positional
  embeddings added) and as the output softmax weights (reference
  `SharedEmbeddingSoftmaxLayer`)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('vocab_size', 0, 'Vocabulary size.')
    p.Define('max_len', 0, 'Max positions (0 ⇒ no learned positional embedding).')
    p.Define('embedding_dim', 0, 'Model dim M.')
    p.Define('z_loss_coef', 1e-4, 'z-loss coefficient.')
    p.Define('num_devices', 1, 'Kept for parity.')
    p.Define('logits_abs_max', None, 'Clip logits to ± this value.')
    p.Define('label_smoothing', 0.1, 'Label smoothing.')
    p.Define('use_tgt_labels_size_as_loss_denominator', True, 'Loss denominator.')
    return p

  def _CreateLayerVariables(self):
    p = self.params
    self.CreateVariable('embedding', WeightParams(
        [p.vocab_size, p.embedding_dim], WeightInit.Gaussian(1.0), p.dtype))
    if p.max_len:
      self.CreateVariable('pos_embedding', WeightParams(
          [p.max_len, p.embedding_dim], WeightInit.Gaussian(1.0), p.dtype))

  def FProp(self, theta, ids, segment_pos=None):
    """ids `[B, L]` → `[B, L, M]`."""
    p = self.params
    y = F.embedding(ids.long(), theta.embedding)
    if p.max_len and segment_pos is not None:
      y = y + F.embedding(segment_pos.long(), theta.pos_embedding)
    return y.to(self.fprop_dtype)

  def ComputeLoss(self, theta, activation, labels, segment_ids):
    """activation `[B, L, M]`, labels/segment_ids `[B, L]` → (loss, per-token stats)."""
    p = self.params
    non_padding = ((segment_ids > 0) & (labels > 0)).float()
    logits = torch.matmul(activation.float() * (p.embedding_dim**-0.5),
                          theta.embedding.float().t())
    if p.logits_abs_max is not None:
      logits = logits.clamp(-p.logits_abs_max, p.logits_abs_max)
    lse = torch.logsumexp(logits, -1)
    true_logit = logits.gather(-1, labels.long().unsqueeze(-1)).squeeze(-1)
    off = p.label_smoothing / p.vocab_size
    on = 1.0 - p.label_smoothing + off
    soft = (on - off) * true_logit + off * logits.sum(-1)
    per_tok = (lse - soft) + p.z_loss_coef * lse.square()
    denom = float(non_padding.numel()) if p.use_tgt_labels_size_as_loss_denominator else (
        non_padding.sum().clamp_min(1.0))
    loss = (per_tok * non_padding).sum() / denom
    return loss, NestedMap(per_token_loss=per_tok * non_padding, non_padding=non_padding,
                           mean_xent=((lse - true_logit) * non_padding).sum() /
                           non_padding.sum().clamp_min(1.0))


# ------------------------------------------------------------------------------------------
# More gating policies (ref gshard_layers.py:2564-2990, 3166-3527). All return the packed
# `GSEC` combine / dispatch pair `FeedForwardNetworksApplyGating` and the indexed movers use.
# ------------------------------------------------------------------------------------------
def ShardedWeightParams(shape, init=None, dtype=None, collections=None,
                        tensor_split_dims_mapping=None):
  """WeightParams that also records how the variable is split over the device mesh (:104)."""
  p = py_utils.WeightParams(shape, init, dtype, collections)
  if tensor_split_dims_mapping is not None:
    assert len(tensor_split_dims_mapping) == len(shape)
    p.tensor_split_dims_mapping = list(tensor_split_dims_mapping)
  return p


def TokenShufflingOnlogitsV2(logits, paddings, num_devices, experts_dim, expert_capacity_dim,
                             fprop_dtype, use_xla_sharding=True, capacity_factor=None,
                             mask_dtype=None):
  """Expert-choice routing on raw gate scores with padded tokens excluded (:2564): each
  expert picks its `C` best non-padded tokens; a token keeps, for every expert that picked
  it, that expert's softmax weight; its slot is its rank among the expert's picks in
  sequence order. Returns (0, combine `GSEC`, dispatch `GSEC`)."""
  del num_devices, use_xla_sharding, mask_dtype
  g, s, e = logits.shape
  gates = torch.softmax(logits.float(), -1)
  nonpad = torch.ones(g, s, device=logits.device) if paddings is None else 1.0 - paddings.float()
  scores = (gates * nonpad.unsqueeze(-1)).transpose(1, 2)                    # GES
  cap = min(ExpertCapacity(s, e, expert_capacity_dim, capacity_factor), s)
  picked = scores.topk(cap, dim=-1).indices                                  # GEC
  mask = torch.zeros(g, e, s, device=logits.device)
  mask.scatter_(2, picked, 1.0)
  mask = mask.transpose(1, 2) * nonpad.unsqueeze(-1)                         # GSE
  pos = (torch.cumsum(mask, dim=1) - mask).long()                            # exclusive, GSE
  keep = mask * (pos < cap)
  combine = (gates * keep).unsqueeze(-1) * F.one_hot(pos.clamp(max=cap - 1), cap)
  combine = combine.to(fprop_dtype)
  return (torch.zeros((), device=logits.device, dtype=fprop_dtype), combine,
          (keep.unsqueeze(-1) * F.one_hot(pos.clamp(max=cap - 1), cap)).to(fprop_dtype))


def OptimalTransportOnlogits(logits, experts_dim, use_xla_sharding=False, epsilon=0.1,
                             num_iterations=50, fprop_dtype=None):
  """Balanced expert-choice routing (:2736): an entropic optimal-transport plan between
  experts (each takes `C = 2S/E` tokens) and tokens (each goes to ≤ 2 experts, the slack
  absorbed by a dummy expert) re-weights the softmax scores before every expert's top-C pick.
  The plan itself is treated as a constant (stop-gradient), as in the reference."""
  del use_xla_sharding
  from lingvo_b200.core import differentiable_assignment
  g, s, e = logits.shape
  assert e == experts_dim
  fprop_dtype = fprop_dtype or logits.dtype
  max_token_capacity = 2
  cap = s * 2 // e
  scores = torch.softmax(logits.float().transpose(1, 2), -1)                 # GES, over tokens
  scores_plus = torch.cat([scores, scores.new_zeros(g, 1, s)], 1)
  upper = torch.cat([torch.ones_like(scores),
                     scores.new_full((g, 1, s), float(max_token_capacity))], 1)
  rows = torch.cat([scores.new_full((g, e), float(cap)),
                    scores.new_full((g, 1), float(max_token_capacity * s - cap * e))], 1)
  cols = scores.new_full((g, s), float(max_token_capacity))
  with torch.no_grad():
    plan = differentiable_assignment.max_assignment(
        scores_plus, elementwise_upper_bound=upper, row_sums=rows, col_sums=cols,
        epsilon=epsilon, num_iterations=num_iterations, use_epsilon_scaling=True)[0][:, :e]
  gate, idx = (plan * scores).topk(cap, dim=-1)                              # GEC
  combine = torch.zeros(g, s, e, cap, device=logits.device, dtype=fprop_dtype)
  gi = torch.arange(g, device=logits.device)[:, None, None].expand(g, e, cap)
  ei = torch.arange(e, device=logits.device)[None, :, None].expand(g, e, cap)
  ci = torch.arange(cap, device=logits.device)[None, None, :].expand(g, e, cap)
  combine = combine.index_put((gi, idx, ei, ci), gate.to(fprop_dtype))
  return (torch.zeros((), device=logits.device, dtype=fprop_dtype), combine,
          (combine != 0).to(fprop_dtype))


def GetSentenceEmbeddings(inputs, segment_id):
  """Mean input embedding of each token's segment (:3293); segment 0 (padding) maps to 0.
  Segments are identified over the WHOLE `[G, S]` block, as in the reference."""
  m = inputs.shape[-1]
  flat = inputs.reshape(-1, m).float()
  seg = segment_id.reshape(-1).long()
  n = flat.shape[0]
  sums = torch.zeros(n + 1, m, device=inputs.device).index_add_(0, seg.clamp(max=n), flat)
  counts = torch.zeros(n + 1, device=inputs.device).index_add_(
      0, seg.clamp(max=n), torch.ones_like(seg, dtype=torch.float32))
  means = sums / counts.clamp(min=1.0).unsqueeze(-1)
  means[0] = 0.0
  return means[seg.clamp(max=n)].reshape(inputs.shape).to(inputs.dtype)


def _GateOnEmbeddings(w, embeddings, orig_inputs, paddings, num_devices, experts_dim,
                      expert_capacity_dim, local_dispatch, fprop_dtype, use_xla_sharding,
                      second_expert_policy, second_expert_threshold, legacy_mtf_behavior,
                      capacity_factor=None, seeds=None):
  logits = torch.einsum('GSM,ME->GSE', embeddings.to(w.dtype), w)
  aux, comb, disp = Top2GatingOnLogits(
      embeddings, paddings, logits, num_devices, experts_dim, expert_capacity_dim,
      fprop_dtype, use_xla_sharding, second_expert_policy, second_expert_threshold,
      legacy_mtf_behavior, capacity_factor, seeds=seeds)
  if not local_dispatch:
    disp = disp.reshape(list(orig_inputs.shape[:2]) + list(disp.shape[2:]))
    comb = comb.reshape(list(orig_inputs.shape[:2]) + list(comb.shape[2:]))
  return NestedMap(combine_tensor=comb, dispatch_tensor=disp, aux_loss=aux)


def SentenceTop2Gating(w, inputs, paddings, segment_id, num_devices, experts_dim,   # pylint: disable=function-redefined
                       expert_capacity_dim, local_dispatch, fprop_dtype,
                       use_xla_sharding=True, second_expert_policy='all',
                       second_expert_threshold=0.0, legacy_mtf_behavior=True,
                       embedding_type='sentence', capacity_factor=None, seeds=None):
  """Top-2 gating on per-sentence mean embeddings: every token of a segment is routed by the
  same logits (:3359)."""
  assert embedding_type == 'sentence'
  orig = inputs
  if not local_dispatch:
    inputs = inputs.reshape(1, inputs.shape[0] * inputs.shape[1], -1)
    segment_id = segment_id.reshape(1, -1)
    paddings = None if paddings is None else paddings.reshape(1, -1)
  emb = GetSentenceEmbeddings(inputs, segment_id)
  return _GateOnEmbeddings(w, emb, orig, paddings, num_devices, experts_dim,
                           expert_capacity_dim, local_dispatch, fprop_dtype, use_xla_sharding,
                           second_expert_policy, second_expert_threshold, legacy_mtf_behavior,
                           capacity_factor, seeds)


def TaskTop2Gating(w, inputs, paddings, task_embeddings, num_devices, experts_dim,
                   expert_capacity_dim, local_dispatch, fprop_dtype, use_xla_sharding=True,
                   second_expert_policy='all', second_expert_threshold=0.0,
                   legacy_mtf_behavior=True, seeds=None):
  """Top-2 gating on task embeddings instead of token activations (:3450)."""
  orig = inputs
  if not local_dispatch:
    task_embeddings = task_embeddings.reshape(
        1, task_embeddings.shape[0] * task_embeddings.shape[1], -1)
    paddings = None if paddings is None else paddings.reshape(1, -1)
  return _GateOnEmbeddings(w, task_embeddings, orig, paddings, num_devices, experts_dim,
                           expert_capacity_dim, local_dispatch, fprop_dtype, use_xla_sharding,
                           second_expert_policy, second_expert_threshold, legacy_mtf_behavior,
                           None, seeds)


_BaseComputeGating = ComputeGating


def ComputeGating(w, inputs, paddings, num_devices, experts_dim, expert_capacity_dim,   # pylint: disable=function-redefined
                  local_dispatch, fprop_dtype, gating_func='top_2', use_xla_sharding=True,
                  second_expert_policy='all', second_expert_threshold=0.0,
                  legacy_mtf_behavior=True, capacity_factor=None,
                  model_dim_reshape_segments=None, mask_dtype=None,
                  gating_logits_dtype=None, expert_id=None, expert_padding_idx=None,
                  seeds=None):
  """`ComputeGating` including the `token_shuffle_v2` and `optimal_transport` policies."""
  if gating_func not in ('token_shuffle_v2', 'optimal_transport'):
    return _BaseComputeGating(
        w, inputs, paddings, num_devices, experts_dim, expert_capacity_dim, local_dispatch,
        fprop_dtype, gating_func, use_xla_sharding, second_expert_policy,
        second_expert_threshold, legacy_mtf_behavior, capacity_factor,
        model_dim_reshape_segments, mask_dtype, gating_logits_dtype, expert_id,
        expert_padding_idx, seeds)
  orig = inputs
  if not local_dispatch:
    inputs = inputs.reshape(1, inputs.shape[0] * inputs.shape[1], -1)
    paddings = None if paddings is None else paddings.reshape(1, -1)
  ldt = gating_logits_dtype or fprop_dtype
  logits = EinsumWithModelDim('GSM,ME->GSE', inputs.to(ldt), w.to(ldt),
                              model_dim_reshape_segments)
  if gating_func == 'token_shuffle_v2':
    aux, comb, disp = TokenShufflingOnlogitsV2(
        logits, paddings, num_devices, experts_dim, expert_capacity_dim, fprop_dtype,
        capacity_factor=capacity_factor)
  else:
    aux, comb, disp = OptimalTransportOnlogits(logits, experts_dim, fprop_dtype=fprop_dtype)
  if not local_dispatch:
    disp = disp.reshape(list(orig.shape[:2]) + list(disp.shape[2:]))
    comb = comb.reshape(list(orig.shape[:2]) + list(comb.shape[2:]))
  return NestedMap(combine_tensor=comb, dispatch_tensor=disp, aux_loss=aux)


def HashGating(*args, **kwargs):
  return ComputeGating(*args, gating_func='hashing', **kwargs)


def Top2Gating(*args, **kwargs):
  return ComputeGating(*args, gating_func='top_2', **kwargs)


def TokenShuffleGating(*args, **kwargs):
  return ComputeGating(*args, gating_func='token_shuffle', **kwargs)


def TokenShuffleGatingV2(*args, **kwargs):
  return ComputeGating(*args, gating_func='token_shuffle_v2', **kwargs)


def OptimalTransportGating(*args, **kwargs):
  return ComputeGating(*args, gating_func='optimal_transport', **kwargs)


def GatherK(selected_pos, values, k, num_devices=1):
  """Packs, per row, the LAST `k` selected positions of every `[B, T, …]` tensor in `values`
  to the right of a `[B, k, …]` output, in sequence order (:3166). Returns (outputs,
  padding `[B, k]` with 1 at unfilled slots; those read position 0, as in the reference)."""
  del num_devices
  b, t = selected_pos.shape
  for v in values:
    assert tuple(v.shape[:2]) == (b, t), (v.shape, selected_pos.shape)
  one_based = torch.arange(1, t + 1, device=selected_pos.device).unsqueeze(0)
  top = (one_based * selected_pos.to(one_based.dtype)).topk(k, dim=-1).values
  idx = top.flip(-1)                                                     # ascending, 0 = empty
  padding = (idx == 0).to(values[0].dtype if values[0].is_floating_point() else torch.float32)
  src = (idx - 1).clamp(min=0)
  outs = []
  for v in values:
    gi = src.reshape(b, k, *([1] * (v.dim() - 2))).expand(b, k, *v.shape[2:])
    outs.append(v.gather(1, gi))
  return outs, padding


ZERO_STATE_MAX_ABS_TOLERANCE = 1e-6


class Conv1DStateLayer(base_layer.BaseLayer):
  """Sliding window of the last `kernel_size` inputs of a causal conv1d during incremental
  (flat-beam) decoding (:1432). Explicit-state API like `MultiHeadAttentionStateLayer`:
  `InitState` → `LoadPrefix` (optional) → `Step` per decoded position."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('shape', [None, None, None], 'batch, time, trailing dims….')
    p.Define('kernel_size', 0, 'Width of the convolution window.')
    p.Define('skip_store_zero_state', False,
             'All-zero inputs (zeroed padding positions) do not enter the window.')
    return p

  def InitState(self, batch, beam, device=None, dtype=None):
    p = self.params
    assert p.kernel_size > 0
    return torch.zeros([batch, beam, p.kernel_size] + list(p.shape[2:]),
                       dtype=dtype or self.fprop_dtype,
                       device=device or py_utils.CurrentDevice())

  def LoadPrefix(self, state, x):
    """x `[B, prefix_len, …]`: the window becomes the prefix's last `kernel_size` inputs
    (left-padded with zeros), shared by all beams."""
    k = self.params.kernel_size
    tail = x[:, -k:]
    if tail.shape[1] < k:
      tail = torch.cat([tail.new_zeros(tail.shape[0], k - tail.shape[1], *tail.shape[2:]),
                        tail], 1)
    return tail.unsqueeze(1).expand_as(state).to(state.dtype).contiguous()

  def Step(self, state, x):
    """x `[B, beam, …]` → (window `[B*beam, kernel_size, …]`, new state)."""
    p = self.params
    new_state = torch.cat([state[:, :, 1:], x.unsqueeze(2).to(state.dtype)], 2)
    if p.skip_store_zero_state:
      is_zero = x.reshape(x.shape[0], x.shape[1], -1).abs().amax(-1) < ZERO_STATE_MAX_ABS_TOLERANCE
      mask = is_zero.reshape(list(is_zero.shape) + [1] * (state.dim() - 2)).to(state.dtype)
      new_state = state * mask + new_state * (1 - mask)
    b, beam = new_state.shape[:2]
    return new_state.reshape(b * beam, *new_state.shape[2:]), new_state

  def FProp(self, theta, x):
    """Training: the convolution sees the whole sequence; nothing to do."""
    return x

  @staticmethod
  def Reorder(state, batch_index, beam_parent):
    """Flat beam search: hypothesis (b, k) continues (b, beam_parent[b, k])."""
    del batch_index
    idx = beam_parent.long().reshape(list(beam_parent.shape) + [1] * (state.dim() - 2))
    return state.gather(1, idx.expand_as(state))
