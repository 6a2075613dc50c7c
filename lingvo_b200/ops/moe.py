"""Front-end of the fused sm_90a MoE kernels (csrc/moe_kernels.cu) with their fp32 oracles.

Buffer convention of the expert exchange (shared with `parallel/symm.py:MoeExchange`):
tokens are `[T = G_l·S, M]` (G_l local groups of S tokens); every token has two expert
choices `k ∈ {0, 1}` described by `index[k, t]` (expert id), `pos[k, t]` (position inside the
expert's capacity buffer) and `gate[k, t]` (combine weight, 0 = dropped). Expert-side buffers
are **slot-major** `[E, G_l, C, M]`: slot `(e, g, c)` holds the c-th token that group g sent to
expert e.

  combine        y[t]      = Σ_k gate[k,t] · yc[index[k,t], g(t), pos[k,t]]
  gather_rows    out[t]    = Σ_k (gate[k,t] ≠ 0) · src[…same slot…]        (backward of scatter)
  combine_bwd_gate dgate[k,t] = ⟨yc[slot_k(t)], dy[t]⟩

`gate_dispatch` (gate + capacity assignment + peer-store dispatch in one kernel) and
`scatter_rows` write into *peer* memory through pointer tables and are driven by the exchange
engine; their math oracle is `core/gshard_layers.Top2GatingIndices` (tested in
`tests/test_kernels_gpu.py`). The row movers below are plain tensor → tensor and are exposed
here with `*_ref` oracles like every other op module.
"""

import torch

from lingvo_b200 import ops


def available() -> bool:
  mod = ops.native(required=False)
  return mod is not None and hasattr(mod, '_has_moe')


def _Slots(index, pos, s, g_l, c):
  """Flat slot id `[2, T]` of each (choice, token) in an `[E, G_l, C]` buffer."""
  t = index.shape[-1]
  g = (torch.arange(t, device=index.device) // s).unsqueeze(0)
  return (index.long() * g_l + g) * c + pos.long()


# ---------------------------------------------------------------------------- combine --
def _K(t, g_l, s):
  """The kernels take the per-choice tables as `[2, G_l, S]` (T = G_l·S is derived from the
  last two dims); callers may hold them flat as `[2, T]`."""
  t = t.contiguous()
  assert t.shape[0] == 2 and t.numel() == 2 * g_l * s, (tuple(t.shape), g_l, s)
  return t.view(2, g_l, s)


def combine(yc, index, pos, gate, s, g_l, c):
  """yc `[E, G_l, C, M]` bf16 (any leading layout with E·G_l·C rows), index/pos `[2, T]`
  int32, gate `[2, T]` fp32 → y `[T, M]` bf16. One warp per token, 16-byte loads, fp32
  accumulate; dropped choices (gate 0) are never read."""
  return ops.native().moe_combine(yc.contiguous(), _K(index, g_l, s), _K(pos, g_l, s),
                                  _K(gate.float(), g_l, s), int(s), int(g_l), int(c))


def combine_ref(yc, index, pos, gate, s, g_l, c):
  m = yc.shape[-1]
  rows = yc.reshape(-1, m).float()
  slots = _Slots(index, pos, s, g_l, c).clamp(0, rows.shape[0] - 1)
  picked = rows[slots]                                           # [2, T, M]
  w = gate.float().unsqueeze(-1)
  return (torch.where(w != 0, picked, torch.zeros_like(picked)) * w).sum(0)


def gather_rows(src, index, pos, gate, s, g_l, c):
  """The transpose of the dispatch scatter: every token sums the rows of its (kept) slots —
  the input gradient of the dispatch."""
  return ops.native().moe_gather_rows(src.contiguous(), _K(index, g_l, s), _K(pos, g_l, s),
                                      _K(gate.float(), g_l, s), int(s), int(g_l), int(c))


def gather_rows_ref(src, index, pos, gate, s, g_l, c):
  keep = (gate != 0).float()
  return combine_ref(src, index, pos, keep, s, g_l, c)


def combine_bwd_gate(yc, dy, index, pos, gate, s, g_l, c):
  """dgate `[2, T]` = ⟨yc[slot], dy[t]⟩ for kept choices (0 for dropped ones)."""
  return ops.native().moe_combine_bwd_gate(yc.contiguous(), dy.contiguous(),
                                           _K(index, g_l, s), _K(pos, g_l, s),
                                           _K(gate.float(), g_l, s), int(s), int(g_l),
                                           int(c)).view(2, -1)


def combine_bwd_gate_ref(yc, dy, index, pos, gate, s, g_l, c):
  m = yc.shape[-1]
  rows = yc.reshape(-1, m).float()
  slots = _Slots(index, pos, s, g_l, c).clamp(0, rows.shape[0] - 1)
  dots = (rows[slots] * dy.float().unsqueeze(0)).sum(-1)
  return torch.where(gate != 0, dots, torch.zeros_like(dots))


# ------------------------------------------------------------------- gating oracle --
def top2_gate_ref(logits, paddings, capacity, legacy_mtf_behavior=False):
  """fp32 oracle of the gate half of `moe_gate_dispatch`: → NestedMap(index `[2, G, S]`,
  pos `[2, G, S]`, gate `[2, G, S]`, aux_loss). Thin adapter over
  `gshard_layers.Top2GatingIndices` (the reference formulation, ref gshard_layers.py:1970)."""
  from lingvo_b200.core import gshard_layers   # pylint: disable=g-import-not-at-top
  e = logits.shape[-1]
  g = gshard_layers.Top2GatingIndices(
      logits.float(), paddings, e, capacity, torch.float32, 'all', 0.0,
      legacy_mtf_behavior, 2.0, None)
  return g
