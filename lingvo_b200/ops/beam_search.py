"""Device-resident beam search step + terminated-hyp ranking (SURVEY K13).

Re-design of the reference's CPU ops `BeamSearchStep` / `TopKTerminatedHyps`
(ref `lingvo/core/ops/beam_search_step_op_kernels.cc:100-950`, `:955-1660`): the
reference runs one host thread per beam over STL heaps and serialises `Hypothesis`
protos; here the whole step is a handful of batched tensor ops on the GPU
(per-hyp top-(K+1), one per-beam top-K over K·(K+1) survivors, masked scatters),
so the decode loop never synchronises with the host and can be captured in a
CUDA graph. Terminated hypotheses are kept as struct-of-arrays
(`done_scores[t, hyp]`) and materialised by back-tracking `prev_hyps` once, at
the end.

Index convention (same as the reference, `…kernels.cc:336`): flat hyp index =
`hyp_id * num_beams + beam_id`.

Semantics kept from the reference:
  * candidate order: global score desc, then word id asc, then hyp id asc;
  * step 0 expands only hyp 0 of each beam;
  * EOS terminates a hyp iff it is among the hyp's own K best tokens (or
    `force_eos_in_top_k`), `global > best_in_hyp − valid_eos_max_logit_delta`
    and `local > local_eos_threshold`;
  * a beam is done when no active hyp scores above
    `best_terminated − beam_size` (and, with `ensure_full_beam`, K hyps have
    terminated).
"""

from __future__ import annotations

from typing import NamedTuple, Optional

import torch

NEG = -1.0e30


class BeamState(NamedTuple):
  best_scores: torch.Tensor        # [num_beams]   best terminated score so far
  cumulative_scores: torch.Tensor  # [num_hyps]
  scores: torch.Tensor             # [T, num_hyps] local score of the token chosen at t
  hyps: torch.Tensor               # [T, num_hyps] token ids
  prev_hyps: torch.Tensor          # [T, num_hyps] flat index of the parent hyp
  done_scores: torch.Tensor        # [T, num_hyps] global score of a hyp terminated at t (NEG: none)
  atten_probs: torch.Tensor        # [T, num_hyps, S]
  beam_done: torch.Tensor          # [num_beams] bool
  num_done: torch.Tensor           # [num_beams] number of terminated hyps


def init_state(num_beams, num_hyps_per_beam, max_steps, src_len, device,
               dtype=torch.float32) -> BeamState:
  n = num_beams * num_hyps_per_beam
  return BeamState(
      best_scores=torch.full((num_beams,), NEG, device=device, dtype=dtype),
      cumulative_scores=torch.zeros(n, device=device, dtype=dtype),
      scores=torch.zeros(max_steps, n, device=device, dtype=dtype),
      hyps=torch.zeros(max_steps, n, device=device, dtype=torch.int64),
      prev_hyps=torch.zeros(max_steps, n, device=device, dtype=torch.int64),
      done_scores=torch.full((max_steps, n), NEG, device=device, dtype=dtype),
      atten_probs=torch.zeros(max_steps, n, max(src_len, 1), device=device, dtype=dtype),
      beam_done=torch.zeros(num_beams, device=device, dtype=torch.bool),
      num_done=torch.zeros(num_beams, device=device, dtype=torch.int64))


def _TopKRef(log_probs, cum, active, k, eos_id):
  """Plain-PyTorch form of `beam_topk` (CPU path and numerics oracle of the kernel).

  Scores are floored at NEG as in the kernel, whose lists start at NEG: a row with fewer than
  k candidates above NEG pads its top-k with (NEG, word 0), and a row whose every score is
  below NEG has best_in_hyp = NEG."""
  lp = log_probs.float()
  glob = cum.unsqueeze(1) + lp
  best_in_hyp = glob.max(1).values.clamp_min(NEG)
  eos_glob = glob[:, eos_id]
  glob_no_eos = glob.clone()
  glob_no_eos[:, eos_id] = NEG
  glob_no_eos = torch.where(active.unsqueeze(1), glob_no_eos, torch.full_like(glob_no_eos, NEG))
  # score desc, word id asc on ties: stable sort of the (ascending-id) row
  order = torch.argsort(glob_no_eos, dim=1, descending=True, stable=True)[:, :k]
  top_s = glob_no_eos.gather(1, order).clamp_min(NEG)
  top_w = torch.where(top_s > NEG / 2, order, torch.zeros_like(order))
  return top_s, top_w, best_in_hyp, eos_glob, lp[:, eos_id]


def _TopK(log_probs, cum, active, k, eos_id):
  """Fused score-add + EOS mask + per-hyp top-K (`csrc/beam_kernels.cu` on the GPU)."""
  from lingvo_b200 import ops  # pylint: disable=g-import-not-at-top
  if (ops.use_cuda_kernels(log_probs) and k <= 16 and
      log_probs.dtype in (torch.float32, torch.bfloat16)):
    return tuple(ops.native().beam_topk(log_probs.contiguous(), cum, active, int(k), int(eos_id)))
  return _TopKRef(log_probs, cum, active, k, eos_id)


def beam_search_step(log_probs, atten_probs, state: BeamState, cur_step: int,
                     eos_id: int, beam_size: float, num_hyps_per_beam: int,
                     valid_eos_max_logit_delta: float = 5.0,
                     local_eos_threshold: float = -100.0,
                     ensure_full_beam: bool = False,
                     force_eos_in_last_step: bool = False,
                     is_last_step: bool = False,
                     allow_empty_terminated_hyp: bool = True,
                     force_eos_in_top_k: bool = False,
                     beam_independence: bool = True,
                     merge_paths: bool = False,
                     eoc_id: int = -1,
                     path_ids: Optional[torch.Tensor] = None):
  """One step. log_probs `[num_hyps, V]`, atten_probs `[num_hyps, S]`.

  Options beyond the basics (reference `beam_search_step_op_kernels.cc:47-76,115,154`):
    * `force_eos_in_top_k`: EOS is always a candidate of its hyp; otherwise (default) a hyp
      can only terminate when EOS is among *its own* K best tokens. The
      `valid_eos_max_logit_delta` / `local_eos_threshold` tests always apply.
    * `beam_independence` (always honoured here): a finished beam's rows are frozen, the
      step is a no-op for it, other beams continue.
    * `merge_paths` (+ `eoc_id`, `path_ids`): for epsilon-emitting models (RNN-T / NT).
      Surviving candidates of a beam whose label sequences are identical once epsilons
      (`eoc_id`) are removed are merged: one survivor keeps the log-sum-exp of their
      scores. `path_ids [num_hyps]` is an int64 hash of each row's epsilon-free prefix
      (maintained by this function; pass the previous step's `state_path_ids`).

  Returns (new_state, all_done [scalar bool tensor]) — and, with `merge_paths`,
  (new_state, all_done, new_path_ids).
  """
  n, v = log_probs.shape
  k = num_hyps_per_beam
  b = n // k
  dev = log_probs.device
  cum = state.cumulative_scores.float()

  # hyp (row) is active unless its beam is done; on step 0 only hyp_id 0 is live.
  beam_of = torch.arange(n, device=dev) % b
  hyp_id = torch.arange(n, device=dev) // b
  active = ~state.beam_done[beam_of]
  if cur_step == 0:
    active = active & (hyp_id == 0)

  # ---- fused: global scores, EOS column, per-hyp top-K --------------------------
  kk = min(k, v - 1) if v > 1 else 1
  top_s, top_w, best_in_hyp, eos_glob, eos_local = _TopK(log_probs, cum, active, kk, eos_id)
  lp = log_probs

  # ---- EOS handling ----------------------------------------------------------
  eos_ok = (eos_glob > best_in_hyp - valid_eos_max_logit_delta) & (
      eos_local > local_eos_threshold) & active
  if not force_eos_in_top_k:
    # EOS must be one of the hyp's own K best tokens: at most K−1 others beat it
    eos_ok = eos_ok & (eos_glob >= top_s[:, kk - 1])
  if not allow_empty_terminated_hyp and cur_step == 0:
    eos_ok = torch.zeros_like(eos_ok)
  if force_eos_in_last_step and is_last_step:
    eos_ok = active
  # regroup rows by beam: [b, k(hyp), kk]
  s_b = top_s.view(k, b, kk).permute(1, 0, 2).reshape(b, k * kk)
  w_b = top_w.view(k, b, kk).permute(1, 0, 2).reshape(b, k * kk)
  h_b = hyp_id.view(k, b, 1).expand(k, b, kk).permute(1, 0, 2).reshape(b, k * kk)
  # deterministic tie-break: score desc, word asc, hyp asc → lexicographic key
  order = torch.argsort(h_b, dim=1, stable=True)
  s_b, w_b, h_b = s_b.gather(1, order), w_b.gather(1, order), h_b.gather(1, order)
  order = torch.argsort(w_b, dim=1, stable=True)
  s_b, w_b, h_b = s_b.gather(1, order), w_b.gather(1, order), h_b.gather(1, order)
  order = torch.argsort(s_b, dim=1, descending=True, stable=True)[:, :k]
  sel_s, sel_w, sel_h = s_b.gather(1, order), w_b.gather(1, order), h_b.gather(1, order)

  new_path_ids = None
  if merge_paths:
    # Epsilon-free label hash of every surviving candidate: emitting `eoc_id` keeps the
    # parent's hash, any other token extends it. Equal hashes inside a beam ⇒ same path:
    # the best one absorbs the probability mass (log-sum-exp), duplicates are dropped.
    assert path_ids is not None, 'merge_paths needs the previous path_ids'
    par = (sel_h * b + torch.arange(b, device=dev).unsqueeze(1))
    ph = path_ids[par]
    ext = (ph * 1000003 + sel_w + 1) & 0x7FFFFFFFFFFFFFF
    cand_hash = torch.where(sel_w == eoc_id, ph, ext)
    same = (cand_hash.unsqueeze(2) == cand_hash.unsqueeze(1)) & (
        sel_s.unsqueeze(2) > NEG / 2) & (sel_s.unsqueeze(1) > NEG / 2)
    earlier = torch.tril(torch.ones(k, k, dtype=torch.bool, device=dev), -1)
    dup = (same & earlier.unsqueeze(0)).any(2)                      # a better twin exists
    merged = torch.logsumexp(
        torch.where(same, sel_s.unsqueeze(1).expand(b, k, k), torch.full_like(same, NEG, dtype=sel_s.dtype)),
        dim=2)
    sel_s = torch.where(dup, torch.full_like(sel_s, NEG), torch.where(
        sel_s > NEG / 2, merged, sel_s))
    new_path_ids = cand_hash.t().reshape(-1)

  # A hyp whose EOS candidate passed the tests above is moved off the beam and recorded
  # as terminated (reference :281-293, :795-812) — it does not compete with continuations.
  eos_keep = eos_ok
  done_row = torch.where(eos_keep, eos_glob, torch.full_like(eos_glob, NEG))
  done_scores = state.done_scores.clone()
  done_scores[cur_step] = done_row.to(done_scores.dtype)
  best_term = torch.full((b,), NEG, device=dev).scatter_reduce(
      0, beam_of, done_row, reduce='amax', include_self=True)
  best_scores = torch.maximum(state.best_scores.float(), best_term)
  num_done = state.num_done + torch.zeros(b, device=dev, dtype=torch.int64).scatter_add(
      0, beam_of, eos_keep.to(torch.int64))

  # ---- write the K new hyps of every beam ---------------------------------------
  # new flat index = new_hyp_id * b + beam
  new_cum = sel_s.t().reshape(-1)                                  # [k*b]
  new_w = sel_w.t().reshape(-1)
  parent = (sel_h * b + torch.arange(b, device=dev).unsqueeze(1)).t().reshape(-1)
  valid = new_cum > NEG / 2
  frozen = state.beam_done[beam_of]                                # done beams keep state
  keep_old = frozen | ~valid
  new_cum = torch.where(keep_old, torch.where(frozen, cum, torch.full_like(cum, NEG)), new_cum)
  local = torch.where(valid, lp[parent, new_w].float(), torch.zeros_like(new_cum))
  scores = state.scores.clone()
  hyps = state.hyps.clone()
  prev = state.prev_hyps.clone()
  attn = state.atten_probs.clone()
  scores[cur_step] = local.to(scores.dtype)
  hyps[cur_step] = torch.where(valid, new_w, torch.zeros_like(new_w))
  prev[cur_step] = torch.where(valid, parent, torch.arange(n, device=dev))
  if atten_probs is not None and attn.shape[-1] == atten_probs.shape[-1]:
    attn[cur_step] = atten_probs[parent].to(attn.dtype)

  # ---- beam termination -----------------------------------------------------------
  best_active = sel_s[:, 0]
  done_now = (best_active <= best_scores - beam_size) | (best_active <= NEG / 2)
  if ensure_full_beam:
    done_now = done_now & (num_done >= k)
  beam_done = state.beam_done | (done_now & (best_scores > NEG / 2)) | (
      best_active <= NEG / 2)
  new_state = BeamState(best_scores.to(state.best_scores.dtype),
                        new_cum.to(state.cumulative_scores.dtype), scores, hyps, prev,
                        done_scores, attn, beam_done, num_done)
  del beam_independence
  if merge_paths:
    keep_ids = torch.where(valid & ~frozen, new_path_ids, path_ids)
    return new_state, beam_done.all(), keep_ids
  return new_state, beam_done.all()


def top_k_terminated_hyps(state: BeamState, src_lens, k: int, num_steps: int,
                          length_normalization: float = 0.0,
                          coverage_penalty: float = 0.0,
                          target_seq_length_ratio: float = 1.0,
                          eos_id: int = 2):
  """Ranks terminated hyps of every beam (ref :955-1100).

  Returns ids `[num_beams, k, T]`, lens `[num_beams, k]`, scores `[num_beams, k]`
  (normalised). Empty slots have len 0 and score NEG.
  """
  t_max, n = state.done_scores.shape
  b = state.best_scores.shape[0]
  dev = state.done_scores.device
  t_used = min(num_steps, t_max)
  done = state.done_scores[:t_used].float()                        # [t, n]
  # Back-track: ancestors[t', t, n] would be big; walk back once per end-time instead.
  # seqs[t_end, n, :] = ids of the path that ends (with EOS) at step t_end from row n.
  ids = torch.zeros(t_used, n, t_used, dtype=torch.int64, device=dev)
  sum_scores = torch.zeros(t_used, n, device=dev)
  cov = None
  if coverage_penalty > 0:
    cov = torch.zeros(t_used, n, state.atten_probs.shape[-1], device=dev)
  for t_end in range(t_used):
    row = torch.arange(n, device=dev)
    ids[t_end, :, t_end] = eos_id
    if coverage_penalty > 0 and t_end < state.atten_probs.shape[0]:
      cov[t_end] += state.atten_probs[t_end].float()      # attention at the EOS step
    for t in range(t_end - 1, -1, -1):
      ids[t_end, :, t] = state.hyps[t, row]
      sum_scores[t_end] += state.scores[t, row].float()
      if coverage_penalty > 0:
        cov[t_end] += state.atten_probs[t, row].float()
      row = state.prev_hyps[t, row]
  length = torch.arange(1, t_used + 1, device=dev).float().unsqueeze(1)   # incl. EOS
  norm = ((length + 5.0) ** length_normalization) / (5.0 ** length_normalization)
  final = done / norm
  if coverage_penalty > 0:
    sl = src_lens.float().clamp_min(1.0)
    beam_of = torch.arange(n, device=dev) % b
    src_mask = (torch.arange(cov.shape[-1], device=dev).unsqueeze(0) <
                sl[beam_of].unsqueeze(1)).float()
    pen = (torch.log((cov / target_seq_length_ratio).clamp(1e-3, 0.5)) *
           src_mask.unsqueeze(0)).sum(-1)
    final = final + target_seq_length_ratio * coverage_penalty * pen
  final = torch.where(done > NEG / 2, final, torch.full_like(final, NEG))
  # candidates of beam j: all (t, hyp_id) with flat index hyp_id*b + j
  cand = final.view(t_used, -1, b).permute(2, 0, 1).reshape(b, -1)         # [b, t*k0]
  # ties → shorter first: candidates are laid out by increasing t, stable sort keeps it
  order = torch.argsort(cand, dim=1, descending=True, stable=True)[:, :k]
  top_scores = cand.gather(1, order)
  k0 = n // b
  t_idx = order // k0
  h_idx = order % k0
  flat = h_idx * b + torch.arange(b, device=dev).unsqueeze(1)
  top_ids = ids[t_idx, flat]                                               # [b, k, T]
  lens = torch.where(top_scores > NEG / 2, t_idx + 1, torch.zeros_like(t_idx))
  mask = torch.arange(t_used, device=dev).view(1, 1, -1) < lens.unsqueeze(-1)
  return top_ids * mask, lens, top_scores
