"""Flat beam search (ref `lingvo/core/flat_beam_search_helper.py:69`).

A beam search whose hypotheses live in ONE flat token buffer per batch element
(`buf_size = beam_size · max_steps`): every step appends `beam_size` tokens, and a
hyp is the chain of buffer positions linked by `parent` indices, so the decoder
callback can attend over the whole buffer with a `[beam, buf]` ancestor mask
instead of re-ordering per-hyp caches. Decoder callback:

  dec_callback(tgt_id [B,K], tgt_pos [B,K], tgt_segment_id, tgt_mask [B,K,buf],
               dec_state, t) → (logits [B,K,V], dec_state)

Returns ((ids, lens, scores) for the n-best, final dec_state).

With a `prefix` (the reference's layout) every row continues its own prompt. Prompts are
right-aligned in `prefix [B, P]` (P a multiple of K) so that the last prompt token P* sits
at the same column in every row. The buffer then holds `P + K · max_steps` slots:

  * one callback `dec_callback(ids [B,P], pos [B,P], segment_id [B,P], None, dec_state, 0)`
    fills the decoder state with the prompt minus P*, shifted one slot right so that it
    ends at slot P−1 (slot s holds prompt token s−1−(P−plen); padding has segment id 0);
  * step i = 0 … max_steps−1 (t = P/K + i) feeds K tokens at slots t·K … t·K+K−1 with the
    mask `[B,K,buf]` of the slots each hypothesis sees (its prompt, its ancestors and its
    own slot). Step 0 feeds P* to all K hypotheses; hypotheses 1…K−1 start at a score of
    −1e30, so the first expansion comes from hypothesis 0 alone.

The returned ids `[B, n, max_steps]` are the continuations only, ending in EOS.
"""

from __future__ import annotations

import torch

NEG = -1.0e30


def einsum_i32(eq, *args):  # pylint: disable=invalid-name
  """Integer einsum (exact for masks / ids): operands and result are int32 (ref :47)."""
  return torch.einsum(eq, *[x.to(torch.int32) for x in args]).to(torch.int32)


def update_nbest(nbest_hyps, cur_hyps):  # pylint: disable=invalid-name
  """Merges (mask, score) n-best lists keeping the best `k` (ref :52)."""
  (m0, s0), (m1, s1) = nbest_hyps, cur_hyps
  k = s0.shape[1]
  score = torch.cat([s0, s1], 1)
  mask = torch.cat([m0, m1], 1)
  top, idx = torch.topk(score, k, 1)
  return mask.gather(1, idx.unsqueeze(-1).expand(-1, -1, mask.shape[-1])), top


def flat_beam_search(batch_size, beam_size, max_steps, dec_callback, dec_state, bos_id=1,  # pylint: disable=invalid-name
                     eos_id=2, length_norm_alpha=0.8, beam_gap=3.0, top_k_fn=None, prefix=None,
                     prefix_len=None, fprop_dtype=torch.float32, ext_size=0, nbest_size=None,
                     debug=False, device=None):
  del top_k_fn, ext_size, debug, fprop_dtype
  if prefix is not None:
    return _PrefixBeamSearch(batch_size, beam_size, max_steps, dec_callback, dec_state, eos_id,
                             length_norm_alpha, beam_gap, prefix, prefix_len, nbest_size,
                             device)
  assert prefix_len is None
  b, k = batch_size, beam_size
  nbest = nbest_size or k
  buf = k * max_steps
  dev = device or torch.device('cpu')
  buf_ids = torch.zeros(b, buf, dtype=torch.int64, device=dev)
  buf_parent = torch.full((b, buf), -1, dtype=torch.int64, device=dev)
  anc = torch.zeros(b, buf, buf, dtype=torch.bool, device=dev)      # anc[b, i, j]: j ∈ path(i)
  score = torch.full((b, k), NEG, device=dev)
  score[:, 0] = 0.0                                                   # only hyp 0 is live
  cur_ids = torch.full((b, k), bos_id, dtype=torch.int64, device=dev)
  cur_slot = torch.full((b, k), -1, dtype=torch.int64, device=dev)   # buffer slot of each hyp
  best_scores = torch.full((b, nbest), NEG, device=dev)
  best_slots = torch.full((b, nbest), -1, dtype=torch.int64, device=dev)
  best_lens = torch.zeros(b, nbest, dtype=torch.int64, device=dev)
  ar = torch.arange(b, device=dev).unsqueeze(1)
  for t in range(max_steps):
    pos = torch.full((b, k), t, dtype=torch.int64, device=dev)
    # ancestors mask of each live hyp over the buffer (+ itself is fed as tgt_id)
    mask = torch.zeros(b, k, buf, dtype=torch.bool, device=dev)
    live = cur_slot >= 0
    if t > 0:
      mask = anc[ar, cur_slot.clamp_min(0)] & live.unsqueeze(-1)
    logits, dec_state = dec_callback(cur_ids, pos, None, mask, dec_state, t)
    logp = torch.log_softmax(logits.float(), -1)
    v = logp.shape[-1]
    total = score.unsqueeze(-1) + logp                               # [B,K,V]
    # finished candidates
    eos_total = total[:, :, eos_id]
    norm = ((5.0 + t + 1) / 6.0) ** length_norm_alpha
    fin = torch.where(score > NEG / 2, eos_total / norm, torch.full_like(eos_total, NEG))
    cand_scores = torch.cat([best_scores, fin], 1)
    cand_slots = torch.cat([best_slots, cur_slot], 1)
    cand_lens = torch.cat([best_lens, torch.full((b, k), t + 1, dtype=torch.int64, device=dev)], 1)
    best_scores, idx = torch.topk(cand_scores, nbest, 1)
    best_slots, best_lens = cand_slots.gather(1, idx), cand_lens.gather(1, idx)
    # continuations
    total[:, :, eos_id] = NEG
    top, flat = torch.topk(total.reshape(b, -1), k, 1)
    parent_hyp, tok = flat // v, flat % v
    slot = t * k + torch.arange(k, device=dev).unsqueeze(0).expand(b, k)
    par_slot = cur_slot.gather(1, parent_hyp)
    buf_ids[ar, slot] = tok
    buf_parent[ar, slot] = par_slot
    par_anc = anc[ar, par_slot.clamp_min(0)] & (par_slot >= 0).unsqueeze(-1)
    new_anc = par_anc.clone()
    new_anc[ar, torch.arange(k, device=dev).unsqueeze(0).expand(b, k), slot] = True
    anc[ar, slot] = new_anc
    score, cur_ids, cur_slot = top, tok, slot
    if beam_gap is not None and (t + 1) % 4 == 0:
      live_best = (score / norm).max(1).values
      if bool(((best_scores[:, 0] - live_best) > beam_gap).all()):
        break
  # materialise the n-best token sequences by walking parents
  out_ids = torch.full((b, nbest, max_steps + 1), eos_id, dtype=torch.int64, device=dev)
  lens = best_lens.clone()
  slot = best_slots.clone()
  for step in range(max_steps - 1, -1, -1):
    take = (slot >= 0) & (best_lens - 1 > step)
    tok = buf_ids[ar, slot.clamp_min(0)]
    # token at position `step` belongs to the hyp iff its depth matches
    depth = slot.clamp_min(0) // k
    here = take & (depth == step)
    out_ids[:, :, step] = torch.where(here, tok, out_ids[:, :, step])
    slot = torch.where(here, buf_parent[ar, slot.clamp_min(0)], slot)
  return (out_ids, lens, best_scores), dec_state


def _PrefixBeamSearch(batch_size, beam_size, max_steps, dec_callback, dec_state, eos_id,  # pylint: disable=invalid-name
                      length_norm_alpha, beam_gap, prefix, prefix_len, nbest_size, device):
  """`flat_beam_search` from right-aligned prompts (see the module docstring)."""
  b, k = batch_size, beam_size
  nbest = nbest_size or k
  dev = device or prefix.device
  pfx = prefix.to(dev).long()
  plen = prefix_len.to(dev).long()
  pmax = pfx.shape[1]
  if pfx.shape[0] != b or plen.shape != (b,):
    raise ValueError('prefix must be [batch, P] and prefix_len [batch]')
  if pmax % k:
    raise ValueError('prefix length %d must be a multiple of beam_size %d' % (pmax, k))
  if bool(((plen < 1) | (plen > pmax)).any()):
    raise ValueError('prefix_len must be in [1, %d]' % pmax)
  t0 = pmax // k
  buf = pmax + k * max_steps
  idx = torch.arange(pmax, device=dev) - pmax + (plen - 1).unsqueeze(1)   # position at a slot
  pad = idx >= 0                                                          # (P* excluded)
  pfx_id = torch.roll(pfx, 1, 1) * pad
  _, dec_state = dec_callback(pfx_id, idx.clamp_min(0), pad.long(), None, dec_state, 0)

  ar_k = torch.arange(k, device=dev)
  cur_ids = pfx[:, -1:].expand(b, k).clone()
  pos = (plen - 1).unsqueeze(1).expand(b, k).clone()
  mask = torch.zeros(b, k, buf, dtype=torch.bool, device=dev)
  mask[:, :, :pmax] = pad.unsqueeze(1)
  mask[:, ar_k, pmax + ar_k] = True
  buf_ids = torch.zeros(b, buf, dtype=torch.int64, device=dev)
  score = torch.full((b, k), NEG, device=dev)
  score[:, 0] = 0.0
  best_scores = torch.full((b, nbest), NEG, device=dev)
  best_masks = torch.zeros(b, nbest, buf, dtype=torch.bool, device=dev)
  for i in range(max_steps):
    t = t0 + i
    buf_ids[:, t * k:(t + 1) * k] = cur_ids
    logits, dec_state = dec_callback(cur_ids, pos, None, mask, dec_state, t)
    logp = torch.log_softmax(logits.float(), -1)
    v = logp.shape[-1]
    total = score.unsqueeze(-1) + logp                               # [B,K,V]
    # finished candidates: i generated tokens + EOS
    norm = ((5.0 + i + 1) / 6.0) ** length_norm_alpha
    fin = torch.where(score > NEG / 2, total[:, :, eos_id] / norm, torch.full_like(score, NEG))
    best_masks, best_scores = update_nbest((best_masks, best_scores), (mask, fin))
    # continuations
    total[:, :, eos_id] = NEG
    top, flat = torch.topk(total.reshape(b, -1), k, 1)
    parent, tok = flat // v, flat % v
    mask = mask.gather(1, parent.unsqueeze(-1).expand(b, k, buf))
    if i + 1 < max_steps:
      mask[:, ar_k, (t + 1) * k + ar_k] = True
    score, cur_ids, pos = top, tok, pos.gather(1, parent) + 1
    if beam_gap is not None and (i + 1) % 4 == 0:
      live_best = (score / norm).max(1).values
      if bool(((best_scores[:, 0] - live_best) > beam_gap).all()):
        break
  # continuation tokens: the tokens fed after P* on each candidate's path, then EOS
  cont = best_masks[:, :, pmax + k:]
  at = torch.where(cont, cont.long().cumsum(-1) - 1, torch.full_like(cont, max_steps, dtype=torch.long))
  out_ids = torch.full((b, nbest, max_steps + 1), eos_id, dtype=torch.int64, device=dev)
  out_ids.scatter_(2, at, buf_ids[:, pmax + k:].unsqueeze(1).expand_as(at))
  lens = torch.where(best_scores > NEG / 2, cont.sum(-1) + 1, torch.zeros_like(best_scores,
                                                                              dtype=torch.long))
  return (out_ids[:, :, :max_steps], lens, best_scores), dec_state
