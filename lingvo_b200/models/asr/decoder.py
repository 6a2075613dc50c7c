"""LAS attention decoder (ref `lingvo/tasks/asr/decoder.py`: `AsrDecoderBase` :48,
`AsrDecoder` :1378).

Embedding → attention LSTM (input `[emb_t ; context_{t-1}]`, its output queries the attention)
→ (N−1) LSTMs that also see the context (residual from `residual_start`) → softmax over
`[rnn_out ; context]`. Features of the reference decoder that are implemented here:

  * **scheduled sampling** (`min_ground_truth_prob < 1`; ref :1286-1376): from
    `prob_decay_start_step` to `min_prob_step` the probability of feeding the ground-truth
    token decays linearly to `min_ground_truth_prob`; otherwise the token *sampled* from the
    previous step's distribution is fed;
  * **LM fusion** (`p.fusion`, `fusion.py`) — the fusion layer steps its LM next to the
    decoder and produces the fused logits, in training and in beam search;
  * **contextualizer** (`p.contextualizer`) — biasing context attended with the same query and
    combined with the audio context;
  * **adapters** (`adapter_task_id_field`): a `MultitaskAdapterLayer` after every RNN layer,
    task ids taken from the encoder outputs;
  * **losses**: label smoothing or `targets.probs`, focal loss (`focal_loss_alpha/gamma`),
    per-token or per-sequence averaging, `token_normalized_per_seq_loss`, several weighted
    logit heads (`logit_types`), per-sequence losses for MWER-style training.

H100 notes. Two execution plans share the same cells and weights:
  * the *sequence plan* (teacher forcing, no per-step feedback): the attention LSTM runs its
    step loop, but the upper LSTMs and the softmax run over the whole `[T, B, ·]` sequence —
    their input GEMMs are hoisted out of the time loop onto the tensor cores;
  * the *step plan* (`SingleDecodeStep`, used whenever a step depends on the previous step's
    prediction: scheduled sampling, fusion, adapters, and always in beam search) keeps every
    tensor on the device; sampling uses `torch.multinomial` on device logits — no host sync.
"""

from __future__ import annotations

import collections

import torch
import torch.nn.functional as F

from lingvo_b200.core import attention
from lingvo_b200.core import base_decoder
from lingvo_b200.core import layers
from lingvo_b200.core import py_utils
from lingvo_b200.core import rnn_cell
from lingvo_b200.core import rnn_layers
from lingvo_b200.core import summary_utils
from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.models.asr import contextualizer_base
from lingvo_b200.models.asr import fusion as fusion_lib


def SoftmaxCrossEntropyFocalLoss(logits, label_ids=None, label_probs=None, alpha=None,
                                 gamma=None):
  """Per-token softmax cross entropy with the focal modulation (1 − p_t)^γ · α_t
  (ref `py_utils.SoftmaxCrossEntropyFocalLoss`). `label_probs` (soft targets) take precedence
  over `label_ids`. With γ = α = None this is the plain cross entropy."""
  lp = F.log_softmax(logits.float(), -1)
  if label_probs is not None:
    lpr = label_probs.float()
    loss = -(lpr * lp)
    if gamma is not None and gamma != 0:
      loss = loss * torch.pow(1.0 - lp.exp(), gamma)
    if alpha is not None:
      a = torch.as_tensor(alpha, dtype=loss.dtype, device=loss.device)
      loss = loss * a
    return loss.sum(-1)
  ll = lp.gather(-1, label_ids.long().unsqueeze(-1)).squeeze(-1)
  loss = -ll
  if gamma is not None and gamma != 0:
    loss = loss * torch.pow(1.0 - ll.exp(), gamma)
  if alpha is not None:
    a = torch.as_tensor(alpha, dtype=loss.dtype, device=loss.device)
    loss = loss * (a[label_ids.long()] if a.dim() else a)
  return loss


class AsrDecoderBase(base_decoder.BaseBeamSearchDecoder):
  """Shared machinery of speech decoders (ref :48)."""

  TargetInfo = collections.namedtuple('TargetInfo',
                                      ['id', 'label', 'weight', 'emb', 'padding', 'misc'])

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('dropout_prob', 0.0, 'Prob at which we do dropout.')
    p.Define('emb', layers.EmbeddingLayer.Params(), 'Embedding layer params.')
    p.Define('emb_dim', 0, 'Dimension of the embedding layer.')
    p.Define('label_smoothing', None, 'Label smoothing class params.')
    p.Define('rnn_cell_tpl', rnn_cell.LSTMCellSimple.Params(), 'RNN cell template.')
    p.Define('rnn_cell_dim', 0, 'Size of the rnn cells.')
    p.Define('rnn_cell_hidden_dim', 0, 'Internal size of the rnn cells (projection if > 0).')
    p.Define('attention', attention.AdditiveAttention.Params(), 'Attention params.')
    p.Define('softmax', layers.SimpleFullSoftmax.Params(), 'Softmax params.')
    p.Define('softmax_uses_attention', True, 'Feed the attention context to the softmax.')
    p.Define('source_dim', 0, 'Dimension of the source encodings.')
    p.Define('atten_context_dim', 0, 'Depth of the attention context (0: source_dim).')
    p.Define('first_rnn_input_dim', 0, 'Kept for parity (derived from emb + context).')
    p.Define('rnn_layers', 1, 'Number of rnn layers.')
    p.Define('residual_start', 0, 'Residual connections from this layer on (0: none).')
    p.Define('fusion', fusion_lib.NullFusion.Params(), 'Fusion class params.')
    p.Define('parallel_iterations', 30, 'Kept for parity (no while-loop on this runtime).')
    p.Define('per_token_avg_loss', True,
             'Per-token average loss; otherwise the mean of the per-sequence losses.')
    p.Define('token_normalized_per_seq_loss', False,
             'Normalise the per-sequence loss by the sequence length.')
    p.Define('min_ground_truth_prob', 1.0,
             'Min probability of feeding the ground truth as the previous token '
             '(scheduled sampling); 1.0 disables sampling.')
    p.Define('min_prob_step', 1e6, 'Step at which min_ground_truth_prob is reached.')
    p.Define('prob_decay_start_step', 1e4, 'Step at which the probability starts decaying.')
    p.Define('use_while_loop_based_unrolling', True,
             'Step-by-step unrolling (required by scheduled sampling).')
    p.Define('logit_types', {'logits': 1.0}, 'logit name → loss weight.')
    p.Define('use_unnormalized_logits_as_log_probs', True,
             'Beam search may use unnormalised (fused) logits as scores.')
    p.Define('contextualizer', contextualizer_base.NullContextualizer.Params(),
             'Contextualizer params.')
    p.Define('focal_loss_alpha', None, 'Focal loss weighting factor α.')
    p.Define('focal_loss_gamma', None, 'Focal loss focusing parameter γ.')
    p.Define('adapter_layer_tpl', layers.MultitaskAdapterLayer.Params(), 'Adapter layer params.')
    p.Define('adapter_task_id_field', None,
             'Field of encoder_outputs holding per-utterance task ids; enables adapters.')
    p.Define('teacher_forcing', True, 'Feed previous-token embeddings (else ones).')
    p.target_seq_len = 300
    return p

  @classmethod
  def UpdateTargetVocabSize(cls, p, vocab_size, wpm_model=None):
    p.emb.vocab_size = vocab_size
    p.softmax.num_classes = vocab_size
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.min_ground_truth_prob <= 1.0 and p.min_ground_truth_prob >= 0.0
    self._max_label_prob = 1.0 - p.min_ground_truth_prob
    self._decay_interval = float(p.min_prob_step - p.prob_decay_start_step)
    if self._max_label_prob > 0:
      assert self._decay_interval > 0
      assert p.use_while_loop_based_unrolling, 'scheduled sampling needs step-wise unrolling'

  # -- scheduled sampling ---------------------------------------------------------
  def GroundTruthProbability(self):
    """P(feed ground truth) at the current global step, a float32 0-d tensor."""
    p = self.params
    gs = py_utils.GetGlobalStep()
    step = gs.float() if isinstance(gs, torch.Tensor) else torch.tensor(float(gs))
    sampling_p = (step - p.prob_decay_start_step) / self._decay_interval
    return torch.clamp(1.0 - self._max_label_prob * sampling_p,
                       min=p.min_ground_truth_prob, max=1.0)

  # -- metrics --------------------------------------------------------------------
  def _ComputeMetrics(self, logits, target_labels, target_weights, target_probs=None):
    """logits `[B, T, V]`, labels/weights `[B, T]`, probs `[B, T, V]` →
    (metrics, per_sequence_loss `[B]`) (ref :638)."""
    p = self.params
    w = target_weights.float()
    wsum = w.sum()
    wsum_eps = wsum + 1e-6
    correct = (logits.argmax(-1) == target_labels.long()).float()
    accuracy = (correct * w).sum() / wsum_eps
    per_example = SoftmaxCrossEntropyFocalLoss(
        logits, label_ids=target_labels, label_probs=target_probs, alpha=p.focal_loss_alpha,
        gamma=p.focal_loss_gamma)
    per_sequence_loss = (per_example * w).sum(1)
    per_token_avg_loss = per_sequence_loss.sum() / wsum_eps
    if p.token_normalized_per_seq_loss:
      per_sequence_loss = per_sequence_loss / (w.sum(1) + 0.001)
    if p.per_token_avg_loss:
      loss, loss_weight = per_token_avg_loss, wsum
    else:
      loss = per_sequence_loss.mean()
      loss_weight = torch.tensor(float(per_sequence_loss.shape[0]), device=loss.device)
    metrics = {
        'loss': (loss, loss_weight),
        'log_pplx': (per_token_avg_loss, wsum),
        'token_normed_prob': (torch.exp(-per_token_avg_loss), wsum),
        'fraction_of_correct_next_step_preds': (accuracy, wsum),
    }
    return metrics, per_sequence_loss

  def ComputeLoss(self, theta, predictions, targets):
    """→ (metrics, {'loss': per-sequence −log p `[B]`}) (ref :721). Every head named in
    `logit_types` contributes with its weight; per-head metrics are kept as `<name>/<head>`."""
    p = self.params
    if 'probs' in targets:
      target_probs = targets.probs
    elif p.label_smoothing is not None:
      target_probs = self.smoother.FProp(theta.smoother, targets.paddings, targets.labels,
                                         targets.ids)
    else:
      target_probs = None
    merged = {}
    per_seq = 0.0
    for name, weight in p.logit_types.items():
      logits = predictions.Get(name)
      if logits is None:
        logits = self._ComputeLogits(theta, predictions.softmax_input).transpose(0, 1)
      metrics, seq_loss = self._ComputeMetrics(logits, targets.labels, targets.weights,
                                               target_probs)
      for k, (v, w) in metrics.items():
        merged['%s/%s' % (k, name)] = (v, w)
        acc = merged.get(k, (0.0, 0.0))
        merged[k] = (acc[0] + weight * v, acc[1] + weight * w)
      per_seq = per_seq + weight * seq_loss
    return NestedMap(merged), NestedMap(loss=per_seq)

  def _ComputeLogits(self, theta, softmax_input):
    return self.softmax.Logits(theta.softmax, softmax_input)


class AsrDecoder(AsrDecoderBase):
  """Listen-Attend-Spell decoder (ref :1378)."""

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.CreateChild('contextualizer', p.contextualizer)
    audio_ctx = p.atten_context_dim or p.source_dim
    ctx = audio_ctx + self.contextualizer.GetContextDim()
    self._audio_ctx, self._ctx = audio_ctx, ctx
    self.CreateChild('emb', p.emb.Copy().Set(embedding_dim=p.emb_dim))
    self.CreateChild('dropout', layers.DropoutLayer.Params().Set(keep_prob=1 - p.dropout_prob))
    atten = p.attention.Copy().Set(source_dim=p.source_dim, query_dim=p.rnn_cell_dim)
    cell = p.rnn_cell_tpl.Copy().Set(num_input_nodes=p.emb_dim + ctx,
                                     num_output_nodes=p.rnn_cell_dim,
                                     num_hidden_nodes=p.rnn_cell_hidden_dim)
    self.CreateChild('atten_rnn', rnn_layers.FRNNWithAttention.Params().Set(
        cell=cell, attention=atten, use_zero_atten_state=True, atten_context_dim=audio_ctx,
        packed_input=p.packed_input))
    rnns = []
    for i in range(1, p.rnn_layers):
      rnns.append(rnn_layers.FRNN.Params().Set(
          name='rnn_%d' % i, cell=p.rnn_cell_tpl.Copy().Set(
              num_input_nodes=p.rnn_cell_dim + ctx, num_output_nodes=p.rnn_cell_dim,
              num_hidden_nodes=p.rnn_cell_hidden_dim)))
    self.CreateChildren('rnn', rnns)
    sm_in = p.rnn_cell_dim + (ctx if p.softmax_uses_attention else 0)
    self.CreateChild('softmax', p.softmax.Copy().Set(input_dim=sm_in))
    fp = p.fusion.Copy()
    if fp.base_model_logits_dim is None:
      fp.base_model_logits_dim = p.softmax.num_classes
    self.CreateChild('fusion', fp)
    if p.label_smoothing is not None:
      self.CreateChild('smoother', p.label_smoothing.Copy().Set(
          num_classes=p.softmax.num_classes))
    if p.adapter_task_id_field:
      self.CreateChildren('adapters', [
          p.adapter_layer_tpl.Copy().Set(name='adapter_%d' % i, input_dim=p.rnn_cell_dim,
                                         data_format='TBC') for i in range(p.rnn_layers)])

  # -- plans ------------------------------------------------------------------------
  def _NeedsStepPlan(self):
    p = self.params
    return (self._max_label_prob > 0 or bool(p.adapter_task_id_field) or
            not isinstance(self.fusion, fusion_lib.NullFusion) or
            self.contextualizer.GetContextDim() > 0 or not p.teacher_forcing)

  def ComputePredictions(self, theta, encoder_outputs, targets):
    """→ NestedMap(softmax_input `[T, B, D]`, logits `[B, T, V]` (step plan),
    attention.probs `[T, B, S]`)."""
    if self._NeedsStepPlan():
      return self.ComputePredictionsDynamic(theta, encoder_outputs, targets)
    p = self.params
    ids = targets.ids.t().long()
    pad = targets.paddings.t().float().unsqueeze(-1)
    emb = self.dropout.FProp(theta.dropout, self.emb.EmbLookup(theta.emb, ids))
    ctx, xs, probs, _ = self.atten_rnn.FProp(
        theta.atten_rnn, encoder_outputs.encoded, encoder_outputs.padding, emb, pad)
    for i, r in enumerate(self.rnn):
      ys, _ = r.FProp(theta.rnn[i], torch.cat([xs, ctx], -1), pad)
      ys = self.dropout.FProp(theta.dropout, ys)
      xs = xs + ys if (p.residual_start and i + 2 >= p.residual_start) else ys
    sm_in = torch.cat([xs, ctx], -1) if p.softmax_uses_attention else xs
    return NestedMap(softmax_input=self.dropout.FProp(theta.dropout, sm_in),
                     attention=NestedMap(probs=probs))

  # -- step plan --------------------------------------------------------------------
  def MiscZeroState(self, theta, encoder_outputs, target_ids, bs):
    """Scheduled-sampling bookkeeping and adapter task ids (ref :1286)."""
    p = self.params
    misc = NestedMap()
    if self._max_label_prob > 0:
      misc.prev_predicted_ids = target_ids[:, 0].reshape(bs).long()
      gp = self.GroundTruthProbability().to(target_ids.device)
      summary_utils.scalar('ground_truth_sampling_probability', gp)
      misc.groundtruth_p = gp
    if p.adapter_task_id_field:
      task_ids = encoder_outputs.Get(p.adapter_task_id_field).reshape(-1).long()
      misc[p.adapter_task_id_field] = task_ids.repeat(bs // task_ids.shape[0])
    return misc

  def DecoderStepZeroState(self, theta, encoder_outputs, target_ids, bs):
    """→ (decoder step state, packed source) (ref :498)."""
    packed = self.atten_rnn.InitForSourcePacked(theta.atten_rnn, encoder_outputs.encoded,
                                                encoder_outputs.padding)
    misc = self.MiscZeroState(theta, encoder_outputs, target_ids, bs)
    self.contextualizer.InitAttention(theta.contextualizer, packed, misc)
    st = self.atten_rnn.zero_state(theta.atten_rnn, encoder_outputs.encoded, packed, bs)
    audio_ctx = st.atten
    ctx = self.contextualizer.ZeroAttention(theta.contextualizer, bs, misc, audio_ctx, packed)
    rnn_states = [st.rnn] + [r.zero_state(theta.rnn[i], bs) for i, r in enumerate(self.rnn)]
    state = NestedMap(rnn_states=rnn_states, atten_context=ctx, atten_probs=st.atten_probs,
                      atten_states=st.atten_state,
                      fusion_states=self.fusion.zero_state(theta.fusion, bs),
                      misc_states=misc)
    return state, packed

  def BaseZeroState(self, theta, encoder_outputs, bs, misc_zero_states,
                    per_step_source_padding=None):
    """→ (rnn_states, atten_context, atten_probs, atten_states, packed_src): the RNN and
    attention part of the initial step state (ref :464)."""
    del per_step_source_padding
    packed = self.atten_rnn.InitForSourcePacked(theta.atten_rnn, encoder_outputs.encoded,
                                                encoder_outputs.padding)
    self.contextualizer.InitAttention(theta.contextualizer, packed, misc_zero_states)
    st = self.atten_rnn.zero_state(theta.atten_rnn, encoder_outputs.encoded, packed, bs)
    ctx = self.contextualizer.ZeroAttention(theta.contextualizer, bs, misc_zero_states,
                                            st.atten, packed)
    rnn_states = [st.rnn] + [r.zero_state(theta.rnn[i], bs) for i, r in enumerate(self.rnn)]
    return rnn_states, ctx, st.atten_probs, st.atten_state, packed

  def InitDecoder(self, theta, encoder_outputs, dec_bs):
    """Initial state for inference-style stepping, as the flat tuple (rnn_states,
    atten_context, atten_probs, atten_states, fusion_states, misc_states, packed_src)
    (ref :696)."""
    sos = torch.full((dec_bs, 1), self.params.target_sos_id, dtype=torch.long,
                     device=encoder_outputs.encoded.device)
    st, packed = self.DecoderStepZeroState(theta, encoder_outputs, sos, dec_bs)
    return (st.rnn_states, st.atten_context, st.atten_probs, st.atten_states,
            st.fusion_states, st.misc_states, packed)

  def CreateTargetInfoMisc(self, targets):
    """The `misc` field of the per-step `TargetInfo` (ref :770): FST bias probabilities when
    the targets carry them."""
    if 'fst_bias_probs' in targets:
      return NestedMap(fst_bias_probs=targets.fst_bias_probs)
    return NestedMap()

  def AddAdditionalDecoderSummaries(self, encoder_outputs, targets, seq_out_tas,
                                    softmax_input):
    """Hook for model-specific summaries (ref :493)."""

  def _AddDecoderActivationsSummary(self, encoder_outputs, targets, atten_probs, rnn_outs,
                                    softmax_input, additional_atten_probs=None,
                                    target_alignments=None):
    """Attention-matrix image + activation-norm scalars of one unrolled batch (ref :511);
    `atten_probs` is `[T, B, S]`."""
    del rnn_outs, additional_atten_probs, target_alignments
    if not summary_utils._ShouldAddSummary():   # pylint: disable=protected-access
      return
    name = self.params.name or 'decoder'
    summary_utils.AddAttentionSummary(name, [atten_probs.detach()],
                                      encoder_outputs.padding, targets.paddings.t())
    summary_utils.scalar('%s/softmax_input_rms' % name,
                         softmax_input.detach().float().square().mean().sqrt())

  def ComputePredictionsFunctional(self, theta, encoder_outputs, targets):
    """The unrolling expressed as ONE step function scanned by `recurrent.Recurrent`
    (ref :1066) — rematerialised backward over long targets instead of T live step graphs.
    Teacher forcing only (`min_ground_truth_prob == 1`, no fusion feedback)."""
    from lingvo_b200.core import recurrent  # pylint: disable=g-import-not-at-top
    p = self.params
    assert p.min_ground_truth_prob == 1.0
    ids = targets.ids.t().long()
    b = ids.shape[1]
    if 'weights' not in targets:
      targets.weights = 1.0 - targets.paddings
    embs = self.dropout.FProp(theta.dropout, self.emb.EmbLookup(theta.emb, ids))
    state0, packed = self.DecoderStepZeroState(theta, encoder_outputs, targets.ids, b)
    misc = self.CreateTargetInfoMisc(targets)
    inputs = NestedMap(id=ids, label=targets.labels.t().long(),
                       weight=targets.weights.t().float(), emb=embs,
                       padding=targets.paddings.t().float().unsqueeze(-1))
    # the per-step output rides along as a state field so that `Recurrent` stacks it
    state0.step_outs = embs.new_zeros(b, p.rnn_cell_dim + state0.atten_context.shape[-1])

    def Step(th, state, inp):
      info = AsrDecoderBase.TargetInfo(id=inp.id, label=inp.label, weight=inp.weight,
                                       emb=inp.emb, padding=inp.padding, misc=misc)
      carried = NestedMap({k: v for k, v in state.items() if k != 'step_outs'})
      step_out, new_state = self.SingleDecodeStep(th, packed, info, carried)
      new_state.step_outs = step_out
      return new_state, NestedMap()

    acc, _ = recurrent.Recurrent(theta, state0, inputs, Step)
    sm_in = acc.step_outs if p.softmax_uses_attention else acc.step_outs[..., :p.rnn_cell_dim]
    return NestedMap(softmax_input=self.dropout.FProp(theta.dropout, sm_in),
                     attention=NestedMap(probs=acc.atten_probs))

  def _Adapt(self, theta, i, x, misc):
    p = self.params
    if not p.adapter_task_id_field:
      return x
    return self.adapters[i].FProp(theta.adapters[i], x.unsqueeze(0),
                                  misc[p.adapter_task_id_field]).squeeze(0)

  def _ComputeAttention(self, theta, rnn_out, packed_src, attention_state):
    return self.atten_rnn.atten.ComputeContextVectorWithSource(
        theta.atten_rnn.atten, packed_src, rnn_out, attention_state)

  def SingleDecodeStep(self, theta, packed_src, cur_target_info, decoder_step_state,
                       per_step_src_padding=None, use_deterministic_random=False):
    """One decoder step (ref :1444) → (step_out `[B, rnn + ctx]`, new state)."""
    del per_step_src_padding, use_deterministic_random
    p = self.params
    st = decoder_step_state
    misc = st.misc_states
    prev_embs = cur_target_info.emb if p.teacher_forcing else torch.ones_like(
        cur_target_info.emb)
    pad = cur_target_info.padding
    s0, _ = self.atten_rnn.cell.FProp(
        theta.atten_rnn.cell, st.rnn_states[0],
        NestedMap(act=[prev_embs, st.atten_context.to(prev_embs.dtype)], padding=pad))
    new_states = [s0]
    rnn_out = self._Adapt(theta, 0, self.atten_rnn.cell.GetOutput(s0), misc)
    audio_ctx, probs, atten_states = self._ComputeAttention(theta, rnn_out, packed_src,
                                                            st.atten_states)
    ctx = self.contextualizer.QueryAttention(theta.contextualizer, rnn_out, misc, audio_ctx,
                                             packed_src)
    for i, r in enumerate(self.rnn, 1):
      si, _ = r.cell.FProp(theta.rnn[i - 1].cell, st.rnn_states[i],
                           NestedMap(act=[rnn_out, ctx.to(rnn_out.dtype)], padding=pad))
      new_states.append(si)
      new_out = self._Adapt(theta, i, r.cell.GetOutput(si), misc)
      new_out = self.dropout.FProp(theta.dropout, new_out)
      rnn_out = rnn_out + new_out if (i + 1 >= p.residual_start > 0) else new_out
    step_out = torch.cat([rnn_out, ctx.to(rnn_out.dtype)], 1)
    return step_out, NestedMap(rnn_states=new_states, atten_context=ctx, atten_probs=probs,
                               atten_states=atten_states, fusion_states=st.fusion_states,
                               misc_states=misc)

  def _StepLogits(self, theta, step_out, state, ids, padding, is_eval=False):
    """Softmax (+ fusion) on one step's output → (logits `[B, V]`, fusion state)."""
    p = self.params
    sm_in = step_out if p.softmax_uses_attention else step_out[:, :p.rnn_cell_dim]
    sm_in = self.dropout.FProp(theta.dropout, sm_in)
    am_logits = self._ComputeLogits(theta, sm_in)
    fused_in, fstate = self.fusion.FProp(theta.fusion, state.fusion_states, am_logits,
                                         ids.reshape(-1, 1), padding.reshape(-1, 1))
    logits = self.fusion.ComputeLogitsWithLM(fstate, fused_in, is_eval=is_eval)
    return logits, fstate, sm_in

  def TargetsToBeFedAtCurrentDecodeStep(self, t, theta, state, ids, labels, weights, embs,
                                        paddings):
    """TargetInfo of step t; with scheduled sampling the previous *prediction* replaces the
    ground-truth token with probability 1 − groundtruth_p (ref :1310)."""
    tid, emb = ids[t], embs[t]
    if self._max_label_prob > 0:
      bs = tid.shape[0]
      pick = torch.rand(bs, device=tid.device) < state.misc_states.groundtruth_p
      prev = state.misc_states.prev_predicted_ids.detach()
      emb = torch.where(pick.unsqueeze(-1), emb, self.emb.EmbLookup(theta.emb, prev).to(
          emb.dtype))
      tid = torch.where(pick, tid, prev)
    return AsrDecoderBase.TargetInfo(id=tid, label=labels[t], weight=weights[t], emb=emb,
                                     padding=paddings[t], misc=NestedMap())

  def PostStepDecoderStateUpdate(self, state, logits=None):
    """Samples the next "previous prediction" for scheduled sampling (ref :1343)."""
    if logits is None:
      raise ValueError('logits cannot be None')
    if self._max_label_prob > 0:
      probs = torch.softmax(logits.detach().float(), -1)
      state.misc_states.prev_predicted_ids = torch.multinomial(probs, 1).reshape(-1)
    return state

  def ComputePredictionsDynamic(self, theta, encoder_outputs, targets):
    """Step-by-step unrolling (ref :958)."""
    ids = targets.ids.t().long()
    t, b = ids.shape
    labels = targets.labels.t().long()
    weights = targets.weights.t().float()
    pads = targets.paddings.t().float().unsqueeze(-1)
    embs = self.dropout.FProp(theta.dropout, self.emb.EmbLookup(theta.emb, ids))
    state, packed = self.DecoderStepZeroState(theta, encoder_outputs, targets.ids, b)
    sm_ins, logits, probs = [], [], []
    for i in range(t):
      info = self.TargetsToBeFedAtCurrentDecodeStep(i, theta, state, ids, labels, weights,
                                                    embs, pads)
      step_out, state = self.SingleDecodeStep(theta, packed, info, state)
      lg, fstate, sm_in = self._StepLogits(theta, step_out, state, info.id, info.padding)
      state.fusion_states = fstate
      state = self.PostStepDecoderStateUpdate(state, lg)
      sm_ins.append(sm_in)
      logits.append(lg)
      probs.append(state.atten_probs)
    return NestedMap(softmax_input=torch.stack(sm_ins, 0),
                     logits=torch.stack(logits, 1),
                     attention=NestedMap(probs=torch.stack(probs, 0)))

  def ComputeLoss(self, theta, predictions, targets):
    if 'logits' not in predictions:
      # sequence plan: one softmax GEMM over the whole [T·B, D] block
      logits = self._ComputeLogits(theta, predictions.softmax_input).transpose(0, 1)
      predictions = NestedMap(predictions)
      predictions.logits = logits
    metrics, per_seq = super().ComputeLoss(theta, predictions, targets)
    return metrics, per_seq

  # -- beam search ------------------------------------------------------------------
  def _InitBeamSearchStateCallback(self, theta, encoder_outputs, num_hyps_per_beam):
    p = self.params
    n = encoder_outputs.encoded.shape[1] * num_hyps_per_beam
    dev = encoder_outputs.encoded.device
    sos = torch.full((n, 1), p.target_sos_id, dtype=torch.long, device=dev)
    state, packed = self.DecoderStepZeroState(theta, encoder_outputs, sos, n)
    encoder_outputs.packed_src = packed
    init = NestedMap(log_probs=torch.zeros(n, p.softmax.num_classes, device=dev),
                     atten_probs=torch.zeros(n, encoder_outputs.encoded.shape[0], device=dev))
    return init, state

  def _PreBeamSearchStepCallback(self, theta, encoder_outputs, step_ids, states,
                                 num_hyps_per_beam, cur_step):
    p = self.params
    n = step_ids.shape[0]
    ids = step_ids.squeeze(1).long()
    emb = self.emb.EmbLookup(theta.emb, ids)
    pad = torch.zeros(n, 1, device=emb.device)
    info = AsrDecoderBase.TargetInfo(id=ids, label=None, weight=None, emb=emb, padding=pad,
                                     misc=NestedMap())
    step_out, new_state = self.SingleDecodeStep(theta, encoder_outputs.packed_src, info, states)
    logits, fstate, _ = self._StepLogits(theta, step_out, new_state, ids, pad, is_eval=True)
    new_state.fusion_states = fstate
    fused = not isinstance(self.fusion, fusion_lib.NullFusion)
    if fused and p.use_unnormalized_logits_as_log_probs:
      log_probs = logits.float()
    else:
      log_probs = torch.log_softmax(logits.float(), -1)
    return (NestedMap(log_probs=log_probs, atten_probs=new_state.atten_probs), new_state)

  def _PostBeamSearchStepCallback(self, theta, encoder_outputs, new_step_ids, states):
    return states
