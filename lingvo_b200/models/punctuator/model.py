"""Punctuator model (ref `lingvo/tasks/punctuator/model.py`): the RNMT+ translation model
from unpunctuated lower-case text to punctuated text, plus the string-in / string-out
inference subgraph the reference exports for serving.

`Inference()['default'](src_strings)` (ref `_InferenceSubgraph_Default` :37): tokenise the raw
strings with the input generator's tokenizer (padded to `source_max_length`), encode, beam
search, and convert the top-k hypotheses back to strings. On the H100 serving path the
encoder/decoder math runs on the device; only tokenisation and detokenisation are host work.
"""

import torch

from lingvo_b200.core.nested_map import NestedMap
from lingvo_b200.models.mt import model as mt_model


class _PunctuatorInferenceMixin:
  """String-level inference shared by the RNMT and Transformer punctuators."""

  def Inference(self):
    """{'default': fn(src_strings) → NestedMap(src_ids, topk_decoded, topk_scores, …)}."""
    return {'default': self._InferenceSubgraph_Default}

  def _InferenceSubgraph_Default(self, src_strings):   # pylint: disable=invalid-name
    gen = self.input_generator
    if isinstance(src_strings, (str, bytes)):
      src_strings = [src_strings]
    src_strings = [s.decode('utf-8') if isinstance(s, bytes) else s for s in src_strings]
    _, src_ids, src_paddings = gen.tokenizer.StringsToIds(
        src_strings, gen.params.source_max_length or 512)
    dev = self.Device()
    src = NestedMap(ids=torch.as_tensor(src_ids).long().to(dev),
                    paddings=torch.as_tensor(src_paddings).float().to(dev))
    with torch.no_grad():
      enc = self.enc.FProp(self.theta.enc, src)
      out = self.dec.BeamSearchDecodeWithTheta(self.theta.dec, enc)
    b = len(src_strings)
    k = out.topk_hyps.ids.shape[1] if hasattr(out.topk_hyps, 'ids') else (
        out.topk_ids.shape[0] // b)
    topk_ids = out.topk_ids.reshape(b * k, -1)
    topk_lens = out.topk_lens.reshape(b * k)
    # topk_lens - 1 drops the end-of-sentence id
    decoded = gen.IdsToStrings(topk_ids.cpu(), (topk_lens - 1).clamp_min(0).cpu())
    decoded = [decoded[i * k:(i + 1) * k] for i in range(b)]
    return NestedMap(src_ids=src.ids, topk_decoded=decoded,
                     topk_scores=out.topk_scores.reshape(b, k), topk_ids=topk_ids.reshape(b, k, -1),
                     topk_lens=topk_lens.reshape(b, k))

  def Punctuate(self, text):
    """Convenience: best hypothesis for one string (or a list of strings)."""
    single = isinstance(text, (str, bytes))
    out = self._InferenceSubgraph_Default([text] if single else list(text))
    best = [hyps[0] for hyps in out.topk_decoded]
    return best[0] if single else best


class RNMTModel(_PunctuatorInferenceMixin, mt_model.RNMTModel):
  """RNMT+ for punctuation restoration (ref :22)."""


class TransformerModel(_PunctuatorInferenceMixin, mt_model.TransformerModel):
  """Transformer variant with the same string-level inference contract."""
