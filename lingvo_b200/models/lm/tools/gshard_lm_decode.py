"""Decoding driver for GShard LMs (ref `lingvo/tasks/lm/tools/gshard_lm_decode.py`).

  python -m lingvo_b200.models.lm.tools.gshard_lm_decode \
      --model=lm.synthetic_packed_input.DenseLm8B2x2Decode --checkpoint=/path/ckpt-00001000 \
      --input=prompts.tsv --output=continuations.tsv --batch_size=16 --prefix_max_len=128 \
      [--beam_size=4]

`GShardLMDecode` serves prompts through the stream-pipelined loop of
`core.gshard_decode.GShardDecode` (pinned H2D infeed → device decode → D2H outfeed);
`GShardLMDecodeBatch` decodes whole TSV files (one prompt per line, space-separated token
ids unless a tokenizer is plugged in by overriding `init_vocab / encode_string_to_ids /
decode_ids_to_string`) and skips files already decoded (restart-safe). With `beam_size` ≥ 1
the continuations come from a flat beam search (`gshard_decode.BeamDecodeIds`) and each line
holds the best hypothesis and its length-normalised score; 0 keeps greedy / sampled decoding.
"""

from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np
import torch

from lingvo_b200 import model_registry
from lingvo_b200.core import cluster_factory
from lingvo_b200.core import gshard_decode
from lingvo_b200.core.nested_map import NestedMap


def read_files_1_col(tsv_files):  # pylint: disable=invalid-name
  """First column of every line of every file (ref :50)."""
  out = []
  for f in tsv_files:
    with open(f, encoding='utf-8') as fh:
      out.append([l.rstrip('\n').split('\t')[0] for l in fh if l.strip()])
  return out


def override_params(model_params, spec):  # pylint: disable=invalid-name
  """`a.b=1,c=x` → sets task params (ref :66)."""
  for kv in filter(None, (spec or '').split(',')):
    k, v = kv.split('=', 1)
    try:
      v = eval(v, {}, {})  # pylint: disable=eval-used
    except Exception:  # pylint: disable=broad-except
      pass
    model_params.task.Set(**{k: v})
  return model_params


class GShardLMDecode(gshard_decode.GShardDecode):
  """Interactive / streaming decoder (ref :82)."""

  def __init__(self, model_name, checkpoint=None, prefix_max_len=128, batch_size=8,
               max_decode_steps=None, temperature=0.0, device=None, params_override='',
               beam_size=0):
    self.prefix_max_len = prefix_max_len
    self.beam_size = beam_size
    self.batch_size = batch_size
    self.temperature = temperature
    try:
      mp = model_registry.GetParams(model_name, 'Test')
    except NotImplementedError:
      mp = model_registry.GetParams(model_name, 'Train')     # synthetic-input models
    mp = override_params(mp, params_override)
    if max_decode_steps:
      mp.task.decoder_max_steps = max_decode_steps
    dev = torch.device(device) if device else torch.device(
        'cuda' if torch.cuda.is_available() else 'cpu')
    with cluster_factory.Cluster(mp.cluster.Copy().Set(do_eval=True)):
      self.task = mp.task.Instantiate()
    self.task.to(dev)
    if checkpoint:
      self.RestoreVariables(checkpoint)
    self.init_vocab(mp)
    super().__init__(self._DecodeFn, device=dev)

  def RestoreVariables(self, checkpoint):
    """Loads every model variable present in a tensor-bundle checkpoint prefix."""
    from lingvo_b200.utils import tensor_bundle
    reader = tensor_bundle.BundleReader(checkpoint)
    missing = []
    with torch.no_grad():
      for v in self.task.vars.Flatten():
        if reader.Has(v.var_name):
          arr = reader.Read(v.var_name)
          v.copy_(torch.as_tensor(np.asarray(arr, np.float32)).reshape(v.shape))
        else:
          missing.append(v.var_name)
    if missing:
      print('warning: %d variables not in checkpoint (e.g. %s)' % (len(missing), missing[0]))

  # -- tokenizer hooks --------------------------------------------------------------
  def init_vocab(self, model_params):  # pylint: disable=invalid-name
    self.bos_token_id = model_params.task.decoder_bos_id
    self.eos_token_id = model_params.task.decoder_eos_id

  def encode_string_to_ids(self, string):  # pylint: disable=invalid-name
    return [int(s) for s in string.split(' ') if s]

  def decode_ids_to_string(self, ids):  # pylint: disable=invalid-name
    return ' '.join(str(int(i)) for i in ids)

  # -- batching ---------------------------------------------------------------------
  def MakeBatch(self, prompts):
    """List of strings → (ids [B,T], paddings [B,T]) numpy, B padded to batch_size."""
    t = self.prefix_max_len
    ids = np.full((self.batch_size, t), self.eos_token_id, np.int64)
    pad = np.ones((self.batch_size, t), np.float32)
    for i, s in enumerate(prompts):
      toks = ([self.bos_token_id] + self.encode_string_to_ids(s))[:t]
      ids[i, :len(toks)] = toks
      pad[i, :len(toks)] = 0.0
    pad[len(prompts):, 0] = 0.0                      # dummy rows: 1-token prefix
    return ids, pad

  def _DecodeFn(self, batch):
    ids, pad = batch
    if self.beam_size:
      out = gshard_decode.BeamDecodeIds(
          self.task, self.task.theta, NestedMap(ids=ids, paddings=pad), beam_size=self.beam_size)
      # the best hypothesis; its ids are the continuation alone, so it starts at column 0
      return (out.topk_ids[:, 0], torch.zeros_like(out.prefix_lens), out.topk_lens[:, 0],
              out.topk_scores[:, 0])
    out = gshard_decode.DecodeIds(
        self.task, self.task.theta, NestedMap(ids=ids, paddings=pad),
        temperature=self.temperature)
    return out.ids, out.prefix_lens, out.lens, out.scores

  def DecodePrompts(self, prompts):
    """→ list of (continuation string, score) in input order."""
    batches, sizes = [], []
    for i in range(0, len(prompts), self.batch_size):
      chunk = prompts[i:i + self.batch_size]
      batches.append(self.MakeBatch(chunk))
      sizes.append(len(chunk))
    results = []
    for n, (ids, plen, lens, scores) in zip(sizes, self.decode(batches)):
      ids, plen, lens, scores = (np.asarray(x) for x in (ids, plen, lens, scores))
      for r in range(n):
        gen = ids[r, plen[r]:lens[r]]
        results.append((self.decode_ids_to_string(gen), float(scores[r])))
    return results


class GShardLMDecodeBatch(GShardLMDecode):
  """File-to-file decoding (ref :256)."""

  def DecodeFiles(self, tsv_files, output_dir, skip_done=True):
    os.makedirs(output_dir, exist_ok=True)
    done = []
    for f, prompts in zip(tsv_files, read_files_1_col(tsv_files)):
      out = os.path.join(output_dir, os.path.basename(f) + '.decoded')
      if skip_done and os.path.exists(out):
        continue
      t0 = time.time()
      res = self.DecodePrompts(prompts)
      tmp = out + '.tmp'
      with open(tmp, 'w', encoding='utf-8') as fh:
        for p, (s, sc) in zip(prompts, res):
          fh.write('%s\t%s\t%.6f\n' % (p, s, sc))
      os.replace(tmp, out)
      done.append(out)
      print('%s: %d prompts in %.1fs' % (f, len(prompts), time.time() - t0))
    return done


def main(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--model', required=True)
  ap.add_argument('--checkpoint', default=None)
  ap.add_argument('--input', required=True, help='comma-separated TSV files')
  ap.add_argument('--output', required=True, help='output directory')
  ap.add_argument('--batch_size', type=int, default=8)
  ap.add_argument('--prefix_max_len', type=int, default=128)
  ap.add_argument('--max_decode_steps', type=int, default=0)
  ap.add_argument('--temperature', type=float, default=0.0)
  ap.add_argument('--params_override', default='')
  ap.add_argument('--beam_size', type=int, default=0,
                  help='flat beam search with this many hypotheses; 0: greedy / sampling')
  a = ap.parse_args(argv)
  dec = GShardLMDecodeBatch(a.model, a.checkpoint, a.prefix_max_len, a.batch_size,
                            a.max_decode_steps or None, a.temperature,
                            params_override=a.params_override, beam_size=a.beam_size)
  dec.DecodeFiles(a.input.split(','), a.output)
  dec.stop()
  return 0


if __name__ == '__main__':
  sys.exit(main())
