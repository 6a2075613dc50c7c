"""Inference export (ref `lingvo/core/inference_graph_exporter.py`).

The reference freezes a TF `GraphDef` plus `subgraphs{name: feeds, fetches}`. The
H100 equivalent of "a frozen graph" is a self-contained **inference bundle**:

  <dir>/inference_graph.json   model name, task, subgraph names + their feed/fetch
                               keys, dtype policy, bundle format version
  <dir>/params.txt             the full model Params (`ToText`) – rebuilds the layers
  <dir>/weights.pt             {var_name: tensor} (optionally bf16, EMA applied)

`Predictor` (predictor.py) rebuilds the model from `params.txt`, loads the weights
and serves the subgraphs returned by `task.Inference()`; static-shape subgraphs are
captured into CUDA graphs on first use.
"""

from __future__ import annotations

import collections
import inspect
import json
import os
from typing import Dict, Optional

import torch

from lingvo_b200.core import hyperparams
from lingvo_b200.core import py_utils
from lingvo_b200.utils import protowire as pw

BUNDLE_VERSION = 1
InferenceDeviceOptions = collections.namedtuple(
    'InferenceDeviceOptions', ['device', 'retain_device_placement', 'var_options',
                               'gen_init_op', 'dtype_override', 'fprop_dtype_override'])
InferenceDeviceOptions.__new__.__defaults__ = ('', False, None, True, None, None)


class InferenceGraph:
  """In-memory description of an exported bundle (the `InferenceGraph` proto's role)."""

  def __init__(self, model_name='', task_name='', subgraphs=None, asset_dir=''):
    self.model_name = model_name
    self.task_name = task_name
    self.subgraphs = subgraphs or {}      # name → {'feeds': [...], 'fetches': [...]}
    self.asset_dir = asset_dir

  def ToJson(self):
    return json.dumps({'version': BUNDLE_VERSION, 'model_name': self.model_name,
                       'task_name': self.task_name, 'subgraphs': self.subgraphs}, indent=1)

  @classmethod
  def FromJson(cls, text, asset_dir=''):
    d = json.loads(text)
    return cls(d.get('model_name', ''), d.get('task_name', ''), d.get('subgraphs', {}),
               asset_dir)

  # -- `tensorflow.lingvo.InferenceGraph` wire format (ref core/inference_graph.proto) ----
  # Serving tools of the reference read subgraph signatures (feeds / fetches and their
  # dtype / shape metadata), the hyper-parameters and the asset list from this message. The
  # `graph_def` field cannot carry a TF graph here; it holds a one-node GraphDef naming the
  # bundle, so that the message stays well-formed for any protobuf reader.
  _DTYPES = {'float32': 1, 'float64': 2, 'int32': 3, 'uint8': 4, 'int16': 5, 'int8': 6,
             'string': 7, 'int64': 9, 'bool': 10, 'bfloat16': 14, 'float16': 19}

  @staticmethod
  def _MapEntry(field, key, value_bytes):
    return pw.f_bytes(field, pw.f_bytes(1, key) + pw.f_bytes(2, value_bytes))

  def _MetaBytes(self, meta):
    out = b''
    dt = self._DTYPES.get(str(meta.get('dtype', '')).replace('torch.', ''))
    if dt is not None:
      out += pw.f_varint(2, dt)
    if meta.get('shape') is not None:
      out += pw.f_packed_varint(3, [int(d) if d is not None and d >= 0 else (1 << 64) - 1
                                    for d in meta['shape']])
    if meta.get('layout'):
      out += pw.f_bytes(4, meta['layout'])
    return out

  def ToProto(self, hyperparameters: str = '', assets=()) -> bytes:
    node = pw.f_bytes(1, 'lingvo_b200/bundle') + pw.f_bytes(2, 'NoOp')
    msg = pw.f_bytes(1, pw.f_bytes(1, node))                     # graph_def { node {…} }
    for name in sorted(self.subgraphs):
      spec = self.subgraphs[name]
      sub = b''
      for fname in spec.get('feeds', []):
        sub += self._MapEntry(2, fname, '%s/%s:0' % (name, fname))
      for fname in spec.get('fetches', []):
        sub += self._MapEntry(3, fname, '%s/%s:0' % (name, fname))
      for fname, meta in sorted((spec.get('feeds_meta') or {}).items()):
        sub += self._MapEntry(4, fname, self._MetaBytes(meta))
      for fname, meta in sorted((spec.get('fetches_meta') or {}).items()):
        sub += self._MapEntry(5, fname, self._MetaBytes(meta))
      msg += self._MapEntry(5, name, sub)
    if hyperparameters:
      msg += pw.f_bytes(7, hyperparameters)
    for fn in assets:
      info = pw.f_bytes(1, 'asset/%s:0' % fn)                    # TensorInfo.name
      msg += pw.f_bytes(10, pw.f_bytes(1, info) + pw.f_bytes(2, fn))
    return msg

  @classmethod
  def FromProto(cls, buf: bytes, asset_dir=''):
    """Parses `ToProto` output (or any InferenceGraph message) → (graph, hyperparameters,
    asset file names)."""
    inv = {v: k for k, v in cls._DTYPES.items()}
    subgraphs, hyper, assets = {}, '', []

    def Str(b):
      return b.decode('utf-8') if isinstance(b, (bytes, bytearray)) else str(b)

    def Meta(mb):
      m = {}
      for f, _, v in pw.parse(mb):
        if f == 2:
          m['dtype'] = inv.get(int(v), int(v))
        elif f == 3:
          vals = pw.parse_packed_varints(v) if isinstance(v, (bytes, bytearray)) else [v]
          m['shape'] = [None if d == (1 << 64) - 1 else int(d) for d in vals]
        elif f == 4:
          m['layout'] = Str(v)
      return m

    for f, _, v in pw.parse(buf):
      if f == 5:
        entry = pw.parse_dict(v)
        name = Str(entry[1][0])
        spec = {'feeds': [], 'fetches': [], 'feeds_meta': {}, 'fetches_meta': {}}
        for sf, _, sv in pw.parse(entry.get(2, [b''])[0]):
          kv = pw.parse_dict(sv)
          k = Str(kv[1][0])
          if sf == 2:
            spec['feeds'].append(k)
          elif sf == 3:
            spec['fetches'].append(k)
          elif sf == 4:
            spec['feeds_meta'][k] = Meta(kv.get(2, [b''])[0])
          elif sf == 5:
            spec['fetches_meta'][k] = Meta(kv.get(2, [b''])[0])
        subgraphs[name] = spec
      elif f == 7:
        hyper = Str(v)
      elif f == 10:
        d = pw.parse_dict(v)
        if 2 in d:
          assets.append(Str(d[2][0]))
    return cls(subgraphs=subgraphs, asset_dir=asset_dir), hyper, assets


def _SubgraphSpec(fn):
  """feeds = the callable's argument names; fetches are discovered at first run."""
  try:
    feeds = [p.name for p in inspect.signature(fn).parameters.values()
             if p.kind in (p.POSITIONAL_OR_KEYWORD, p.KEYWORD_ONLY)]
  except (TypeError, ValueError):
    feeds = []
  return {'feeds': feeds, 'fetches': []}


class InferenceGraphExporter:

  @classmethod
  def Export(cls, model_cfg, model_task_name=None, device_options=InferenceDeviceOptions(),
             freeze_checkpoint=None, freeze_defaults=False, export_path=None,
             subgraph_filter=None, random_seed=None, disable_packed_input=True,
             prune_graph=True, export_graph_collections=False, model=None) -> InferenceGraph:
    """Builds the model (or uses `model`), optionally loads `freeze_checkpoint`, and
    writes the bundle to `export_path` (a directory). Returns the InferenceGraph."""
    del freeze_defaults, prune_graph, export_graph_collections
    if random_seed is not None:
      torch.manual_seed(random_seed)
    cfg = model_cfg.Copy()
    if disable_packed_input:
      def _Off(p):
        if isinstance(p, hyperparams.Params) and 'packed_input' in p:
          p.packed_input = False
      _Off(cfg.task) if 'task' in cfg and cfg.task is not None else None
    cfg.is_inference = True
    if model is None:
      model = cfg.Instantiate()
    task = model.GetTask(model_task_name) if model_task_name else model.tasks[0]
    if freeze_checkpoint:
      from lingvo_b200.core import checkpointer  # pylint: disable=g-import-not-at-top
      checkpointer.Checkpointer(os.path.dirname(freeze_checkpoint), model).RestoreFromPath(
          checkpoint_path=freeze_checkpoint)
    subgraphs = task.Inference()
    if subgraph_filter:
      keep = set(subgraph_filter if isinstance(subgraph_filter, (list, tuple))
                 else [subgraph_filter])
      subgraphs = {k: v for k, v in subgraphs.items() if k in keep}
    graph = InferenceGraph(
        model_name=str(model_cfg.get('model', '') if hasattr(model_cfg, 'get') else ''),
        task_name=model_task_name or '', subgraphs={k: _SubgraphSpec(v)
                                                    for k, v in subgraphs.items()})
    if export_path:
      os.makedirs(export_path, exist_ok=True)
      dtype = device_options.dtype_override
      weights = {}
      for v in model.vars.Flatten():
        t = v.detach().cpu()
        if dtype is not None and t.is_floating_point():
          t = t.to(dtype)
        weights[v.var_name] = t
      torch.save(weights, os.path.join(export_path, 'weights.pt'))
      with open(os.path.join(export_path, 'params.txt'), 'w') as f:
        f.write(model_cfg.ToText())
      with open(os.path.join(export_path, 'inference_graph.json'), 'w') as f:
        f.write(graph.ToJson())
      # the reference's `InferenceGraph` proto next to the bundle manifest
      with open(os.path.join(export_path, 'inference_graph.pb'), 'wb') as f:
        f.write(graph.ToProto(hyperparameters=model_cfg.ToText(),
                              assets=('weights.pt', 'params.txt', 'inference_graph.json')))
      graph.asset_dir = export_path
    return graph


def LoadInferenceGraph(path) -> InferenceGraph:
  """Loads a bundle directory, its `inference_graph.json`, or its `inference_graph.pb`."""
  d = path if os.path.isdir(path) else os.path.dirname(path)
  if not os.path.isdir(path) and path.endswith('.pb'):
    with open(path, 'rb') as f:
      graph, _, _ = InferenceGraph.FromProto(f.read(), d)
    js = os.path.join(d, 'inference_graph.json')
    if os.path.exists(js):                     # names of model / task live in the manifest
      with open(js) as f:
        full = InferenceGraph.FromJson(f.read(), d)
      graph.model_name, graph.task_name = full.model_name, full.task_name
    return graph
  with open(os.path.join(d, 'inference_graph.json')) as f:
    return InferenceGraph.FromJson(f.read(), d)
