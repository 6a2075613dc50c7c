"""Input generators.

Reference `lingvo/core/base_input_generator.py`: `BaseInputGenerator` params
(:141-257), `GetPreprocessedInputBatch` (:395), `SplitInputBatch` (:1006),
`GlobalBatchSize/InfeedBatchSize` (:350-364), file-based generators
(:1223-1296), sequence generators (:1465-1697), `BaseTinyDatasetInput`
(:1706-1767).

H100-first: a batch is a NestedMap of **pinned host tensors** produced by
native C++ threads (`lingvo_b200.ops.native_input`); `DevicePrefetcher`
overlaps the H2D copy of batch i+1 with the compute of batch i on a side
stream — the analogue of the reference's TPU infeed queues.
"""

from __future__ import annotations

import os
import queue
import threading
from typing import Any, Callable, Dict, List, Optional

import numpy as np
import torch

from lingvo_b200.core import base_layer
from lingvo_b200.core import batch_utils
from lingvo_b200.core import cluster_factory
from lingvo_b200.core import hyperparams
from lingvo_b200.core import py_utils
from lingvo_b200.core.nested_map import NestedMap


class BaseInputGenerator(base_layer.BaseLayer):
  """The abstract base input generator."""

  @classmethod
  def DefineInfeedParams(cls, p):
    p.Define('use_per_host_infeed', False, 'Kept for parity (per-rank input).')
    p.Define('use_per_core_infeed', False, 'Kept for parity.')
    p.Define('tpu_infeed_parallelism', 1, 'Prefetch depth of the H2D queue.')
    p.Define('use_partitioned_infeed_queue', False, 'Kept for parity.')
    p.Define('num_partitions', None, 'Kept for parity.')

  @classmethod
  def Params(cls):
    p = super().Params()
    p.name = 'input'
    p.Define('file_datasource', None, 'DataSource params to read from.')
    p.Define('batch_size', 0, 'Batch size for a device split.')
    p.Define('num_samples', 0,
             'If non-zero, the dataset contains these many samples.')
    p.Define('resettable', False, 'Input can be reset (epoch-exact eval).')
    p.Define('eval_samples_per_summary', None, 'Overrides task.eval value.')
    p.Define('decoder_samples_per_summary', None, 'Overrides task.eval value.')
    p.Define('filter_sparse_tensors', False, 'Kept for parity.')
    p.Define('input_stats_summary_interval_steps', 10, 'Stats interval.')
    p.Define('cpu_passthrough_keys', [], 'Keys kept on host (strings etc.).')
    p.Define('pin_memory', True, 'Produce batches in pinned host memory.')
    cls.DefineInfeedParams(p)
    p.Define('remote', hyperparams.Params(), 'Kept for parity.')
    p.remote.Define('max_inflights_per_target', 32, 'Kept for parity.')
    p.Define('skip_tpu_embedding_enqueue_ops', False, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self._made_iter = False
    self._batch_cache = None
    if self.params.file_datasource is not None:
      self.CreateChild('datasource', self.params.file_datasource)
      # the reference does this in `CreateDatasource` (:296): sources call back into the
      # generator (`LoadDataset`, `GetSequenceLength`, custom transforms …)
      self.datasource.SetInputGenerator(self)

  # ----------------------------------------------------------- batch sizing --
  def GlobalBatchSize(self) -> int:
    """Batch size summed over all splits of all replicas."""
    return self.InfeedBatchSize() * max(self.cluster.world_size, 1)

  def InfeedBatchSize(self) -> int:
    """Batch size produced by this process per step."""
    p = self.params
    return batch_utils.scale_split_to_infeed(p.batch_size,
                                             p.use_per_host_infeed)

  def Initialize(self, sess=None):
    pass

  def Reset(self, sess=None):
    pass

  def CommonInputOpArgs(self) -> Dict[str, Any]:
    return {}

  # ----------------------------------------------------------------- batches --
  def _InputBatch(self) -> NestedMap:
    """Subclasses produce one (infeed) batch as a NestedMap of tensors."""
    raise NotImplementedError('Abstract method')

  def _PreprocessInputBatch(self, batch: NestedMap) -> NestedMap:
    return batch

  def GetPreprocessedInputBatch(self) -> NestedMap:
    return self._PreprocessInputBatch(self._InputBatch())

  def SplitInputBatch(self, num_splits: int) -> List[NestedMap]:
    """One infeed batch split along dim 0 into `num_splits` shards (:1006)."""
    batch = self.GetPreprocessedInputBatch()
    if num_splits <= 1:
      return [batch]
    return SplitBatch(batch, num_splits)

  def FProp(self, theta=None):
    return self.GetPreprocessedInputBatch()

  def __iter__(self):
    while True:
      try:
        yield self.GetPreprocessedInputBatch()
      except StopIteration:
        return


def SplitBatch(batch: NestedMap, num_splits: int) -> List[NestedMap]:
  """Splits every tensor's leading dim into `num_splits` equal parts."""
  flat = batch.FlattenItems()
  outs = [[] for _ in range(num_splits)]
  for k, v in flat:
    if isinstance(v, torch.Tensor) and v.dim() > 0:
      assert v.shape[0] % num_splits == 0, (
          'batch dim %d of %s not divisible by %d' % (v.shape[0], k, num_splits))
      parts = torch.chunk(v, num_splits, dim=0)
    elif isinstance(v, np.ndarray) and v.ndim > 0:
      parts = np.array_split(v, num_splits)
    else:
      parts = [v] * num_splits
    for i in range(num_splits):
      outs[i].append(parts[i])
  return [batch.Pack(o) for o in outs]


class DevicePrefetcher:
  """Host→device double-buffering on a side stream (infeed analogue).

  `Next()` returns a NestedMap already resident on `device`; the copy of the
  following batch is issued immediately on `copy_stream` from pinned memory so
  it overlaps the caller's compute. Also accounts the H2D bytes per step.
  """

  def __init__(self, input_gen: BaseInputGenerator, device, depth: int = 2,
               passthrough_keys=()):
    self._gen = input_gen
    self._device = torch.device(device)
    self._cuda = self._device.type == 'cuda'
    self._stream = torch.cuda.Stream(self._device) if self._cuda else None
    self._depth = max(1, depth)
    self._q: List = []
    self._passthrough = set(passthrough_keys)
    self.h2d_bytes_last = 0

  def _Issue(self):
    host = self._gen.GetPreprocessedInputBatch()
    nbytes = 0

    def pin(x):
      if isinstance(x, np.ndarray) and x.dtype.kind not in 'OUS':
        x = torch.from_numpy(x)
      if isinstance(x, torch.Tensor) and self._cuda and not x.is_cuda and not (
          x.is_pinned()):
        x = x.pin_memory()
      return x

    host = host.Transform(pin)
    if not self._cuda:
      self._q.append((host, None, 0))
      return
    with torch.cuda.stream(self._stream):
      def move(k, x):
        nonlocal nbytes
        if isinstance(x, torch.Tensor) and k not in self._passthrough:
          nbytes += x.numel() * x.element_size()
          return x.to(self._device, non_blocking=True)
        return x
      dev = host.TransformWithKey(move)
      ev = torch.cuda.Event()
      ev.record(self._stream)
    self._q.append((dev, ev, nbytes))

  def Next(self) -> NestedMap:
    while len(self._q) < self._depth:
      self._Issue()
    batch, ev, nbytes = self._q.pop(0)
    if ev is not None:
      torch.cuda.current_stream(self._device).wait_event(ev)
      for t in batch.Flatten():
        if isinstance(t, torch.Tensor) and t.is_cuda:
          t.record_stream(torch.cuda.current_stream(self._device))
    self.h2d_bytes_last = nbytes
    self._Issue()
    return batch


def MaybeOffsetDataSourceId(ds, p, offset):
  """Gives datasource params `ds` the source-id offset unless the legacy all-zero behaviour
  is requested (ref :1055)."""
  if not p.all_zero_source_id_without_within_batch_mixing:
    ds.Set(source_id_offset=offset)


def PartitionFilePatternsIntoDataSources(p):
  """`batch_mixing_partition_boundaries` → (list of SimpleDataSource params, one per
  partition, each mixing its patterns within a batch; the partitions' summed weights)
  (ref :1065)."""
  from lingvo_b200.core import datasource  # pylint: disable=g-import-not-at-top
  if max(len(e) for e in p.file_pattern) >= 3:
    raise ValueError('Cannot use batch_mixing_partition_boundaries with backprop filters, '
                     'i.e. file_pattern cannot have triplets: %s' % (p.file_pattern,))
  bounds = list(p.batch_mixing_partition_boundaries)
  if any(b <= a for a, b in zip([0] + bounds, bounds)):
    raise ValueError('batch_mixing_partition_boundaries must be an increasing series '
                     'greater than 0. Values were: %s' % bounds)
  if bounds[-1] >= len(p.file_pattern):
    raise ValueError('batch_mixing_partition_boundaries cannot have a boundary >= the number '
                     'of file patterns: %s vs %d' % (bounds, len(p.file_pattern)))
  datasources, weights = [], []
  for start, end in zip([0] + bounds, bounds + [len(p.file_pattern)]):
    pats = [e[0] for e in p.file_pattern[start:end]]
    ws = [float(e[1]) for e in p.file_pattern[start:end]]
    ds = datasource.SimpleDataSource.Params().Set(file_pattern=pats, weights=ws)
    MaybeOffsetDataSourceId(ds, p, start)
    datasources.append(ds)
    weights.append(float(np.sum(ws)))
  return datasources, weights


def FilePatternToDataSource(p):
  """The (deprecated) `file_pattern` forms → datasource params (ref :1144):

  * `'type:glob'` or a list of them → one `SimpleDataSource`;
  * `[(pattern, weight), …]` with `use_within_batch_mixing` → one weighted source;
  * `[(pattern, weight[, bprop_filter]), …]` otherwise → `CrossBatchMixingDataSource`
    (optionally partitioned by `batch_mixing_partition_boundaries`).
  """
  from lingvo_b200.core import datasource  # pylint: disable=g-import-not-at-top
  fp = p.file_pattern
  if isinstance(fp, str):
    ds = datasource.SimpleDataSource.Params().Set(file_pattern=fp)
  elif isinstance(fp, (list, tuple)):
    if all(isinstance(x, str) for x in fp):
      ds = datasource.SimpleDataSource.Params().Set(file_pattern=list(fp))
    elif p.use_within_batch_mixing:
      if max(len(e) for e in fp) >= 3:
        raise ValueError('Expected a list of pairs, got %s' % (fp,))
      pats, weights = (list(x) for x in zip(*fp))
      ds = datasource.SimpleDataSource.Params().Set(file_pattern=pats, weights=weights)
    else:
      for e in fp:
        if isinstance(e, str):
          raise ValueError('Should explicitly specify weights, got string: %s' % e)
      if p.Get('batch_mixing_partition_boundaries') is not None:
        subs, weights = PartitionFilePatternsIntoDataSources(p)
        ds = datasource.CrossBatchMixingDataSource.Params().Set(sub=subs, weights=weights)
      else:
        subs, weights, filters = [], [], []
        for source_id, e in enumerate(fp):
          subs.append(datasource.SimpleDataSource.Params().Set(file_pattern=e[0]))
          MaybeOffsetDataSourceId(subs[-1], p, source_id)
          weights.append(e[1])
          filters.append(e[2] if len(e) > 2 else '')
        ds = datasource.CrossBatchMixingDataSource.Params().Set(
            sub=subs, weights=weights, bprop_variable_filters=filters)
  else:
    raise ValueError('Cannot parse p.file_pattern into a datasource.')
  cluster = cluster_factory.Current()
  if (getattr(cluster, 'tf_data_service_address', '') and not cluster.do_eval and
      p.Get('use_tf_data_service')):
    ds = datasource.TFDataServiceSource.Params().Set(
        sub=ds, bucket_upper_bound=p.Get('bucket_upper_bound'))
    ds = datasource.TFDatasetPrefetch.Params().Set(sub=ds)
  return ds


class BaseInputGeneratorFromFiles(BaseInputGenerator):
  """Base class for input generators that read from files (:1223-1460)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('file_pattern', '', '`type:glob` or list of them / (pattern, '
             'weight) pairs. Deprecated in favour of file_datasource.')
    p.Define('file_random_seed', 301, 'Shuffle seed; 0 ⇒ system-random.')
    p.Define('file_buffer_size', 10000, 'Shuffle buffer size (records).')
    p.Define('file_buffer_size_in_seconds', 0, 'Adaptive buffer (seconds).')
    p.Define('file_parallelism', 16, 'Number of files read in parallel.')
    p.Define('bucket_adjust_every_n', 0, 'Re-tune buckets every n records.')
    p.Define('flush_every_n', 0, 'Flush partial buckets every n records.')
    p.Define('num_batcher_threads', 1, 'Processor threads.')
    p.Define('repeat_count', -1, 'Epochs to produce; -1 = forever.')
    p.Define('require_sequential_order', False, 'Read files sequentially.')
    p.Define('use_within_batch_mixing', False, 'Mix sources within a batch.')
    p.Define('batch_mixing_partition_boundaries', None,
             'With cross-batch mixing: ascending indices into file_pattern that start a new '
             'partition; patterns inside a partition are mixed WITHIN a batch, partitions '
             'are mixed across batches with the summed weights (ref :1268).')
    p.Define('all_zero_source_id_without_within_batch_mixing', True,
             'Legacy behaviour: every cross-batch source reports source_id 0. False gives '
             'source k the id k.')
    p.Define('use_tf_data_service', True, 'Allow the host-parallel data service wrapper.')
    p.Define('use_chaining', False, 'Chain sources sequentially.')
    p.Define('fatal_errors', [], 'Error substrings that abort the pipeline.')
    p.Define('bucket_upper_bound', [], 'Bucketing scheme: upper bounds.')
    p.Define('bucket_batch_limit', [], 'Per-bucket batch limits.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    if p.file_datasource is None and p.file_pattern:
      self.CreateChild('datasource', FilePatternToDataSource(p).Set(name='datasource'))
      self.datasource.SetInputGenerator(self)
    self._input_op = None

  def CommonInputOpArgs(self):
    p = self.params
    args = super().CommonInputOpArgs()
    num_threads = p.num_batcher_threads
    if self.cluster.require_sequential_input_order:
      num_threads = 1
    args.update({
        'file_random_seed': p.file_random_seed,
        'file_buffer_size': p.file_buffer_size,
        'file_buffer_size_in_seconds': p.file_buffer_size_in_seconds,
        'file_parallelism': p.file_parallelism,
        'bucket_adjust_every_n': p.bucket_adjust_every_n,
        'flush_every_n': p.flush_every_n,
        'num_threads': num_threads,
        'repeat_count': p.repeat_count,
        'require_sequential_order': (p.require_sequential_order or
                                     self.cluster.require_sequential_input_order),
        'fatal_errors': p.fatal_errors,
        'bucket_upper_bound': list(p.bucket_upper_bound),
        'bucket_batch_limit': self.infeed_bucket_batch_limit,
    })
    return args

  @property
  def infeed_bucket_batch_limit(self) -> List[int]:
    p = self.params
    return [batch_utils.scale_split_to_infeed(b, p.use_per_host_infeed)
            for b in p.bucket_batch_limit]

  def InfeedBatchSize(self):
    lim = self.infeed_bucket_batch_limit
    return max(lim) if lim else super().InfeedBatchSize()

  def ProcessRecord(self, record: bytes, source_id: int = 0):
    """Subclass hook: one serialized record → `(NestedMap of np arrays, bucket_key)`
    or None to drop it. Used by the default `_DataSourceFromFilePattern`."""
    raise NotImplementedError(
        '%s must implement ProcessRecord or _DataSourceFromFilePattern' %
        type(self).__name__)

  def _DataSourceFromFilePattern(self, file_pattern, input_source_weights=None,
                                 **extra_input_kwargs):
    """Returns a callable producing one batch NestedMap per call. Default: the
    native yielder + bucketing batcher (`core/generic_input.py`) over
    `self.ProcessRecord` (the role of the per-task `generic_input_op` wrappers in
    the reference, e.g. `tasks/mt/input_generator.py`)."""
    from lingvo_b200.core import generic_input  # pylint: disable=g-import-not-at-top
    args = self.CommonInputOpArgs()
    gi = generic_input.GenericInput(
        self.ProcessRecord, file_pattern=file_pattern,
        bucket_upper_bound=args['bucket_upper_bound'] or [1 << 30],
        bucket_batch_limit=args['bucket_batch_limit'] or [self.InfeedBatchSize()],
        file_random_seed=args['file_random_seed'],
        file_buffer_size=args['file_buffer_size'],
        file_parallelism=args['file_parallelism'], num_threads=args['num_threads'],
        flush_every_n=args['flush_every_n'], repeat_count=args['repeat_count'],
        require_sequential_order=args['require_sequential_order'],
        input_source_weights=input_source_weights,
        bucket_adjust_every_n=args['bucket_adjust_every_n'],
        fatal_errors=(list(args['fatal_errors']) if args['fatal_errors'] else None),
        file_buffer_size_in_seconds=args['file_buffer_size_in_seconds'],
        **extra_input_kwargs)
    self._generic_input = gi

    def _Next():
      batch, keys = gi.GetNext()
      batch = batch if isinstance(batch, NestedMap) else NestedMap(data=batch)
      batch = batch.Transform(
          lambda x: torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x)
      batch.bucket_keys = torch.from_numpy(np.asarray(keys))
      return batch
    return _Next

  def _InputBatch(self):
    ds = self.datasource
    if getattr(ds, '_input_generator', None) is None:
      ds.SetInputGenerator(self)
    return ds.GetNext()


class BaseSequenceInputGenerator(BaseInputGeneratorFromFiles):
  """Sequence inputs with tokenizers and bucketing (:1465-1697)."""

  @classmethod
  def Params(cls):
    from lingvo_b200.core import tokenizers
    p = super().Params()
    p.Define('pad_to_max_seq_length', False, 'Pad every batch to max length.')
    p.Define('source_max_length', None, 'Max source length.')
    p.Define('target_max_length', 300, 'Max target length.')
    p.Define('tokenizer', tokenizers.AsciiTokenizer.Params(), 'Tokenizer.')
    p.Define('tokenizer_dict', {}, 'key → tokenizer params.')
    p.bucket_upper_bound = [10, 20, 30, 60, 120]
    p.bucket_batch_limit = [128, 128, 128, 32, 16]
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    self.tokenizer_dict = {}
    if p.tokenizer:
      assert 'default' not in p.tokenizer_dict
      td = dict(p.tokenizer_dict)
      td['default'] = p.tokenizer
    else:
      td = dict(p.tokenizer_dict)
    names = []
    for k, tp in td.items():
      if tp:
        names.append(k)
        self.CreateChild('tokenizer_%s' % k, tp.Copy().Set(
            name='tokenizer_%s' % k))
    for k in names:
      self.tokenizer_dict[k] = self.children['tokenizer_%s' % k]
    if 'default' in self.tokenizer_dict:
      self.tokenizer = self.tokenizer_dict['default']

  @property
  def scaled_bucket_batch_limit(self):
    return self.infeed_bucket_batch_limit

  def StringsToIds(self, strs, is_source=False, external_max_length=None,
                   external_append_eos=None, key=None, languages=None):
    """strings → (ids, labels, paddings), each `[batch, maxlen]` (:1565)."""
    p = self.params
    if external_max_length is not None:
      maxlen = external_max_length
    elif is_source:
      maxlen = p.source_max_length
    else:
      maxlen = p.target_max_length
    tok = self.tokenizer_dict[key or 'default']
    return tok.StringsToIds(strs, maxlen, external_append_eos, languages)

  def StringsToIdsWithOffsets(self, strs, **kwargs):
    return self.StringsToIds(strs, **kwargs)

  def IdsToStrings(self, ids, lens, key=None):
    return self.tokenizer_dict[key or 'default'].IdsToStrings(ids, lens)


class TFDataSequenceInputGenerator(BaseSequenceInputGenerator):
  """Sequence inputs assembled from `datasource.Dataset` pipelines (ref :1770): subclasses
  provide `LoadDataset(file_pattern)` (examples without a batch dim), `ProcessDataset`,
  `GetSequenceLength`, `_InputShape`; this class adds eval truncation, length bucketing +
  padding, optional host-parallel service and prefetch. A drop-in for generators derived
  from `BaseSequenceInputGenerator` (file_pattern / bucket params keep their meaning)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('prefetch_buffer_size', 1, 'Local prefetch buffer size (batches).')
    p.resettable = True
    return p

  def __init__(self, params):
    from lingvo_b200.core import datasource  # pylint: disable=g-import-not-at-top
    p = params.Copy()
    ds = p.file_datasource
    if not ds:
      ds = self.ConvertFilePatternToDataSource(p, p.file_pattern)
      p.file_pattern = ''
    ds = datasource.CustomTFDatasetTransform.Params().Set(sub=ds, fn='TakeEvalSamples')
    ds = datasource.TFDatasetBatchBySequenceLength.Params().Set(
        sub=ds, seqlen_fn='GetSequenceLength', input_shape_fn='_InputShape',
        input_padding_fn='_InputPaddingValue', bucket_upper_bound=p.bucket_upper_bound,
        bucket_batch_limit=p.bucket_batch_limit)
    cluster = cluster_factory.Current()
    if getattr(cluster, 'tf_data_service_address', '') and not cluster.do_eval:
      ds = datasource.TFDataServiceSource.Params().Set(
          sub=ds, bucket_upper_bound=p.bucket_upper_bound)
    p.file_datasource = datasource.TFDatasetPrefetch.Params().Set(
        sub=ds, buffer_size=p.prefetch_buffer_size)
    super().__init__(p)

  @classmethod
  def ConvertFilePatternToDataSource(cls, p, file_pattern):
    from lingvo_b200.core import datasource  # pylint: disable=g-import-not-at-top
    weights = None
    if isinstance(file_pattern, str):
      patterns = file_pattern.split(',')
    elif all(isinstance(x, str) for x in file_pattern):
      patterns = list(file_pattern)
    elif all(isinstance(x, tuple) for x in file_pattern):
      patterns, weights = (list(x) for x in zip(*file_pattern))
    else:
      raise ValueError('file_pattern must be all strings or all tuples, but got: %s.' %
                       (file_pattern,))
    for fp in patterns:
      if ',' in fp:
        raise ValueError('file_pattern should not contain comma: %s' % fp)
    subs = [datasource.TFDatasetFnInput.Params().Set(
        load_fn='LoadDataset', kwargs=dict(file_pattern=fp),
        shuffle_buffer_size=p.file_buffer_size) for fp in patterns]
    if len(subs) > 1:
      if not p.use_within_batch_mixing:
        raise ValueError('Only p.use_within_batch_mixing is supported with multiple '
                         'file_patterns.')
      subs = [datasource.TFDatasetMixer.Params().Set(sub=subs, weights=weights)]
    return datasource.CustomTFDatasetTransform.Params().Set(sub=subs[0], fn='ProcessDataset')

  def Reset(self, sess=None):
    self.datasource.Reset(sess)

  def _InputBatch(self):
    return self.datasource.GetNext()

  def LoadDataset(self, file_pattern):
    """→ `datasource.Dataset` of single examples (no batch dim) read from `file_pattern`."""
    raise NotImplementedError()

  def TakeEvalSamples(self, dataset):
    p = self.params
    if self.do_eval and p.num_samples > 0:
      dataset = dataset.take(p.num_samples)
    return dataset

  def ProcessDataset(self, dataset):
    """→ Dataset of processed example NestedMaps (still no batch dim)."""
    raise NotImplementedError()

  def GetSequenceLength(self, example):
    raise NotImplementedError()

  def _InputShape(self, key):
    """Final per-example shape of tensor `key` (None entries = pad to the bucket bound)."""
    if key in ('source_id', 'bucket_keys'):
      return ()
    raise ValueError('Unexpected key %s' % key)

  def _InputPaddingValue(self, key, tensorspec):
    dtype = getattr(tensorspec, 'dtype', None) or np.float32
    return np.ones([], dtype) if key.endswith('_paddings') else np.zeros([], dtype)


class BaseDataExampleInputGenerator(BaseInputGenerator):
  """Batches of parsed `tf.Example` features read from record files (ref :1916):
  list files → interleaved readers → shuffle → take → repeat → batch → parse with
  `GetFeatureSpec()` → `_PreprocessInputBatch`."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('input_files', None, 'Comma-delimited glob(s) of input files.')
    p.Define('dataset_type', None, 'Callable filename → iterable of serialized records '
             '(e.g. `lingvo_b200.utils.tfrecord.ReadRecords`).')
    p.Define('randomize_order', True, 'Shuffle files and records.')
    p.Define('parallel_readers', 1, 'Files read concurrently (round-robin interleave).')
    p.Define('num_examples', -1, 'Number of examples (-1 for unlimited).')
    p.Define('num_epochs', -1, 'Passes over the data (-1 for unlimited); the input raises '
             'StopIteration afterwards.')
    p.Define('randomize_shuffle_size', 500, 'Size of the random shuffle buffer.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    assert p.input_files, 'input_files is required for an example input generator'
    assert p.dataset_type, 'dataset_type is required for an example input generator'
    self._iterator = iter(self._InitDataset())

  def GetFeatureSpec(self):
    """→ {feature name: (dtype, shape) | FixedLenFeature-like with .dtype/.shape}; an empty
    spec keeps every feature of the record as a 1-D array."""
    return {}

  def _AdditionalPreprocessInputBatch(self, batch):
    return batch

  def _ParseBatch(self, records):
    from lingvo_b200.utils import tf_example  # pylint: disable=g-import-not-at-top
    spec = self.GetFeatureSpec()
    parsed = [tf_example.ParseExample(r) for r in records]
    names = list(spec) if spec else sorted(parsed[0])
    out = NestedMap()
    for name in names:
      cols = []
      for ex in parsed:
        if name not in ex:
          raise KeyError('Feature %r missing from a record' % name)
        v = ex[name]
        if spec:
          sp = spec[name]
          dtype, shape = (sp.dtype, sp.shape) if hasattr(sp, 'dtype') else sp
          if v.dtype.kind not in 'OSU':
            v = v.astype(dtype)
          v = v.reshape(list(shape))
        cols.append(v)
      arr = np.stack(cols)
      out[name] = arr if arr.dtype.kind in 'OSU' else torch.from_numpy(
          np.ascontiguousarray(arr))
    return out

  def _InitDataset(self):
    import glob  # pylint: disable=g-import-not-at-top
    from lingvo_b200.core import datasource  # pylint: disable=g-import-not-at-top
    p = self.params
    files = sorted(f for pat in p.input_files.split(',') for f in glob.glob(pat))
    assert files, 'No files match %s' % p.input_files
    rng = np.random.RandomState(p.random_seed)

    def Records():
      order = list(files)
      if p.randomize_order:
        rng.shuffle(order)
      pending = list(order)
      readers = []
      while pending or readers:
        while pending and len(readers) < max(p.parallel_readers, 1):
          readers.append(iter(p.dataset_type(pending.pop(0))))
        for r in list(readers):
          try:
            yield next(r)
          except StopIteration:
            readers.remove(r)

    ds = datasource.Dataset.FromGenerator(Records)
    if p.randomize_order:
      ds = ds.shuffle(p.randomize_shuffle_size, seed=p.random_seed)
    if p.num_examples >= 0:
      ds = ds.take(p.num_examples)
    ds = ds.repeat(None if p.num_epochs < 0 else p.num_epochs)
    bs = self.InfeedBatchSize()

    def Batches():
      buf = []
      for rec in ds:
        buf.append(rec)
        if len(buf) == bs:
          yield self._ParseBatch(buf)
          buf = []          # remainder dropped, as drop_remainder=True

    return datasource.Dataset.FromGenerator(Batches).prefetch(2)

  def _InputBatch(self):
    return next(self._iterator)

  def GetPreprocessedInputBatch(self):
    return self._AdditionalPreprocessInputBatch(super().GetPreprocessedInputBatch())

  def Reset(self, sess=None):
    self._iterator = iter(self._InitDataset())


class BaseTinyDatasetInput(BaseInputGenerator):
  """Whole tiny dataset in memory (MNIST) (reference :1706-1767).

  `ckpt` names a data file holding named tensors (`.npz`, or a tensor-bundle
  checkpoint prefix as the reference uses); `data`/`label` name the tensors.
  Batches are random permutations per epoch (`repeat`) or one sequential pass
  with the last batch zero-padded and `weight` masking the padding.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('ckpt', None, 'Path of the data file.')
    p.Define('data', 'x_train', 'Name of the data tensor.')
    p.Define('data_dtype', torch.uint8, 'Type of the data tensor.')
    p.Define('data_shape', (0, 0, 0), 'Shape of one example.')
    p.Define('label', 'y_train', 'Name of the label tensor.')
    p.Define('label_dtype', torch.uint8, 'Type of the label tensor.')
    p.Define('repeat', True, 'Go through the dataset repeatedly.')
    p.use_per_host_infeed = True
    return p

  def __init__(self, params):
    super().__init__(params)
    self._cached = None
    self._perm = None

  def _Load(self):
    if self._cached is None:
      p = self.params
      from lingvo_b200.ops import native_input
      tensors = native_input.CachedLoadTensors(p.ckpt, [p.data, p.label])
      self._cached = (torch.as_tensor(tensors[p.data]),
                      torch.as_tensor(tensors[p.label]))
    return self._cached

  def _InputBatch(self):
    p = self.params
    data, label = self._Load()
    n = min(p.num_samples or data.shape[0], data.shape[0])
    bs = self.InfeedBatchSize()
    if self._perm is None:
      from lingvo_b200.ops import native_input
      self._perm = native_input.RandomPermutationSequence(
          num=n, batch=bs, repeat=p.repeat,
          seed=p.random_seed if p.random_seed is not None else 0)
    idx = self._perm.Next()  # raises StopIteration at epoch end if not repeat
    idx_t = torch.as_tensor(idx, dtype=torch.long)
    raw = data[idx_t].to(torch.float32)
    raw = raw.reshape([len(idx)] + list(p.data_shape))
    lab = label[idx_t].to(torch.float32)
    pad = bs - len(idx)
    weight = torch.ones([bs])
    if pad > 0:
      raw = torch.cat([raw, torch.zeros([pad] + list(raw.shape[1:]))], 0)
      lab = torch.cat([lab, torch.zeros([pad] + list(lab.shape[1:]))], 0)
      weight[len(idx):] = 0
    return NestedMap(raw=raw, data=raw, label=lab, weight=weight,
                     sample_ids=torch.nn.functional.pad(idx_t, (0, pad)))

  def _PreprocessInputBatch(self, batch):
    # Image data is in [0, 255]; normalise to [-1, 1].
    batch.data = (batch.raw - 128.0) / 128.0
    return batch

  def Reset(self, sess=None):
    self._perm = None


def DefineTFDataInput(name, func, ignore_args=None, map_args=None,
                      base_class=BaseInputGenerator):
  """Defines an InputGenerator class from a dataset-pipeline function (reference :2022).

  `func(**args)` returns a `datasource.Dataset` (or any re-iterable) of dict-like elements;
  its signature is analysed to generate `Params().args` so the pipeline's configuration
  lives in Params like everything else. `map_args = {func_param: layer_param}` feeds existing
  params (e.g. `batch_size`) into the function instead. The generated generator behaves like
  a one-shot iterator of the pipeline (`GetPreprocessedInputBatch()` yields its elements in
  order, as `NestedMap`s); with `cluster.tf_data_service_address` set, training inputs are
  produced by the background worker pool (`TFDataServiceSource`) behind a prefetch.

    def my_dataset(begin=0, end=10):
      return datasource.Dataset.FromElements({'value': i} for i in range(begin, end))
    MyInput = DefineTFDataInput('MyInput', my_dataset)
    p = MyInput.Params(); p.args.end = 3
    MyInput(p).GetPreprocessedInputBatch()      # NestedMap(value=0), then 1, 2
  """
  import inspect  # pylint: disable=g-import-not-at-top
  from lingvo_b200.core import cluster_factory  # pylint: disable=g-import-not-at-top
  from lingvo_b200.core import datasource  # pylint: disable=g-import-not-at-top
  from lingvo_b200.core import hyperparams  # pylint: disable=g-import-not-at-top
  from lingvo_b200.core import inspect_utils  # pylint: disable=g-import-not-at-top
  ignore_args = set(ignore_args or ())
  map_args = dict(map_args or {})
  generated_cls = type(name, (base_class,), {})

  @classmethod
  def _Params(cls):
    p = super(generated_cls, cls).Params()
    p.Define('args', hyperparams.Params(), 'Parameter list of the pipeline.')
    inspect_utils.DefineParams(func, p.args, ignore_args | set(map_args.keys()))
    ds = datasource.TFDatasetFnInput.Params().Set(load_fn='GetDataset', shuffle_buffer_size=1)
    cur = cluster_factory.Current()
    if getattr(cur.params, 'tf_data_service_address', None) and not cur.do_eval:
      ds = datasource.TFDataServiceSource.Params().Set(sub=ds)
      ds = datasource.TFDatasetPrefetch.Params().Set(sub=ds)
    p.file_datasource = ds
    return p

  def _GetDataset(self):
    p = self.params
    overrides = {k: p.Get(v) for k, v in map_args.items()}
    dataset = inspect_utils.CallWithParams(func, p.args, **overrides)
    if not isinstance(dataset, datasource.Dataset):
      src = dataset
      assert hasattr(src, '__iter__') or callable(src), (
          'DefineTFDataInput must take a callable which returns a Dataset / iterable. '
          'The given callable `%s` returned `%s`' % (func, dataset))
      dataset = datasource.Dataset(lambda: iter(src() if callable(src) else src))
    return dataset

  def _GetPreprocessedInputBatch(self):
    data = self.datasource.GetNext()
    assert isinstance(data, dict), (
        'DefineTFDataInput accepts only datasets that return a dict or its subclasses.')
    if not isinstance(data, NestedMap):
      data = NestedMap.FromNestedDict(data) if hasattr(NestedMap, 'FromNestedDict') else (
          NestedMap(data))
    return data

  generated_cls.Params = _Params
  generated_cls.GetDataset = _GetDataset
  generated_cls.GetPreprocessedInputBatch = _GetPreprocessedInputBatch
  generated_cls.__module__ = inspect.stack()[1].frame.f_globals.get('__name__', '__main__')
  return generated_cls
