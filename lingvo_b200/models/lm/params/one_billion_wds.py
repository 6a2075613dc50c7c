"""One Billion Words LM configs (ref `lingvo/tasks/lm/params/one_billion_wds.py`)."""

import os

from lingvo_b200 import model_registry
from lingvo_b200.core import base_model_params
from lingvo_b200.core import layers
from lingvo_b200.core import optimizer
from lingvo_b200.core import py_utils
from lingvo_b200.core import schedule
from lingvo_b200.core import tokenizers
from lingvo_b200.models.lm import input_generator as lm_inp
from lingvo_b200.models.lm import layers as lm_layers
from lingvo_b200.models.lm import model

DATADIR = os.environ.get('LINGVO_B200_1BWDS', '/tmp/lm1b/1-billion-word-language-modeling-benchmark-r13output')


class WordLevelOneBwdsBase(base_model_params.SingleTaskModelParams):
  """Word-level LSTM LM with the 793k-word vocabulary (ref :49)."""

  CORPUS_DIR = DATADIR
  EMBEDDING_DIM = 1024
  MAX_TOKENS = 1024
  NUM_EMBEDDING_SHARDS = 8
  NUM_SAMPLED = 8192
  NUM_SOFTMAX_SHARDS = 8
  RNN_STATE_DIM = 2048
  VOCAB_SIZE = 793472
  WORD_VOCAB = os.path.join(DATADIR, 'vocab.txt')

  @classmethod
  def _Input(cls, pattern, training):
    p = lm_inp.LmInput.Params()
    p.bucket_upper_bound = [10, 20, 30, 40, 50, 100, 256, 512, 1024]
    p.bucket_batch_limit = [max(1, cls.MAX_TOKENS // b) for b in p.bucket_upper_bound]
    p.file_buffer_size = 10000000 if training else 1
    p.file_parallelism = 10 if training else 1
    p.file_pattern = 'text:' + os.path.join(cls.CORPUS_DIR, pattern)
    p.name = '1bwds_train_set' if training else '1bwds_dev_set'
    p.tokenizer = tokenizers.VocabFileTokenizer.Params().Set(
        token_vocab_filepath=cls.WORD_VOCAB, target_sos_id=1, target_eos_id=2,
        target_unk_id=3, load_token_ids_from_vocab=False)
    p.num_batcher_threads = 16 if training else 1
    p.target_max_length = 1024
    p.tokenizer.vocab_size = cls.VOCAB_SIZE
    if not training:
      p.num_samples = 6206
      p.require_sequential_order = True
    return p

  def Train(self):
    return self._Input('training-monolingual.tokenized.shuffled/news.en*', True)

  def Dev(self):
    return self._Input('heldout-monolingual.tokenized.shuffled/news.en.heldout-00001*', False)

  def Test(self):
    return self._Input('heldout-monolingual.tokenized.shuffled/news.en.heldout-00000*', False)

  def Task(self):
    p = model.LanguageModel.Params()
    p.name = '1bwds_word_level_lm'
    p.eval.samples_per_summary = 10000
    p.lm = lm_layers.RnnLm.CommonParams(
        vocab_size=self.VOCAB_SIZE, emb_dim=self.EMBEDDING_DIM, num_layers=2,
        residual_start=3, rnn_dims=self.EMBEDDING_DIM,
        rnn_hidden_dims=self.RNN_STATE_DIM)
    p.lm.embedding_dropout_keep_prob = 0.75
    p.lm.output_dropout_prob = 0.25
    for tpl in ([p.lm.rnns.cell_tpl] if not isinstance(p.lm.rnns.cell_tpl, list)
                else p.lm.rnns.cell_tpl):
      tpl.params_init = py_utils.WeightInit.Uniform(0.05)
    tp = p.train
    tp.sum_loss_across_tokens_in_batch = True
    tp.l2_regularizer_weight = None
    tp.vn_std = 0.0
    tp.learning_rate = 0.2
    tp.max_lstm_gradient_norm = 16
    tp.clip_gradient_norm_to_value = 0.0
    tp.optimizer = optimizer.Adagrad.Params()
    tp.lr_schedule = schedule.PiecewiseConstantSchedule.Params().Set(boundaries=[], values=[1.0])
    return p


@model_registry.RegisterSingleTaskModel
class WordLevelOneBwdsSimpleSampledSoftmax(WordLevelOneBwdsBase):
  """Sampled-softmax variant (ref :134). On H100 the full 793k softmax fits the
  fused chunked LM-head kernel, so `NUM_SAMPLED` only bounds its chunk size."""

  def Task(self):
    p = super().Task()
    p.lm.softmax.chunk_size = max(1, self.NUM_SAMPLED // 8)
    return p


@model_registry.RegisterSingleTaskModel
class WordLevelOneBwdsSimpleSampledSoftmaxTiny(WordLevelOneBwdsSimpleSampledSoftmax):
  """Unit-test sized config (ref :170)."""

  EMBEDDING_DIM = 7
  MAX_TOKENS = 1024
  NUM_EMBEDDING_SHARDS = 1
  NUM_SAMPLED = 8
  NUM_SOFTMAX_SHARDS = 8
  RNN_STATE_DIM = 32
  VOCAB_SIZE = 32


@model_registry.RegisterSingleTaskModel
class OneBwdsTransformerLm(WordLevelOneBwdsBase):
  """Transformer LM on the same data (H100 flagship-style stack)."""

  VOCAB_SIZE = 32000
  MODEL_DIM = 1024
  HIDDEN_DIM = 4096
  NUM_HEADS = 8
  NUM_LAYERS = 12

  def Task(self):
    p = model.LanguageModel.Params()
    p.name = '1bwds_transformer_lm'
    p.lm = lm_layers.TransformerLm.CommonParams(
        model_dim=self.MODEL_DIM, hidden_dim=self.HIDDEN_DIM, num_heads=self.NUM_HEADS,
        num_layers=self.NUM_LAYERS, vocab_size=self.VOCAB_SIZE)
    tp = p.train
    tp.learning_rate = 1e-3
    tp.optimizer = optimizer.Adam.Params().Set(beta1=0.9, beta2=0.98, epsilon=1e-9)
    tp.lr_schedule = schedule.TransformerSchedule.Params().Set(
        warmup_steps=4000, model_dim=self.MODEL_DIM)
    return p


@model_registry.RegisterSingleTaskModel
class OneBWdsGPipeTransformerWPM(WordLevelOneBwdsBase):
  """32-layer, d=2048 Transformer LM trained with GPipe (ref :181). The reference reports
  relative throughput 1.0 / 0.93 / 0.85 / 0.775 on 1 / 2 / 4 / 8 V100s; here the stack is
  cut into `GPUS` cells run by `parallel.pp.PipelineEngine` (one rank per cell, P2P
  activations over NVLink)."""

  VOCAB_SIZE = 32000
  EMBEDDING_DIM = 2048
  BATCH_SIZE = 32
  MAX_TOKENS = 1024
  GPUS = 4
  SPLITS = [8 * (i + 1) for i in range(GPUS)]     # cumulative layer index per cell
  LAYERS = SPLITS[-1]
  NUM_MICRO_BATCHES = 32

  def Train(self):
    p = super().Train()
    p.tokenizer = tokenizers.AsciiTokenizer.Params().Set(
        target_sos_id=1, target_eos_id=2, target_unk_id=0, vocab_size=self.VOCAB_SIZE)
    p.target_max_length = self.MAX_TOKENS
    p.bucket_upper_bound = [self.MAX_TOKENS]
    p.bucket_batch_limit = [self.BATCH_SIZE]
    p.fixed_input_shape = True
    return p

  def _Heldout(self, shard, name, n):
    p = self.Train()
    p.file_pattern = 'text:' + os.path.join(
        self.CORPUS_DIR, 'heldout-monolingual.tokenized.shuffled', shard)
    p.Set(name=name, num_batcher_threads=1, num_samples=n)
    return p

  def Dev(self):
    return self._Heldout('news.en.heldout-00001*', '1bwds_dev_set', 6206)

  def Test(self):
    return self._Heldout('news.en.heldout-00000*', '1bwds_test_set', 6075)

  def Task(self):
    p = model.BatchMajorLanguageModel.Params()
    p.eval.samples_per_summary = 0
    p.name = '1bwds_wpm_level_lm'
    p.lm = lm_layers.GPipeTransformerLm.CommonParams(
        model_dim=self.EMBEDDING_DIM, vocab_size=self.VOCAB_SIZE,
        hidden_dim=self.EMBEDDING_DIM * 4, num_layers=self.LAYERS, num_heads=16,
        softmax_max_alloc=128 * (2 ** 20), atten_dropout_prob=0.1,
        residual_dropout_prob=0.1)
    p.lm.Set(num_splits=len(self.SPLITS), num_micro_batches=self.NUM_MICRO_BATCHES)
    p.train.Set(
        learning_rate=0.5, optimizer=optimizer.Adam.ParamsA(),
        clip_gradient_norm_to_value=0.0, grad_norm_to_clip_to_zero=0.0,
        lr_schedule=schedule.TransformerSchedule.Params().Set(
            warmup_steps=40000, worker_replicas=1, model_dim=self.EMBEDDING_DIM))
    return p
