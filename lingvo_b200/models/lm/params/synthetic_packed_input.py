"""DenseBuilder-based LMs with synthetic packed inputs.

Reference `tasks/lm/params/synthetic_packed_input.py` (`SyntheticTrain`
:29-50, `DenseLmTemplate` :53-160 and the registered `DenseLm*` configs) plus
the GShard **MoE** LM the north-star benchmark names (assembled as
`gshard_builder_test.py:631-666` does: `UniTransformer(moe=True)` +
`DenseBuilder(e_dim=8, capacity_factor, moe_hidden_dim)`).
"""

import numpy as np
import torch

from lingvo_b200 import model_registry
from lingvo_b200.core import base_input_generator
from lingvo_b200.core import base_model_params
from lingvo_b200.core import gshard_builder
from lingvo_b200.core import optimizer
from lingvo_b200.core import program
from lingvo_b200.core import py_utils
from lingvo_b200.core import schedule
from lingvo_b200.core.nested_map import NestedMap


class SyntheticTrain(base_input_generator.BaseInputGenerator):
  """Synthetic data in the packed-input LM format.

  `random_ids=False` reproduces the reference (all-ones targets). With
  `random_ids=True` token ids are uniform in [1, vocab) — needed for MoE
  benchmarks, where identical tokens would all route to one expert — and each
  row is packed as `segments_per_row` equal-length segments.
  """

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('seq_len', 0, 'Number of tokens in one example.')
    p.Define('random_ids', False, 'Uniform random ids instead of ones.')
    p.Define('vocab_size', 32000, 'Vocabulary for random ids.')
    p.Define('segments_per_row', 1, 'Packed segments per row.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self._step = 0

  def _InputBatch(self):
    p = self.params
    b, l = self.InfeedBatchSize(), p.seq_len
    if p.random_ids:
      gen = torch.Generator()
      gen.manual_seed((p.random_seed or 0) * 1000003 + self._step +
                      7919 * self.cluster.rank)
      self._step += 1
      targets = torch.randint(1, p.vocab_size, (b, l), generator=gen,
                              dtype=torch.int32)
    else:
      targets = torch.ones(b, l, dtype=torch.int32)
    seg_len = l // p.segments_per_row
    pos = torch.arange(l, dtype=torch.int32)
    seg_ids = (pos // seg_len + 1).clamp(max=p.segments_per_row)
    seg_pos = pos - (seg_ids - 1) * seg_len
    if not p.random_ids and p.segments_per_row == 1:
      # Reference quirk: segment_pos = targets (all ones).
      seg_pos = torch.ones(l, dtype=torch.int32)
    batch = NestedMap()
    batch.tgt = NestedMap(
        ids=torch.roll(targets, 1, dims=1), labels=targets,
        segment_ids=seg_ids.unsqueeze(0).expand(b, l).contiguous(),
        segment_pos=seg_pos.unsqueeze(0).expand(b, l).contiguous())
    if p.pin_memory and torch.cuda.is_available():
      batch = batch.Transform(lambda t: t.pin_memory())
    # Host-side knowledge: every position belongs to a segment (ids ≥ 1), so the model
    # may skip its padding masks. Computed from host data, no device sync involved.
    batch.tgt.all_valid = True
    return batch


class DenseLmTemplate(base_model_params.SingleTaskModelParams):
  """DenseBuilder-based LM Template (reference :53-160)."""
  BATCH_DIM_PER_DEVICE = 0.0625
  NUM_DEVICES_PER_SPLIT = 64
  SEQUENCE_LENGTH = 1024
  HIDDEN_DIM = 65536
  ATTENTION_KEY_VALUE_DIM = 128
  MODEL_DIM = 8192
  NUM_HEADS = 128
  NUM_KV_HEADS = None        # grouped-query / multi-query attention; None = NUM_HEADS
  NUM_TRANSFORMER_LAYERS = 32
  LABEL_SMOOTHING = 0.0
  VOCAB_SIZE = 32000
  DEVICE_MESH_SHAPE = [64, 1]
  DEVICE_MESH = None
  DEBUG = False
  ATTEN_LOGIT_CAP = 0
  ATTENTION_EXTRA_LOGIT = None
  MODEL_DIM_RESHAPE_SEGMENTS = None
  GATED_GELU = True
  POSITIONAL_EMBEDDING = False
  USE_REPEAT_LAYER = False
  TRAIN_STEPS_PER_LOOP = 100

  def _Builder(self):
    return gshard_builder.DenseBuilder.Params().Set(
        device_mesh_shape=self.DEVICE_MESH_SHAPE,
        device_mesh=self.DEVICE_MESH,
        relative_attention_num_buckets=32,
        relative_attention_type='bias',
        relative_attention_max_distance=128,
        dtype=torch.float32,
        fprop_dtype=torch.bfloat16,
        atten_logit_cap=self.ATTEN_LOGIT_CAP,
        attention_logits_dtype=torch.float32,
        dropout_rate=0.0,
        num_devices=1,
        attention_dropout_prob=0.0,
        attention_key_value_dim=self.ATTENTION_KEY_VALUE_DIM,
        attention_extra_logit=self.ATTENTION_EXTRA_LOGIT,
        relative_attention_use_universal_1d_position=True,
        model_dim_reshape_segments=self.MODEL_DIM_RESHAPE_SEGMENTS,
        model_dim=self.MODEL_DIM,
        attention_num_heads=self.NUM_HEADS,
        attention_num_memory_heads=self.NUM_KV_HEADS,
        ff_dim=self.HIDDEN_DIM,
        attention_combine_dims=True)

  def _BatchSize(self):
    return max(1, int(self.BATCH_DIM_PER_DEVICE * self.NUM_DEVICES_PER_SPLIT))

  def Task(self):
    p = gshard_builder.UniTransformer.Params().Set(
        gated_gelu=self.GATED_GELU,
        debug=self.DEBUG,
        positional_embedding=self.POSITIONAL_EMBEDDING,
        use_repeat_layer=self.USE_REPEAT_LAYER,
        dtype=torch.float32,
        fprop_dtype=torch.bfloat16,
        name='transformer',
        builder=self._Builder(),
        batch_size=self._BatchSize(),
        sequence_length=self.SEQUENCE_LENGTH,
        num_transformer_layers=self.NUM_TRANSFORMER_LAYERS,
        aux_loss_coef=0.0,
        label_smoothing=self.LABEL_SMOOTHING,
        vocab_size=self.VOCAB_SIZE,
        max_length=self.SEQUENCE_LENGTH)
    p.train.optimizer = optimizer.XLAShardingAdafactor.Params().Set(
        beta1=0.0, beta2=0.99, multiply_by_parameter_scale=True,
        clipping_threshold=1.0, factored=True, decay_exponent_pow=0.8)
    p.train.learning_rate = 1.0
    p.train.lr_schedule = schedule.SqrtDecay.Params().Set(
        warmup_steps=10000, multiplier=1.0)
    p.train.max_steps = 2000000
    p.train.save_max_to_keep = 100
    return p

  def Train(self):
    p = SyntheticTrain.Params()
    p.batch_size = self._BatchSize()
    p.seq_len = self.SEQUENCE_LENGTH
    return p

  def ProgramSchedule(self):
    p = program.SimpleProgramScheduleForTask(
        train_dataset_name='Train',
        train_steps_per_loop=self.TRAIN_STEPS_PER_LOOP,
        eval_dataset_names=[], eval_steps_per_loop=0, decode_steps_per_loop=0)
    p.train_program.spmd = True
    p.train_executions_per_eval = 5
    return p


@model_registry.RegisterSingleTaskModel
class DenseLm8B2x2(DenseLmTemplate):
  """8B params LM model with 1D split."""
  SEQUENCE_LENGTH = 1024
  NUM_DEVICES_PER_SPLIT = 128
  BATCH_DIM_PER_DEVICE = 0.125
  NUM_TRANSFORMER_LAYERS = 4
  DEVICE_MESH_SHAPE = [1, 8]
  DEVICE_MESH = np.arange(8).reshape(DEVICE_MESH_SHAPE)

  def Task(self):
    p = super().Task()
    p.train.tpu_device_order_mode = 2
    p.builder.model_dim_reshape_segments = self.DEVICE_MESH_SHAPE[1]
    p.builder.emb_w_split = [-1, 1]
    p.builder.emb_out_split = [0, -1, 1]
    p.builder.blm_split = [0, -1, 1]
    p.builder.logits_split = [0, -1, 1]
    return p


@model_registry.RegisterSingleTaskModel
class DenseLm8B2x2Decode(DenseLm8B2x2):
  """8B params LM decoding config."""

  def Task(self):
    p = super().Task()
    p.builder.relative_attention_use_universal_1d_position = False
    return p


@model_registry.RegisterSingleTaskModel
class DenseLm128B8x8(DenseLmTemplate):
  """128B params LM model with 2D split (~3.7k tokens/s on TPU v3-128)."""
  SEQUENCE_LENGTH = 1024
  NUM_DEVICES_PER_SPLIT = 128
  BATCH_DIM_PER_DEVICE = 0.125
  NUM_TRANSFORMER_LAYERS = 64
  DEVICE_MESH_SHAPE = [8, 16]
  DEVICE_MESH = np.arange(128).reshape(DEVICE_MESH_SHAPE)

  def Task(self):
    p = super().Task()
    p.train.tpu_device_order_mode = 2
    p.builder.model_dim_reshape_segments = self.DEVICE_MESH_SHAPE[1]
    p.builder.emb_w_split = [-1, 1]
    p.builder.emb_out_split = [0, -1, 1]
    p.builder.blm_split = [0, -1, 1]
    p.builder.logits_split = [0, -1, 1]
    return p


@model_registry.RegisterSingleTaskModel
class DenseLm128B16x16(DenseLm128B8x8):
  """128B LM on a 16x16 mesh (~18k tokens/s on TPU v3-512)."""
  NUM_DEVICES_PER_SPLIT = 512
  BATCH_DIM_PER_DEVICE = 0.25
  DEVICE_MESH_SHAPE = [16, 32]
  DEVICE_MESH = np.arange(512).reshape(DEVICE_MESH_SHAPE)


@model_registry.RegisterSingleTaskModel
class DenseLm175B32x32(DenseLm128B16x16):
  """175B LM (seq 2048, 2M-token batch; ~51.53k tokens/s on TPU v3-2048)."""
  HIDDEN_DIM = 12288 * 4
  MODEL_DIM = 12288
  NUM_HEADS = 96
  NUM_TRANSFORMER_LAYERS = 96
  GATED_GELU = False
  POSITIONAL_EMBEDDING = False
  SEQUENCE_LENGTH = 2048
  NUM_DEVICES_PER_SPLIT = 2048
  BATCH_DIM_PER_DEVICE = 0.5
  DEVICE_MESH_SHAPE = [64, 32]
  DEVICE_MESH = np.arange(2048).reshape(DEVICE_MESH_SHAPE)


@model_registry.RegisterSingleTaskModel
class DenseLm175B32x32DP(DenseLm175B32x32):
  """175B LM with data + model parallelism."""
  DEVICE_MESH_SHAPE = [8, 8, 32]
  DEVICE_MESH = np.arange(2048).reshape(DEVICE_MESH_SHAPE)


@model_registry.RegisterSingleTaskModel
class DenseLm175B1K(DenseLm175B32x32):
  """175B LM on a 1024-device [64, 16] mesh (ref :280)."""
  DEVICE_MESH_SHAPE = [64, 16]
  DEVICE_MESH = np.arange(1024).reshape(DEVICE_MESH_SHAPE)


@model_registry.RegisterSingleTaskModel
class DenseLm175B8x8Decode2D(DenseLm175B32x32):
  """175B LM decoding on 128 devices with a 2-D logical mesh (ref :297): heads do not divide
  the device count, so both the model dim and the heads are sharded. Loads
  `DenseLm175B32x32` checkpoints."""
  BATCH_DIM_PER_DEVICE = 0.125
  NUM_DEVICES_PER_SPLIT = 128
  DEVICE_MESH_SHAPE = [8, 16]
  DEVICE_MESH = np.arange(128).reshape(DEVICE_MESH_SHAPE)

  def Task(self):
    p = super().Task()
    b = p.builder
    # packed relative positions are per example when decoding
    b.relative_attention_use_universal_1d_position = False
    b.model_dim_reshape_segments = self.DEVICE_MESH_SHAPE[0]
    b.emb_w_split = [1, 0]
    b.emb_out_split = [-1, -1, 0]
    b.blm_split = [-1, -1, 0]
    b.blh_split = [-1, -1, 1]
    b.qkv_split = [0, -1, 1, -1]
    b.logits_split = [-1, -1, 1]
    return p


@model_registry.RegisterSingleTaskModel
class DenseLM13B32x32(DenseLm128B16x16):
  """13B LM."""
  HIDDEN_DIM = 5120 * 4
  MODEL_DIM = 5120
  NUM_HEADS = 40
  NUM_TRANSFORMER_LAYERS = 40
  GATED_GELU = False


@model_registry.RegisterSingleTaskModel
class DenseLm1T16x16(DenseLm128B16x16):
  """1T params LM (~1.4k tokens/s on TPU v3-512)."""
  NUM_TRANSFORMER_LAYERS = 128
  HIDDEN_DIM = 131072
  MODEL_DIM = 16384
  NUM_HEADS = 256


@model_registry.RegisterSingleTaskModel
class DenseLm128B32x32(DenseLm128B16x16):
  """128B LM on v3-2048 (~62k tokens/s)."""
  NUM_DEVICES_PER_SPLIT = 2048
  BATCH_DIM_PER_DEVICE = 0.25
  DEVICE_MESH_SHAPE = [64, 32]
  DEVICE_MESH = np.arange(2048).reshape(DEVICE_MESH_SHAPE)


class ShardedAdamOptimizer(optimizer.Adam):
  """Adam whose slot variables inherit the variable sharding, with optional accumulation of
  `num_micro_batches` gradients before every update (reference :358-405)."""

  SLOT_SUFFIX = dict(getattr(optimizer.Adam, 'SLOT_SUFFIX', {}), grad_accum='grad_accum')
  COUNTER_ATTRS = tuple(getattr(optimizer.Adam, 'COUNTER_ATTRS', ())) + ('_micro_count',)

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('num_micro_batches', 1, 'Number of accumulated micro-batches per update.')
    return p

  def __init__(self, params):
    super().__init__(params)
    self._micro_count = 0

  def Apply(self, lr, var_grad, grad_scale=None):
    n = self.params.num_micro_batches
    if n <= 1:
      return super().Apply(lr, var_grad, grad_scale=grad_scale)
    pairs = optimizer._Pairs(var_grad)   # pylint: disable=protected-access
    with torch.no_grad():
      accs = [self._Slot(v, 'grad_accum') for v, _ in pairs]
      torch._foreach_add_(accs, optimizer._ScaledF32(pairs, grad_scale))   # pylint: disable=protected-access
    self._micro_count += 1
    if self._micro_count % n:
      return None
    with torch.no_grad():
      avg = torch._foreach_div(accs, float(n))
    super().Apply(lr, [py_utils.VarGrad(v, g) for (v, _), g in zip(pairs, avg)])
    with torch.no_grad():
      torch._foreach_zero_(accs)
    return None


@model_registry.RegisterSingleTaskModel
class DenseLm12kWide41BAdam16x16(DenseLm128B16x16):
  """41B LM with Adam (~53.8k tokens/s on TPU v3-512)."""
  MODEL_DIM = 12288
  HIDDEN_DIM = 12288 * 4
  NUM_HEADS = 96
  NUM_TRANSFORMER_LAYERS = 36
  GATED_GELU = False
  NUM_MICRO_BATCHES = 1

  def Task(self):
    p = super().Task()
    p.train.optimizer = ShardedAdamOptimizer.Params().Set(
        beta1=0.9, beta2=0.999, epsilon=1e-6, num_micro_batches=self.NUM_MICRO_BATCHES)
    p.train.learning_rate = 0.005
    return p


@model_registry.RegisterSingleTaskModel
class DenseLm12kWide41BAdam8x8(DenseLm12kWide41BAdam16x16):
  """41B LM, Adam, v3-128 (~17.4k tokens/s)."""
  NUM_DEVICES_PER_SPLIT = 128
  DEVICE_MESH_SHAPE = [8, 16]
  DEVICE_MESH = np.arange(128).reshape(DEVICE_MESH_SHAPE)


@model_registry.RegisterSingleTaskModel
class DenseLm12kWide162BAdam16x16(DenseLm12kWide41BAdam16x16):
  """162B LM, Adam, v3-512 (~12.5k tokens/s)."""
  NUM_TRANSFORMER_LAYERS = 144


@model_registry.RegisterSingleTaskModel
class DenseLm12kWide162BAdamBS25616x16(DenseLm12kWide162BAdam16x16):
  """Same model, global batch 256 as 4 micro-batches of 64 (ref :469)."""
  BATCH_DIM_PER_DEVICE = 0.125
  NUM_MICRO_BATCHES = 4


@model_registry.RegisterSingleTaskModel
class DenseLm12kWide162BAdam32x32(DenseLm12kWide162BAdam16x16):
  """162B LM, Adam, 2048 devices on a [64, 32] mesh (heads sharded 32 ways) (ref :481)."""
  TRAIN_STEPS_PER_LOOP = 20
  NUM_DEVICES_PER_SPLIT = 2048
  BATCH_DIM_PER_DEVICE = 0.125
  DEVICE_MESH_SHAPE = [64, 32]
  DEVICE_MESH = np.reshape(np.arange(2048), [32, 64]).transpose()


ShardedAdam = ShardedAdamOptimizer


class MoELmTemplate(DenseLmTemplate):
  """GShard MoE LM: [attn, moe, attn, ffw] × (L/2), top-2 gating."""
  NUM_EXPERTS = 8
  MOE_HIDDEN_DIM = 8192
  CAPACITY_FACTOR = 2.0
  GATED_GELU = False
  BATCH_SIZE_PER_GPU = 8
  AUX_LOSS_COEF = 0.01

  def _BatchSize(self):
    return self.BATCH_SIZE_PER_GPU

  def _Builder(self):
    b = super()._Builder()
    b.Set(e_dim=self.NUM_EXPERTS, c_dim=0,
          capacity_factor=self.CAPACITY_FACTOR,
          moe_hidden_dim=self.MOE_HIDDEN_DIM, moe_activation='RELU',
          second_expert_policy='all', gating_logits_dtype=torch.float32,
          mask_dtype=torch.float32, legacy_mtf_behavior=True)
    return b

  def Task(self):
    p = super().Task()
    p.moe = True
    p.aux_loss_coef = self.AUX_LOSS_COEF
    return p

  def Train(self):
    p = super().Train()
    p.random_ids = True
    p.vocab_size = self.VOCAB_SIZE
    p.random_seed = 1234
    return p


@model_registry.RegisterSingleTaskModel
class MoELm8E(MoELmTemplate):
  """The north-star benchmark model: GShard MoE LM with 8 experts.

  8 sub-layer pairs → 4 MoE + 4 dense FFN + 8 attention blocks; M = 2048,
  16 heads × 128, FFN/expert hidden 8192, vocab 32000, seq 1024, 8 sequences
  per GPU; experts are partitioned over the ranks (EP = min(world, 8)).
  ≈1.4 B parameters.
  """
  SEQUENCE_LENGTH = 1024
  MODEL_DIM = 2048
  HIDDEN_DIM = 8192
  MOE_HIDDEN_DIM = 8192
  NUM_HEADS = 16
  ATTENTION_KEY_VALUE_DIM = 128
  NUM_TRANSFORMER_LAYERS = 8
  NUM_EXPERTS = 8
  BATCH_SIZE_PER_GPU = 8
  TRAIN_STEPS_PER_LOOP = 20


@model_registry.RegisterSingleTaskModel
class MoELm8EKv4(MoELm8E):
  """MoELm8E with grouped-query attention: 16 query heads share 4 KV heads (wk, wv
  [2048, 512]), which makes the decoding KV cache 4x smaller."""
  NUM_KV_HEADS = 4


@model_registry.RegisterSingleTaskModel
class MoELm8ESoftCap(MoELm8E):
  """MoELm8E with the reference's attention options: the logits soft-capped at 50
  (cap·tanh(q·k / cap), before the relative bias) and an extra logit of 0 in every softmax.
  Both run inside our flash attention kernels."""
  ATTEN_LOGIT_CAP = 50.0
  ATTENTION_EXTRA_LOGIT = 0.0


@model_registry.RegisterSingleTaskModel
class MoELm8ETiny(MoELmTemplate):
  """Tiny MoE LM for tests / smoke runs."""
  SEQUENCE_LENGTH = 64
  MODEL_DIM = 64
  HIDDEN_DIM = 128
  MOE_HIDDEN_DIM = 128
  NUM_HEADS = 4
  ATTENTION_KEY_VALUE_DIM = 16
  NUM_TRANSFORMER_LAYERS = 2
  NUM_EXPERTS = 8
  BATCH_SIZE_PER_GPU = 4
  VOCAB_SIZE = 256
  TRAIN_STEPS_PER_LOOP = 2


@model_registry.RegisterSingleTaskModel
class DenseLmTiny(DenseLmTemplate):
  """Tiny dense LM for tests (data-parallel / ZeRO-Adam checks)."""
  SEQUENCE_LENGTH = 64
  MODEL_DIM = 64
  HIDDEN_DIM = 128
  NUM_HEADS = 4
  ATTENTION_KEY_VALUE_DIM = 16
  NUM_TRANSFORMER_LAYERS = 2
  VOCAB_SIZE = 256
  BATCH_DIM_PER_DEVICE = 4
  NUM_DEVICES_PER_SPLIT = 1
  DEVICE_MESH_SHAPE = [1, 1]
  TRAIN_STEPS_PER_LOOP = 2
  GATED_GELU = False
