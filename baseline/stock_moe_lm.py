"""Stock-PyTorch comparator for the headline benchmark (`bench.py --impl reference`).

tensorflow/lingvo itself cannot run in this image (no TensorFlow, no bazel, the
pip package refuses Python 3.12 — see DESIGN.md §7), so this file re-states the
*reference's own GPU code path* for the benchmark model with nothing but stock
library calls:

  * GShard MoE Transformer LM assembled like `gshard_builder_test.py:631-666`
    (`UniTransformer(moe=True)` + `DenseBuilder(e_dim=8, capacity_factor=2,
    moe_hidden_dim=8192)`): [attn, moe, attn, ffw] × 4, M = 2048, 16 × 128
    heads, T5 relative attention bias, RMS pre-norm, tied embedding/softmax;
  * top-2 gating and the **dense one-hot dispatch/combine einsums** the
    reference executes on GPUs (`gshard_layers.py:1932-2364` gating,
    `:3072-3086` `GSEC,GSM->EGCM`, `:3154-3158` `GSEC,GECM->GSM`);
  * `torch.matmul`/`einsum` (cuBLAS), `F.scaled_dot_product_attention`,
    `dist.all_to_all_single` for the expert exchange, `dist.all_reduce` for the
    replicated gradients, and an unfused Adafactor written with ordinary
    tensor ops (`optimizer.py:905-1218` semantics: factored second moment,
    parameter scale, update clipping, decay 1 - t^-0.8, beta1 = 0).

NOTHING from `lingvo_b200` is imported here: no kernels, no engine, no model.
bf16 compute with fp32 master weights, the same as the measured arm.
"""

from __future__ import annotations

import math
import os
import time

import torch
import torch.distributed as dist
import torch.nn.functional as F


class Config:
  vocab = 32000
  model_dim = 2048
  heads = 16
  head_dim = 128
  ff_dim = 8192
  moe_hidden = 8192
  experts = 8
  capacity_factor = 2.0
  layers = 8               # [attn, moe, attn, ffw] × layers/2
  seq_len = 1024
  batch = 8                # sequences per GPU
  rel_buckets = 32
  rel_max_distance = 128
  z_loss = 1e-4
  aux_loss_coef = 0.01
  label_smoothing = 0.0
  norm_eps = 1e-6
  # Adafactor (synthetic_packed_input.py:126-133)
  lr = 1.0
  warmup_steps = 10000
  decay_pow = 0.8
  clip_threshold = 1.0
  eps1 = 1e-30
  eps2 = 1e-3
  min_dim_size_to_factor = 128
  compute_dtype = torch.bfloat16


def _RelBucket(rel, num_buckets, max_distance):
  """T5 unidirectional bucket of key_pos - query_pos."""
  n = (-rel).clamp(min=0)
  max_exact = num_buckets // 2
  is_small = n < max_exact
  large = max_exact + (torch.log(n.float().clamp(min=1) / max_exact) /
                       math.log(max_distance / max_exact) *
                       (num_buckets - max_exact)).to(torch.int32)
  large = large.clamp(max=num_buckets - 1)
  return torch.where(is_small, n.to(torch.int32), large)


class _AllToAll(torch.autograd.Function):
  """Differentiable `dist.all_to_all_single` over dim 0 (equal splits)."""

  @staticmethod
  def forward(ctx, x, group, timer):
    ctx.group, ctx.timer = group, timer
    x = x.contiguous()
    out = torch.empty_like(x)
    if timer is not None:
      timer.Begin()
    dist.all_to_all_single(out, x, group=group)
    if timer is not None:
      timer.End()
    return out

  @staticmethod
  def backward(ctx, dy):
    dy = dy.contiguous()
    out = torch.empty_like(dy)
    if ctx.timer is not None:
      ctx.timer.Begin()
    dist.all_to_all_single(out, dy, group=ctx.group)
    if ctx.timer is not None:
      ctx.timer.End()
    return out, None, None


class A2ATimer:
  """CUDA-event brackets around every all-to-all (all on the compute stream ⇒ exposed)."""

  def __init__(self):
    self.pairs = []
    self.enabled = False

  def Begin(self):
    if self.enabled:
      e = torch.cuda.Event(enable_timing=True)
      e.record()
      self._e0 = e

  def End(self):
    if self.enabled:
      e = torch.cuda.Event(enable_timing=True)
      e.record()
      self.pairs.append((self._e0, e))

  def TotalMs(self):
    t = sum(a.elapsed_time(b) for a, b in self.pairs)
    self.pairs = []
    return t


class StockMoeLm:
  """Parameters are plain fp32 tensors; forward casts them to bf16 (theta cast)."""

  def __init__(self, cfg: Config, device, rank=0, world=1, seed=1234):
    self.cfg, self.dev, self.rank, self.world = cfg, device, rank, world
    self.ep = min(world, cfg.experts)
    self.e_local = cfg.experts // self.ep
    self.ep_group = None
    if world > cfg.experts:
      # consecutive EP groups of `experts` ranks; replicas of the experts across groups
      for g0 in range(0, world, cfg.experts):
        grp = dist.new_group(list(range(g0, g0 + cfg.experts)))
        if g0 <= rank < g0 + cfg.experts:
          self.ep_group = grp
    self.a2a_timer = A2ATimer()
    gen = torch.Generator(device='cpu').manual_seed(seed)
    m, h, d = cfg.model_dim, cfg.heads, cfg.head_dim
    P = {}

    def normal(shape, std):
      return (torch.randn(shape, generator=gen) * std).to(device)

    def uniform(shape, scale):
      return ((torch.rand(shape, generator=gen) * 2 - 1) * scale).to(device)

    P['emb'] = normal((cfg.vocab, m), 1.0)
    self.kinds = []
    for li in range(cfg.layers // 2):
      for kind in ('attn', 'moe', 'attn', 'ffw'):
        i = len(self.kinds)
        self.kinds.append(kind)
        P['l%d/ln' % i] = torch.ones(m, device=device)
        if kind == 'attn':
          P['l%d/wq' % i] = normal((m, h * d), (m * d)**-0.5)
          P['l%d/wk' % i] = normal((m, h * d), m**-0.5)
          P['l%d/wv' % i] = normal((m, h * d), m**-0.5)
          P['l%d/wo' % i] = normal((h * d, m), (h * d)**-0.5)
          P['l%d/wrb' % i] = normal((h, cfg.rel_buckets), 1.0)
        elif kind == 'ffw':
          P['l%d/wi' % i] = uniform((m, cfg.ff_dim), (3.0 / m)**0.5)
          P['l%d/wo' % i] = uniform((cfg.ff_dim, m), (3.0 / cfg.ff_dim)**0.5)
        else:
          P['l%d/gw' % i] = normal((m, cfg.experts), m**-0.5)
          wi = uniform((cfg.experts, m, cfg.moe_hidden), (3.0 / m)**0.5)
          wo = uniform((cfg.experts, cfg.moe_hidden, m), (3.0 / cfg.moe_hidden)**0.5)
          lo = (rank % self.ep) * self.e_local
          P['l%d/moe_wi' % i] = wi[lo:lo + self.e_local].contiguous()
          P['l%d/moe_wo' % i] = wo[lo:lo + self.e_local].contiguous()
    P['final_ln'] = torch.ones(m, device=device)
    self.params = {k: v.requires_grad_(True) for k, v in P.items()}
    self.expert_keys = {k for k in P if '/moe_w' in k}
    if world > 1:
      with torch.no_grad():
        for k, v in self.params.items():
          if k not in self.expert_keys:
            dist.broadcast(v, src=0)
    self.opt = StockAdafactor(cfg, self.params)
    self.step_count = 0

  # ------------------------------------------------------------------ layers --
  def _Rms(self, x, scale):
    xf = x.float()
    y = xf * torch.rsqrt(xf.square().mean(-1, keepdim=True) + self.cfg.norm_eps)
    return (y * scale).to(x.dtype)

  def _Attention(self, i, x, mask):
    cfg = self.cfg
    bsz, l, m = x.shape
    h, d = cfg.heads, cfg.head_dim
    p = self.params
    bf = x.dtype
    q = torch.matmul(x, p['l%d/wq' % i].to(bf)).view(bsz, l, h, d)
    k = torch.matmul(x, p['l%d/wk' % i].to(bf)).view(bsz, l, h, d)
    v = torch.matmul(x, p['l%d/wv' % i].to(bf)).view(bsz, l, h, d)
    # relative bias: one-hot bucket einsum of the reference (`HX,LJX->HLJ`)
    pos = torch.arange(l, device=x.device)
    bucket = _RelBucket(pos[None, :] - pos[:, None], cfg.rel_buckets,
                        cfg.rel_max_distance)
    onehot = F.one_hot(bucket.long(), cfg.rel_buckets).to(torch.float32)
    rb = torch.einsum('HX,LJX->HLJ', p['l%d/wrb' % i], onehot)
    bias = (mask + rb.unsqueeze(0)).to(bf)
    o = F.scaled_dot_product_attention(
        q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=bias,
        scale=1.0)
    o = o.transpose(1, 2).reshape(bsz, l, h * d)
    return torch.matmul(o, p['l%d/wo' % i].to(bf))

  def _Ffw(self, i, x):
    p = self.params
    hmid = F.relu(torch.matmul(x, p['l%d/wi' % i].to(x.dtype)))
    return torch.matmul(hmid, p['l%d/wo' % i].to(x.dtype))

  def _Top2Gating(self, logits, capacity):
    """GSE fp32 logits → combine GSEC (fp32), dispatch GSEC (bool), aux loss."""
    e = logits.shape[-1]
    raw = torch.softmax(logits, -1)
    idx1 = raw.argmax(-1)
    mask1 = F.one_hot(idx1, e).to(raw.dtype)
    gate1 = (raw * mask1).sum(-1)
    without1 = raw * (1.0 - mask1)
    idx2 = without1.argmax(-1)
    mask2 = F.one_hot(idx2, e).to(raw.dtype)
    gate2 = (without1 * mask2).sum(-1)
    denom = gate1 + gate2 + 1e-9           # legacy_mtf_behavior
    gate1, gate2 = gate1 / denom, gate2 / denom
    density1 = mask1.mean(1)
    proxy = raw.mean(1)
    aux = (proxy * density1).mean() * float(e * e)
    pos1 = (torch.cumsum(mask1, 1) - mask1) * mask1
    mask1 = mask1 * (pos1 < capacity).to(raw.dtype)
    count1 = mask1.sum(1, keepdim=True)
    pos2 = (torch.cumsum(mask2, 1) - mask2 + count1) * mask2
    mask2 = mask2 * (pos2 < capacity).to(raw.dtype)
    gate1 = gate1 * mask1.sum(-1)
    gate2 = gate2 * mask2.sum(-1)
    p1 = (pos1 * mask1).sum(-1).long()
    p2 = (pos2 * mask2).sum(-1).long()
    c1 = F.one_hot(p1, capacity).to(raw.dtype)
    c2 = F.one_hot(p2, capacity).to(raw.dtype)
    combine = (gate1[..., None, None] * mask1[..., :, None] * c1[..., None, :] +
               gate2[..., None, None] * mask2[..., :, None] * c2[..., None, :])
    return combine, combine != 0, aux

  def _Moe(self, i, x):
    cfg = self.cfg
    p = self.params
    g, s, m = x.shape            # one group per sequence
    e = cfg.experts
    cap = int(s * cfg.capacity_factor / e)
    logits = torch.matmul(x.float(), p['l%d/gw' % i])
    combine, dispatch, aux = self._Top2Gating(logits, cap)
    bf = x.dtype
    xe = torch.einsum('GSEC,GSM->EGCM', dispatch.to(bf), x)
    if self.ep > 1:
      xe = _AllToAll.apply(xe, self.ep_group, self.a2a_timer)       # [ep·E_l, G, C, M]
      xe = xe.view(self.ep, self.e_local, g, cap, m).transpose(0, 1)
    xe = xe.reshape(self.e_local, -1, m)
    hmid = F.relu(torch.bmm(xe, p['l%d/moe_wi' % i].to(bf)))
    ye = torch.bmm(hmid, p['l%d/moe_wo' % i].to(bf))
    if self.ep > 1:
      ye = ye.view(self.e_local, self.ep, g, cap, m).transpose(0, 1).reshape(
          e, g, cap, m)
      ye = _AllToAll.apply(ye, self.ep_group, self.a2a_timer)
    ye = ye.reshape(e, g, cap, m)
    y = torch.einsum('GSEC,EGCM->GSM', combine.to(bf), ye)
    return y, aux

  # -------------------------------------------------------------------- step --
  def Loss(self, ids, labels, segment_ids, segment_pos):
    cfg = self.cfg
    p = self.params
    bf = cfg.compute_dtype
    x = F.embedding(ids.long(), p['emb']).to(bf)
    a, c = segment_ids.unsqueeze(-1), segment_ids.unsqueeze(-2)
    not_vis = (a != c) | (segment_pos.unsqueeze(-1) < segment_pos.unsqueeze(-2))
    mask = (not_vis.float() * -1e9).unsqueeze(1)
    aux_total = torch.zeros((), device=x.device)
    for i, kind in enumerate(self.kinds):
      hn = self._Rms(x, p['l%d/ln' % i])
      if kind == 'attn':
        x = x + self._Attention(i, hn, mask)
      elif kind == 'ffw':
        x = x + self._Ffw(i, hn)
      else:
        y, aux = self._Moe(i, hn)
        x = x + y
        aux_total = aux_total + aux
    x = self._Rms(x, p['final_ln']) * (cfg.model_dim**-0.5)
    logits = torch.matmul(x, p['emb'].to(bf).t()).float()
    lse = torch.logsumexp(logits, -1)
    true_logit = logits.gather(-1, labels.long().unsqueeze(-1)).squeeze(-1)
    loss = lse - true_logit + cfg.z_loss * lse.square()
    nonpad = ((segment_ids != 0) & (labels > 0)).float()
    avg = (loss * nonpad).sum() / float(nonpad.numel())
    return avg + cfg.aux_loss_coef * aux_total

  def _SyncGrads(self):
    if self.world <= 1:
      return
    keys = [k for k in self.params if k not in self.expert_keys]
    grads = [self.params[k].grad for k in keys]
    flat = torch.cat([g.reshape(-1).to(torch.bfloat16) for g in grads])
    dist.all_reduce(flat)
    flat = flat.float().div_(self.world)
    off = 0
    for g in grads:
      n = g.numel()
      g.copy_(flat[off:off + n].view_as(g))
      off += n
    if self.world > self.cfg.experts:
      # expert replicas across EP groups (not used at ≤ 8 GPUs)
      raise NotImplementedError('world > experts')
    # Tokens of all ranks reach each expert: match the mean-reduced dense gradients.
    for k in self.expert_keys:
      self.params[k].grad.div_(self.world)

  def TrainStep(self, batch):
    """batch: dict of device int32 tensors `[B, L]`. Returns the loss (device scalar)."""
    for v in self.params.values():
      v.grad = None
    loss = self.Loss(batch['ids'], batch['labels'], batch['segment_ids'],
                     batch['segment_pos'])
    loss.backward()
    self._SyncGrads()
    self.step_count += 1
    self.opt.Step(self.step_count, ep_world=self.world if self.world > 1 else 1,
                  expert_keys=self.expert_keys)
    return loss.detach()


class StockAdafactor:
  """Unfused Adafactor (factored, beta1 = 0, parameter scaling, update clipping)."""

  def __init__(self, cfg: Config, params):
    self.cfg = cfg
    self.params = params
    self.state = {}
    for k, v in params.items():
      # factored second moment only when both factored dims are ≥ 128
      # (`min_dim_size_to_factor`, optimizer.py:905-1218)
      if v.dim() >= 2 and min(v.shape[-2:]) >= cfg.min_dim_size_to_factor:
        self.state[k] = (torch.zeros(v.shape[:-1], device=v.device),
                         torch.zeros(v.shape[:-2] + v.shape[-1:], device=v.device))
      else:
        self.state[k] = (torch.zeros_like(v),)

  def Step(self, t, ep_world=1, expert_keys=()):
    cfg = self.cfg
    lr = cfg.lr / math.sqrt(max(float(t), cfg.warmup_steps))
    decay = 1.0 - float(t)**(-cfg.decay_pow) if t > 1 else 0.0
    # global gradient norm + finiteness guard (learner.py:395-500 semantics)
    with torch.no_grad():
      norms = torch._foreach_norm([v.grad for v in self.params.values()])  # pylint: disable=protected-access
      sq = torch.stack(norms).square()
      if ep_world > 1:
        keys = list(self.params.keys())
        is_exp = torch.tensor([k in expert_keys for k in keys], device=sq.device)
        exp_sq = (sq * is_exp).sum()
        dist.all_reduce(exp_sq)
        gsq = (sq * ~is_exp).sum() + exp_sq
      else:
        gsq = sq.sum()
      ok = torch.isfinite(gsq).float()
      for k, v in self.params.items():
        g = v.grad * ok
        g2 = g.square() + cfg.eps1
        scale = torch.clamp(v.square().mean().sqrt(), min=cfg.eps2)
        st = self.state[k]
        if len(st) == 2:
          vr, vc = st
          vr.mul_(decay).add_(g2.mean(-1), alpha=1.0 - decay)
          vc.mul_(decay).add_(g2.mean(-2), alpha=1.0 - decay)
          r = (vr / vr.mean(-1, keepdim=True)).rsqrt().unsqueeze(-1)
          c = vc.rsqrt().unsqueeze(-2)
          u = g * r * c
        else:
          vv, = st
          vv.mul_(decay).add_(g2, alpha=1.0 - decay)
          u = g * vv.rsqrt()
        rms = u.square().mean().sqrt()
        u = u / torch.clamp(rms / cfg.clip_threshold, min=1.0)
        v.sub_(u * (lr * scale) * ok)


def SyntheticBatch(cfg: Config, step, rank, pin=True):
  """Uniform random token ids in the packed-input LM format (one segment per row)."""
  gen = torch.Generator().manual_seed(1234 * 1000003 + step + 7919 * rank)
  b, l = cfg.batch, cfg.seq_len
  labels = torch.randint(1, cfg.vocab, (b, l), generator=gen, dtype=torch.int32)
  pos = torch.arange(l, dtype=torch.int32).unsqueeze(0).expand(b, l).contiguous()
  out = {'ids': torch.roll(labels, 1, dims=1), 'labels': labels,
         'segment_ids': torch.ones(b, l, dtype=torch.int32), 'segment_pos': pos}
  if pin and torch.cuda.is_available():
    out = {k: v.pin_memory() for k, v in out.items()}
  return out


def RunBenchmark(args, clock_sampler_cls):
  """Same protocol as the measured arm: W warm-up steps, K device-timed steps, max over
  ranks; then K end-to-end steps with per-step pinned H2D + D2H loss read."""
  world = int(os.environ.get('WORLD_SIZE', '1'))
  rank = int(os.environ.get('RANK', '0'))
  local_rank = int(os.environ.get('LOCAL_RANK', '0'))
  torch.cuda.set_device(local_rank)
  dev = torch.device('cuda', local_rank)
  if world > 1:
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    dist.init_process_group('nccl', device_id=dev)
  torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = True
  cfg = Config()
  model = StockMoeLm(cfg, dev, rank, world)
  tokens_per_step = cfg.batch * cfg.seq_len * world

  def sync():
    if world > 1:
      dist.barrier()
    torch.cuda.synchronize()

  n_stage = min(args.warmup + args.steps, 8)
  staged = [{k: v.to(dev) for k, v in SyntheticBatch(cfg, i, rank).items()}
            for i in range(n_stage)]
  for i in range(args.warmup):
    model.TrainStep(staged[i % n_stage])
  sync()
  model.a2a_timer.enabled = True
  model.a2a_timer.pairs = []
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  with clock_sampler_cls(local_rank) as clocks:
    sync()
    e0.record()
    for i in range(args.steps):
      loss = model.TrainStep(staged[(args.warmup + i) % n_stage])
    e1.record()
    sync()
  ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
  a2a = torch.tensor([model.a2a_timer.TotalMs() / args.steps], device=dev)
  model.a2a_timer.enabled = False
  if world > 1:
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    dist.all_reduce(a2a, op=dist.ReduceOp.MAX)
  ms_total = float(ms.item())
  value = tokens_per_step * args.steps / (ms_total / 1e3)

  # end to end: fresh pinned host batch each step, H2D copy + D2H loss read in the region
  host = [SyntheticBatch(cfg, 1000 + i, rank) for i in range(args.steps + 2)]
  for i in range(2):
    model.TrainStep({k: v.to(dev, non_blocking=True) for k, v in host[i].items()})
  sync()
  t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  h2d = d2h = 0
  t0.record()
  for i in range(args.steps):
    hb = host[2 + i]
    batch = {k: v.to(dev, non_blocking=True) for k, v in hb.items()}
    h2d = sum(v.numel() * v.element_size() for v in hb.values())
    loss = model.TrainStep(batch)
    host_loss = loss.float().cpu()
    d2h = host_loss.numel() * host_loss.element_size()
  t1.record()
  sync()
  ems = torch.tensor([t0.elapsed_time(t1)], device=dev)
  if world > 1:
    dist.all_reduce(ems, op=dist.ReduceOp.MAX)
  out = None
  if rank == 0:
    out = {
        'metric': 'tokens/sec (whole job, device-timed, max over ranks) '
                  'GShard-MoE 8-expert LM training step',
        'value': value, 'unit': 'tokens/s', 'n_gpus': world, 'steps': args.steps,
        'warmup': args.warmup, 'ms_per_step': ms_total / args.steps,
        'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
        'dtype': 'bf16', 'data': 'synthetic (uniform random token ids, packed LM '
                                 'format; random-init weights)',
        'impl': 'reference',
        'reference_kind': 'stock PyTorch (cuBLAS matmul/einsum + SDPA + NCCL all_to_all/'
                          'all_reduce + unfused Adafactor) re-statement of the reference GPU '
                          'code path; TF lingvo itself is not installable here (no '
                          'TensorFlow/bazel; pip package requires Python < 3.11)',
        'config': {'model': 'lm.synthetic_packed_input.MoELm8E',
                   'global_batch': cfg.batch * world, 'seq_len': cfg.seq_len,
                   'parallelism': 'dp%d+ep%d' % (world, min(world, cfg.experts)),
                   'experts': cfg.experts, 'model_dim': cfg.model_dim,
                   'layers': cfg.layers, 'optimizer': 'Adafactor (unfused torch ops)',
                   'l2_flush': 'working set (1.4B fp32 params + activations) >> 50 MB '
                               'L2; no explicit flush'},
        'clocks': clocks.Summary(),
        'exposed_a2a_ms_per_step': float(a2a.item()),
        'gpu_launches': 0,
        'final_loss': float(loss),
        'e2e': {'value': tokens_per_step * args.steps / (float(ems.item()) / 1e3),
                'unit': 'tokens/s', 'h2d_bytes_per_step': int(h2d),
                'd2h_bytes_per_step': int(d2h)},
    }
  if world > 1:
    dist.barrier()
    torch.cuda.synchronize()
    dist.destroy_process_group()
  return out
