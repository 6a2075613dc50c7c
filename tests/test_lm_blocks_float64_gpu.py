"""The blocks of the MoELm8E step outside the MoE layer, run as the model wires them, stage by
stage against float64 written from the formulas: the LM head and loss (embedding lookup,
final norm, M^-0.5 scale, `_LmHeadXent`, `UniTransformer.ComputeLoss`), the attention block
(`DecoderBlock` with `SelfAttentionLayer`) and the dense FFN block (`DecoderBlock` with
`DenseReluDenseLayer`).

Contract of the head. For the decoder output h [T, M] (bf16), token ids and labels [T],
segment ids, the final norm's scale and the shared embedding E [V, M]:

    xs = rms_norm(h)·scale·M^-0.5 (zeroed where segment_id = 0 unless `all_valid`)
    l  = xs·Eᵀ,  lse = log Σ_v exp l_v,  soft_t = lse − ((on − off)·l_y + off·Σ_v l_v)
    loss = Σ_t (soft_t + z·lse_t²)·np_t / denom + aux_loss_coef·aux

with off = ls/V, on = 1 − ls + off for label smoothing ls, np_t = [segment_id ≠ 0 and
label > 0] and denom = T (`use_tgt_labels_size_as_loss_denominator`, the model's default) or
Σ np. mean_xent = Σ (lse − l_y)·np / Σ np, acc1 = Σ [argmax l = y]·np / Σ np. The gradient of
the shared embedding is the LM head's dW plus the lookup's Σ of the upstream rows per id.

Where the fused path rounds, and what is checked at each stage, from the stage's own recorded
inputs (every function is wrapped with `monkeypatch`; gshard_builder and ops/xent.py look them
up at call time):

    norm out   bf16 rms_norm: the bound of tests/test_norm_gpu.py (`_Oracle`, `_AssertBf16`)
    xs         bf16(norm·M^-0.5): correctly rounded up to 2u of the float64 product
    logits     the wgmma GEMM: the bound of tests/test_gemm_float64_gpu.py (`_Check`)
    lse        fp32 online softmax with __expf / __logf: within 2^-16·(1 + max|l|), the flash
               test's `_LSE_REL` form
    argmax     bitwise the first maximum of the recorded bf16 logits; on rows whose float64
               top two (of xs·Eᵀ) are further apart than twice the GEMM bound, the float64 one
    loss, mean_xent, soft xent, z increment: the masked means, from the recorded logits in
               float64; the kernel's lse error (bounded above) enters once, its fp32 Σ_v l_v
               with V·u·Σ|l|, and the fp32 arithmetic and token sums with T·u of the sum of
               |terms|. Per-token entropy and soft xent are not checked one by one here (the
               stats kernel's per-row values are, in tests/test_xent_gpu.py).
    a, b, c    the per-row coefficients handed to `xent_bwd`: a = d_soft + 2z·lse·d_z,
               b = off·d_soft, c = (on − off)·d_soft, d_soft = d_z = np/denom, each within 4u
    dlogits    bf16(exp(l − lse)·a − b − [v = y]·c) from the recorded l, lse, a, b, c: the
               result must be a correct rounding of some value within e of the float64 one,
               e = 2·(|p·a|·(|l − lse| + 5)·u + u·(|b| + |c|)) (the __expf argument and result
               error and the fp32 products). That window is far below one bf16 ulp, so a
               term of relative size 2^-9 — the z-loss gradient at z = 1e-4 — changes the
               rounding of a large share of the elements and fails it.
    dxs, dW    the GEMM bound, from the recorded dlogits, E and xs
    d norm out bf16(dxs·M^-0.5), correctly rounded up to 2u
    dh, dscale the norm backward's bound. The layers run on `theta`, the fp32 masters cast to
               bf16 (fprop_dtype), so `_NormFn` returns dscale in bf16 and the master gets
               that bf16 value: the bound plus ½ bf16 ulp, and a bf16-representable result.
    dE         `_EmbedRows` returns the fp32 lookup sum cast to the bf16 theta's dtype, and
               autograd adds it to the bf16 LM-head dW of the same theta tensor: the master
               gets bf16(bf16(lookup Σ) + dW), a bf16 value (asserted), within
               2·(½ ulp(Σ) + R·u·Σ|g| + ½ ulp(dE)) of lookup64 + dW
    daux       exactly aux_loss_coef in fp32

The head runs through `ComputePredictions` with every decoder block replaced by the identity,
so the stack's final norm, its padding mask and the M^-0.5 scale are the model's own code;
g, the gradient reaching the lookup, is recorded at the decoder input. Three cases at the
benchmark's shape (T 8192, M 2048, V 32000): `all_valid` with the benchmark's settings, packed
rows with trailing padding, and the smoothed case below; each has label-0 tokens, duplicate
ids, and 200 tokens a row labelled with the float64 argmax, so acc1 is far from 0.

Controls, each of which must fail the stage bound it targets (on the GPU in every head case, on
the CPU with a bf16 stand-in): the z-loss term dropped from a; label smoothing's b dropped (the
smoothed case); the other loss denominator (padded tokens counted, or not); the M^-0.5 scale
missing from the backward; the embedding gradient without its LM-head part, or without its
lookup part. The smoothed case uses ls = 0.1 and z = 0.05, so 2·z·lse ≈ 1 and every term of a,
b and c is of the same size as the others.

The attention block, at B 8, L 1024, M 2048, H 16 x 128 (`all_valid` as the benchmark runs,
and packed), grouped KV (Hk = 4, packed), L = 128 with B = 1 and L = 384. Each stage is checked
from the block's recorded bf16 values under the bound of the kernel's own test:

    x_in, norm out, dx   the norm test's bounds; dx with the residual stream's gradient
                         (`dres`), exactly 0 on padded tokens; dscale as for the head
    residual gradient    bitwise the block's upstream gradient
    qkv, dxn, dwqkv      the GEMM test's `_Check` for each projection GEMM; with grouped KV,
                         dxn is the bf16 sum of three dgrads: their bounds plus an ulp per add
    rel table            bitwise wrb gathered by the float64 T5 decoder buckets of query − key
    o, dq, dk, dv, d rel the flash test's `_Oracle` bounds (`_GqaOracle` for grouped KV)
    d wrb                the recorded d rel folded by bucket: within 2·(R·u·Σ|d rel| + ½ ulp)
                         of the float64 fold, a bf16 value
    y, d o, dwo          `_Check` with the residual added in the epilogue; d o bitwise the
                         flash kernel's upstream gradient

A padded token contributes exactly nothing: another input on the padded rows leaves every
weight gradient and dx bitwise unchanged. Controls: the k − q table differs from the recorded
one; k and v swapped (packed case) fail the o bound; the residual dropped or added twice fails
the y bound; dx without the residual stream's gradient fails the norm bound; d wrb folded into
the next bucket fails its bound.

The FFN block (M 2048, H 8192, `all_valid` and packed): the norm pass as above, the residual
gradient bitwise, and y = relu(xn·wi)·wo + x_in against float64 within the GEMM bound of y
plus the bf16 rounding of h (2^-8·|h|·|wo|) and its fp32 accumulation; the residual dropped
or added twice fails that bound.

Not covered here: an end-to-end comparison of each block against pure float64 (outputs and
weight gradients compared under one composed bound), and a check that the blocks chain
bitwise inside the two-layer model's `FProp`.

The float64 oracles (`_Bucket64`, `_AttnBlock64`, `_Head64`) never call the repository's layer
code; CPU tests check them against `RelativePositionBucket` (exactly, every distance at
L ∈ {128, 1024}), the layers' fp32 CPU path (`_Bias` + `_AttentionCore`) and the unfused
branch of `ComputeLoss`.

Measured on an H100 80GB HBM3 (700 W limit, 1980 MHz max SM clock), seeded so these repeat.
Worst err/bound per checked quantity ("0" is below 0.001):

              logits lse   loss,xents,z  a     b     c     dxs   dW    dE
    bench     0.498  0     0             0.240 0     0     0.471 0.492 0.500
    padded    0.498  0.007 0             0.240 0     0     0.471 0.492 0.500
    smoothed  0.498  0.007 0             0.275 0.001 0.126 0.481 0.494 0.500

              qkv   o     dv    dk    dq    d rel d wrb y     d o   dwo
    bench     0.485 0.451 0.489 0.270 0.109 0.022 0.497 0.498 0.485 0.419
    packed    0.485 0.451 0.478 0.255 0.112 0.042 0.498 0.497 0.485 0.418
    kv4       0.484 0.424 0.550 0.214 0.111 0.032 0.497 0.497 0.485 0.420
    one_block 0.479 0.397 0.461 0.159 0.116 0.034 0.494 0.491 0.472 0.499
    ragged    0.484 0.419 0.489 0.214 0.115 0.044 0.499 0.496 0.471 0.495
    FFN y     0.053 (bench), 0.052 (packed)

dlogits, xs and d norm out pass their rounding windows on every element, and every control
fails its bound. dE and d wrb sit at ½: their one bf16 rounding. The bf16 stand-in on the CPU
stays below 0.4 everywhere. The whole module takes ~30 s on the H100, with a peak of 30 GiB of
device memory.
"""
import math

import pytest
import torch

from lingvo_b200.core.nested_map import NestedMap

import test_flash_attn_gpu as TF
import test_flash_attn_gqa_gpu as TG
import test_gemm_float64_gpu as gemm64
import test_norm_gpu as N

_U = 2.0**-24              # fp32 unit roundoff
_U8 = 2.0**-8              # bf16 unit roundoff
_BUCKETS, _MAX_DISTANCE = 32, 128
_EPS = 1e-6


# ------------------------------------------------------------------ the oracles ----
def _Bucket64(qk):
  """T5 decoder bucket of the relative position query − key (one-directional): the exact
  offsets below 16, then 16 log-spaced buckets up to distance 128, clamped to bucket 31."""
  n = qk.double().clamp_min(0)
  exact = _BUCKETS // 2
  large = exact + torch.floor(torch.log(n.clamp_min(1) / exact) /
                              math.log(_MAX_DISTANCE / exact) * (_BUCKETS - exact))
  return torch.where(n < exact, n, large.clamp(max=_BUCKETS - 1)).long()


def _Rms64(x, scale):
  return x * torch.rsqrt((x * x).mean(-1, keepdim=True) + _EPS) * scale


def _Visible64(seg, pos, causal_shift=0):
  """[B, L, L]: query i sees key j iff same non-zero segment and pos_j ≤ pos_i."""
  same = (seg[:, :, None] == seg[:, None, :]) & (seg[:, :, None] != 0)
  return same & (pos[:, None, :] <= pos[:, :, None] + causal_shift)


def _AttnBlock64(x, scale, wq, wk, wv, wo, wrb, seg, pos, all_valid):
  """Float64 pre-norm decoder self-attention block with the T5 relative bias:
  x_in + softmax(q·kᵀ + bias + mask)·v·wo, x_in = x masked by segment_id ≠ 0."""
  b, l, m = x.shape
  h = wrb.shape[0]
  hk = wk.shape[1] * h // wq.shape[1]
  d = wq.shape[1] // h
  x_in = x if all_valid else x * (seg != 0)[..., None].to(x.dtype)
  xn = _Rms64(x_in, scale)
  q = (xn @ wq).view(b, l, h, d)
  k = (xn @ wk).view(b, l, hk, d).repeat_interleave(h // hk, 2)
  v = (xn @ wv).view(b, l, hk, d).repeat_interleave(h // hk, 2)
  i = torch.arange(l)
  bias = wrb[:, _Bucket64(i[:, None] - i[None, :])]                       # [H, L, L]
  s = torch.einsum('bqhd,bkhd->bhqk', q, k) + bias
  vis = _Visible64(seg, pos)[:, None]
  s = torch.where(vis, s, torch.full_like(s, -math.inf))
  p = torch.softmax(s, -1).nan_to_num(0.0)
  o = torch.einsum('bhqk,bkhd->bqhd', p, v).reshape(b, l, h * d)
  return x_in + o @ wo


def _Head64(h, scale, emb, ids, labels, seg, aux, g_emb, ls, z, coef, count_all,
            all_valid):
  """Float64 head and loss of the module docstring, with the upstream rows g_emb of the
  embedding lookup: returns the loss terms and metrics (the objective is loss + Σ emb·g)."""
  t, m = h.shape
  v = emb.shape[0]
  live = (seg != 0).to(h.dtype)[:, None]
  xn = _Rms64(h, scale)
  xs = (xn if all_valid else xn * live) * m**-0.5
  logits = xs @ emb.t()
  lse = torch.logsumexp(logits, -1)
  ly = logits.gather(-1, labels[:, None])[:, 0]
  off = ls / v
  on = 1.0 - ls + off
  soft = lse - ((on - off) * ly + off * logits.sum(-1))
  zinc = z * lse * lse
  npd = ((seg != 0) & (labels > 0)).to(h.dtype)
  denom = float(t) if count_all else npd.sum()
  loss = ((soft + zinc) * npd).sum() / denom + coef * aux
  rows = emb[ids]
  obj = loss + (rows * g_emb).sum()
  safe = npd.sum().clamp_min(1.0)
  return NestedMap(obj=obj, loss=loss, mean_xent=((lse - ly) * npd).sum() / safe,
                   soft_labels_xent=(soft * npd).sum() / safe,
                   avg_z=(zinc * npd).sum() / denom, logits=logits, npd=npd, denom=denom)


# ------------------------------------------------------------------- the model ----
def _Task(m=2048, heads=16, d=128, kv=None, ff=8192, vocab=32000, ls=0.0, z=1e-4,
          count_all=True, fprop=torch.bfloat16, seed=1):
  """The MoELm8E task cut to one attention/MoE and one attention/FFN pair, optionally at
  smaller dims, with the model's own weight init."""
  from lingvo_b200 import model_registry
  import lingvo_b200.models.lm.params.synthetic_packed_input  # noqa: F401
  tp = model_registry.GetParams('lm.synthetic_packed_input.MoELm8E', 'Train').task
  tp.num_transformer_layers = 2
  tp.random_seed = seed
  tp.builder.Set(model_dim=m, attention_num_heads=heads, attention_key_value_dim=d,
                 attention_num_memory_heads=kv, ff_dim=ff, moe_hidden_dim=ff)
  tp.vocab_size = vocab
  tp.label_smoothing = ls
  tp.z_loss = z
  tp.use_tgt_labels_size_as_loss_denominator = count_all
  tp.fprop_dtype = fprop
  tp.builder.fprop_dtype = fprop
  return tp.Instantiate()


def _Packed(b, l, seed):
  """seg / pos [b, l]: three unequal segments per row and trailing padding."""
  gen = torch.Generator().manual_seed(seed)
  seg = torch.zeros(b, l, dtype=torch.int32)
  pos = torch.zeros(b, l, dtype=torch.int32)
  for bi in range(b):
    cuts = sorted(torch.randint(1, l - 8, (3,), generator=gen).tolist())
    bounds = [0, cuts[0], cuts[1] + 1, cuts[2] + 2]
    for si in range(3):
      s, e = bounds[si], min(bounds[si + 1], l)
      seg[bi, s:e] = si + 1
      pos[bi, s:e] = torch.arange(e - s, dtype=torch.int32)
  return seg, pos


# ------------------------------------------------------------------ CPU checks ----
@pytest.mark.parametrize('l', [128, 1024])
def test_bucket_oracle_equals_the_model_bucket_at_every_distance(l):
  from lingvo_b200.core.gshard_builder import RelativePositionBucket
  qk = torch.arange(-(l - 1), l)
  got = RelativePositionBucket(-qk, _BUCKETS, _MAX_DISTANCE, bidirectional=False)
  assert torch.equal(got.long(), _Bucket64(qk))


def _SmallBatch(b, l, vocab, seed):
  gen = torch.Generator().manual_seed(seed)
  seg, pos = _Packed(b, l, seed)
  ids = torch.randint(1, vocab, (b, l), generator=gen)
  labels = torch.randint(0, vocab, (b, l), generator=gen) * (seg != 0)
  return seg, pos, ids, labels, gen


def test_attention_oracle_matches_the_layer_fp32_path():
  """`DecoderBlock` + `SelfAttentionLayer` in fp32 on the CPU (`_Bias` + `_AttentionCore`)
  against `_AttnBlock64`: output and every gradient, packed rows, grouped KV heads."""
  for kv in (None, 2):
    task = _Task(m=64, heads=4, d=16, kv=kv, ff=128, vocab=256, fprop=torch.float32)
    blk = task.dec.layers[0]
    b, l = 2, 160
    seg, pos, _, _, gen = _SmallBatch(b, l, 256, 3)
    x = torch.randn(b, l, 64, generator=gen, requires_grad=True)
    live = (seg != 0)[..., None]
    dy = torch.randn(b, l, 64, generator=gen) * live     # the model's upstream is 0 there
    out = blk.FProp(blk.theta, NestedMap(vec=x, segment_id=seg, segment_pos=pos,
                                         aux_loss=torch.zeros(()), all_valid=False))
    th = blk.vars
    leaves = [th.ln.scale, th.layer.wq, th.layer.wk, th.layer.wv, th.layer.wo, th.layer.wrb]
    got = torch.autograd.grad((out.vec * dy).sum(), [x] + leaves)
    w64 = [t.detach().double().requires_grad_() for t in [x] + leaves]
    y64 = _AttnBlock64(*w64, seg, pos, False)
    want = torch.autograd.grad((y64 * dy.double()).sum(), w64)
    # A padded query's output is unspecified (the layer averages every key there).
    torch.testing.assert_close((out.vec * live).double(), y64 * live, rtol=1e-4, atol=1e-4)
    for name, g, w in zip(['x', 'scale', 'wq', 'wk', 'wv', 'wo', 'wrb'], got, want):
      torch.testing.assert_close(g.double(), w, rtol=1e-4, atol=1e-4, msg=name)


def _RunHead(task, ids, labels, seg, pos, h, aux, g_emb):
  theta = task.theta
  emb = task.dec_emb.FProp(theta.dec_emb, ids)
  x = task.dec.final_layer_norm.FProp(theta.dec.final_layer_norm, h)
  x = x * (seg != 0)[..., None].to(x.dtype)
  pred = NestedMap(dec_outputs=x * task.params.builder.model_dim**-0.5, aux_loss=aux)
  batch = NestedMap(tgt=NestedMap(ids=ids, labels=labels, segment_ids=seg, segment_pos=pos))
  metrics, _ = task.ComputeLoss(theta, pred, batch)
  (metrics['loss'][0] + (emb * g_emb).sum()).backward()
  return metrics


@pytest.mark.parametrize('ls,z,count_all', [(0.0, 1e-4, True), (0.1, 0.05, False)])
def test_head_oracle_matches_the_unfused_compute_loss(ls, z, count_all):
  """The unfused fp32 branch of `ComputeLoss` with the embedding lookup and the final norm
  against `_Head64`: loss, metrics and the gradients of h, scale, embedding and aux."""
  b, l, m, v = 2, 96, 64, 256
  task = _Task(m=m, heads=4, d=16, ff=128, vocab=v, ls=ls, z=z, count_all=count_all,
               fprop=torch.float32)
  seg, pos, ids, labels, gen = _SmallBatch(b, l, v, 5)
  ids[0, :8] = 7                                                   # duplicate ids
  h = torch.randn(b, l, m, generator=gen, requires_grad=True)
  aux = torch.tensor(0.37, requires_grad=True)
  g_emb = torch.randn(b, l, m, generator=gen) * (seg != 0)[..., None]
  metrics = _RunHead(task, ids, labels, seg, pos, h, aux, g_emb)
  th = task.vars
  leaves = [h, th.dec.final_layer_norm.scale, th.dec_emb.embedding, aux]
  w64 = [t.detach().double().requires_grad_() for t in leaves]
  o = _Head64(w64[0].reshape(-1, m), w64[1], w64[2], ids.reshape(-1), labels.reshape(-1),
              seg.reshape(-1), w64[3], g_emb.double().reshape(-1, m), ls, z, 0.01, count_all,
              False)
  o.obj.backward()
  for name in ('loss', 'mean_xent', 'soft_labels_xent'):
    torch.testing.assert_close(metrics[name][0].double(), o[name].detach(), rtol=1e-5,
                               atol=1e-6, msg=name)
  torch.testing.assert_close(metrics['avg_z_loss_increment'][0].double(), o.avg_z.detach(),
                             rtol=1e-5, atol=1e-7)
  for name, g, w in zip(['h', 'scale', 'emb', 'aux'], leaves, w64):
    torch.testing.assert_close(g.grad.double(), w.grad, rtol=1e-4, atol=1e-6, msg=name)


# ------------------------------------------------------------ head stage checks ----
def _Within(got, ref, e):
  """bf16 `got` is a round-to-nearest of some value within e of the float64 ref."""
  lo = (ref - e).to(torch.bfloat16).double()
  hi = (ref + e).to(torch.bfloat16).double()
  g = got.double()
  return (g >= lo) & (g <= hi)


def _Coefs64(rec, z=None, ls=None, denom=None):
  """Float64 a, b, c of `xent_bwd` from the recorded lse (the controls pass other z, ls or
  denominators)."""
  z = rec.z if z is None else z
  ls = rec.ls if ls is None else ls
  denom = rec.denom if denom is None else denom
  off = ls / rec.v
  on = 1.0 - ls + off
  d = rec.npd / denom
  lse = rec.lse.double()
  return d * (1.0 + 2.0 * z * lse), d * off, d * (on - off)


def _DLogits64(rec, a, b, c):
  x = rec.logits.double() - rec.lse.double()[:, None]
  pa = torch.exp(x) * a[:, None]
  ref = pa - b[:, None]
  ref.scatter_add_(1, rec.labels[:, None], -c[:, None])
  cy = torch.zeros_like(ref).scatter_(1, rec.labels[:, None], c.abs()[:, None])
  e = 2 * (pa.abs() * (x.abs() + 5) * _U + _U * (b.abs()[:, None] + cy)) + 2 * _U * ref.abs()
  return ref, e


def _LossRefs(rec, denom=None, z=None):
  """Float64 loss and metrics from the recorded bf16 logits, and their bounds."""
  denom = rec.denom if denom is None else denom
  z = rec.z if z is None else z
  l64 = rec.logits.double()
  v = rec.v
  off = rec.ls / v
  on = 1.0 - rec.ls + off
  lse = torch.logsumexp(l64, -1)
  ly = l64.gather(-1, rec.labels[:, None])[:, 0]
  lsum = l64.sum(-1)
  d_lse = TF._LSE_REL * (1 + l64.abs().amax(-1))
  d_sum = v * _U * l64.abs().sum(-1)
  soft = lse - ((on - off) * ly + off * lsum)
  zinc = z * lse * lse
  e_soft = d_lse + off * d_sum + 4 * _U * (lse.abs() + ly.abs() + off * lsum.abs())
  e_z = 2 * z * lse.abs() * d_lse + 3 * _U * zinc
  npd, t = rec.npd, l64.shape[0]
  safe = max(float(npd.sum()), 1.0)

  def Mean(val, err, den):
    return (val * npd).sum() / den, ((err + t * _U * val.abs()) * npd).sum() / den

  out = {}
  loss, e = Mean(soft + zinc, e_soft + e_z, denom)
  out['loss'] = (loss + rec.coef * rec.aux, e + 2 * _U * (abs(rec.coef * rec.aux) + loss.abs()))
  out['mean_xent'] = Mean(lse - ly, d_lse + 2 * _U * (lse.abs() + ly.abs()), safe)
  out['soft_labels_xent'] = Mean(soft, e_soft, safe)
  out['avg_z_loss_increment'] = Mean(zinc, e_z, denom)
  return out


def _HeadStages(rec, metrics):
  """Asserts the loss, coefficient and dlogits stages; returns the worst err/bound of each."""
  res = {}
  for name, (ref, bound) in _LossRefs(rec).items():
    err = abs(float(metrics[name][0]) - float(ref))
    assert err <= float(bound), '%s: err %g bound %g' % (name, err, float(bound))
    res[name] = err / float(bound)
  for name, got, ref in zip('abc', (rec.a, rec.b, rec.c), _Coefs64(rec)):
    err = (got.double() - ref).abs()
    bound = 4 * _U * ref.abs()
    assert bool((err <= bound).all()), 'coefficient %s: %d rows outside 4u' % (
        name, int((err > bound).sum()))
    res[name] = float(torch.where(err > 0, err / bound, torch.zeros_like(err)).max())
  ref, e = _DLogits64(rec, *_Coefs64(rec))
  ok = _Within(rec.dlogits, ref, e)
  assert bool(ok.all()), 'dlogits: %d elements are no rounding of the float64 value' % int(
      (~ok).sum())
  return res


def _HeadControls(rec, metrics):
  """(name, rejected) of the head's controls."""
  out = []
  other = float(rec.npd.numel()) if rec.denom != float(rec.npd.numel()) else float(
      rec.npd.sum())
  ref, bound = _LossRefs(rec, denom=other)['loss']
  out.append(('the other denominator (loss)',
              abs(float(metrics['loss'][0]) - float(ref)) > float(bound)))
  a_ok = _Coefs64(rec)[0]
  out.append(('the other denominator (a)', bool(
      ((rec.a.double() - _Coefs64(rec, denom=other)[0]).abs() > 4 * _U * a_ok.abs()).any())))
  a_noz = _Coefs64(rec, z=0.0)[0]
  out.append(('z-loss dropped from a', bool(
      ((rec.a.double() - a_noz).abs() > 4 * _U * a_ok.abs()).any())))
  a, b, c = _Coefs64(rec)
  ref, e = _DLogits64(rec, a_noz, b, c)
  out.append(('z-loss dropped from dlogits', not bool(_Within(rec.dlogits, ref, e).all())))
  if rec.ls:
    ref, e = _DLogits64(rec, a, torch.zeros_like(b), c)
    out.append(('b dropped from dlogits', not bool(_Within(rec.dlogits, ref, e).all())))
  return out


def _EmbGrad(got, dw_head, ids, g_emb, v, lookup=True, head=True):
  """(err/bound worst, rejected?) of the embedding's master gradient against
  lookup64 + dW_head (either part may be left out for the controls)."""
  m = g_emb.shape[-1]
  look = torch.zeros(v, m, dtype=torch.float64, device=g_emb.device)
  look.index_add_(0, ids, g_emb.double())
  absum = torch.zeros_like(look).index_add_(0, ids, g_emb.double().abs())
  cnt = torch.zeros(v, dtype=torch.float64, device=g_emb.device).index_add_(
      0, ids, torch.ones_like(ids, dtype=torch.float64))
  ref = (look if lookup else 0.0) + (dw_head.double() if head else 0.0)
  g = got.double()
  bound = 2 * (0.5 * gemm64._Ulp(look) * (look != 0) + cnt[:, None] * _U * absum +
               0.5 * gemm64._Ulp(torch.maximum(ref.abs(), g.abs())))
  err = (g - ref).abs()
  return float((err / bound).max()), bool((err > bound).any())


# ---------------------------------------------------------- the bf16 stand-in ----
def _Bf(t):
  return t.to(torch.bfloat16)


def _StandInHead(xs, emb, labels, npd, ls, z, coef, aux, count_all):
  """The fused head's arithmetic in float64, rounded where the kernels round: bf16 logits,
  fp32 statistics and coefficients, bf16 dlogits."""
  t = xs.shape[0]
  v = emb.shape[0]
  logits = _Bf(xs.double() @ emb.double().t())
  l32 = logits.float()
  lse = torch.logsumexp(l32, -1)
  ly = l32.gather(-1, labels[:, None])[:, 0]
  off = ls / v
  on = 1.0 - ls + off
  soft = lse - ((on - off) * ly + off * l32.sum(-1))
  zinc = z * lse * lse
  np32 = npd.float()
  denom = float(t) if count_all else np32.sum()
  loss = ((soft + zinc) * np32).sum() / denom + coef * aux
  safe = np32.sum().clamp_min(1.0)
  metrics = {'loss': (loss, None), 'mean_xent': (((lse - ly) * np32).sum() / safe, None),
             'soft_labels_xent': ((soft * np32).sum() / safe, None),
             'avg_z_loss_increment': ((zinc * np32).sum() / denom, None)}
  d = np32 * (1.0 / torch.as_tensor(denom, dtype=torch.float32))
  a = d + d * (2.0 * z) * lse
  b = d * off
  c = d * (on - off)
  dl = torch.exp(l32 - lse[:, None]) * a[:, None] - b[:, None]
  dl.scatter_add_(1, labels[:, None], -c[:, None])
  rec = NestedMap(logits=logits, labels=labels, lse=lse, a=a, b=b, c=c, dlogits=_Bf(dl),
                  npd=npd.double(), denom=float(denom), v=v, ls=ls, z=z, coef=coef, aux=aux)
  return rec, metrics


@pytest.mark.parametrize('ls,z,count_all', [(0.0, 1e-4, True), (0.1, 0.05, False)],
                         ids=['bench', 'smoothed'])
def test_head_bounds_pass_the_stand_in_and_reject_the_controls(ls, z, count_all):
  t, m, v = 512, 64, 1024
  gen = torch.Generator().manual_seed(9)
  seg, _, ids, labels, gen = _SmallBatch(1, t, v, 13)
  seg, ids, labels = seg[0], ids[0], labels[0]
  labels[:5] = 0
  npd = ((seg != 0) & (labels > 0))
  xs = _Bf(torch.randn(t, m, generator=gen) * m**-0.5 * (seg != 0)[:, None])
  emb = _Bf(torch.randn(v, m, generator=gen))
  rec, metrics = _StandInHead(xs, emb, labels, npd, ls, z, 0.01, 0.3, count_all)
  res = _HeadStages(rec, metrics)
  print('stand-in', {k: round(x, 3) for k, x in res.items()})
  missed = [n for n, rejected in _HeadControls(rec, metrics) if not rejected]
  assert not missed, missed
  # the embedding gradient: bf16(bf16(lookup) + dW) passes, either part alone fails
  g_emb = _Bf(torch.randn(t, m, generator=gen) * (seg != 0)[:, None])
  dw = _Bf(rec.dlogits.double().t() @ xs.double())
  look = torch.zeros(v, m).index_add_(0, ids, g_emb.float())
  got = (_Bf(look) + dw).float()
  assert not _EmbGrad(got, dw, ids, g_emb, v)[1]
  assert _EmbGrad(got, dw, ids, g_emb, v, lookup=False)[1]
  assert _EmbGrad(got, dw, ids, g_emb, v, head=False)[1]


# ------------------------------------------------------------------- GPU: head ----
class _HeadSpy:
  """Records the final norm, the LM head's GEMMs, the stats and `xent_bwd`'s operands."""

  def __init__(self, monkeypatch):
    from lingvo_b200 import ops
    from lingvo_b200.ops import gemm, norm, xent
    self.gemms, self.norms, self.stats, self.bwd = [], [], [], []
    real_gemm, real_norm, real_xent = gemm.gemm, norm.rms_norm, xent.lm_head_xent
    nat = ops.native()
    real_bwd = nat.xent_bwd

    def Gemm(*args, **kw):
      out = real_gemm(*args, **kw)
      self.gemms.append((args, out.clone()))
      return out

    def Norm(x, scale, eps):
      y = real_norm(x, scale, eps)
      rec = NestedMap(x=x.detach(), scale=scale.detach(), y=y.detach())
      y.register_hook(lambda g: rec.update(dy=g.detach().clone()))
      self.norms.append(rec)
      return y

    def Xent(*args, **kw):
      st = real_xent(*args, **kw)
      self.stats.append(st)
      return st

    def Bwd(logits, labels, lse, a, b, c):
      rec = NestedMap(logits=logits.clone(), lse=lse.clone(), a=a.clone(), b=b.clone(),
                      c=c.clone())
      real_bwd(logits, labels, lse, a, b, c)
      rec.dlogits = logits.clone()
      self.bwd.append(rec)
    monkeypatch.setattr(gemm, 'gemm', Gemm)
    monkeypatch.setattr(norm, 'rms_norm', Norm)
    monkeypatch.setattr(xent, 'lm_head_xent', Xent)
    monkeypatch.setattr(nat, 'xent_bwd', Bwd)


_HEAD_CASES = [('bench', 0.0, 1e-4, True, True), ('padded', 0.0, 1e-4, True, False),
               ('smoothed', 0.1, 0.05, False, False)]


def _RunModelHead(task, ids, labels, seg, pos, aux, all_valid, monkeypatch):
  """`ComputePredictions` and `ComputeLoss` of the task with every decoder block replaced by
  the identity, so that the embedding output is the stack's output: the lookup, the stack's
  final norm and padding mask and the M^-0.5 scale all run the model's own code. The first
  block adds `aux` to the aux loss and records the decoder input h and its gradient."""
  from lingvo_b200.core import gshard_builder
  rec = NestedMap()

  def Identity(self, theta, i):
    o = i.copy()
    if 'h' not in rec:
      rec.h = i.vec.detach()
      i.vec.register_hook(lambda g: rec.update(dh=g.detach().clone()))
      o.aux_loss = i.aux_loss + aux
    return o
  monkeypatch.setattr(gshard_builder.DecoderBlock, 'FProp', Identity)
  theta = task.theta
  batch = NestedMap(tgt=NestedMap(ids=ids, labels=labels, segment_ids=seg, segment_pos=pos,
                                  all_valid=all_valid))
  pred = task.ComputePredictions(theta, batch)
  metrics, _ = task.ComputeLoss(theta, pred, batch)
  metrics['loss'][0].backward()
  return metrics, rec


@pytest.mark.gpu
@pytest.mark.parametrize('case', _HEAD_CASES, ids=[c[0] for c in _HEAD_CASES])
def test_head_against_float64(case, monkeypatch):
  """Embedding lookup, final norm, M^-0.5, fused LM head and `ComputeLoss` at the benchmark's
  shape (T 8192, M 2048, V 32000): `all_valid` as the benchmark runs, and packed rows with
  trailing padding; label-0 tokens, duplicate ids, and labels set to the float64 argmax on a
  share of the tokens. Every stage of the module docstring, and the controls."""
  name, ls, z, count_all, all_valid = case
  dev = torch.device('cuda', torch.cuda.current_device())
  b, l, m, v = 8, 1024, 2048, 32000
  task = _Task(ls=ls, z=z, count_all=count_all).to(dev)
  seg, pos, ids, labels, gen = _SmallBatch(b, l, v, 21)
  if all_valid:
    seg = torch.ones(b, l, dtype=torch.int32)
    pos = torch.arange(l, dtype=torch.int32).expand(b, l).contiguous()
    labels = torch.randint(1, v, (b, l), generator=gen)
  ids[:, :64] = ids[:, :1]                                          # duplicate ids
  labels[:, 100:110] = 0                                            # live tokens with label 0
  seg, pos, ids, labels = (t.to(dev) for t in (seg, pos, ids, labels))
  live = (seg != 0)[..., None]
  with torch.no_grad():                      # labels = the float64 argmax on 200 tokens a row
    th = task.theta
    x64 = _Rms64(th.dec_emb.embedding[ids].double(), th.dec.final_layer_norm.scale.double())
    l64 = (x64 * live * m**-0.5).reshape(-1, m) @ th.dec_emb.embedding.double().t()
    top = l64.argmax(-1).view(b, l)
    labels[:, 200:400] = torch.where(seg[:, 200:400] != 0, top[:, 200:400], 0)
    del x64, l64, th
  aux = torch.tensor(0.3, device=dev, requires_grad=True)
  spy = _HeadSpy(monkeypatch)
  metrics, hr = _RunModelHead(task, ids, labels, seg, pos, aux, all_valid, monkeypatch)
  monkeypatch.undo()
  g_emb = hr.dh
  assert len(spy.stats) == 1 and len(spy.bwd) == 1, 'the fused LM head did not run'
  assert len(spy.gemms) == 3 and len(spy.norms) == 1, (len(spy.gemms), len(spy.norms))
  (xs, emb_b, _, _), logits = spy.gemms[0]
  (dl_in, _, _, _), dxs = spy.gemms[1]
  (_, xs2, _, _), dw_head = spy.gemms[2]
  bw = spy.bwd[0]
  nrec = spy.norms[0]
  t = b * l
  labels_f = labels.reshape(-1)
  npd = ((seg != 0) & (labels > 0)).reshape(-1)
  res = {}
  # final norm, xs, logits
  o = N._Oracle(nrec.x.reshape(t, m), None, nrec.scale.float(), None, False)
  N._AssertBf16(nrec.y.reshape(t, m), o['y'], o['slack_y'] + N._Ulp(o['y']), 'norm out')
  xs_ref = nrec.y.reshape(t, m).double() * live.reshape(t, 1) * m**-0.5
  assert bool(_Within(xs, xs_ref, 2 * _U * xs_ref.abs()).all()), 'xs'
  res['logits'] = gemm64._Check(logits, xs, emb_b, True, True, what='logits')[0]
  assert torch.equal(gemm64._Bits(bw.logits), gemm64._Bits(logits))
  # lse and argmax
  l64 = logits.double()
  lse64 = torch.logsumexp(l64, -1)
  d_lse = TF._LSE_REL * (1 + l64.abs().amax(-1))
  res['lse'] = float(((bw.lse.double() - lse64).abs() / d_lse).max())
  assert res['lse'] <= 1.0, res['lse']
  amax = spy.stats[0].argmax
  assert torch.equal(amax, logits.argmax(-1)), 'argmax of the bf16 logits'
  s64 = xs.double() @ emb_b.double().t()
  top = s64.topk(2, -1).values
  kk = math.ceil(m / 16) + 16
  p_abs = (xs.double().abs() @ emb_b.double().abs().t()).amax(-1)
  clear = (top[:, 0] - top[:, 1]) > 2 * gemm64._C * (
      gemm64._Ulp(top[:, 0]) + kk * gemm64._U_ACC * p_abs)
  assert float(clear.double().mean()) > 0.3
  assert torch.equal(amax[clear], s64.argmax(-1)[clear]), 'argmax on clear rows'
  acc1 = float(((amax == labels_f) & npd).double().sum() / max(1, int(npd.sum())))
  assert acc1 > 0.1, acc1
  assert abs(float(metrics['acc1'][0]) - acc1) <= 4 * _U * acc1
  del s64, l64
  # loss, coefficients, dlogits
  rec = NestedMap(logits=logits, labels=labels_f, lse=bw.lse, a=bw.a, b=bw.b, c=bw.c,
                  dlogits=bw.dlogits, npd=npd.double(),
                  denom=float(t) if count_all else float(npd.sum()), v=v, ls=ls, z=z,
                  coef=task.params.aux_loss_coef, aux=float(aux.detach()))
  res.update(_HeadStages(rec, metrics))
  assert torch.equal(gemm64._Bits(dl_in), gemm64._Bits(bw.dlogits))
  # dxs, dW, d norm out, dh, dscale, dE, daux
  res['dxs'] = gemm64._Check(dxs, bw.dlogits, emb_b, True, False, what='dxs')[0]
  res['dW'] = gemm64._Check(dw_head, bw.dlogits, xs2, False, False, what='dW')[0]
  dxn_ref = dxs.double() * m**-0.5 * live.reshape(t, 1)
  dxn = nrec.dy.reshape(t, m)
  assert bool(_Within(dxn, dxn_ref, 2 * _U * dxn_ref.abs()).all()), 'd norm out'
  o = N._Oracle(nrec.x.reshape(t, m), dxn, nrec.scale.float(), None, False)
  assert torch.equal(gemm64._Bits(nrec.x), gemm64._Bits(hr.h))
  N._AssertBf16(hr.dh.reshape(t, m), o['dx'], o['slack_dx'] + N._Ulp(o['dx']), 'dh')
  _AssertScaleGrad(task.vars.dec.final_layer_norm.scale, o, name)
  # the embedding master gets bf16(bf16(lookup) + dW): a bf16 value
  g = task.vars.dec_emb.embedding.grad
  assert torch.equal(g, g.bfloat16().float()), 'dE is not a bf16 value'
  res['dE'], bad = _EmbGrad(task.vars.dec_emb.embedding.grad, dw_head, ids.reshape(-1),
                            g_emb.reshape(t, m), v)
  assert not bad, 'embedding gradient: worst err/bound %g' % res['dE']
  assert float(aux.grad) == float(torch.tensor(task.params.aux_loss_coef, dtype=torch.float32))
  # controls
  missed = [n for n, rejected in _HeadControls(rec, metrics) if not rejected]
  if bool(_Within(dxn, dxs.double() * live.reshape(t, 1), 2 * _U * dxn_ref.abs()).all()):
    missed.append('M^-0.5 missing from the backward')
  for kw, what in ((dict(lookup=False), 'lookup part'), (dict(head=False), 'LM-head part')):
    if not _EmbGrad(task.vars.dec_emb.embedding.grad, dw_head, ids.reshape(-1),
                    g_emb.reshape(t, m), v, **kw)[1]:
      missed.append('embedding gradient without its ' + what)
  assert not missed, '%s: the bounds do not reject: %s' % (name, ', '.join(missed))
  print('%s: %s' % (name, ' '.join('%s %.3f' % kv for kv in res.items())))


@pytest.mark.gpu
def test_second_backward_through_the_lm_head_raises():
  """xent_bwd overwrites the saved logits with dlogits: a second backward through a retained
  graph must raise, and the first one's gradients must be those of a fresh run."""
  from lingvo_b200.ops import xent
  dev = torch.device('cuda', torch.cuda.current_device())
  gen = torch.Generator(device=dev).manual_seed(5)
  x0 = torch.randn(256, 512, device=dev, generator=gen).to(torch.bfloat16)
  w0 = torch.randn(2048, 512, device=dev, generator=gen).to(torch.bfloat16) * 0.05
  labels = torch.randint(0, 2048, (256,), device=dev, generator=gen)

  def Run():
    x, w = x0.clone().requires_grad_(), w0.clone().requires_grad_()
    st = xent.lm_head_xent(x, w, labels, 0.1, 1e-4)
    return x, w, (st.soft_xent + st.z_inc).sum()
  x, w, loss = Run()
  loss.backward(retain_graph=True)
  first = (x.grad.clone(), w.grad.clone())
  with pytest.raises(RuntimeError, match='modified by an inplace operation'):
    loss.backward()
  assert torch.equal(x.grad, first[0]) and torch.equal(w.grad, first[1])
  x2, w2, loss2 = Run()
  loss2.backward()
  assert torch.equal(x2.grad, first[0]) and torch.equal(w2.grad, first[1])


# -------------------------------------------------------- GPU: decoder blocks ----
class _BlockSpy:
  """Records the norm pass, the linear layers, the fused FFN and flash attention of a
  `DecoderBlock`, with the gradients that reach each of their inputs and outputs."""

  def __init__(self, monkeypatch):
    from lingvo_b200.ops import attention, gemm, norm
    self.norm, self.linears, self.ffn, self.flash = None, [], None, None
    real_pass, real_linear = norm.rms_norm_pass, gemm.linear
    real_ffn, real_flash = gemm.ffn_relu, attention.flash_attention

    def Hook(rec, key, t):
      if t is not None and t.requires_grad:
        t.register_hook(lambda g: rec.update({key: g.detach().clone()}))

    def Pass(x, scale, eps):
      xn, xp = real_pass(x, scale, eps)
      self.norm = NestedMap(x=x.detach(), scale=scale.detach(), xn=xn.detach())
      Hook(self.norm, 'dxn', xn)
      Hook(self.norm, 'dpass', xp)
      return xn, xp

    def Linear(x, w, bias=None, act=None, residual=None):
      y = real_linear(x, w, bias, act, residual)
      rec = NestedMap(x=x.detach(), w=w.detach(), y=y.detach(),
                      res=None if residual is None else residual.detach())
      for key, t in (('dx', x), ('dw', w), ('dy', y)):
        Hook(rec, key, t)
      self.linears.append(rec)
      return y

    def Ffn(x, wi, wo, residual=None):
      y = real_ffn(x, wi, wo, residual)
      self.ffn = NestedMap(x=x.detach(), y=y.detach())
      Hook(self.ffn, 'dy', y)
      return y

    def Flash(q, k, v, rel, seg, pos, scale, causal):
      o = real_flash(q, k, v, rel, seg, pos, scale, causal)
      self.flash = NestedMap(q=q.detach(), k=k.detach(), v=v.detach(), rel=rel.detach(),
                             seg=seg, pos=pos, scale=scale, causal=causal, o=o.detach())
      for key, t in (('dq', q), ('dk', k), ('dv', v), ('drel', rel), ('do', o)):
        Hook(self.flash, key, t)
      return o
    monkeypatch.setattr(norm, 'rms_norm_pass', Pass)
    monkeypatch.setattr(gemm, 'linear', Linear)
    monkeypatch.setattr(gemm, 'ffn_relu', Ffn)
    monkeypatch.setattr(attention, 'flash_attention', Flash)


def _ZeroGrads(task):
  for v in task.vars.Flatten():
    v.grad = None


def _Flat(t):
  return t.reshape(-1, t.shape[-1])


def _RunBlock(blk, x, seg, pos, dy, all_valid):
  """One forward and backward of the block as the stack runs it → (out, theta)."""
  theta = blk.theta
  out = blk.FProp(theta, NestedMap(vec=x, segment_id=seg, segment_pos=pos,
                                   aux_loss=torch.zeros((), device=x.device),
                                   all_valid=all_valid))
  out.vec.backward(dy)
  return out.vec.detach()


def _NormPassStages(spy, x, live, what):
  """Norm pass forward, and dx with the residual stream's gradient, under the norm test's
  bounds; the residual gradient dropped must fail them. → the master dscale bound check."""
  nr = spy.norm
  t, m = _Flat(x).shape
  assert torch.equal(gemm64._Bits(nr.x), gemm64._Bits(x.detach() * live)), what + ' x_in'
  o = N._Oracle(_Flat(nr.x), None, nr.scale.float(), None, False)
  N._AssertBf16(_Flat(nr.xn), o['y'], o['slack_y'] + N._Ulp(o['y']), what + ' norm out')
  o = N._Oracle(_Flat(nr.x), _Flat(nr.dxn), nr.scale.float(), None, False,
                dres=_Flat(nr.dpass))
  dx = _Flat(x.grad)
  N._AssertBf16(dx, o['dx'] * _Flat(live), o['slack_dx'] + N._Ulp(o['dx']), what + ' dx')
  assert bool((dx[_Flat(live)[:, 0] == 0] == 0).all()), what + ": dx of a padded token"
  o2 = N._Oracle(_Flat(nr.x), _Flat(nr.dxn), nr.scale.float(), None, False)
  with pytest.raises(AssertionError):
    N._AssertBf16(dx, o2['dx'] * _Flat(live), o2['slack_dx'] + N._Ulp(o2['dx']), 'control')
  return o


def _AssertScaleGrad(master, o, what):
  """The fp32 master of a bf16 parameter gets the kernel's fp32 dscale rounded to bf16 once
  (`_NormFn`/`_NormPassFn` return ds in the theta's dtype): the norm test's bound plus that
  rounding, and a value that bf16 represents exactly."""
  g = master.grad
  assert torch.equal(g, g.bfloat16().float()), what + ': dscale is not a bf16 value'
  bound = o['d_ds'] + 0.5 * gemm64._Ulp(torch.maximum(o['ds'].abs(), g.double().abs()))
  assert bool(((g.double() - o['ds']).abs() <= bound).all()), what + ' dscale'


_ATTN_CASES = [
    ('bench', 8, 1024, None, True),        # what bench.py runs
    ('packed', 8, 1024, None, False),
    ('kv4', 8, 1024, 4, False),            # MoELm8EKv4: three q / k / v GEMMs
    ('one_block', 1, 128, None, False),
    ('ragged', 2, 384, None, False),
]


@pytest.fixture(scope='module')
def bench_tasks():
  """MHA and grouped-KV MoELm8E tasks (two layers) on the device, built once."""
  dev = torch.device('cuda', torch.cuda.current_device())
  return {kv: _Task(kv=kv, seed=7).to(dev) for kv in (None, 4)}


def _BlockInputs(b, l, m, all_valid, dev, seed):
  if all_valid:
    seg = torch.ones(b, l, dtype=torch.int32)
    pos = torch.arange(l, dtype=torch.int32).expand(b, l).contiguous()
  else:
    seg, pos = _Packed(b, l, seed)
  seg, pos = seg.to(dev), pos.to(dev)
  gen = torch.Generator(device=dev).manual_seed(seed)
  live = (seg != 0)[..., None].to(torch.bfloat16)
  x = torch.randn(b, l, m, device=dev, generator=gen).to(torch.bfloat16)
  dy = torch.randn(b, l, m, device=dev, generator=gen).to(torch.bfloat16) * live
  return seg, pos, live, x, dy


@pytest.mark.gpu
@pytest.mark.parametrize('case', _ATTN_CASES, ids=[c[0] for c in _ATTN_CASES])
def test_attention_block_stages(case, bench_tasks, monkeypatch):
  """`DecoderBlock` + `SelfAttentionLayer` as the MoELm8E stack runs it: every stage of the
  module docstring under the kernels' own bounds, the controls, and padded tokens."""
  from lingvo_b200.ops import gemm as G
  name, b, l, kv, all_valid = case
  dev = torch.device('cuda', torch.cuda.current_device())
  m = 2048
  task = bench_tasks[kv]
  blk = task.dec.layers[0]
  _ZeroGrads(task)
  seg, pos, live, x0, dy = _BlockInputs(b, l, m, all_valid, dev, 40 + b + l)
  x = x0.clone().requires_grad_()
  spy = _BlockSpy(monkeypatch)
  y = _RunBlock(blk, x, seg, pos, dy, all_valid)
  monkeypatch.undo()
  fl, lin = spy.flash, spy.linears
  assert fl is not None, 'the flash kernel did not run'
  assert len(lin) == (2 if kv is None else 4), len(lin)
  assert bool(torch.isfinite(y).all())
  res = {}
  # norm pass and the residual stream's gradient
  o_norm = _NormPassStages(spy, x, live, name)
  assert torch.equal(gemm64._Bits(spy.norm.dpass), gemm64._Bits(dy)), 'residual gradient'
  _AssertScaleGrad(blk.vars.ln.scale, o_norm, name)
  # q / k / v projections and their backward
  for rec in lin[:-1]:
    res['qkv'] = max(res.get('qkv', 0), gemm64._Check(_Flat(rec.y), _Flat(rec.x), rec.w, True,
                                                       False, what='qkv')[0])
    gemm64._Check(rec.dw, _Flat(rec.x), _Flat(rec.dy), False, False, what='dwqkv')
  if len(lin) == 2:
    gemm64._Check(_Flat(lin[0].dx), _Flat(lin[0].dy), lin[0].w, True, True, what='dxn')
  else:
    # three projections read xn: autograd adds their bf16 dgrads in bf16. Each is within
    # the GEMM bound; each of the two adds rounds by at most an ulp of its terms.
    ref, slack = 0.0, 0.0
    for rec in lin[:-1]:
      dyd, wd = _Flat(rec.dy).double(), rec.w.double()
      si = dyd @ wd.t()
      n = math.ceil(wd.shape[1] / 16) + 16
      ref = ref + si
      slack = slack + gemm64._Ulp(si) + n * gemm64._U_ACC * (dyd.abs() @ wd.abs().t())
    got = _Flat(spy.norm.dxn).double()
    bound = gemm64._C * (slack + gemm64._Ulp(torch.maximum(ref.abs(), got.abs())))
    err = (got - ref).abs()
    assert bool((err <= bound).all()), 'dxn: worst err/bound %g' % float((err / bound).max())
  # the relative-bias table: bitwise the float64 gather of wrb by the buckets of q − k
  wrb = blk.theta.layer.wrb.detach().double()
  qk = torch.arange(2 * l - 1, device=dev) - (l - 1)
  assert torch.equal(fl.rel.double(), wrb[:, _Bucket64(qk)]), 'rel table'
  assert not torch.equal(fl.rel.double(), wrb[:, _Bucket64(-qk)])    # the k − q table differs
  # flash attention forward and backward, from its recorded inputs
  with torch.no_grad():
    r = TG._GqaOracle(fl.q, fl.k, fl.v, fl.rel, fl.seg, fl.pos, fl.scale, fl.causal, fl.do)
  u = _U8
  rows = r['live'][:, :, None, None].expand_as(fl.o)
  TF._CheckBound(name, 'o', fl.o, r['out'], TF._C_O * u * r['a_out'] + TF._Bf16Ulp(r['out']),
                 rows)
  TF._CheckBound(name, 'dv', fl.dv, r['dv'], TF._C_DV * u * r['a_dv'] + TF._Bf16Ulp(r['dv']))
  TF._CheckBound(name, 'dk', fl.dk, r['dk'], TF._C_DQK * u * r['a_dk'] + TF._Bf16Ulp(r['dk']))
  TF._CheckBound(name, 'dq', fl.dq, r['dq'], TF._C_DQK * u * r['a_dq'] + TF._Bf16Ulp(r['dq']))
  drel_bound = TF._C_DREL * u * r['drel_delta'] + TF._DREL_FLOOR * r['drel_abs']
  TF._CheckBound(name, 'drel', fl.drel, r['drel'], drel_bound)
  if name == 'packed':
    with torch.no_grad():
      r2 = TF._Oracle(fl.q[:1], fl.v[:1], fl.k[:1], fl.rel, fl.seg[:1], fl.pos[:1], fl.scale,
                      fl.causal, fl.do[:1])
    with pytest.raises(AssertionError):          # control: k and v swapped
      TF._CheckBound(name, 'o', fl.o[:1], r2['out'],
                     TF._C_O * u * r2['a_out'] + TF._Bf16Ulp(r2['out']), rows[:1])
    del r2
  del r
  # d wrb: the recorded d rel folded by bucket in fp32, rounded once to the bf16 theta
  bucket = _Bucket64(qk)
  g = blk.vars.layer.wrb.grad
  assert torch.equal(g, g.bfloat16().float()), 'd wrb is not a bf16 value'

  def Fold(bk):
    f = torch.zeros(g.shape, dtype=torch.float64, device=dev).index_add_(
        1, bk, fl.drel.double())
    fa = torch.zeros_like(f).index_add_(1, bk, fl.drel.double().abs())
    cnt = torch.bincount(bk, minlength=_BUCKETS).double()
    return f, 2 * (cnt * _U * fa + 0.5 * gemm64._Ulp(torch.maximum(f.abs(), g.double().abs())))
  fold, bound = Fold(bucket)
  err = (g.double() - fold).abs()
  assert bool((err <= bound).all()), 'd wrb: worst err/bound %g' % float((err / bound).max())
  res['dwrb'] = float((err / bound).max())
  nfold, nbound = Fold((bucket + 1) % _BUCKETS)
  assert bool(((g.double() - nfold).abs() > nbound).any()), 'control: d wrb in the next bucket'
  # the output projection with the residual, and its backward
  out = lin[-1]
  res['y'] = gemm64._Check(_Flat(out.y), _Flat(out.x), out.w, True, False, aux=_Flat(out.res),
                           aux_mode=G.AUX_ADD, what='y')[0]
  for mult in (0, 2):                            # controls: residual dropped / added twice
    with pytest.raises(AssertionError):
      gemm64._Check(_Flat(out.y), _Flat(out.x), out.w, True, False,
                    aux=_Flat(out.res) * mult, aux_mode=G.AUX_ADD, what='control')
  assert torch.equal(gemm64._Bits(out.dy), gemm64._Bits(dy))
  assert torch.equal(gemm64._Bits(out.dx.reshape(-1)), gemm64._Bits(fl.do.reshape(-1))), 'd o'
  res['do'] = gemm64._Check(_Flat(out.dx), _Flat(dy), out.w, True, True, what='do')[0]
  res['dwo'] = gemm64._Check(out.dw, _Flat(out.x), _Flat(dy), False, False, what='dwo')[0]
  if not all_valid:
    # a padded token contributes nothing: another input there leaves every gradient unchanged
    grads = {k: v.grad.clone() for k, v in blk.vars.FlattenItems()}
    _ZeroGrads(task)
    gen = torch.Generator(device=dev).manual_seed(99)
    other = torch.randn(x0.shape, device=dev, generator=gen).to(torch.bfloat16)
    x2 = torch.where(live > 0, x0, other).requires_grad_()
    y2 = _RunBlock(blk, x2, seg, pos, dy, all_valid)
    for k, v in blk.vars.FlattenItems():
      assert torch.equal(v.grad, grads[k]), '%s: a padded token changed d%s' % (name, k)
    assert torch.equal(gemm64._Bits(x2.grad), gemm64._Bits(x.grad))
    assert torch.equal(gemm64._Bits(y2 * live), gemm64._Bits(y * live))
  print('%s: %s' % (name, ' '.join('%s %.3f' % kv for kv in res.items())))


@pytest.mark.gpu
@pytest.mark.parametrize('all_valid', [True, False], ids=['bench', 'packed'])
def test_ffn_block_stages(all_valid, bench_tasks, monkeypatch):
  """`DecoderBlock` + `DenseReluDenseLayer` (M 2048, H 8192): the norm pass and the
  residual stream's gradient under the norm test's bounds, the fused FFN's output with the
  residual added once, and the residual gradient passed to the norm pass unchanged."""
  dev = torch.device('cuda', torch.cuda.current_device())
  task = bench_tasks[None]
  blk = task.dec.layers[3]
  _ZeroGrads(task)
  seg, pos, live, x0, dy = _BlockInputs(8, 1024, 2048, all_valid, dev, 77)
  x = x0.clone().requires_grad_()
  spy = _BlockSpy(monkeypatch)
  y = _RunBlock(blk, x, seg, pos, dy, all_valid)
  monkeypatch.undo()
  assert spy.ffn is not None and not spy.linears, 'the fused FFN did not run'
  o = _NormPassStages(spy, x, live, 'ffn')
  assert torch.equal(gemm64._Bits(spy.norm.dpass), gemm64._Bits(dy)), 'residual gradient'
  _AssertScaleGrad(blk.vars.ln.scale, o, 'ffn')
  th = blk.theta.layer
  xn = _Flat(spy.norm.xn).double()
  wi, wo = th.wi.detach().double(), th.wo.detach().double()
  res_in = _Flat(spy.norm.x).double()
  h = torch.relu(xn @ wi)
  s = h @ wo
  ref = s + res_in
  # The fused FFN rounds h to bf16 (≤ 2^-8·|h|) after an fp32 accumulation over M
  # (n_h·u′·|xn|·|wi|, the GEMM test's model); both reach y through |wo|. Then the GEMM
  # bound of y itself over K = H.
  n_h, n_o = math.ceil(xn.shape[1] / 16) + 16, math.ceil(h.shape[1] / 16) + 16
  p = h @ wo.abs()
  q = (n_h * gemm64._U_ACC * (xn.abs() @ wi.abs())) @ wo.abs()
  e = n_o * gemm64._U_ACC * p + 3 * _U * (s.abs() + res_in.abs()) + _U8 * p + q
  del q
  bound = gemm64._Bound(ref, _Flat(y).double(), e)
  err = (_Flat(y).double() - ref).abs()
  assert bool((err <= bound).all()), 'ffn y: worst err/bound %g' % float((err / bound).max())
  for mult in (0.0, 2.0):                        # controls: residual dropped / added twice
    bad = (_Flat(y).double() - (s + mult * res_in)).abs() > bound
    assert bool(bad.any()), 'control: residual x%g' % mult
  print('ffn %s: y %.3f' % ('bench' if all_valid else 'packed', float((err / bound).max())))
