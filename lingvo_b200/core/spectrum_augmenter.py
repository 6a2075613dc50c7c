"""SpecAugment (ref `lingvo/core/spectrum_augmenter.py`, arXiv:1904.08779).

`FProp(theta, inputs [B, T, F, C], paddings [B, T], domain_ids=None)` applies, in this order
(ref `_AugmentationNetwork` :955): frequency warp → time warp → frequency noise → time mask
(optionally filled with noise) → frequency mask → block mask. Feature parity with the
reference:

  * multi-masks with static / length-proportional widths, `time_mask_max_ratio`, adaptive
    multiplicity `time_masks_per_frame` (ref `_GetMask` :209),
  * piecewise-linear time / frequency warping that fixes both ends of the valid region and
    moves one random anchor (ref `_GetWarpMatrix` :341, `_ConstructWarpMatrix` :449),
  * multiplicative frequency noise N(1, σ), σ ~ U(0, max·warm-up weight) (ref :877),
  * block masking on a (t, f) block grid with a per-utterance drop probability (ref :705),
  * stacked-frame handling `unstack / stack_height` (ref :942),
  * per-domain settings: every augmentation parameter may be a list aligned with
    `p.domain_ids`; utterances of other domains pass through (ref FProp :1023),
  * `use_input_dependent_random_seed`: randomness is a pure function of the input features
    (counter-based hash evaluated on the device — no host round trip), which is what
    federated / replayable training needs (ref :145).

H100 design. All randomness is drawn on the device (torch generator, or the stateless
hash), every mask is built by broadcast comparisons, and nothing synchronises with the host,
so augmentation is a handful of elementwise kernels inside the captured train step. This
base class keeps the reference's explicit `[B, N, N]` warp matrices (small batched GEMMs on
the tensor cores — fine for N of a few hundred); `SpectrumAugmenterOnDevice`
(`spectrum_augmenter_on_device.py`) replaces them with an O(N) two-tap gather and fuses all
multiplicative masks into one pass. In eval mode the layer is the identity.
"""

from __future__ import annotations

import torch
import torch.nn.functional as F

from lingvo_b200.core import base_layer
from lingvo_b200.core import py_utils

_SPECAUGMENT_ARGS = (
    'freq_mask_max_bins', 'freq_mask_count', 'use_dynamic_time_mask_max_frames',
    'time_mask_max_frames', 'time_mask_count', 'time_mask_max_ratio', 'time_masks_per_frame',
    'block_mask_prob', 'block_mask_size', 'freq_warp_max_bins', 'time_warp_bound',
    'time_warp_max_frames', 'time_warp_max_ratio', 'freq_noise_max_stddev')


def _Hat(x):
  """Hat function: 1 − |x| on [−1, 1], 0 elsewhere (linear-interpolation weights)."""
  return F.relu(x + 1) - 2 * F.relu(x) + F.relu(x - 1)


def _Lsr(x, k):
  """Logical right shift of an int64 tensor (torch's >> is arithmetic)."""
  return (x >> k) & ((1 << (64 - k)) - 1)


def _Mix64(x):
  """splitmix64-style finaliser on int64 tensors (wrap-around arithmetic)."""
  x = (x ^ _Lsr(x, 30)) * -4658895280553007687      # 0xBF58476D1CE4E5B9
  x = (x ^ _Lsr(x, 27)) * -7723592293110705685      # 0x94D049BB133111EB
  return x ^ _Lsr(x, 31)


def StatelessUniform(shape, seed, salt, device):
  """U[0, 1) of `shape` as a pure function of the 0-d int64 tensor `seed` and int `salt`
  (counter-based: hash(seed, salt, element index)); evaluated on `device`."""
  n = 1
  for s in shape:
    n *= int(s)
  idx = torch.arange(n, dtype=torch.int64, device=device)
  h = _Mix64(idx * -7046029254386353131 + seed.to(device) + int(salt) * 0x632BE59B)
  h = _Mix64(h + int(salt))
  u = _Lsr(h, 11).to(torch.float64) * (1.0 / (1 << 53))
  return u.to(torch.float32).reshape(tuple(int(s) for s in shape))


def StatelessNormal(shape, seed, salt, device):
  """N(0, 1) via Box–Muller over two stateless uniform streams."""
  u1 = StatelessUniform(shape, seed, 2 * salt + 101, device).clamp_min(1e-12)
  u2 = StatelessUniform(shape, seed, 2 * salt + 102, device)
  return torch.sqrt(-2.0 * torch.log(u1)) * torch.cos(6.283185307179586 * u2)


class _Rng:
  """Random source of one FProp: a seeded generator, the default CUDA/CPU generator, or the
  stateless input-dependent hash. `salt` names the stream (the reference's seed_1…seed_7)."""

  def __init__(self, layer, inputs):
    p = layer.params
    self.device = inputs.device
    self.stateless_seed = None
    self.gen = None
    if p.use_input_dependent_random_seed:
      s = inputs.detach().abs().double().sum()
      self.stateless_seed = (s * 1000.0).to(torch.int64) + int(p.random_seed or 0)
    elif p.random_seed is not None:
      self.gen = torch.Generator(device=self.device)
      gs = py_utils.GetGlobalStep()
      self.gen.manual_seed(int(p.random_seed) + (int(gs) if not isinstance(gs, torch.Tensor)
                                                 else 0))

  def Uniform(self, shape, salt):
    if self.stateless_seed is not None:
      return StatelessUniform(shape, self.stateless_seed, salt, self.device)
    return torch.rand(tuple(shape), device=self.device, generator=self.gen)

  def Normal(self, shape, salt):
    if self.stateless_seed is not None:
      return StatelessNormal(shape, self.stateless_seed, salt, self.device)
    return torch.randn(tuple(shape), device=self.device, generator=self.gen)


class SpectrumAugmenter(base_layer.BaseLayer):
  """SpecAugment layer (ref :82)."""

  @classmethod
  def Params(cls):
    p = super().Params()
    p.Define('freq_mask_max_bins', 15, 'Maximum number of frequency bins of a frequency mask.')
    p.Define('freq_mask_count', 1, 'Number of masks applied on the frequency axis.')
    p.Define('use_dynamic_time_mask_max_frames', False,
             'If true, the max time-mask width is time_mask_max_ratio * utterance_length.')
    p.Define('time_mask_max_frames', 50, 'Maximum number of frames of a time mask (ignored '
             'when use_dynamic_time_mask_max_frames).')
    p.Define('time_mask_count', 1, 'Number of masks on the time axis (upper bound when '
             'time_masks_per_frame > 0).')
    p.Define('time_mask_max_ratio', 1.0, 'Maximum portion of the utterance a mask may cover.')
    p.Define('time_masks_per_frame', 0.0, 'If > 0, the number of time masks is '
             'min(time_masks_per_frame * utterance_length, time_mask_count).')
    p.Define('block_mask_prob', 0.0, 'Block-mask drop probability upper bound.')
    p.Define('block_mask_size', dict(t=32, f=32), 'Block size of the block mask.')
    p.Define('freq_warp_max_bins', 0, 'Maximum shift (bins) of frequency warping.')
    p.Define('time_warp_bound', 'static', "'static': bound = min(time_warp_max_frames, "
             "ratio*length); 'dynamic': bound = time_warp_max_ratio * length.")
    p.Define('time_warp_max_frames', 0, 'Maximum shift (frames) of time warping.')
    p.Define('time_warp_max_ratio', 0.0, 'Maximum shift of time warping as a portion of length.')
    p.Define('use_noise', False, 'Fill time-masked regions with noise.')
    p.Define('gaussian_noise', False, 'Noise stddev 1 (else stddev ~ U(0.1, 0.2)).')
    p.Define('freq_noise_max_stddev', 0.0, 'Max stddev of the multiplicative frequency noise.')
    p.Define('freq_noise_warmup_steps', 0, 'Steps over which that stddev ramps up linearly.')
    p.Define('unstack', False, 'Unstack stacked frames before augmenting.')
    p.Define('stack_height', 3, 'Frames stacked per input frame (with `unstack`).')
    p.Define('domain_ids', [0], 'Domains to augment; per-domain parameters are lists aligned '
             'with this one. Other domains pass through unchanged.')
    p.Define('use_input_dependent_random_seed', False,
             'Randomness is a pure function of the input features (stateless hash).')
    p.Define('eval_data_in_domains', False, 'Kept for parity.')
    return p

  def __init__(self, params):
    super().__init__(params)
    p = self.params
    n = len(p.domain_ids)
    self._dom = {}
    for field in _SPECAUGMENT_ARGS:
      v = p.Get(field)
      if isinstance(v, (list, tuple)):
        assert len(v) == n, ('Length: %d of field: %s does not match total domains: %d' %
                             (len(v), field, n))
        self._dom[field] = list(v)
      else:
        self._dom[field] = [v] * n
    d = self._dom
    assert d['freq_mask_max_bins'][0] > -1
    assert d['time_mask_max_frames'][0] > -1
    assert d['freq_warp_max_bins'][0] > -1
    assert d['time_warp_max_frames'][0] > -1
    assert d['freq_noise_max_stddev'][0] >= 0.0

  # ---------------------------------------------------------------------------------
  @property
  def augment_weight(self):
    """Warm-up weight of the frequency noise: min(step, warmup) / warmup (ref :200)."""
    p = self.params
    if p.freq_noise_warmup_steps == 0:
      return 1.0
    gs = py_utils.GetGlobalStep()
    if isinstance(gs, torch.Tensor):
      return torch.clamp(gs.float(), max=float(p.freq_noise_warmup_steps)) / float(
          p.freq_noise_warmup_steps)
    return min(float(gs), float(p.freq_noise_warmup_steps)) / float(p.freq_noise_warmup_steps)

  def _GetMask(self, rng, batch_size, choose_range, mask_size, max_length=None,
               masks_per_frame=0.0, multiplicity=1, max_ratio=1.0, salts=(1, 2)):
    """Multi-mask `[B, mask_size]`, 0 inside masked spans, 1 elsewhere (ref :209).

    Widths ~ U[0, max_length) (or U[0, choose_range·max_ratio) when max_length is None),
    truncated to choose_range·max_ratio; starts uniform so the span stays inside
    [0, choose_range). With masks_per_frame > 0 only the first
    min(masks_per_frame·choose_range, multiplicity) masks of each row are active.
    """
    dev = rng.device
    cr = choose_range.to(device=dev, dtype=torch.float32)
    if max_length is not None and max_length > 0:
      max_len = torch.full((batch_size,), float(max_length), device=dev)
    else:
      max_len = cr * max_ratio
    portion = rng.Uniform((batch_size, multiplicity), salts[0])
    size = torch.floor(max_len.unsqueeze(1) * portion)
    bound = torch.floor(max_ratio * cr).clamp_min(1.0).unsqueeze(1)
    length = torch.minimum(size, bound)
    start = torch.floor(rng.Uniform((batch_size, multiplicity), salts[1]) *
                        (cr.unsqueeze(1) - length + 1.0))
    end = start + length                                     # exclusive
    pos = torch.arange(mask_size, device=dev, dtype=torch.float32).view(1, 1, mask_size)
    inside = (pos >= start.unsqueeze(-1)) & (pos < end.unsqueeze(-1))
    if masks_per_frame > 0:
      k = torch.arange(multiplicity, device=dev, dtype=torch.float32).view(1, multiplicity)
      active = k < (masks_per_frame * cr).unsqueeze(1)
      inside = inside & active.unsqueeze(-1)
    return 1.0 - inside.any(1).to(torch.float32)

  def _WarpEndpoints(self, rng, batch_size, choose_range, max_warp_frames=None,
                     max_ratio=1.0, salts=(3, 4, 5)):
    """(origin, destination) `[B]` float: a random anchor in [1, range−1) and where it moves
    (shift bounded by max_warp_frames and by max_ratio·range) (ref :341)."""
    dev = rng.device
    cr = choose_range.to(device=dev, dtype=torch.float32)
    upper = torch.floor(max_ratio * cr)
    if max_warp_frames is not None and max_warp_frames > 0:
      shift = torch.floor(rng.Uniform((batch_size,), salts[0]) * (2 * max_warp_frames + 1)
                          ) - max_warp_frames
    else:
      shift = torch.trunc((rng.Uniform((batch_size,), salts[1]) * 2.0 - 1.0) * upper)
    shift = torch.maximum(-upper, torch.minimum(shift, upper))
    mid = (cr - 2.0).clamp_min(0.0)
    origin = torch.floor(rng.Uniform((batch_size,), salts[2]) * mid) + 1.0
    return origin, origin + shift

  @staticmethod
  def _SourceCoordinates(matrix_size, origin, destination, choose_range):
    """orig_i `[B, N]`: the source coordinate sampled by output position i. Piecewise linear:
    fixes 0 and choose_range, maps destination → origin; identity beyond choose_range."""
    cr = choose_range.to(torch.float32)
    destination = torch.minimum(destination.clamp_min(1.0), cr - 1.0)
    slope_0 = origin / destination
    slope_1 = (cr - origin) / (cr - destination)
    x = torch.arange(matrix_size, device=origin.device, dtype=torch.float32).unsqueeze(0)
    return (slope_0.unsqueeze(1) * x +
            (slope_1 - slope_0).unsqueeze(1) * F.relu(x - destination.unsqueeze(1)) +
            (1.0 - slope_1).unsqueeze(1) * F.relu(x - cr.unsqueeze(1)))

  def _ConstructWarpMatrix(self, batch_size, matrix_size, origin, destination, choose_range,
                           dtype=torch.float32):
    """`[B, N, N]` with warp[b, i, j] = hat(orig_i − j): row i linearly interpolates the two
    source pixels around orig_i (ref :449)."""
    del batch_size
    src = self._SourceCoordinates(matrix_size, origin, destination, choose_range)
    j = torch.arange(matrix_size, device=src.device, dtype=torch.float32).view(1, 1, -1)
    return _Hat(src.unsqueeze(-1) - j).to(dtype)

  def _GetWarpMatrix(self, rng, batch_size, choose_range, matrix_size, max_warp_frames=None,
                     dtype=torch.float32, max_ratio=1.0):
    origin, destination = self._WarpEndpoints(rng, batch_size, choose_range, max_warp_frames,
                                              max_ratio)
    return self._ConstructWarpMatrix(batch_size, matrix_size, origin, destination,
                                     choose_range.to(rng.device), dtype)

  # -- the six augmentations ---------------------------------------------------------
  def _FrequencyMask(self, inputs, rng, di=0):
    d = self._dom
    bins, count = d['freq_mask_max_bins'][di], d['freq_mask_count'][di]
    if bins == 0 or count == 0:
      return inputs
    b, _, f, _ = inputs.shape
    mask = self._GetMask(rng, b, torch.full((b,), f, device=inputs.device), f, max_length=bins,
                         multiplicity=count, salts=(11, 12))
    return inputs * mask.to(inputs.dtype).view(b, 1, f, 1)

  def _TimeMaskArrays(self, inputs, seq_lengths, rng, di):
    d = self._dom
    max_frames = d['time_mask_max_frames'][di]
    dynamic = d['use_dynamic_time_mask_max_frames'][di]
    count, ratio = d['time_mask_count'][di], d['time_mask_max_ratio'][di]
    if (max_frames == 0 and not dynamic) or ratio <= 0.0 or count == 0:
      return None
    b, t = inputs.shape[:2]
    return self._GetMask(rng, b, seq_lengths, t, max_length=None if dynamic else max_frames,
                         masks_per_frame=d['time_masks_per_frame'][di], multiplicity=count,
                         max_ratio=ratio, salts=(1, 2))

  def _TimeMask(self, inputs, seq_lengths, rng, noisify=False, gaussian_noise=False, di=0):
    mask = self._TimeMaskArrays(inputs, seq_lengths, rng, di)
    if mask is None:
      return inputs
    b, t, f, _ = inputs.shape
    out = inputs * mask.to(inputs.dtype).view(b, t, 1, 1)
    if noisify:
      if gaussian_noise:
        stddev = 1.0
      else:
        stddev = (1.0 + rng.Uniform((), 6)) * 0.1 + 0.0001
      noise = rng.Normal((b, t, f), 7) * stddev
      out = out + (noise * (1.0 - mask).unsqueeze(-1)).to(inputs.dtype).unsqueeze(-1)
    return out

  def _BlockMask(self, inputs, rng, di=0):
    d = self._dom
    prob, size = d['block_mask_prob'][di], d['block_mask_size'][di]
    if prob == 0.0:
      return inputs
    b, t0, f0, c = inputs.shape
    fl = f0 * c
    tb, fb = int(size['t']), int(size['f'])
    nt, nf = -(-t0 // tb), -(-fl // fb)
    batch_prob = rng.Uniform((b,), 21) * prob
    keep = rng.Uniform((b, nt, nf), 22) > batch_prob.view(b, 1, 1)
    keep = keep.repeat_interleave(tb, 1).repeat_interleave(fb, 2)[:, :t0, :fl]
    return inputs * keep.to(inputs.dtype).reshape(b, t0, f0, c)

  def _ApplyWarp(self, inputs, axis, origin, destination, choose_range):
    """Applies the warp along `axis` (1: time, 2: frequency) with explicit matrices."""
    n = inputs.shape[axis]
    w = self._ConstructWarpMatrix(inputs.shape[0], n, origin, destination, choose_range,
                                  inputs.dtype)
    if axis == 1:
      return torch.einsum('bxyc,bzx->bzyc', inputs, w)
    return torch.einsum('bxyc,bzy->bxzc', inputs, w)

  def _FrequencyWarp(self, inputs, rng, di=0):
    bins = self._dom['freq_warp_max_bins'][di]
    if bins == 0:
      return inputs
    b, _, f, _ = inputs.shape
    cr = torch.full((b,), f, device=inputs.device)
    origin, dest = self._WarpEndpoints(rng, b, cr, bins, 1.0, salts=(31, 32, 33))
    return self._ApplyWarp(inputs, 2, origin, dest, cr)

  def _TimeWarp(self, inputs, seq_lengths, rng, di=0):
    d = self._dom
    frames, ratio, bound = (d['time_warp_max_frames'][di], d['time_warp_max_ratio'][di],
                            d['time_warp_bound'][di])
    assert bound in ('static', 'dynamic')
    if (frames == 0 and bound == 'static') or ratio <= 0.0:
      return inputs
    b = inputs.shape[0]
    origin, dest = self._WarpEndpoints(rng, b, seq_lengths,
                                       None if bound == 'dynamic' else frames, ratio)
    return self._ApplyWarp(inputs, 1, origin, dest, seq_lengths)

  def _FrequencyNoise(self, inputs, rng, di=0):
    """x · N(1, σ) per (utterance, frequency bin), σ ~ U(0, max·warm-up) (ref :877):
    multiplication in frequency imitates additive coloured noise in time."""
    max_std = self._dom['freq_noise_max_stddev'][di]
    if max_std <= 0.0:
      return inputs
    b, _, f, _ = inputs.shape
    w = self.augment_weight
    w = w.to(inputs.device) if isinstance(w, torch.Tensor) else w
    stddev = rng.Uniform((b, 1, 1, 1), 41) * (max_std * w)
    scale = 1.0 + rng.Normal((b, 1, f, 1), 42) * stddev
    return inputs * scale.to(inputs.dtype)

  def UnstackFeatures(self, src_inputs, src_paddings):
    """`[B, T, F·h, C]` stacked frames → `[B, T·h, F, C]` and the matching paddings."""
    sh = self.params.stack_height
    b, t, _, c = src_inputs.shape
    src_inputs = src_inputs.reshape(b, t * sh, -1, c)
    lengths = (sh * (1 - src_paddings.float()).sum(1)).long()
    pos = torch.arange(t * sh, device=src_inputs.device).unsqueeze(0)
    return src_inputs, (pos >= lengths.unsqueeze(1)).to(src_paddings.dtype)

  def _AugmentationNetwork(self, inputs, paddings, rng, di=0):
    p = self.params
    shape = inputs.shape
    if p.unstack:
      inputs, paddings = self.UnstackFeatures(inputs, paddings)
    lengths = (1.0 - paddings.float()).sum(1)
    inputs = self._FrequencyWarp(inputs, rng, di)
    inputs = self._TimeWarp(inputs, lengths, rng, di)
    inputs = self._FrequencyNoise(inputs, rng, di)
    inputs = self._TimeMask(inputs, lengths, rng, noisify=p.use_noise,
                            gaussian_noise=p.gaussian_noise, di=di)
    inputs = self._FrequencyMask(inputs, rng, di)
    inputs = self._BlockMask(inputs, rng, di)
    if p.unstack:
      inputs = inputs.reshape(shape)
    return inputs

  def FProp(self, theta, inputs, paddings, domain_ids=None):
    """inputs `[B, T, F, C]` (or `[B, T, F]`), paddings `[B, T]`, domain_ids `[B(, 1)]`.
    Returns (augmented inputs, paddings)."""
    p = self.params
    if self.do_eval:
      return inputs, paddings
    squeeze = inputs.dim() == 3
    if squeeze:
      inputs = inputs.unsqueeze(-1)
    rng = _Rng(self, inputs)
    if len(p.domain_ids) > 1:
      assert domain_ids is not None, 'domain_ids are required with several p.domain_ids'
      dom = domain_ids.reshape(inputs.shape[0]).to(inputs.device)
      out = inputs
      for i, domain_id in enumerate(p.domain_ids):
        aug = self._AugmentationNetwork(inputs, paddings, rng, i)
        sel = (dom == domain_id).view(-1, 1, 1, 1)
        out = torch.where(sel, aug, out)
    else:
      out = self._AugmentationNetwork(inputs, paddings, rng, 0)
    return (out.squeeze(-1) if squeeze else out), paddings


def _AttachEinsumHooks(cls):
  """The overridable contraction hooks of the reference (:178-197); subclasses replace them
  with quantised or sharded einsums."""
  specs = {'EinsumBBmBm': 'b,bm->bm', 'EinsumBmtBmBt': 'bmt,bm->bt',
           'EinsumBxycByBxyc': 'bxyc,by->bxyc', 'EinsumBxycBxBxyc': 'bxyc,bx->bxyc',
           'EinsumBxyBxBxy': 'bxy,bx->bxy', 'EinsumBxycBzxBzyc': 'bxyc,bzx->bzyc',
           'EinsumBxycBzyBxzc': 'bxyc,bzy->bxzc'}
  for name, eq in specs.items():
    if not hasattr(cls, name):
      def _Fn(self, a, b, name=None, _eq=eq):
        del name
        return torch.einsum(_eq, a, b.to(a.dtype))
      _Fn.__name__ = name
      setattr(cls, name, _Fn)
  return cls


_AttachEinsumHooks(SpectrumAugmenter)
