"""SpecAugment tuned for running inside the accelerator step
(ref `lingvo/core/spectrum_augmenter_on_device.py`).

The reference's on-device variant rewrites the base layer's einsums into forms its target
accelerator executes well. The H100 equivalent changes the *algorithms* that were shaped by
a matrix unit into memory-lean ones, keeping the sampled augmentation identical to
`SpectrumAugmenter` for the same random stream:

  * warping: instead of materialising a `[B, N, N]` interpolation matrix and a batched GEMM
    (O(N²) bytes per utterance), each output row gathers its two source rows and blends them
    — O(N), one pass over the spectrogram;
  * masking: frequency noise, time mask, frequency mask and block mask are folded into one
    `[B, T, F]` multiplier applied in a single pass (the base class makes one pass per
    augmentation), the optional time-mask noise is added in the same expression.
"""

from __future__ import annotations

import torch

from lingvo_b200.core import spectrum_augmenter


class SpectrumAugmenterOnDevice(spectrum_augmenter.SpectrumAugmenter):
  """Drop-in replacement of `SpectrumAugmenter` with O(N) warps and a single masking pass."""

  def _ApplyWarp(self, inputs, axis, origin, destination, choose_range):
    n = inputs.shape[axis]
    src = self._SourceCoordinates(n, origin, destination, choose_range.to(inputs.device))
    # hat(orig − j) is non-zero only for j ∈ {floor(orig), floor(orig)+1}
    lo = torch.floor(src)
    frac = (src - lo).to(inputs.dtype)
    lo = lo.long()
    hi = lo + 1
    w_lo = torch.where((lo >= 0) & (lo < n), 1.0 - frac, torch.zeros_like(frac))
    w_hi = torch.where((hi >= 0) & (hi < n), frac, torch.zeros_like(frac))
    lo, hi = lo.clamp(0, n - 1), hi.clamp(0, n - 1)
    b = inputs.shape[0]
    view = [b, 1, 1, 1]
    view[axis] = n

    def Take(idx):
      return inputs.gather(axis, idx.view(view).expand_as(inputs))

    return Take(lo) * w_lo.view(view) + Take(hi) * w_hi.view(view)

  def _AugmentationNetwork(self, inputs, paddings, rng, di=0):
    p = self.params
    d = self._dom
    shape = inputs.shape
    if p.unstack:
      inputs, paddings = self.UnstackFeatures(inputs, paddings)
    lengths = (1.0 - paddings.float()).sum(1)
    inputs = self._FrequencyWarp(inputs, rng, di)
    inputs = self._TimeWarp(inputs, lengths, rng, di)
    b, t, f, c = inputs.shape
    dev = inputs.device
    mult = None                                    # [B, T|1, F|1] combined multiplier

    def Fold(m):
      nonlocal mult
      mult = m if mult is None else mult * m

    # frequency noise (same streams / order as the base class)
    max_std = d['freq_noise_max_stddev'][di]
    if max_std > 0.0:
      w = self.augment_weight
      w = w.to(dev) if isinstance(w, torch.Tensor) else w
      stddev = rng.Uniform((b, 1, 1, 1), 41) * (max_std * w)
      Fold((1.0 + rng.Normal((b, 1, f, 1), 42) * stddev).view(b, 1, f))
    tmask = self._TimeMaskArrays(inputs, lengths, rng, di)
    noise = None
    if tmask is not None:
      Fold(tmask.view(b, t, 1))
      if p.use_noise:
        stddev = 1.0 if p.gaussian_noise else (1.0 + rng.Uniform((), 6)) * 0.1 + 0.0001
        noise = rng.Normal((b, t, f), 7) * stddev * (1.0 - tmask).unsqueeze(-1)
    bins, count = d['freq_mask_max_bins'][di], d['freq_mask_count'][di]
    fmask = None
    if bins != 0 and count != 0:
      fmask = self._GetMask(rng, b, torch.full((b,), f, device=dev), f, max_length=bins,
                            multiplicity=count, salts=(11, 12)).view(b, 1, f)
      Fold(fmask)
    out = inputs
    if mult is not None:
      out = out * mult.to(inputs.dtype).unsqueeze(-1)
    if noise is not None:
      # the base class adds the noise before the frequency mask, which therefore masks it too
      if fmask is not None:
        noise = noise * fmask
      out = out + noise.to(inputs.dtype).unsqueeze(-1)
    out = self._BlockMask(out, rng, di)
    if p.unstack:
      out = out.reshape(shape)
    return out
