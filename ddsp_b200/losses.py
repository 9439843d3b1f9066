"""Multi-scale spectral loss with the reference's constructor and semantics
(`ddsp/losses.py:102-243`), in torch (cuFFT on the GPU)."""
import functools

import torch

from ddsp_b200 import spectral_ops


def mean_difference(target, value, loss_type='L1', weights=None):
  """losses.mean_difference (losses.py:102-127)."""
  difference = target - value
  weights = 1.0 if weights is None else weights
  loss_type = loss_type.upper()
  if loss_type == 'L1':
    return torch.mean(torch.abs(difference * weights))
  elif loss_type == 'L2':
    return torch.mean(difference**2 * weights)
  elif loss_type == 'COSINE':
    cos = torch.nn.functional.cosine_similarity(target, value, dim=-1)
    return torch.mean((1.0 - cos) * weights)   # weights is 1.0 when none were given
  else:
    raise ValueError('Loss type ({}), must be '
                     '"L1", "L2", or "COSINE"'.format(loss_type))


class SpectralLoss:
  """Multi-scale spectrogram loss (losses.py:130-243)."""

  def __init__(self,
               fft_sizes=(2048, 1024, 512, 256, 128, 64),
               loss_type='L1',
               mag_weight=1.0,
               delta_time_weight=0.0,
               delta_freq_weight=0.0,
               cumsum_freq_weight=0.0,
               logmag_weight=0.0,
               loudness_weight=0.0,
               name='spectral_loss'):
    self.name = name
    self.fft_sizes = fft_sizes
    self.loss_type = loss_type
    self.mag_weight = mag_weight
    self.delta_time_weight = delta_time_weight
    self.delta_freq_weight = delta_freq_weight
    self.cumsum_freq_weight = cumsum_freq_weight
    self.logmag_weight = logmag_weight
    self.loudness_weight = loudness_weight
    self.spectrogram_ops = [
        functools.partial(spectral_ops.compute_mag, size=size)
        for size in self.fft_sizes]

  def __call__(self, target_audio, audio, weights=None):
    return self.call(target_audio, audio, weights=weights)

  def get_losses_dict(self, target_audio, audio, **kwargs):
    """losses.Loss.get_losses_dict (losses.py:60-66)."""
    return {self.name: self.call(target_audio, audio, **kwargs)}

  def _fusable(self, target_audio, audio, weights):
    """The ae.gin configuration (L1 on magnitudes and log-magnitudes,
    ae.gin:39-41) on CUDA tensors runs through three hand-written kernels per FFT
    size around cuFFT instead of ~70 elementwise launches."""
    return (torch.is_tensor(audio) and audio.is_cuda and torch.is_tensor(target_audio)
            and target_audio.is_cuda and weights is None
            and self.loss_type.upper() == 'L1'
            and self.delta_time_weight <= 0 and self.delta_freq_weight <= 0
            and self.cumsum_freq_weight <= 0
            and (self.mag_weight > 0 or self.logmag_weight > 0)
            and audio.dim() == 2 and target_audio.shape == audio.shape
            and all(int(sz) >= 16 and (int(sz) & (int(sz) - 1)) == 0
                    for sz in self.fft_sizes))

  def _call_fused(self, target_audio, audio):
    return spectral_ops.SpectralLossFn.apply(
        target_audio.detach(), audio, tuple(int(s) for s in self.fft_sizes),
        max(self.mag_weight, 0.0), max(self.logmag_weight, 0.0))

  def call(self, target_audio, audio, weights=None):
    if self._fusable(target_audio, audio, weights):
      loss = self._call_fused(target_audio, audio)
    else:
      loss = self._call_spectrograms(target_audio, audio, weights)
    if self.loudness_weight > 0:
      # losses.py:236-241: n_fft = 2048 and every other argument at its default,
      # whatever the audio's sample rate
      target = spectral_ops.compute_loudness(target_audio, n_fft=2048)
      value = spectral_ops.compute_loudness(audio, n_fft=2048)
      loss = loss + self.loudness_weight * mean_difference(
          target, value, self.loss_type, weights=weights)
    return loss

  def _call_spectrograms(self, target_audio, audio, weights):
    loss = 0.0
    diff = lambda x, axis: torch.diff(x, dim=axis)
    for loss_op in self.spectrogram_ops:
      target_mag = loss_op(target_audio)
      value_mag = loss_op(audio)
      if self.mag_weight > 0:
        loss = loss + self.mag_weight * mean_difference(
            target_mag, value_mag, self.loss_type, weights=weights)
      if self.delta_time_weight > 0:
        loss = loss + self.delta_time_weight * mean_difference(
            diff(target_mag, 1), diff(value_mag, 1), self.loss_type,
            weights=weights)
      if self.delta_freq_weight > 0:
        loss = loss + self.delta_freq_weight * mean_difference(
            diff(target_mag, 2), diff(value_mag, 2), self.loss_type,
            weights=weights)
      if self.cumsum_freq_weight > 0:
        loss = loss + self.cumsum_freq_weight * mean_difference(
            torch.cumsum(target_mag, 2), torch.cumsum(value_mag, 2),
            self.loss_type, weights=weights)
      if self.logmag_weight > 0:
        loss = loss + self.logmag_weight * mean_difference(
            spectral_ops.safe_log(target_mag), spectral_ops.safe_log(value_mag),
            self.loss_type, weights=weights)
    return loss
