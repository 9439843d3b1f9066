"""Float64 torch restatement of the reference's `losses.SpectralLoss.call`
(losses.py:194-243) with every spectrogram term and 'L1' or 'L2': per FFT size,
weight * mean_difference of the magnitudes, their core.diff along time and along
frequency, their cumsum along frequency, and their safe_log.  Its gradients are torch
autograd's.  Pinned to the unmodified reference by tests/golden/spectral_terms.npz."""
import torch

from tests import grad_ref

TERMS = ('mag', 'delta_time', 'delta_freq', 'cumsum_freq', 'logmag')


def _diff(x, axis):
  n = x.shape[axis] - 1
  return x.narrow(axis, 1, n) - x.narrow(axis, 0, n)


_OPS = {
    'mag': lambda m: m,
    'delta_time': lambda m: _diff(m, 1),
    'delta_freq': lambda m: _diff(m, 2),
    'cumsum_freq': lambda m: torch.cumsum(m, 2),
    'logmag': grad_ref.safe_log,
}


def mean_difference(target, value, loss_type):
  d = target - value
  return torch.mean(d.abs()) if loss_type == 'L1' else torch.mean(d**2)


def spectral_loss(target, value, fft_sizes, loss_type='L1', spectra=None, **weights):
  """The loss for weights `<term>_weight` (mag_weight defaults to 1, the others to
  0, as in the reference's constructor).  `spectra`: optional (target STFT, value
  STFT) per FFT size, at which the loss is evaluated as in grad_ref.spectral_loss."""
  w = {t: float(weights.get(t + '_weight', 1.0 if t == 'mag' else 0.0)) for t in TERMS}
  target, value = (torch.as_tensor(x) for x in (target, value))
  loss = 0.0
  for i, size in enumerate(fft_sizes):
    xt = torch.fft.rfft(grad_ref.stft_frames(target, size), dim=-1)
    xv = torch.fft.rfft(grad_ref.stft_frames(value, size), dim=-1)
    if spectra is not None:
      xt = spectra[i][0].to(xt.dtype).to(xt.device).detach()
      xv = xv + (spectra[i][1].to(xv.dtype).to(xv.device) - xv).detach()
    t, v = xt.abs(), xv.abs()
    for term in TERMS:
      if w[term] > 0:
        op = _OPS[term]
        loss = loss + w[term] * mean_difference(op(t), op(v), loss_type)
  return loss
