"""Float64 torch restatement of core.sinusoidal_to_harmonic (core.py:733-781), formula
for formula on the reference's broadcast [B, T, K, S] tensors, with get_harmonic_frequencies
(core.py:1028-1045), safe_divide (core.py:207-210) and remove_above_nyquist
(core.py:869-891).  Differentiable: the tests take float64 autograd gradients of it,
which follow TensorFlow's (sign(0) = 0 in abs, nothing through a `where` branch not
taken, nothing through safe_divide's constant).  Pinned to the unmodified reference by
tests/golden/sinusoidal_to_harmonic.npz."""
import torch

from tests.consistency_ref import F64, safe_divide, t64


def harmonic_frequencies(f0_hz, n_harmonics):
  """f0 [B, T, 1] * [1 .. K]: tf.linspace(1, K, K) gives exact integers."""
  return f0_hz * torch.arange(1, n_harmonics + 1, dtype=F64)[None, None, :]


def sinusoidal_to_harmonic(sin_amps, sin_freqs, f0_hz, harmonic_width=0.1, n_harmonics=100,
                           sample_rate=16000, normalize=False):
  a, f, f0 = t64(sin_amps), t64(sin_freqs), t64(f0_hz)
  harm_freqs = harmonic_frequencies(f0, n_harmonics)
  freqs_diff = f[:, :, None, :] - harm_freqs[..., None]
  freqs_ratio = torch.abs(safe_divide(freqs_diff, f0[..., None]))
  weights = torch.exp(-(freqs_ratio / harmonic_width)**2)
  if normalize:
    # where(sum > 1, safe_divide(w, sum), w).  The branch not taken gets no gradient,
    # but torch's division backward forms w / sum^2, which is 0 / 0 where a sum of
    # underflowing weights squares to 0; dividing by 1 there instead changes no value.
    weights_sum = torch.sum(weights, -1, keepdim=True)
    sel = weights_sum > 1.0
    weights = torch.where(sel, safe_divide(weights, torch.where(sel, weights_sum, 1.0)),
                          weights)
  harm_amps = torch.sum(weights * a[:, :, None, :], -1)
  harm_amps = torch.where(harm_freqs >= sample_rate / 2.0, torch.zeros_like(harm_amps),
                          harm_amps)
  harm_amp = torch.sum(harm_amps, -1, keepdim=True)
  return harm_amp, safe_divide(harm_amps, harm_amp)
