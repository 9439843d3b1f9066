"""Float64 torch restatement of the reference's consistency losses
(losses.py:492-578, 689-1076) and core.harmonic_to_sinusoidal (core.py:784-794),
formula for formula, including tfp's MixtureSameFamily(Categorical, Normal).log_prob
on the reference's broadcast pairwise tensors.  Differentiable: the tests take
float64 autograd gradients of it.  Pinned to the unmodified reference by
tests/golden/consistency.npz.

`ShimMixtureSameFamily`, `ShimCategorical` and `ShimNormal` restate the same three
tfp distributions in NumPy for the reference run on the NumPy TensorFlow shim
(tests/golden/make_consistency_golden.py installs them there for that run only).
"""
import math

import numpy as np
import torch

F64 = torch.float64
HALF_LOG_2PI = 0.5 * math.log(2.0 * math.pi)


def t64(x):
  return x.to(F64) if torch.is_tensor(x) else torch.as_tensor(np.asarray(x), dtype=F64)


# ---- core ------------------------------------------------------------------------
def safe_divide(numerator, denominator, eps=1e-7):
  """eps enters as the float32 constant TensorFlow makes of it."""
  eps = float(np.float32(eps))
  return numerator / torch.where(denominator == 0.0, torch.full_like(denominator, eps),
                                 denominator)


def safe_log(x, eps=1e-5):
  x = t64(x)
  return torch.log(torch.where(x <= 0.0, torch.full_like(x, eps), x))


def logb(x, base=2.0, eps=1e-5):
  return safe_divide(safe_log(x, eps), safe_log(base, eps), eps)


def log10(x, eps=1e-5):
  return logb(x, base=10, eps=eps)


def hz_to_midi(frequencies):
  frequencies = t64(frequencies)
  notes = 12.0 * (logb(frequencies, 2.0) - logb(440.0, 2.0)) + 69.0
  return torch.where(frequencies <= 0.0, torch.zeros_like(notes), notes)


def harmonic_to_sinusoidal(harm_amp, harm_dist, f0_hz, sample_rate=16000):
  harm_amp, harm_dist, f0_hz = t64(harm_amp), t64(harm_dist), t64(f0_hz)
  k = int(harm_dist.shape[-1])
  freqs = f0_hz * torch.linspace(1.0, float(k), k, dtype=F64)[None, None, :]
  harm_dist = torch.where(freqs >= sample_rate / 2.0, torch.zeros_like(harm_dist),
                          harm_dist)
  harm_dist = safe_divide(harm_dist, torch.sum(harm_dist, -1, keepdim=True))
  return harm_amp * harm_dist, freqs


# ---- tfp -------------------------------------------------------------------------
def normal_log_prob(x, loc, scale):
  """tfd.Normal(loc, scale).log_prob(x)."""
  return -0.5 * ((x - loc) / scale)**2 - math.log(scale) - HALF_LOG_2PI


def mixture_log_prob(x, logits, loc, scale):
  """tfd.MixtureSameFamily(tfd.Categorical(logits=logits), tfd.Normal(loc, scale))
  .log_prob(x): x is padded with a component axis, and the component log-probs plus
  log_softmax(logits) are reduced by a max-shifted logsumexp (tf.reduce_logsumexp)."""
  lp = normal_log_prob(x[..., None], loc, scale)
  return torch.logsumexp(lp + torch.log_softmax(logits, dim=-1), dim=-1)


# ---- losses ----------------------------------------------------------------------
def mean_difference(target, value, loss_type='L1', weights=None):
  difference = target - value
  weights = 1.0 if weights is None else weights
  if loss_type.upper() == 'L1':
    return torch.mean(torch.abs(difference * weights))
  assert loss_type.upper() == 'L2'
  return torch.mean(difference**2 * weights)


def amp_loss(amp, amp_target, loss_type='L1', weights=None, log=False, amin=1e-5):
  amp, amp_target = t64(amp), t64(amp_target)
  if log:
    amp = log10(torch.clamp(amp, min=amin))
    amp_target = log10(torch.clamp(amp_target, min=amin))
  return mean_difference(amp, amp_target, loss_type, weights)


def freq_loss(f_hz, f_hz_target, loss_type='L1', weights=None):
  return mean_difference(hz_to_midi(f_hz), hz_to_midi(f_hz_target), loss_type, weights)


def harmonic_consistency(harm_amp, harm_amp_target, harm_dist, harm_dist_target, f0_hz,
                         f0_hz_target, amp_weight=1.0, dist_weight=1.0, f0_weight=1.0,
                         amp_threshold=1e-4):
  weights = (t64(harm_amp_target) >= amp_threshold).to(F64)
  return {
      'harm_amp_loss': amp_weight * amp_loss(harm_amp, harm_amp_target),
      'harm_dist_loss': dist_weight * amp_loss(harm_dist, harm_dist_target,
                                               weights=weights),
      'f0_hz_loss': f0_weight * freq_loss(f0_hz, f0_hz_target, weights=weights),
  }


def _amps_probs(amps):
  amps = torch.where(amps == 0.0, torch.full_like(amps, 1e-7), amps)
  return safe_divide(amps, torch.sum(amps, -1, keepdim=True))


def kde_nll(amps, freqs, amps_target, freqs_target, scale_target):
  """KDEConsistencyLoss.nll: [batch, time]."""
  amps, freqs, amps_target, freqs_target = map(t64, (amps, freqs, amps_target,
                                                     freqs_target))
  logits = torch.log(_amps_probs(amps_target))          # Categorical(probs=...)
  loc = hz_to_midi(freqs_target)
  x = hz_to_midi(freqs).permute(2, 0, 1)                # [freq, batch, time]
  nll = -mixture_log_prob(x, logits, loc, scale_target).permute(1, 2, 0)
  amps_norm = safe_divide(amps, torch.sum(amps, -1, keepdim=True))
  return torch.mean(nll * amps_norm, -1)


def kde_loss(amps_a, freqs_a, amps_b, freqs_b, weight_a=1.0, weight_b=1.0,
             weight_mean_amp=1.0, scale_a=0.1, scale_b=0.1):
  amps_a, freqs_a, amps_b, freqs_b = map(t64, (amps_a, freqs_a, amps_b, freqs_b))
  loss = torch.zeros((), dtype=F64)
  if weight_a > 0.0:
    loss = loss + torch.mean(weight_a * kde_nll(amps_a, freqs_a, amps_b, freqs_b, scale_b))
  if weight_b > 0.0:
    loss = loss + torch.mean(weight_b * kde_nll(amps_b, freqs_b, amps_a, freqs_a, scale_a))
  if weight_mean_amp > 0.0:
    loss = loss + weight_mean_amp * torch.mean(
        torch.abs(torch.mean(amps_a, -1) - torch.mean(amps_b, -1)))
  return loss


TWM_DEFAULTS = dict(sinusoids_weight=1.0, harmonics_weight=1.0, sinusoids_scale=0.5,
                    harmonics_scale=0.2, n_harmonic_points=10, n_harmonic_gaussians=30,
                    softmin_temperature=1.0, sample_rate=16000)


def twm_loss_tensors(f0_candidates, freqs, amps, **kw):
  """TWMLoss.get_loss_tensors: (sinusoids_loss, harmonics_loss), [batch, time, cand]."""
  p = dict(TWM_DEFAULTS, **kw)
  f0_candidates, freqs, amps = map(t64, (f0_candidates, freqs, amps))
  g = p['n_harmonic_gaussians']
  # p(sinusoids | harmonics): Categorical(ones / G) passes the probs as logits
  ratios = safe_divide(freqs[:, :, None, :], f0_candidates[:, :, :, None])
  nll_sinusoids = -mixture_log_prob(ratios, torch.full((g,), 1.0 / g, dtype=F64),
                                    torch.arange(1, g + 1, dtype=F64),
                                    p['harmonics_scale'])
  a = amps[:, :, None, :]
  sinusoids_loss = safe_divide(torch.sum(nll_sinusoids * a, -1), torch.sum(a, -1))
  # p(harmonics | sinusoids)
  n_points = p['n_harmonic_points']
  logits = torch.log(_amps_probs(amps))
  loc = hz_to_midi(freqs)
  n = torch.arange(1, n_points + 1, dtype=F64)
  harmonics = hz_to_midi(f0_candidates[:, :, :, None] * n)
  nll_h = -mixture_log_prob(harmonics.permute(2, 3, 0, 1), logits, loc,
                            p['sinusoids_scale']).permute(2, 3, 0, 1)
  amps_prior = torch.linspace(1.0, 1.0 / n_points, n_points, dtype=F64)
  harmonics_loss = nll_h * amps_prior
  nyquist_mask = (harmonics < hz_to_midi(p['sample_rate'] / 2.0)).to(F64)
  harmonics_loss = harmonics_loss * safe_divide(
      nyquist_mask, torch.mean(nyquist_mask, -1, keepdim=True))
  return sinusoids_loss, torch.mean(harmonics_loss, -1)


def twm_loss(f0_candidates, freqs, amps, **kw):
  p = dict(TWM_DEFAULTS, **kw)
  s, h = twm_loss_tensors(f0_candidates, freqs, amps, **kw)
  combined = p['sinusoids_weight'] * s + p['harmonics_weight'] * h
  return torch.mean(combined * torch.softmax(-combined / p['softmin_temperature'], -1))


def twm_predict_f0(f0_candidates, freqs, amps, **kw):
  p = dict(TWM_DEFAULTS, **kw)
  with torch.no_grad():
    s, h = twm_loss_tensors(f0_candidates, freqs, amps, **kw)
  loss = (p['sinusoids_weight'] * s + p['harmonics_weight'] * h).numpy()
  idx = np.nanargmin(loss, axis=-1)[..., np.newaxis]
  return np.take_along_axis(np.asarray(f0_candidates, np.float64), idx, axis=-1)


# ---- the three tfp distributions on the NumPy shim --------------------------------
def _np(x):
  return np.asarray(x)


class ShimCategorical:
  """tfd.Categorical(logits=None, probs=None): logits_parameter() is log(probs)."""

  def __init__(self, logits=None, probs=None):
    self._logits = None if logits is None else _np(logits)
    self._probs = None if probs is None else _np(probs)

  def logits_parameter(self):
    if self._logits is not None:
      return self._logits
    with np.errstate(divide='ignore'):
      return np.log(self._probs)


class ShimNormal:

  def __init__(self, loc, scale):
    self.loc = _np(loc)
    self.scale = scale

  def log_prob(self, x):
    scale = _np(self.scale).astype(x.dtype)
    z = (x - self.loc) / scale
    return -0.5 * z * z - np.log(scale) - x.dtype.type(HALF_LOG_2PI)


def _logsumexp(v, axis):
  m = np.max(v, axis=axis, keepdims=True)
  m = np.where(np.isfinite(m), m, 0.0)
  return np.log(np.sum(np.exp(v - m), axis=axis)) + np.squeeze(m, axis)


class ShimMixtureSameFamily:
  """tfd.MixtureSameFamily(Categorical, Normal).log_prob, returning a shim tensor of
  the query's dtype."""

  def __init__(self, mixture_distribution, components_distribution):
    self.mixture_distribution = mixture_distribution
    self.components_distribution = components_distribution

  def log_prob(self, x):
    import tensorflow as tf   # the shim, imported by the generator before this call
    xa = _np(x)
    lp = self.components_distribution.log_prob(xa[..., None])
    logits = self.mixture_distribution.logits_parameter().astype(xa.dtype)
    mix = logits - _logsumexp(logits, -1)[..., None]
    return tf.constant(_logsumexp(lp + mix, -1).astype(xa.dtype))
