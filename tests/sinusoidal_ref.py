"""Reference of the fused Sinusoidal synthesis (core.sinusoidal_synthesis:
synths.Sinusoidal.get_signal, synths.py:305-323, on the reference's
core.resample and core.oscillator_bank, core.py:573-714, 911-962) for the tests
of its backward kernel.

TEST INFRASTRUCTURE.
* `nyquist_mask`: the forward kernel's float32 Nyquist decision, per sample and
  sinusoid.  The gradient of the audio the kernel produced takes this decision
  as given (TensorFlow's tf.where has subgradient 0 in the condition).
* `torch_sinusoidal`: a float64, differentiable torch restatement for
  'window' / 'linear' amplitudes and an integer hop, pinned to the float64
  oracle at <= 1e-12 by tests/test_sinusoidal_backward.py on the CPU.  With
  frame i, offset r and frame F := frame F-1:
    fe(t)  = f_i + (f_{i+1} - f_i) r / hop,     phase(t) = sum_{s<=t} fe(s) / sr
    amp(t) = A_i w0(r) + A_{i+1} w1(r),         audio = sum_k m amp sin(2 pi phase)
  with w1 = 0.5 - 0.5 cos(pi r / hop) ('window', the Hann overlap-add) or r / hop
  ('linear') and w0 = 1 - w1.
"""
import math

import numpy as np
import torch


def _next_frame(x):
  """Frame i + 1 of a [B, F, K] tensor, frame F being a copy of frame F - 1."""
  return torch.cat([x[:, 1:], x[:, -1:]], dim=1)


def nyquist_mask(frequencies, n_samples, sample_rate):
  """[B, N, K] bool, True = silenced: fe >= sr / 2 with fe = lo + (hi - lo) * frac
  in float32, one rounding per operation (no FMA), frac = float32(r) *
  float32(1 / hop) - the forward kernel's arithmetic."""
  f = np.asarray(frequencies, np.float32)
  b, n_frames, k = f.shape
  hop = n_samples // n_frames
  inv_hop = np.float32(1.0) / np.float32(hop)
  frac = (np.arange(hop, dtype=np.float32) * inv_hop)[None, None, :, None]
  lo = f[:, :, None, :]
  hi = np.concatenate([f[:, 1:], f[:, -1:]], axis=1)[:, :, None, :]
  fe = lo + (hi - lo) * frac
  return (fe >= np.float32(sample_rate) * np.float32(0.5)).reshape(b, n_frames * hop, k)


def torch_sinusoidal(frequencies, amplitudes, n_samples, sample_rate=16000,
                     amp_resample_method='window', mask=None):
  """float64 frequencies, amplitudes [B, F, K] -> audio [B, N].  mask: [B, N, K]
  bool tensor (True = silenced) or None for the float64 comparison fe >= sr / 2."""
  b, n_frames, k = frequencies.shape
  hop = n_samples // n_frames
  assert hop * n_frames == n_samples, 'the fused route needs an integer hop'
  r = torch.arange(hop, dtype=frequencies.dtype, device=frequencies.device)
  frac = (r / hop)[None, None, :, None]
  f0 = frequencies[:, :, None, :]
  fe = f0 + (_next_frame(frequencies)[:, :, None, :] - f0) * frac      # [B, F, hop, K]
  if amp_resample_method == 'window':
    w1 = 0.5 - 0.5 * torch.cos(math.pi * frac)
  elif amp_resample_method == 'linear':
    w1 = frac
  else:
    raise ValueError(amp_resample_method)
  amp = (amplitudes[:, :, None, :] * (1.0 - w1) +
         _next_frame(amplitudes)[:, :, None, :] * w1)
  fe = fe.reshape(b, n_samples, k)
  amp = amp.reshape(b, n_samples, k)
  if mask is None:
    mask = fe >= sample_rate / 2.0
  amp = torch.where(mask, torch.zeros_like(amp), amp)
  # the oracle's order: omega = f * 2 pi / sr, then the running sum in radians
  phase = torch.cumsum(fe * (2.0 * math.pi) / sample_rate, dim=1)
  return (amp * torch.sin(phase)).sum(-1)
