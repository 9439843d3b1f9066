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
* `regime`: the frequency regimes the kernel tests sweep.
* `float64_grads`: audio and gradients of float64 autograd through
  `torch_sinusoidal`, with the forward kernel's float32 mask.
* `harmonic_sinusoidal64`: core.harmonic_synthesis on its sinusoidal route
  ((f0 k)(1 + shifts), amplitudes * distribution) restated on `torch_sinusoidal`.
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


def regime(name, B, F, K, sr, seed):
  """Frequencies [B, F, K] in Hz, float32."""
  rng = np.random.default_rng(seed)
  nyq = sr / 2.0
  f = rng.uniform(20.0, 7900.0, (B, F, K))
  if name == 'zero':              # silent sinusoids and silent frames
    f[..., ::2] = 0.0
    f[:, ::3, :] = 0.0
  elif name == 'glide':           # every other frame across Nyquist, both ways
    up = np.where(np.arange(F) % 2 == 0, 0.9, 1.1)[None, :, None]
    f[..., ::2] = nyq * up * rng.uniform(0.95, 1.05, (B, F, 1))
  elif name == 'above':           # sinusoid 0 above Nyquist in every frame
    f[..., 0] = rng.uniform(1.01 * nyq, 1.9 * nyq, (B, F))
  return f.astype(np.float32)


def float64_grads(f32, a32, g, n_samples, sample_rate, method):
  """(audio, d frequencies, d amplitudes) of float64 autograd through
  `torch_sinusoidal` on the device of f32, with the forward kernel's float32 mask."""
  mask = torch.from_numpy(nyquist_mask(f32.cpu().numpy(), n_samples,
                                       sample_rate)).to(f32.device)
  f64 = f32.detach().double().requires_grad_(True)
  a64 = a32.detach().double().requires_grad_(True)
  out = torch_sinusoidal(f64, a64, n_samples, sample_rate, method, mask=mask)
  out.backward(g.double())
  return out.detach(), f64.grad, a64.grad


def harmonic_sinusoidal64(f0, amps, hd, shifts, n_samples, sample_rate, method):
  """core.harmonic_synthesis through its frame-rate oscillator bank in float64.
  The harmonic frequencies take the values of the float32 products the kernel is
  given, (f0 k)(1 + shifts), with their float64 derivatives: a float64 product
  differs by up to half a float32 ulp, which over thousands of cycles of a harmonic
  near Nyquist drifts the phase by 1e-3 rad.  The audio-rate mask is decided on the
  same float32 frequencies."""
  k = hd.shape[-1]
  ratios32 = torch.linspace(1.0, float(k), k, device=f0.device)
  hf32 = f0.detach().float() * ratios32
  if shifts is not None:
    hf32 = hf32 * (1.0 + shifts.detach().float())
  mask = torch.from_numpy(nyquist_mask(hf32.cpu().numpy(), n_samples,
                                       sample_rate)).to(f0.device)
  hf = f0 * ratios32.double()
  if shifts is not None:
    hf = hf * (1.0 + shifts)
  hf = hf + (hf32.double() - hf).detach()
  return torch_sinusoidal(hf, amps * hd, n_samples, sample_rate, method, mask=mask)
