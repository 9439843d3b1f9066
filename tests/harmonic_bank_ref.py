"""float64 torch restatements of core.harmonic_oscillator_bank (core.py:966-1025) and
core.linear_lookup (core.py:1168-1214), differentiable: the references of the kernels'
forward and backward ("what TF autodiff gives the reference").  torch's cumsum, remainder,
abs and relu have TensorFlow's gradients (remainder passes 1, abs'(0) = relu'(0) = 0).
tests/test_harmonic_oscillator_bank.py and tests/test_linear_lookup.py pin them to the
unmodified reference run on the shim (tests/golden/*.npz).
"""
import numpy as np
import torch

TWO_PI = 2.0 * np.pi


def harmonic_oscillator_bank(frequency, amplitude_envelopes, initial_phase=None,
                             sample_rate=16000, use_angular_cumsum=True):
  """(audio [B, N], final_phase [B, 1, 1]) in float64.  use_angular_cumsum wraps the
  running phase into [0, 2 pi) exactly; the audio does not depend on it."""
  f = torch.as_tensor(frequency, dtype=torch.float64)
  a = torch.as_tensor(amplitude_envelopes, dtype=torch.float64)
  phases = torch.cumsum(f * (TWO_PI / sample_rate), dim=1)
  if use_angular_cumsum:
    phases = torch.remainder(phases, TWO_PI)
  if initial_phase is not None:
    phases = phases + torch.as_tensor(initial_phase, dtype=torch.float64)
  final_phase = phases[:, -1:, 0:1]
  k = torch.arange(1, a.shape[-1] + 1, dtype=torch.float64, device=a.device)
  return (a * torch.sin(phases * k)).sum(-1), final_phase


def float32_grid(w):
  """TensorFlow's float32 linspace(0, 1, w + 1): delta * j, then 1 (as float64)."""
  delta = np.float32(1.0) / np.float32(w)
  lin = np.concatenate([delta * np.arange(w, dtype=np.float32), np.ones(1, np.float32)])
  return lin.astype(np.float64)


def linear_lookup(phase, wavetables):
  """[B, N] in float64 over the float32 grid: relu(1 - |phase - lin_j| W) weights over the
  W + 1 columns, column W being column 0 again."""
  p = torch.as_tensor(phase, dtype=torch.float64)
  t = torch.as_tensor(wavetables, dtype=torch.float64)
  if t.dim() == 2:
    t = t[:, None, :]
  if p.dim() == 2:
    p = p[..., None]
  w = t.shape[-1]
  t = torch.cat([t, t[..., 0:1]], dim=-1)
  lin = torch.as_tensor(float32_grid(w), device=p.device)
  weights = torch.relu(1.0 - torch.abs(p - lin) * w)
  return (weights * t).sum(-1)
