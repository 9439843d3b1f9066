"""Float64 references of core.wavetable_synthesis (core.py:1238-1282): a NumPy
oracle and a differentiable torch restatement, both written from the maths, not
from the reference's tensors.  Neither builds the [B, N, W + 1] weights: each
sample reads two columns of the (time-interpolated) table.

  phi(t) = sum_{s<t} f0(s) / sr  mod 1      f0 resampled 'linear' to N
  pos = phi W,  j0 = floor(pos),  j1 = (j0 + 1) mod W
  out(t) = amp(t) ((1 - frac) T_t[j0] + frac T_t[j1])     amp resampled 'window'

T_t is the table interpolated in time with the 'linear' resample taps (Fw > 1), or
the one static table.  The torch restatement's d phase is 0 where pos is an
integer (TensorFlow's subgradients of |.| and relu at 0)."""
import numpy as np
import torch


def linear_taps(F, N, index32=False):
  """core.resample 'linear' with add_endpoint: per sample the two frames and their
  weights, from the float64 index (the wide reference) or, with index32, from the
  float32 index of the library's resample kernel."""
  if index32:
    scale = np.float32(F) / np.float32(N)
    src = (np.arange(N, dtype=np.float32) * scale).astype(np.float64)
  else:
    src = np.arange(N, dtype=np.float64) * (F / N)
  fl = np.floor(src)
  i0 = np.clip(fl.astype(np.int64), 0, F - 1)
  i1 = np.minimum(np.ceil(src).astype(np.int64), F - 1)
  return i0, i1, src - fl


def window_taps(F, N):
  """core.upsample_with_windows with add_endpoint (N % F == 0, F < N)."""
  hop = N // F
  t = np.arange(N)
  i = t // hop
  w1 = 0.5 - 0.5 * np.cos(np.pi * (t - i * hop) / hop)
  return i, np.minimum(i + 1, F - 1), w1


def _tables(wavetables):
  w = np.asarray(wavetables, np.float64)
  return w[:, None, :] if w.ndim == 2 else w


def wavetable_synthesis(f0, amps, wavetables, n_samples, sample_rate):
  """NumPy float64 oracle.  f0 [B, Ff(, 1)], amps [B, Fa(, 1)], wavetables
  [B, W] or [B, Fw, W] -> [B, N]."""
  f0 = np.asarray(f0, np.float64).reshape(len(f0), -1)
  amps = np.asarray(amps, np.float64).reshape(len(amps), -1)
  tab = _tables(wavetables)
  B, Fw, W = tab.shape
  N = int(n_samples)
  i0, i1, fr = linear_taps(f0.shape[1], N)
  f = f0[:, i0] + (f0[:, i1] - f0[:, i0]) * fr
  a0, a1, w1 = window_taps(amps.shape[1], N)
  amp = amps[:, a0] * (1 - w1) + amps[:, a1] * w1
  cum = np.concatenate([np.zeros((B, 1)), np.cumsum(f / sample_rate, axis=1)[:, :-1]], 1)
  pos = (cum % 1.0) * W
  j0 = np.floor(pos).astype(np.int64)
  frac = pos - j0
  j1 = (j0 + 1) % W
  b = np.arange(B)[:, None]
  if Fw == 1:
    v0, v1 = tab[b, 0, j0], tab[b, 0, j1]
  else:
    k0, k1, tw = linear_taps(Fw, N)
    v0 = tab[b, k0, j0] + (tab[b, k1, j0] - tab[b, k0, j0]) * tw
    v1 = tab[b, k0, j1] + (tab[b, k1, j1] - tab[b, k0, j1]) * tw
  return amp * ((1 - frac) * v0 + frac * v1)


def torch_wavetable_synthesis(f0, amps, wavetables, n_samples, sample_rate,
                              f0_index32=False):
  """Differentiable float64 torch restatement (same arguments as the oracle, torch
  tensors [B, Ff], [B, Fa], [B, Fw, W]).  f0_index32: resample f0 with the float32
  index of the library's resample kernel, as core.wavetable_synthesis does when the
  f0 and amplitude frame counts differ or do not divide N."""
  B, Fw, W = wavetables.shape
  N = int(n_samples)
  i0, i1, fr = (torch.as_tensor(v, device=f0.device)
                for v in linear_taps(f0.shape[1], N, f0_index32))
  f = f0[:, i0] + (f0[:, i1] - f0[:, i0]) * fr
  a0, a1, w1 = (torch.as_tensor(v, device=f0.device) for v in window_taps(amps.shape[1], N))
  amp = amps[:, a0] * (1 - w1) + amps[:, a1] * w1
  cum = torch.cumsum(f / sample_rate, dim=1)
  cum = torch.cat([torch.zeros_like(cum[:, :1]), cum[:, :-1]], 1)
  pos = torch.remainder(cum, 1.0) * W
  j0 = torch.floor(pos).detach()
  frac = pos - j0
  frac = torch.where(frac == 0, frac.detach(), frac)      # subgradient 0 on the knots
  j0 = j0.long().clamp(0, W - 1)
  j1 = (j0 + 1) % W
  b = torch.arange(B, device=f0.device)[:, None]
  if Fw == 1:
    v0, v1 = wavetables[b, 0, j0], wavetables[b, 0, j1]
  else:
    k0, k1, tw = (torch.as_tensor(v, device=f0.device) for v in linear_taps(Fw, N))
    v0 = wavetables[b, k0, j0] + (wavetables[b, k1, j0] - wavetables[b, k0, j0]) * tw
    v1 = wavetables[b, k0, j1] + (wavetables[b, k1, j1] - wavetables[b, k0, j1]) * tw
  return amp * ((1 - frac) * v0 + frac * v1)


def knot_margin(f0, n_samples, sample_rate, W):
  """Smallest distance, in columns, of a float64 lookup position from a knot."""
  f0 = np.asarray(f0, np.float64).reshape(len(f0), -1)
  i0, i1, fr = linear_taps(f0.shape[1], int(n_samples))
  f = f0[:, i0] + (f0[:, i1] - f0[:, i0]) * fr
  cum = np.concatenate([np.zeros((len(f0), 1)), np.cumsum(f / sample_rate, 1)[:, :-1]], 1)
  pos = (cum % 1.0) * W
  d = np.abs(pos - np.round(pos))
  return float(d[:, 1:].min()) if d.shape[1] > 1 else 1.0
