"""InverseSynthesis's self-supervised training data (training/data_preparation/
synthetic_data.py): generate_notes_v2 on the CUDA kernel of csrc/synthetic_notes.cuh,
generate_notes with numpy's own draws rendered on the GPU, and the seed list of the
reference's dataset job.

Both generators draw from numpy's legacy RandomState exactly as the reference does, so
for the same seed or the same numpy state they return the reference's examples, and in
state mode leave numpy's global state where the reference leaves it.  Outputs are CUDA
tensors; nothing here requires or records grad (this is a data source).
"""
import numbers
import warnings

import numpy as np
import torch

from ddsp_b200 import _lib
from ddsp_b200 import core


def example_seeds(num_examples, random_seed=42):
  """The per-example seeds of the reference's dataset job:
  np.random.seed(random_seed); np.random.randint(2**32, size=num_examples).  Seeds
  numpy's global state as that job does."""
  np.random.seed(random_seed)
  return np.random.randint(2**32, size=num_examples)


def _count(name, value, low=1):
  if isinstance(value, bool) or not isinstance(value, numbers.Integral) or value < low:
    raise ValueError(f'{name} must be an integer >= {low}, got {value!r}.')
  return int(value)


def _check_shape(n_timesteps, n_harmonics, n_mags):
  t = _count('n_timesteps', n_timesteps)
  k = _count('n_harmonics', n_harmonics)
  m = _count('n_mags', n_mags)
  if not _lib.load().ddsp_b200_synthetic_notes_takes(t, k, m):
    raise ValueError(
        f'generate_notes_v2: n_timesteps={t}, n_harmonics={k}, n_mags={m} is beyond the '
        f'kernel (n_timesteps <= {_lib.SYNTHETIC_MAX_T}, n_harmonics and n_mags <= '
        f'{_lib.SYNTHETIC_MAX_BANDS}).')
  return t, k, m


def _device(device):
  if device is None:
    return torch.device('cuda', torch.cuda.current_device())
  device = torch.device(device)
  if device.type != 'cuda':
    raise ValueError(f'generate_notes_v2 runs on a CUDA device, got {device}.')
  if device.index is None:
    device = torch.device('cuda', torch.cuda.current_device())
  return device


def _seeds(seeds, device):
  """The seeds as an int64 tensor on `device`, checked to lie in [0, 2**32).  Host
  seeds go through pinned memory without a synchronisation; a CUDA tensor is checked
  with one read of its extremes."""
  if isinstance(seeds, torch.Tensor) and seeds.is_cuda:
    if seeds.dtype.is_floating_point or seeds.dtype == torch.bool or seeds.dim() != 1:
      raise ValueError('seeds must be a 1-D integer tensor.')
    s = seeds.to(device=device, dtype=torch.int64).contiguous()
    if s.numel() and (int(s.min()) < 0 or int(s.max()) >= 2**32):
      raise ValueError('Seed must be between 0 and 2**32 - 1')
    return s
  arr = np.asarray(seeds.cpu() if isinstance(seeds, torch.Tensor) else seeds)
  if arr.ndim != 1 or not (arr.size == 0 or np.issubdtype(arr.dtype, np.integer)):
    raise ValueError('seeds must be a 1-D sequence of integers.')
  arr = arr.astype(object) if arr.dtype == object else arr
  if arr.size and (min(int(x) for x in arr) < 0 or max(int(x) for x in arr) >= 2**32):
    raise ValueError('Seed must be between 0 and 2**32 - 1')
  host = torch.tensor(np.asarray(arr, dtype=np.int64), dtype=torch.int64)
  return host.pin_memory().to(device, non_blocking=True)


def _controls(harm_amp, harm_dist, f0_midi, mags, divisor, get_controls):
  """The reference's TF steps after its numpy arrays (harm_amp [B, T], f0_midi [B, T]
  float64): exp_sigmoid and the divisor, midi_to_hz, a float64 softmax,
  remove_above_nyquist of f0 itself (the reference's comparison), safe_divide and
  harmonic_to_sinusoidal."""
  harm_amp = harm_amp[..., None]
  if get_controls:
    harm_amp = core.exp_sigmoid(harm_amp) / divisor.to(torch.float32)[:, None, None]
  f0_hz = core.midi_to_hz(f0_midi[..., None])
  if get_controls:
    harm_dist = torch.softmax(harm_dist, dim=-1)
    harm_dist = core.remove_above_nyquist(f0_hz, harm_dist)
    harm_dist = core.safe_divide(harm_dist, torch.sum(harm_dist, dim=-1, keepdim=True))
    mags = core.exp_sigmoid(mags)
  sin_amps, sin_freqs = core.harmonic_to_sinusoidal(harm_amp, harm_dist, f0_hz)
  return {'harm_amp': harm_amp, 'harm_dist': harm_dist, 'f0_hz': f0_hz,
          'sin_amps': sin_amps, 'sin_freqs': sin_freqs, 'noise_magnitudes': mags}


@torch.no_grad()
def generate_notes_v2(n_batch=1, n_timesteps=125, n_harmonics=100, n_mags=65,
                      min_note_length=5, max_note_length=25, p_silent=0.1, p_vibrato=0.5,
                      get_controls=True, *, seeds=None, device=None):
  """synthetic_data.generate_notes_v2: notes of random length with blended amplitude,
  harmonic distribution, f0 (with or without vibrato) and noise magnitudes.

  seeds=None continues numpy's global RandomState, as the reference does, and returns
  with numpy's state where the reference leaves it (one synchronisation).  A sequence
  or tensor of seeds gives item b the reference's np.random.seed(seeds[b]);
  generate_notes_v2(n_batch=1) (its n_batch is len(seeds)), leaves numpy's state
  alone and does not synchronise.  Returns the reference's dict of CUDA tensors:
  float32, except harm_amp, harm_dist and noise_magnitudes, which stay float64 without
  get_controls."""
  t, k, m = _check_shape(n_timesteps, n_harmonics, n_mags)
  lo = _count('min_note_length', min_note_length)
  hi = _count('max_note_length', max_note_length)
  if lo > hi:
    raise ValueError('low >= high')
  get_controls = bool(get_controls)
  dev = _device(device)
  state = seeds is None
  if state:
    b = _count('n_batch', n_batch, low=0)
    seed_t = None
  else:
    seed_t = _seeds(seeds, dev)
    b = seed_t.numel()
  with torch.cuda.device(dev):
    # the kernel writes every element; the package's uninitialised allocations are
    # confined to the modules its memory guard covers, so these are zeros
    f64 = dict(dtype=torch.float64, device=dev)
    harm_amp = torch.zeros((b, t), **f64)
    harm_dist = torch.zeros((b, t, k), **f64)
    f0_midi = torch.zeros((b, t), **f64)
    mags = torch.zeros((b, t, m), **f64)
    divisor = torch.zeros((b,), **f64) if get_controls else None
    key = pos = gauss = None
    if state:
      _, key_np, pos_np, has_gauss, cached = np.random.get_state()
      key = torch.tensor(np.ascontiguousarray(key_np, np.uint32).view(np.int32), device=dev)
      pos = torch.tensor([int(pos_np), int(has_gauss)], dtype=torch.int32, device=dev)
      gauss = torch.tensor([float(cached)], **f64)
    if b or state:
      core._launch('ddsp_b200_synthetic_notes', seed_t, key, pos, gauss, harm_amp,
                   harm_dist, f0_midi, mags, divisor, b, t, k, m, lo, hi, float(p_silent),
                   float(p_vibrato), int(get_controls))
    if state:
      key_out = key.cpu().numpy().view(np.uint32)
      pos_out = pos.cpu().numpy()
      np.random.set_state(('MT19937', key_out, int(pos_out[0]), int(pos_out[1]),
                           float(gauss.cpu()[0])))
    return _controls(harm_amp, harm_dist, f0_midi, mags, divisor, get_controls)


def _line_table(n_harmonics, exponents):
  """-tf.linspace(0.0, float(i), K) ** exponents[i] for i < 10, in float32 as TF's
  linspace computes it: start + (stop - start) / (K - 1) * [0..K-2], then stop."""
  rows = []
  for i, e in enumerate(exponents):
    stop = np.float32(i)
    if n_harmonics == 1:
      line = np.zeros(1, np.float32)
    else:
      delta = (stop - np.float32(0.0)) / np.float32(n_harmonics - 1)
      body = np.float32(0.0) + delta * np.arange(n_harmonics - 1, dtype=np.float32)
      line = np.concatenate([body, [stop]]).astype(np.float32)
    rows.append(-(line ** np.float32(e)))
  return np.stack(rows)


@torch.no_grad()
def generate_notes(n_batch, n_timesteps, n_harmonics=100, n_mags=65, get_controls=True,
                   *, device=None):
  """synthetic_data.generate_notes (v1): n_notes uniform segments resampled to
  n_timesteps.  Its few array-shaped draws are numpy's own, made on the host in the
  reference's order (so numpy's global state advances as the reference's does); the
  resampling, the line table sum and the controls run on the GPU."""
  b = _count('n_batch', n_batch, low=0)
  t, k, m = _check_shape(n_timesteps, n_harmonics, n_mags)
  dev = _device(device)
  rs = np.random
  with warnings.catch_warnings():   # random_integers is deprecated; the reference calls it
    warnings.simplefilter('ignore', DeprecationWarning)
    n_notes = rs.random_integers(1, 20)
  amp_method = 'nearest' if rs.uniform() <= 0.5 else 'linear'
  amp = rs.uniform(-2, 2, [b, n_notes, 1])
  note_midi = rs.uniform(24.0, 84.0, [b, n_notes, 1])
  dist_method = 'nearest' if rs.uniform() <= 0.5 else 'linear'
  exponents = [rs.uniform(1.0, 6.0) for _ in range(10)]
  lines_dist = rs.uniform(0.0, 1.0, [b, n_notes, 10])
  mags_method = 'nearest' if rs.uniform() <= 0.5 else 'linear'
  mags_hi = rs.uniform(-4.0, 0.0)
  mags = rs.uniform(-6.0, mags_hi, [b, n_notes, m])

  def up(x, method):
    return core.resample(torch.tensor(x, dtype=torch.float32, device=dev), t, method=method)

  with torch.cuda.device(dev):
    harm_amp = up(amp, amp_method)
    if get_controls:
      harm_amp = core.exp_sigmoid(harm_amp)
    f0_hz = core.midi_to_hz(up(note_midi, 'nearest'))
    lines = torch.tensor(_line_table(k, exponents), device=dev)
    harm_dist = torch.sum(up(lines_dist, dist_method)[..., None] * lines[None, None], dim=-2)
    if get_controls:
      harm_dist = core.exp_sigmoid(harm_dist)
      harm_dist = core.remove_above_nyquist(f0_hz, harm_dist)
      harm_dist = core.safe_divide(harm_dist, torch.sum(harm_dist, dim=-1, keepdim=True))
    mags = up(mags, mags_method)
    if get_controls:
      mags = core.exp_sigmoid(mags)
    sin_amps, sin_freqs = core.harmonic_to_sinusoidal(harm_amp, harm_dist, f0_hz)
  return {'harm_amp': harm_amp, 'harm_dist': harm_dist, 'f0_hz': f0_hz,
          'sin_amps': sin_amps, 'sin_freqs': sin_freqs, 'noise_magnitudes': mags}
