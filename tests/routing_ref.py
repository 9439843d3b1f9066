"""float64 references for the routing ops: core.resample (core.py:573-714),
processors.Mix (processors.py:179-233), processors.Crop (236-263),
synths.TensorToAudio (synths.py:23-52) and effects.ExpDecayReverb
(effects.py:121-199).

TEST INFRASTRUCTURE.  Differentiable float64 torch restatements: autograd of them
is "what TF autodiff gives the reference", the yardstick of the backward kernels.
tests/test_routing.py pins each one to the unmodified reference run wide (float64)
on the NumPy shim at <= 1e-12.

`resample` takes its sample -> frame indices from TensorFlow's float32 index math
(scale and src = t * scale in float32), as the legacy resize kernels and the CUDA
kernel do; the weights are float64 ('window': the Hann overlap-add's raised cosine,
'linear': src - floor(src), 'cubic': TensorFlow's float32 coefficient table).  It
is a sparse linear map, out[t] = sum_k w[t, k] x[idx[t, k]], so its autograd is the
transpose that scatters every tap, clamped ones included (a NaN upstream gradient
reaches every frame its sample touches, as in TensorFlow's resize gradients).
"""
import numpy as np
import torch


def _cubic_table():
  """resize_bicubic_op.cc InitCoeffsTable(A = -0.75), float32 entries."""
  a = -0.75
  x = np.arange(1025) / 1024.0
  t0 = ((a + 2) * x - (a + 3)) * x * x + 1
  y = x + 1.0
  t1 = ((a * y - 5 * a) * y + 8 * a) * y - 4 * a
  return t0.astype(np.float32).astype(np.float64), t1.astype(np.float32).astype(np.float64)


def resample_taps(n_frames, n_timesteps, method, add_endpoint=True):
  """(idx [N, k] int64, w [N, k] float64) of core.resample from F frames to N
  samples: k = 2 ('window', 'linear'), 1 ('nearest'), 4 ('cubic')."""
  F, N = int(n_frames), int(n_timesteps)
  t = np.arange(N)
  if method == 'window':
    hop = N // F if add_endpoint else N // (F - 1)
    i = t // hop
    r = t - i * hop
    w1 = 0.5 - 0.5 * np.cos(np.pi * r / hop)
    return (np.stack([i, np.minimum(i + 1, F - 1)], 1),
            np.stack([1.0 - w1, w1], 1))
  align = not add_endpoint and N > 1
  scale = np.float32(F - 1) / np.float32(N - 1) if align else np.float32(F) / np.float32(N)
  src = (t.astype(np.float32) * scale).astype(np.float32)
  fl = np.floor(src)
  if method == 'linear':
    frac = (src - fl).astype(np.float64)
    lo = np.minimum(np.maximum(fl.astype(np.int64), 0), F - 1)
    hi = np.minimum(np.ceil(src).astype(np.int64), F - 1)
    return np.stack([lo, hi], 1), np.stack([1.0 - frac, frac], 1)
  if method == 'nearest':
    # C roundf: halves away from zero (src >= 0; the + 0.5 is exact in float64)
    i = np.floor(src.astype(np.float64) + 0.5) if align else fl
    return np.minimum(i.astype(np.int64), F - 1)[:, None], np.ones((N, 1))
  if method == 'cubic':
    t0, t1 = _cubic_table()
    loc = fl.astype(np.int64)
    off = np.rint((src - fl).astype(np.float32) * np.float32(1024)).astype(np.int64)
    w = np.stack([t1[off], t0[off], t0[1024 - off], t1[1024 - off]], 1)
    idx = np.clip(loc[:, None] + np.arange(-1, 3)[None, :], 0, F - 1)
    return idx, w
  raise ValueError(method)


def resample(inputs, n_timesteps, method='linear', add_endpoint=True):
  """core.resample of a 1-D ... 4-D float64 torch tensor (4-D: the 3-D case over
  n_freq * channels, core.py:616-621)."""
  x = inputs.to(torch.float64)
  shape = tuple(x.shape)
  if x.dim() == 1:
    x = x[None, :, None]
  elif x.dim() == 2:
    x = x[:, :, None]
  elif x.dim() == 4:
    x = x.reshape(shape[0], shape[1], shape[2] * shape[3])
  idx, w = resample_taps(x.shape[1], n_timesteps, method, add_endpoint)
  idx = torch.from_numpy(idx).to(x.device)
  w = torch.from_numpy(w).to(x.device)
  out = sum(x[:, idx[:, k], :] * w[None, :, k, None] for k in range(idx.shape[1]))
  if len(shape) == 1:
    return out[0, :, 0]
  if len(shape) == 2:
    return out[:, :, 0]
  if len(shape) == 4:
    return out.reshape(shape[0], int(n_timesteps), shape[2], shape[3])
  return out


def mix(signal_one, signal_two, mix_level):
  """processors.Mix.get_signal (processors.py:217-233)."""
  return (torch.sqrt(torch.abs(mix_level)) * signal_one +
          (1.0 - torch.sqrt(torch.abs(mix_level - 1.0))) * signal_two)


def mix_processor(signal_one, signal_two, nn_out_mix_level):
  """processors.Mix end to end: sigmoid, 'linear' resample to N, crossfade."""
  level = resample(torch.sigmoid(nn_out_mix_level.to(torch.float64)), signal_one.shape[1])
  return mix(signal_one, signal_two, level)


def crop(audio, frame_size, crop_location='back'):
  """processors.Crop.get_signal (processors.py:253-263)."""
  half = int(frame_size // 2)
  pad = 2 * half
  if crop_location == 'front':
    return audio[:, pad:]
  if crop_location == 'center':
    return audio[:, half:-half]
  if crop_location == 'back':
    return audio[:, :-pad]
  raise ValueError(crop_location)


def linspace01(n, device=None):
  """tf.linspace(0, 1, n) in float64: delta * [0 .. n-2], then 1 appended."""
  if n == 1:
    return torch.zeros(1, dtype=torch.float64, device=device)
  delta = 1.0 / (n - 1)
  body = delta * torch.arange(n - 1, dtype=torch.float64, device=device)
  return torch.cat([body, torch.ones(1, dtype=torch.float64, device=device)])


def exp_decay_ir(gain, decay, reverb_length, noise):
  """ExpDecayReverb._get_ir (effects.py:144-151) on the SCALED gain [rows, 1], raw
  decay [rows, 1] and one noise row [1, L]."""
  gain = gain.to(torch.float64).reshape(-1, 1)
  decay = decay.to(torch.float64).reshape(-1, 1)
  time = linspace01(int(reverb_length), gain.device)[None, :]
  return gain * torch.exp(-(2.0 + torch.exp(decay)) * time) * noise.to(torch.float64)


def exp_sigmoid(x, exponent=10.0, max_value=2.0, threshold=1e-7):
  """core.exp_sigmoid (core.py:386-404)."""
  return max_value * torch.sigmoid(x)**np.log(exponent) + threshold


def reverb(audio, ir, add_dry=True):
  """Reverb.get_signal (effects.py:103-117): the dry tap zeroed, 'same'
  convolution with zero delay compensation, plus the dry signal."""
  audio = audio.to(torch.float64)
  ir = ir.to(torch.float64)
  ir = torch.cat([torch.zeros_like(ir[:, :1]), ir[:, 1:]], 1)
  n, s = audio.shape[-1], ir.shape[-1]
  m = n + s - 1
  wet = torch.fft.irfft(torch.fft.rfft(audio, m) * torch.fft.rfft(ir, m), m)[:, :n]
  return wet + audio if add_dry else wet


def exp_decay_reverb(audio, gain, decay, noise, reverb_length, add_dry=True,
                     scale_fn=exp_sigmoid):
  """effects.ExpDecayReverb end to end from the raw gain and decay ([rows, 1];
  rows 1 is the trainable variant, tiled over the batch)."""
  g = scale_fn(gain.to(torch.float64)) if scale_fn is not None else gain
  ir = exp_decay_ir(g, decay, reverb_length, noise)
  if ir.shape[0] == 1 and audio.shape[0] > 1:
    ir = ir.repeat(audio.shape[0], 1)
  return reverb(audio, ir, add_dry)
