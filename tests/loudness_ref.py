"""Float64 torch restatement of spectral_ops.compute_loudness (spectral_ops.py:254-324)
and compute_power (spectral_ops.py:223-249), differentiable, with TensorFlow's tie
rule for tf.maximum: the gradient goes to the FIRST argument on ties, so
max(pmin, p) passes a gradient to p only where p > pmin, and max(dB, -range_db) passes
one to dB where dB >= -range_db.  torch.maximum would split ties in half, so the
clamps are torch.where.  Pinned to the unmodified reference by
tests/golden/loudness.npz."""
import numpy as np
import torch

DB_RANGE = 80.0


def fft_frequencies(*, sr=22050, n_fft=2048):
  """librosa.fft_frequencies: centre frequencies of the rfft bins, k * sr / n_fft."""
  return np.fft.rfftfreq(n=n_fft, d=1.0 / sr)


def A_weighting(frequencies, *, min_db=-80.0):  # noqa: N802 (librosa's name)
  """librosa.A_weighting: IEC 61672 A-weighting in dB from librosa's closed form,
  clipped below at min_db."""
  f_sq = np.asanyarray(frequencies) ** 2.0
  c = np.array([12194.217, 20.598997, 107.65265, 737.86223]) ** 2.0
  with np.errstate(divide='ignore'):
    a = 2.0 + 20.0 * (np.log10(c[0]) + 2 * np.log10(f_sq) - np.log10(f_sq + c[0])
                      - np.log10(f_sq + c[1]) - 0.5 * np.log10(f_sq + c[2])
                      - 0.5 * np.log10(f_sq + c[3]))
  return a if min_db is None else np.maximum(min_db, a)


def a_weights(sample_rate, n_fft):
  """10^(A / 10) of A_weighting(fft_frequencies(sr, n_fft)), min_db = -80, float64
  [n_fft // 2 + 1]."""
  a = A_weighting(fft_frequencies(sr=sample_rate, n_fft=n_fft))
  return torch.from_numpy(10.0 ** (a / 10.0))


def power_to_db(power, ref_db=0.0, range_db=DB_RANGE):
  """core.power_to_db (core.py:258-272) with tf.maximum's gradient."""
  pmin = 10.0 ** (-range_db / 10.0)
  power = torch.where(power > pmin, power, torch.full_like(power, pmin))
  db = 10.0 * torch.log10(power) - ref_db
  return torch.where(db >= -range_db, db, torch.full_like(db, -range_db))


def frames(audio, frame_size, hop, padding):
  """spectral_ops.pad + tf.signal.frame(pad_end=False): [B, N] -> [B, T, frame]."""
  n = audio.shape[-1]
  if padding == 'center':
    audio = torch.nn.functional.pad(audio, (frame_size // 2, frame_size // 2))
  elif padding == 'same':
    n_frames = -(-n // hop)
    audio = torch.nn.functional.pad(audio, (0, (n_frames - 1) * hop + frame_size - n))
  if audio.shape[-1] < frame_size:
    return audio.new_zeros(audio.shape[0], 0, frame_size)
  return audio.unfold(-1, frame_size, hop)


def compute_loudness(audio, sample_rate=16000, frame_rate=250, n_fft=512,
                     range_db=DB_RANGE, ref_db=0.0, padding='center'):
  """[B, N] or [N] float64 -> loudness in dB, [B, T] or [T]."""
  x = audio.to(torch.float64)
  is_1d = x.dim() == 1
  x = x[None] if is_1d else x
  hop = sample_rate // frame_rate
  window = torch.hann_window(n_fft, periodic=True, dtype=torch.float64, device=x.device)
  spec = torch.fft.rfft(frames(x, n_fft, hop, padding) * window, dim=-1)
  power = spec.real ** 2 + spec.imag ** 2
  weighted = power * a_weights(sample_rate, n_fft).to(x.device)
  out = power_to_db(weighted.mean(-1), ref_db=ref_db, range_db=range_db)
  return out[0] if is_1d else out


def compute_power(audio, sample_rate=16000, frame_rate=250, frame_size=512, ref_db=0.0,
                  range_db=DB_RANGE, padding='center'):
  """amplitude_to_db(mean(frame^2)^0.5) = power_to_db(mean(frame^2))."""
  x = audio.to(torch.float64)
  is_1d = x.dim() == 1
  x = x[None] if is_1d else x
  ms = (frames(x, frame_size, sample_rate // frame_rate, padding) ** 2).mean(-1)
  out = power_to_db(ms, ref_db=ref_db, range_db=range_db)
  return out[0] if is_1d else out
