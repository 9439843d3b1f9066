"""Float64 torch restatement of spectral_ops.compute_mel / compute_logmel / compute_mfcc /
compute_logmag (spectral_ops.py:67-133), differentiable, with a dense mel matrix from
tf.signal.linear_to_mel_weight_matrix's formula and mfccs_from_log_mel_spectrograms'
DCT as a matrix.  The gradients are TensorFlow's: torch's complex abs passes 0 at
|X| = 0 (div_no_nan) and the log's torch.where passes nothing where mel <= 0.  Pinned to
the unmodified reference by tests/golden/mel.npz; tests/golden/make_mel_golden.py
installs linear_to_mel_weight_matrix and mfccs_from_log_mel_spectrograms from here on
the NumPy TensorFlow shim, which lacks them."""
import numpy as np
import torch


def hertz_to_mel(f):
  """The HTK mel scale TensorFlow uses: 1127 ln(1 + f / 700)."""
  return 1127.0 * np.log(1.0 + np.asarray(f, np.float64) / 700.0)


def linear_to_mel_weight_matrix(num_mel_bins=20, num_spectrogram_bins=129, sample_rate=8000,
                                lower_edge_hertz=125.0, upper_edge_hertz=3800.0, dtype=None,
                                name=None):
  """tf.signal.linear_to_mel_weight_matrix (TF <= 2.11) in float64: [K, bins]."""
  if num_mel_bins <= 0:
    raise ValueError('num_mel_bins must be positive. Got: %s' % num_mel_bins)
  if lower_edge_hertz < 0.0:
    raise ValueError('lower_edge_hertz must be non-negative. Got: %s' % lower_edge_hertz)
  if lower_edge_hertz >= upper_edge_hertz:
    raise ValueError('lower_edge_hertz %.1f >= upper_edge_hertz %.1f' %
                     (lower_edge_hertz, upper_edge_hertz))
  if sample_rate <= 0.0:
    raise ValueError('sample_rate must be positive. Got: %s' % sample_rate)
  if upper_edge_hertz > sample_rate / 2:
    raise ValueError('upper_edge_hertz must not be larger than the Nyquist frequency '
                     '(sample_rate / 2). Got %s for sample_rate: %s' %
                     (upper_edge_hertz, sample_rate))
  # HTK excludes the DC bin; it is padded back as a zero row
  freqs = np.linspace(0.0, sample_rate / 2.0, int(num_spectrogram_bins))[1:]
  spec_mel = hertz_to_mel(freqs)[:, None]
  edges = np.linspace(hertz_to_mel(lower_edge_hertz), hertz_to_mel(upper_edge_hertz),
                      int(num_mel_bins) + 2)
  lower, center, upper = edges[None, :-2], edges[None, 1:-1], edges[None, 2:]
  lower_slopes = (spec_mel - lower) / (center - lower)
  upper_slopes = (upper - spec_mel) / (upper - center)
  w = np.maximum(0.0, np.minimum(lower_slopes, upper_slopes))
  return np.pad(w, [[1, 0], [0, 0]])


def dct_matrix(bins):
  """[bins, bins] C with x @ C = dct_II(x, norm=None) * rsqrt(2 bins):
  C[n, k] = 2 cos(pi k (2n + 1) / (2 bins)) / sqrt(2 bins)."""
  n = np.arange(bins, dtype=np.float64)[:, None]
  k = np.arange(bins, dtype=np.float64)[None, :]
  return 2.0 * np.cos(np.pi * k * (2.0 * n + 1.0) / (2.0 * bins)) / np.sqrt(2.0 * bins)


def mfccs_from_log_mel_spectrograms(log_mel_spectrograms, name=None):
  """tf.signal.mfccs_from_log_mel_spectrograms on a NumPy array or torch tensor."""
  x = log_mel_spectrograms
  c = dct_matrix(x.shape[-1])
  if torch.is_tensor(x):
    return x @ torch.from_numpy(c).to(x.device, x.dtype)
  return np.asarray(x) @ c


def stft(audio, frame_size=2048, overlap=0.75, pad_end=True):
  """tf.signal.stft as spectral_ops.stft calls it, float64: [B, N] / [N] / [B, N, 1] ->
  complex [B, T, K] / [T, K]."""
  x = audio.to(torch.float64)
  if x.dim() == 3:
    x = x[..., 0]
  is_1d = x.dim() == 1
  x = x[None] if is_1d else x
  frame_size = int(frame_size)
  step = int(frame_size * (1.0 - overlap))
  fft_length = 1 << (frame_size - 1).bit_length()
  n = x.shape[-1]
  if pad_end:
    n_frames = -(-n // step)
    x = torch.nn.functional.pad(x, (0, max(0, (n_frames - 1) * step + frame_size - n)))
  else:
    n_frames = max(0, 1 + (n - frame_size) // step)
  if n_frames == 0:
    s = x.new_zeros((x.shape[0], 0, fft_length // 2 + 1), dtype=torch.complex128)
    return s[0] if is_1d else s
  frames = x.unfold(-1, frame_size, step)[:, :n_frames]
  window = torch.hann_window(frame_size, periodic=frame_size % 2 == 0, dtype=torch.float64,
                             device=x.device)
  s = torch.fft.rfft(frames * window, n=fft_length, dim=-1)
  return s[0] if is_1d else s


def safe_log(x, eps=1e-5):
  return torch.log(torch.where(x <= 0.0, torch.full_like(x, eps), x))


def compute_mag(audio, size=2048, overlap=0.75, pad_end=True):
  return stft(audio, size, overlap, pad_end).abs()


def compute_logmag(audio, size=2048, overlap=0.75, pad_end=True):
  return safe_log(compute_mag(audio, size, overlap, pad_end))


def compute_mel(audio, lo_hz=0.0, hi_hz=8000.0, bins=64, fft_size=2048, overlap=0.75,
                pad_end=True, sample_rate=16000):
  mag = compute_mag(audio, fft_size, overlap, pad_end)
  w = linear_to_mel_weight_matrix(bins, mag.shape[-1], sample_rate, lo_hz, hi_hz)
  return mag @ torch.from_numpy(w).to(mag.device)


def compute_logmel(audio, lo_hz=80.0, hi_hz=7600.0, bins=64, fft_size=2048, overlap=0.75,
                   pad_end=True, sample_rate=16000):
  return safe_log(compute_mel(audio, lo_hz, hi_hz, bins, fft_size, overlap, pad_end,
                              sample_rate))


def compute_mfcc(audio, lo_hz=20.0, hi_hz=8000.0, fft_size=1024, mel_bins=128, mfcc_bins=13,
                 overlap=0.75, pad_end=True, sample_rate=16000):
  logmel = compute_logmel(audio, lo_hz, hi_hz, mel_bins, fft_size, overlap, pad_end,
                          sample_rate)
  return mfccs_from_log_mel_spectrograms(logmel)[..., :mfcc_bins]
