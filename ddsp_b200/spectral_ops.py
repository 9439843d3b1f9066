"""STFT magnitude helpers with the semantics of `ddsp/spectral_ops.py:34-70`.

Consumer of the decoder's audio in the C4 configuration (decoder -> multi-scale
SpectralLoss).  Built on torch's cuFFT-backed FFT as SURVEY.md section 8f-1
prescribes ("torch (cuFFT) first, not a hand kernel"); device-agnostic, so the
CPU tests can pin it against the NumPy oracle.

compute_loudness and compute_power run on hand-written CUDA kernels
(csrc/loudness.cuh) instead: the framed audio would be 32x the input.  So do
compute_mel, compute_logmel and compute_mfcc (csrc/mel.cuh), and everything
PretrainedCREPE does around its network (csrc/crepe.cuh).
"""
import math
import os

import numpy as np
import torch

from ddsp_b200 import _lib
from ddsp_b200 import core


def safe_log(x, eps=1e-5):
  """core.safe_log (core.py:213-216)."""
  return torch.log(torch.where(x <= 0.0, torch.full_like(x, eps), x))


def stft(audio, frame_size=2048, overlap=0.75, pad_end=True):
  """spectral_ops.stft (spectral_ops.py:34-47) = tf.signal.stft with a periodic
  Hann window, frame_step = frame_size * (1 - overlap), fft_length = enclosing
  power of two, and `pad_end` zero padding so that n_frames = ceil(N / step).
  Returns complex [batch, n_frames, fft_length // 2 + 1]."""
  if audio.dim() == 3:
    audio = audio.squeeze(-1)
  audio = audio.to(torch.float32)
  frame_size = int(frame_size)
  step = int(frame_size * (1.0 - overlap))
  n = audio.shape[-1]
  fft_length = 1 << (frame_size - 1).bit_length()
  if pad_end:
    n_frames = -(-n // step)
    padded = (n_frames - 1) * step + frame_size
    audio = torch.nn.functional.pad(audio, (0, max(0, padded - n)))
  else:
    n_frames = max(0, 1 + (n - frame_size) // step)
  frames = audio.unfold(-1, frame_size, step)[..., :n_frames, :]
  window = _hann(frame_size, audio.device)
  return torch.fft.rfft(frames * window, n=fft_length, dim=-1)


def compute_mag(audio, size=2048, overlap=0.75, pad_end=True):
  """spectral_ops.compute_mag (spectral_ops.py:67-70)."""
  return torch.abs(stft(audio, frame_size=size, overlap=overlap, pad_end=pad_end))


def stft_np(audio, frame_size=2048, overlap=0.75, pad_end=True):
  """spectral_ops.stft_np (spectral_ops.py:50-64): the non-differentiable NumPy STFT of
  audio [N] or [batch, N] -> [n_frames, frame_size // 2 + 1] or [batch, n_frames, ...],
  complex64 for float32 audio.  The reference calls librosa.stft(y, n_fft=frame_size,
  hop_length=hop, center=False).T on each example; this restates those semantics
  without librosa: frames of frame_size samples every hop = frame_size * (1 - overlap)
  samples from the first, not centred, times librosa's default window (a periodic Hann
  of length frame_size, in float64), then an rfft of frame_size points.  pad_end pads
  the end with pad(..., 'same') first."""
  assert frame_size * overlap % 2.0 == 0.0
  frame_size = int(frame_size)
  hop_size = int(frame_size * (1.0 - overlap))
  is_2d = (len(audio.shape) == 2)
  if pad_end:
    audio = pad(audio, frame_size, hop_size, 'same', axis=int(is_2d)).cpu().numpy()
  audio = np.asarray(audio)
  window = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(frame_size) / frame_size)
  frames = np.lib.stride_tricks.sliding_window_view(audio, frame_size, axis=-1)
  s = np.fft.rfft(frames[..., ::hop_size, :] * window, axis=-1)
  return s.astype(np.result_type(audio.dtype, np.complex64))


# ---- CUDA pieces of the spectrogram loss (include/ddsp_b200.h) ---------------
_WINDOWS = {}


def _hann(frame_size, device):
  key = (int(frame_size), str(device))
  if key not in _WINDOWS:
    # tf.signal.hann_window: periodic for even lengths, symmetric for odd ones
    _WINDOWS[key] = torch.hann_window(int(frame_size),
                                      periodic=(int(frame_size) % 2 == 0),
                                      dtype=torch.float32, device=device)
  return _WINDOWS[key]


class FrameWindowFn(torch.autograd.Function):
  """stft's framing + periodic Hann window (pad_end=True) as one CUDA kernel,
  and its transpose (windowed overlap-add of the frame gradients) for backward.
  audio [B, N] -> frames [B, ceil(N / step), frame_size]."""

  @staticmethod
  def forward(ctx, audio, frame_size, step):
    frames = _frame_window(audio, frame_size, step)
    ctx.meta = (audio.shape[0], audio.shape[1], frames.shape[1], frame_size, step)
    return frames

  @staticmethod
  def backward(ctx, grad_frames):
    b, n, n_frames, frame_size, step = ctx.meta
    grad_frames = grad_frames.contiguous()
    grad_audio = torch.empty((b, n), dtype=torch.float32, device=grad_frames.device)
    core._launch('ddsp_b200_frame_window_adjoint', grad_frames,
                 _hann(frame_size, grad_frames.device), grad_audio, b, n, n_frames,
                 frame_size, step, None, 0)
    return grad_audio, None, None


def _frame_window(audio, frame_size, step):
  audio = audio.contiguous()
  b, n = audio.shape
  n_frames = -(-n // step)
  frames = torch.empty((b, n_frames, frame_size), dtype=torch.float32,
                       device=audio.device)
  core._launch('ddsp_b200_frame_window', audio, _hann(frame_size, audio.device), frames,
               b, n, n_frames, frame_size, step)
  return frames


class SpectralTermFn(torch.autograd.Function):
  """One FFT size of the 'L1' spectrogram loss (losses.py:102-127, 190-243):
  mag_weight * mean|mag_t - mag_v| + logmag_weight * mean|safe_log mag_t -
  safe_log mag_v| of audio [B, N] against the target's complex STFT.

  forward : framing + Hann (one kernel), cuFFT r2c, ONE pass over both STFTs that
            also leaves the gradient w.r.t. the value STFT, pre-scaled so that the
            transpose of rfft is a plain irfft.
  backward: cuFFT c2r, windowed overlap-add of the frame gradients (one kernel)."""

  @staticmethod
  def forward(ctx, stft_target, audio, frame_size, step, mag_weight, logmag_weight):
    with core._on_device_of(stft_target, audio):
      audio = audio.to(torch.float32).contiguous()
      frames = _frame_window(audio, frame_size, step)
      xv = torch.fft.rfft(frames, n=frame_size, dim=-1)
      del frames
      xt = stft_target.to(torch.complex64).contiguous()
      if xt.data_ptr() % 16:
        xt = xt.clone()   # spectral_l1 reads 16-byte vectors: a view at an odd offset
      if xt.shape != xv.shape:
        raise ValueError(f'target STFT {tuple(xt.shape)} vs value STFT {tuple(xv.shape)}')
      grad = torch.empty_like(xv)
      sums = torch.zeros(2, dtype=torch.float64, device=xv.device)
      m = xv.numel()
      core._launch('ddsp_b200_spectral_l1', xt, xv, grad, sums, m, float(mag_weight),
                   float(logmag_weight), xv.shape[-1], frame_size)
      ctx.save_for_backward(grad)
      ctx.meta = (audio.shape[0], audio.shape[1], xv.shape[1], frame_size, step)
      w = _loss_weights((m,), mag_weight, logmag_weight, xv.device)
      return (sums * w).sum().to(torch.float32)

  @staticmethod
  def backward(ctx, grad_out):
    (grad,) = ctx.saved_tensors
    b, n, n_frames, frame_size, step = ctx.meta
    grad_frames = torch.fft.irfft(grad, n=frame_size, dim=-1).contiguous()
    grad_audio = torch.empty((b, n), dtype=torch.float32, device=grad.device)
    core._launch('ddsp_b200_frame_window_adjoint', grad_frames,
                 _hann(frame_size, grad.device), grad_audio, b, n, n_frames, frame_size,
                 step, None, 0)
    return None, grad_audio * grad_out, None, None, None, None


_LOSS_WEIGHTS = {}


def _loss_weights(counts, mag_weight, logmag_weight, device):
  """[[mag_weight / m, logmag_weight / m] per term] in float64, cached per device: a
  host-to-device copy on every call would keep the loss out of CUDA graph capture."""
  key = (tuple(counts), float(mag_weight), float(logmag_weight), str(device))
  if key not in _LOSS_WEIGHTS:
    _LOSS_WEIGHTS[key] = torch.tensor(
        [[mag_weight / m, logmag_weight / m] for m in counts], dtype=torch.float64,
        device=device)
  return _LOSS_WEIGHTS[key]


# the terms of losses.SpectralLoss in the order of their bits in `terms`
# (DDSP_B200_TERM_*) and of their slots in spectral_terms' sums
_TERMS = (_lib.TERM_MAG, _lib.TERM_DELTA_TIME, _lib.TERM_DELTA_FREQ, _lib.TERM_CUMSUM_FREQ,
          _lib.TERM_LOGMAG)
_TERM_WEIGHTS = {}


def _term_weights(shapes, weights, device):
  """[[weight / element count per term] per FFT size] in float64, cached per device.
  An inactive term (weight <= 0) weighs 0; an active one with no elements (delta_time
  of a single frame) weighs NaN: the mean of nothing, as in the reference."""
  key = (tuple(shapes), tuple(weights), str(device))
  if key not in _TERM_WEIGHTS:
    rows = []
    for b, t, f in shapes:
      counts = (b * t * f, b * (t - 1) * f, b * t * (f - 1), b * t * f, b * t * f)
      rows.append([0.0 if w <= 0 else (w / m if m > 0 else math.nan)
                   for w, m in zip(weights, counts)])
    _TERM_WEIGHTS[key] = torch.tensor(rows, dtype=torch.float64, device=device)
  return _TERM_WEIGHTS[key]


class SpectralLossFn(torch.autograd.Function):
  """The whole multi-scale spectrogram loss (losses.SpectralLoss.call,
  losses.py:194-243) as ONE autograd node: per FFT size framing + Hann (kernel),
  cuFFT r2c of target and value, one pass leaving the loss sums and the value-STFT
  gradient; backward is cuFFT c2r plus a windowed overlap-add per size that
  accumulates, already scaled by the upstream gradient (read on the device), into a
  single dL/d audio buffer.  No elementwise torch op on either pass.

  The `ae.gin` configuration ('L1', mag and logmag only) runs spectral_l1, which
  writes the gradient in place of the value STFT.  Any other configuration ('L1' or
  'L2', any of the five terms) runs spectral_terms; with delta_time its gradient
  goes to a buffer of its own (the kernel reads neighbouring frames)."""

  @staticmethod
  def forward(ctx, target, audio, fft_sizes, mag_weight, logmag_weight,
              delta_time_weight=0.0, delta_freq_weight=0.0, cumsum_freq_weight=0.0,
              loss_type='L1'):
    weights = tuple(float(w) for w in (mag_weight, delta_time_weight, delta_freq_weight,
                                       cumsum_freq_weight, logmag_weight))
    loss_type = loss_type.upper()
    if loss_type not in ('L1', 'L2'):
      raise ValueError(f"SpectralLossFn: loss_type must be 'L1' or 'L2', got {loss_type!r}")
    l1_only = loss_type == 'L1' and max(weights[1:4]) <= 0
    terms = sum(bit for bit, w in zip(_TERMS, weights) if w > 0)
    with core._on_device_of(target, audio):
      audio = audio.to(torch.float32).contiguous()
      target = target.to(torch.float32).contiguous()
      b, n = audio.shape
      sums = torch.zeros((len(fft_sizes), 2 if l1_only else 5), dtype=torch.float64,
                         device=audio.device)
      grads, counts, shapes = [], [], []
      for idx, size in enumerate(fft_sizes):
        size = int(size)
        step = int(size * 0.25)
        xt = torch.fft.rfft(_frame_window(target, size, step), n=size, dim=-1)
        xv = torch.fft.rfft(_frame_window(audio, size, step), n=size, dim=-1)
        m = xv.numel()
        if l1_only:
          core._launch('ddsp_b200_spectral_l1', xt, xv, xv, sums[idx], m, float(mag_weight),
                       float(logmag_weight), xv.shape[-1], -1)
          grad = xv
        else:
          grad = torch.empty_like(xv) if weights[1] > 0 else xv
          core._launch('ddsp_b200_spectral_terms', xt, xv, grad, sums[idx], *xv.shape,
                       terms, getattr(_lib, 'LOSS_' + loss_type), *weights)
        del xt, xv
        grads.append(grad)               # now holds d loss_size / d X_value, irfft-ready
        counts.append(m)
        shapes.append(tuple(grad.shape))
      ctx.save_for_backward(*grads)
      ctx.meta = (b, n, tuple(int(sz) for sz in fft_sizes))
      if l1_only:
        w = _loss_weights(counts, mag_weight, logmag_weight, audio.device)
      else:
        w = _term_weights(shapes, weights, audio.device)
      return (sums * w).sum().to(torch.float32)

  @staticmethod
  def backward(ctx, grad_out):
    b, n, sizes = ctx.meta
    grads = ctx.saved_tensors
    go = grad_out.to(torch.float32).contiguous()
    grad_audio = torch.empty((b, n), dtype=torch.float32, device=go.device)
    for idx, size in enumerate(sizes):
      step = int(size * 0.25)
      n_frames = -(-n // step)
      # unnormalised inverse (the 1/n pass would be an elementwise kernel over the
      # frames; the loss kernels left the spectrum scaled for exactly this)
      gf = torch.fft.irfft(grads[idx], n=size, dim=-1, norm='forward').contiguous()
      core._launch('ddsp_b200_frame_window_adjoint', gf, _hann(size, go.device), grad_audio,
                   b, n, n_frames, size, step, go, int(idx > 0))
    return None, grad_audio, None, None, None, None, None, None, None


def stft_cuda(audio, frame_size, overlap=0.75):
  """stft(pad_end=True) for CUDA tensors through FrameWindowFn + cuFFT."""
  step = int(frame_size * (1.0 - overlap))
  fft_length = 1 << (int(frame_size) - 1).bit_length()
  frames = FrameWindowFn.apply(core.torch_float32(audio), int(frame_size), step)
  return torch.fft.rfft(frames, n=fft_length, dim=-1)


# ---- loudness and RMS power (spectral_ops.py:136-324, csrc/loudness.cuh) ------
F0_RANGE = 127.0  # MIDI
DB_RANGE = core.DB_RANGE  # dB (80.0)
_A_WEIGHTS = {}


def get_framed_lengths(input_length, frame_size, hop_size, padding='center'):
  """spectral_ops.get_framed_lengths (spectral_ops.py:136-170): (n_frames,
  padded_length) of a strided framing.  'valid' frames the signal as it is,
  'center' adds frame_size samples (n_t / hop + 1 frames) and 'same' pads the end
  so that n_frames = ceil(n_t / hop)."""
  def n_frames(length):
    return (length - frame_size) // hop_size + 1
  if padding == 'valid':
    return n_frames(input_length), input_length
  if padding == 'center':
    return n_frames(input_length + frame_size), input_length + frame_size
  if padding == 'same':
    n = -(-input_length // hop_size)
    return n, (n - 1) * hop_size + frame_size
  raise ValueError('`padding` must be one of [\'center\', \'same\', \'valid\'], '
                   f'received ({padding}).')


def _framing(audio, frame_size, hop_size, padding):
  """spectral_ops.pad's checks in its order, on the shape alone: returns (B, N,
  is_1d, n_frames, padding code).  n_frames is what tf.signal.frame gives on the
  padded signal, 0 when 'valid' audio is shorter than a frame."""
  shape = tuple(audio.shape) if torch.is_tensor(audio) else np.shape(audio)
  if len(shape) == 3 and shape[-1] == 1:
    shape = shape[:2]
  if len(shape) not in (1, 2) or shape[-1] < 1:
    raise ValueError(f'audio must be [batch, n_samples], [n_samples] or '
                     f'[batch, n_samples, 1], got shape {tuple(shape)}')
  _padding_check(frame_size, hop_size, padding)
  n = shape[-1]
  if padding == 'same':
    n_frames = -(-n // hop_size)
  else:
    padded = n + 2 * (frame_size // 2) if padding == 'center' else n
    n_frames = 1 + (padded - frame_size) // hop_size if padded >= frame_size else 0
  return ((1 if len(shape) == 1 else shape[0]), n, len(shape) == 1, n_frames,
          _lib.PADDING[padding])


def _audio_2d(audio, b, n):
  return core.torch_float32(audio).reshape(b, n)


def a_weighting(sample_rate, n_fft, device):
  """10^(A_k / 10) of librosa.A_weighting(librosa.fft_frequencies(sr, n_fft)) with its
  min_db = -80 clip, computed in float64 and cached per (sr, n_fft, device): the
  [n_fft // 2 + 1] float32 weights compute_loudness applies to |X_k|^2."""
  key = (float(sample_rate), int(n_fft), str(device))
  if key not in _A_WEIGHTS:
    f_sq = (np.arange(n_fft // 2 + 1, dtype=np.float64) * (sample_rate / n_fft)) ** 2
    c = np.array([12194.217, 20.598997, 107.65265, 737.86223]) ** 2
    with np.errstate(divide='ignore'):
      a = 2.0 + 20.0 * (np.log10(c[0]) + 2 * np.log10(f_sq) - np.log10(f_sq + c[0])
                        - np.log10(f_sq + c[1]) - 0.5 * np.log10(f_sq + c[2])
                        - 0.5 * np.log10(f_sq + c[3]))
    a = np.maximum(-80.0, a)
    _A_WEIGHTS[key] = torch.as_tensor(10.0 ** (a / 10.0), dtype=torch.float32,
                                      device=device)
  return _A_WEIGHTS[key]


class LoudnessFn(torch.autograd.Function):
  """compute_loudness as one CUDA kernel, and its gradient w.r.t. the audio [B, N]
  (csrc/loudness.cuh: the spectrum is recomputed, never saved)."""

  @staticmethod
  def forward(ctx, audio, weights, n_frames, n_fft, hop, padding, range_db, ref_db):
    b, n = audio.shape
    out = torch.empty((b, n_frames), dtype=torch.float32, device=audio.device)
    core._launch('ddsp_b200_loudness_forward', audio, weights, out, b, n, n_frames, n_fft,
                 hop, padding, range_db, ref_db)
    ctx.save_for_backward(audio, weights)
    ctx.meta = (n_frames, n_fft, hop, padding, range_db, ref_db)
    return out

  @staticmethod
  def backward(ctx, grad):
    audio, weights = ctx.saved_tensors
    n_frames, n_fft, hop, padding, range_db, ref_db = ctx.meta
    b, n = audio.shape
    grad = grad.to(torch.float32).contiguous()
    grad_audio = torch.empty_like(audio)
    core._launch('ddsp_b200_loudness_backward', audio, weights, grad, grad_audio, b, n,
                 n_frames, n_fft, hop, padding, range_db, ref_db)
    return grad_audio, None, None, None, None, None, None, None


def compute_loudness(audio, sample_rate=16000, frame_rate=250, n_fft=512,
                     range_db=DB_RANGE, ref_db=0.0, use_tf=True, padding='center'):
  """spectral_ops.compute_loudness (spectral_ops.py:254-324): A-weighted power in dB,
  [B, N] -> [B, T] and [N] -> [T] ([B, N, 1] is read as [B, N]).  Differentiable
  through LoudnessFn; use_tf=False returns the same values as a NumPy array.  n_fft
  must be a power of two (the reference's weighting only broadcasts then)."""
  hop = int(sample_rate // frame_rate)
  n_fft = int(n_fft)
  b, n, is_1d, n_frames, code = _framing(audio, n_fft, hop, padding)
  if n_fft < 2 or n_fft & (n_fft - 1):
    raise ValueError(f'n_fft ({n_fft}) must be a power of two')
  x = _audio_2d(audio, b, n)
  out = LoudnessFn.apply(x, a_weighting(sample_rate, n_fft, x.device), n_frames, n_fft, hop,
                         code, float(range_db), float(ref_db))
  out = out[0] if is_1d else out
  return out if use_tf else out.detach().cpu().numpy()


def _rms(audio, sample_rate, frame_rate, frame_size, padding, in_db, range_db, ref_db,
         name):
  hop = int(sample_rate // frame_rate)
  frame_size = int(frame_size)
  b, n, is_1d, n_frames, code = _framing(audio, frame_size, hop, padding)
  core._no_grad_path(name, audio)
  x = _audio_2d(audio, b, n)
  out = torch.empty((b, n_frames), dtype=torch.float32, device=x.device)
  core._launch('ddsp_b200_rms_power', x, out, b, n, n_frames, frame_size, hop, code,
               int(in_db), float(range_db), float(ref_db))
  return out[0] if is_1d else out


def compute_rms_energy(audio, sample_rate=16000, frame_rate=250, frame_size=512,
                       padding='center'):
  """spectral_ops.compute_rms_energy (spectral_ops.py:223-231): mean(frame^2)^0.5 per
  frame.  Forward only: an input that requires grad raises."""
  return _rms(audio, sample_rate, frame_rate, frame_size, padding, False, DB_RANGE, 0.0,
              'compute_rms_energy')


def compute_power(audio, sample_rate=16000, frame_rate=250, frame_size=512, ref_db=0.0,
                  range_db=DB_RANGE, padding='center'):
  """spectral_ops.compute_power (spectral_ops.py:234-249): amplitude_to_db of the RMS
  energy, i.e. power_to_db(mean(frame^2)).  Forward only."""
  return _rms(audio, sample_rate, frame_rate, frame_size, padding, True, range_db, ref_db,
              'compute_power')


# ---- mel, log-mel, MFCC and log magnitude (spectral_ops.py:67-133, csrc/mel.cuh) --
MAX_MEL_FFT = 16384
MAX_MEL_BINS = 1024
_MEL_TABLES = {}
_MEL_WINDOWS = {}


def compute_logmag(audio, size=2048, overlap=0.75, pad_end=True):
  """spectral_ops.compute_logmag (spectral_ops.py:92-94): safe_log of compute_mag."""
  return safe_log(compute_mag(audio, size, overlap, pad_end))


def _mel_arguments(num_mel_bins, sample_rate, lower_edge_hertz, upper_edge_hertz):
  """The checks of tf.signal.linear_to_mel_weight_matrix, in its order."""
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


def linear_to_mel_weight_matrix(num_mel_bins=20, num_spectrogram_bins=129,
                                sample_rate=8000, lower_edge_hertz=125.0,
                                upper_edge_hertz=3800.0):
  """tf.signal.linear_to_mel_weight_matrix in float64 NumPy, [K, bins]: HTK mel scale
  1127 ln(1 + f / 700), bin frequencies linspace(0, sr / 2, K) with the DC row zero,
  band edges linspace(mel(lo), mel(hi), bins + 2), and each weight
  max(0, min(rising, falling)) in mel space."""
  _mel_arguments(num_mel_bins, sample_rate, lower_edge_hertz, upper_edge_hertz)
  def mel(f):
    return 1127.0 * np.log(1.0 + np.asarray(f, np.float64) / 700.0)
  freqs = np.linspace(0.0, sample_rate / 2.0, num_spectrogram_bins)[1:]
  spec_mel = mel(freqs)[:, None]
  edges = np.linspace(mel(lower_edge_hertz), mel(upper_edge_hertz), num_mel_bins + 2)
  lower, center, upper = edges[None, :-2], edges[None, 1:-1], edges[None, 2:]
  rising = (spec_mel - lower) / (center - lower)
  falling = (upper - spec_mel) / (upper - center)
  w = np.maximum(0.0, np.minimum(rising, falling))
  return np.pad(w, [[1, 0], [0, 0]])


def mel_table(bins, n_spectrogram_bins, sample_rate, lo_hz, hi_hz, device):
  """linear_to_mel_weight_matrix in the sparse layout csrc/mel.cuh reads (one int32
  tensor of 3 K + 2 bins words, include/ddsp_b200.h): per bin its first band and the
  float32 weights into that band and the next, per band its bin range.  Computed in
  float64 and cached per (bins, K, sr, lo, hi, device)."""
  key = (int(bins), int(n_spectrogram_bins), float(sample_rate), float(lo_hz),
         float(hi_hz), str(device))
  if key not in _MEL_TABLES:
    w = linear_to_mel_weight_matrix(bins, n_spectrogram_bins, sample_rate, lo_hz, hi_hz)
    nz = w != 0.0
    rows = np.arange(w.shape[0])
    count = nz.sum(1)
    first = np.where(count > 0, nz.argmax(1), -1)
    nxt = np.minimum(first + 1, bins - 1)
    if (count > 2).any() or ((count == 2) & ~nz[rows, nxt]).any():
      raise AssertionError('mel weights outside two adjacent bands')
    pair = np.zeros((w.shape[0], 2), np.float64)
    pair[:, 0] = np.where(first >= 0, w[rows, np.maximum(first, 0)], 0.0)
    pair[:, 1] = np.where((first >= 0) & (first + 1 < bins), w[rows, nxt], 0.0)
    band_lo = np.zeros(bins, np.int32)
    band_hi = np.zeros(bins, np.int32)
    for j in range(bins):
      ks = np.flatnonzero(nz[:, j])
      if ks.size:
        if ks[-1] + 1 - ks[0] != ks.size:
          raise AssertionError('mel band %d is not one run of bins' % j)
        band_lo[j], band_hi[j] = ks[0], ks[-1] + 1
    words = np.concatenate([pair.astype(np.float32).reshape(-1).view(np.int32),
                            first.astype(np.int32), band_lo, band_hi])
    _MEL_TABLES[key] = torch.as_tensor(words, device=device)
  return _MEL_TABLES[key]


def mel_window(fft_size, device):
  """tf.signal.hann_window(fft_size): periodic for even lengths, symmetric for odd
  ones, computed in float64 and cached as float32 per (fft_size, device)."""
  key = (int(fft_size), str(device))
  if key not in _MEL_WINDOWS:
    n = np.arange(fft_size, dtype=np.float64)
    d = fft_size if fft_size % 2 == 0 else fft_size - 1
    w = 0.5 - 0.5 * np.cos(2.0 * np.pi * n / d) if fft_size > 1 else np.ones(1)
    _MEL_WINDOWS[key] = torch.as_tensor(w, dtype=torch.float32, device=device)
  return _MEL_WINDOWS[key]


class MelFn(torch.autograd.Function):
  """compute_mel / compute_logmel / compute_mfcc as one CUDA kernel, and the gradient
  w.r.t. the audio [B, N] (csrc/mel.cuh: the spectrum and the mel values are
  recomputed, never saved).  meta = (n_frames, fft_size, fft_length, hop, pad_end,
  bins, n_out, mode)."""

  @staticmethod
  def forward(ctx, audio, window, table, meta):
    n_frames, fft_size, fft_length, hop, pad_end, bins, n_out, mode = meta
    b, n = audio.shape
    out = torch.empty((b, n_frames, n_out), dtype=torch.float32, device=audio.device)
    core._launch('ddsp_b200_mel_forward', audio, window, table, out, b, n, n_frames,
                 fft_size, fft_length, hop, pad_end, bins, n_out, mode)
    ctx.save_for_backward(audio, window, table)
    ctx.meta = meta
    return out

  @staticmethod
  def backward(ctx, grad):
    audio, window, table = ctx.saved_tensors
    n_frames, fft_size, fft_length, hop, pad_end, bins, n_out, mode = ctx.meta
    b, n = audio.shape
    if n_frames == 0 or n_out == 0:
      return torch.zeros_like(audio), None, None, None
    grad = grad.to(torch.float32).contiguous()
    grad_audio = torch.empty_like(audio)
    core._launch('ddsp_b200_mel_backward', audio, window, table, grad, grad_audio, b, n,
                 n_frames, fft_size, fft_length, hop, pad_end, bins, n_out, mode)
    return grad_audio, None, None, None


def _mel(audio, lo_hz, hi_hz, bins, fft_size, overlap, pad_end, sample_rate, mode,
         mfcc_bins=None, name='compute_mel'):
  """The shape and argument checks (all before any device work), then MelFn."""
  shape = tuple(audio.shape) if torch.is_tensor(audio) else np.shape(audio)
  if len(shape) == 3 and shape[-1] == 1:
    shape = shape[:2]
  if len(shape) not in (1, 2) or shape[-1] < 1:
    raise ValueError(f'audio must be [batch, n_samples], [n_samples] or '
                     f'[batch, n_samples, 1], got shape {tuple(shape)}')
  fft_size = int(fft_size)
  if fft_size < 1:
    raise ValueError(f'fft_size must be positive, got {fft_size}')
  hop = int(fft_size * (1.0 - overlap))
  if hop < 1:
    raise ValueError(f'frame_step = int(fft_size * (1 - overlap)) must be positive, got '
                     f'{hop} (fft_size {fft_size}, overlap {overlap})')
  bins = int(bins)
  _mel_arguments(bins, sample_rate, lo_hz, hi_hz)
  fft_length = 1 << (fft_size - 1).bit_length()
  if not 2 <= fft_length <= MAX_MEL_FFT:
    raise NotImplementedError(f'{name}: fft_size={fft_size} gives fft_length={fft_length}, '
                              f'outside the 2..{MAX_MEL_FFT} supported')
  if bins > MAX_MEL_BINS:
    raise NotImplementedError(f'{name}: bins={bins} exceeds the {MAX_MEL_BINS} supported')
  n = shape[-1]
  b = 1 if len(shape) == 1 else shape[0]
  n_frames = -(-n // hop) if pad_end else max(0, 1 + (n - fft_size) // hop)
  n_out = len(range(bins)[:mfcc_bins]) if mode == _lib.MFCC else bins
  x = _audio_2d(audio, b, n)
  meta = (n_frames, fft_size, fft_length, hop, int(bool(pad_end)), bins, n_out, mode)
  out = MelFn.apply(x, mel_window(fft_size, x.device),
                    mel_table(bins, fft_length // 2 + 1, sample_rate, lo_hz, hi_hz,
                              x.device), meta)
  return out[0] if len(shape) == 1 else out


def compute_mel(audio, lo_hz=0.0, hi_hz=8000.0, bins=64, fft_size=2048, overlap=0.75,
                pad_end=True, sample_rate=16000):
  """spectral_ops.compute_mel (spectral_ops.py:73-89): |stft| projected on
  linear_to_mel_weight_matrix, [B, N] -> [B, T, bins] and [N] -> [T, bins] ([B, N, 1]
  is read as [B, N]).  Differentiable through MelFn."""
  return _mel(audio, lo_hz, hi_hz, bins, fft_size, overlap, pad_end, sample_rate,
              _lib.MEL)


def compute_logmel(audio, lo_hz=80.0, hi_hz=7600.0, bins=64, fft_size=2048, overlap=0.75,
                   pad_end=True, sample_rate=16000):
  """spectral_ops.compute_logmel (spectral_ops.py:97-109): safe_log of compute_mel."""
  return _mel(audio, lo_hz, hi_hz, bins, fft_size, overlap, pad_end, sample_rate,
              _lib.LOGMEL, name='compute_logmel')


def compute_mfcc(audio, lo_hz=20.0, hi_hz=8000.0, fft_size=1024, mel_bins=128,
                 mfcc_bins=13, overlap=0.75, pad_end=True, sample_rate=16000):
  """spectral_ops.compute_mfcc (spectral_ops.py:112-133):
  tf.signal.mfccs_from_log_mel_spectrograms of compute_logmel (the unnormalised DCT-II
  times rsqrt(2 mel_bins)), cut to [..., :mfcc_bins] with Python's slice rules."""
  return _mel(audio, lo_hz, hi_hz, mel_bins, fft_size, overlap, pad_end, sample_rate,
              _lib.MFCC, mfcc_bins=mfcc_bins, name='compute_mfcc')


# ---- pad and CREPE (spectral_ops.py:171-220, 432-566, csrc/crepe.cuh) -------------
CREPE_SAMPLE_RATE = 16000
CREPE_FRAME_SIZE = 1024
_CREPE_BINS = _lib.CREPE_BINS
_CREPE_SIZES = ('full', 'large', 'small', 'tiny')


def pad(x, frame_size, hop_size, padding='center', axis=1, mode='CONSTANT',
        constant_values=0):
  """spectral_ops.pad (spectral_ops.py:171-220): pads `x` (any shape; axis 0 when it has
  one axis) for strided framing, on the device it is on.  'valid' returns x as float32
  unchecked; 'same' pads the end to get_framed_lengths' padded length; 'center' pads
  frame_size // 2 on both sides.  mode is tf.pad's: 'CONSTANT' (constant_values),
  'REFLECT' (the edge not repeated) or 'SYMMETRIC' (the edge repeated), any case."""
  x = core._as_f32(x)
  if padding == 'valid':
    return x
  _padding_check(frame_size, hop_size, padding)
  if x.dim() <= 1:
    axis = 0
  axis = axis % max(x.dim(), 1)
  n_t = x.shape[axis]
  if padding == 'same':
    _, n_t_padded = get_framed_lengths(n_t, frame_size, hop_size, padding)
    left, right = 0, int(n_t_padded - n_t)
  else:
    left = right = int(frame_size // 2)
  mode = mode.upper()
  if mode == 'CONSTANT':
    shape = list(x.shape)
    parts = []
    for amount in (left, right):
      shape[axis] = amount
      parts.append(torch.full(shape, constant_values, dtype=x.dtype, device=x.device))
    return torch.cat([parts[0], x, parts[1]], dim=axis)
  if mode not in ('REFLECT', 'SYMMETRIC'):
    raise ValueError(f'mode must be one of CONSTANT, REFLECT or SYMMETRIC, got {mode!r}')
  # tf.pad's limits: REFLECT pads less than the axis, SYMMETRIC at most the axis
  limit = n_t - 1 if mode == 'REFLECT' else n_t
  if max(left, right) > limit:
    raise ValueError(f'{mode} padding of {max(left, right)} on an axis of {n_t} elements')
  i = torch.arange(-left, n_t + right, device=x.device)
  if mode == 'REFLECT':
    i = torch.where(i < 0, -i, torch.where(i >= n_t, 2 * (n_t - 1) - i, i))
  else:
    i = torch.where(i < 0, -i - 1, torch.where(i >= n_t, 2 * n_t - 1 - i, i))
  return x.index_select(axis, i)


def _padding_check(frame_size, hop_size, padding):
  """pad's checks for the padding modes that pad, in its order."""
  if padding != 'valid' and hop_size > frame_size:
    raise ValueError(f'During padding, frame_size ({frame_size}) must be greater '
                     f'than hop_size ({hop_size}).')
  if padding not in ('center', 'same', 'valid'):
    raise ValueError('`padding` must be one of [\'center\', \'same\', \'valid\'], '
                     f'received ({padding}).')


def _crepe_frames(audio, hop_size, padding):
  """pad + batch_frames + normalize_frames as one kernel: [B * n_frames, 1024]."""
  b, n, _, n_frames, code = _framing(audio, CREPE_FRAME_SIZE, hop_size, padding)
  x = _audio_2d(audio, b, n)
  frames = torch.empty((b * n_frames, CREPE_FRAME_SIZE), dtype=torch.float32,
                       device=x.device)
  core._launch('ddsp_b200_crepe_frames', x, frames, b, n, n_frames, hop_size, code)
  return frames, b


class PretrainedCREPE:
  """spectral_ops.PretrainedCREPE (spectral_ops.py:432-566): pitch from a CREPE network,
  with everything around the network on CUDA kernels (csrc/crepe.cuh).

  model_size_or_path is the network, mapping normalised frames [M, 1024] to activations
  [M, 360]: a torch.nn.Module or any callable, or the path of a TorchScript file (the
  reference's SavedModel branch).  The sizes 'full', 'large', 'small' and 'tiny' name
  the weights of the `crepe` package, which are not shipped here: they raise
  NotImplementedError.  Nothing here is differentiable: inputs that require grad raise,
  and the network runs under torch.no_grad()."""

  def __init__(self, model_size_or_path, hop_size=160):
    self.hop_size = int(hop_size)
    self.frame_size = CREPE_FRAME_SIZE
    self.sample_rate = CREPE_SAMPLE_RATE
    if isinstance(model_size_or_path, str) and model_size_or_path in _CREPE_SIZES:
      raise NotImplementedError(
          f"PretrainedCREPE: the '{model_size_or_path}' weights come with the crepe "
          'package and are not available here; pass the network as a torch module or '
          'callable, or the path of a TorchScript file.')
    if isinstance(model_size_or_path, (str, os.PathLike)):
      self.core_model = torch.jit.load(os.fspath(model_size_or_path))
    elif callable(model_size_or_path):
      self.core_model = model_size_or_path
    else:
      raise TypeError('PretrainedCREPE: model_size_or_path must be a callable network or '
                      f'a path, got {type(model_size_or_path).__name__}')
    self.model_size_or_path = model_size_or_path

  @classmethod
  def activations_to_f0_and_confidence(cls, activations, centers=None):
    """(f0_hz [M], confidence [M, 1]) of activations [M, 360]: the row max, and the
    activation-weighted mean of the cents of the 10 bins centre - 4 .. centre + 5 (each
    clamped into 0 .. 359) in Hz.  The centre is each row's first argmax, or centers [M]
    (cast to int32 as the reference does).  Weights summing to 0 give NaN (0 / 0), as
    in the reference."""
    shape = core._shape(activations)
    if len(shape) != 2 or shape[1] != _CREPE_BINS:
      raise ValueError(f'activations must be [n_frames, {_CREPE_BINS}], got {shape}')
    if centers is not None and tuple(core._shape(centers)) != shape[:1]:
      raise ValueError(f'centers must be [{shape[0]}], got {tuple(core._shape(centers))}')
    core._no_grad_path('PretrainedCREPE.activations_to_f0_and_confidence', activations)
    acts = core.torch_float32(activations)
    if centers is not None:
      centers = torch.as_tensor(centers, device=acts.device).to(torch.int32).contiguous()
    m = shape[0]
    f0 = torch.empty((m,), dtype=torch.float32, device=acts.device)
    confidence = torch.empty((m, 1), dtype=torch.float32, device=acts.device)
    core._launch('ddsp_b200_crepe_decode', acts, centers, f0, confidence, m)
    return f0, confidence

  def batch_frames(self, audio):
    """Frames of 1024 every hop_size of padded audio [B, N], stacked into [B * F, 1024]
    (tf.signal.frame, pad_end=False); audio of exactly 1024 samples is one frame."""
    audio = core._as_f32(audio)
    if audio.shape[-1] == self.frame_size:
      return audio
    if audio.shape[-1] < self.frame_size:
      return audio.new_zeros((0, self.frame_size))
    frames = audio.unfold(-1, self.frame_size, self.hop_size)
    return frames.reshape(-1, self.frame_size)

  def normalize_frames(self, frames):
    """(frames - mean) / std per frame [M, 1024], with tf.nn.moments' mean and
    population variance (summed in double) and std = 1e-8 where the variance is 0."""
    shape = core._shape(frames)
    if len(shape) != 2 or shape[1] != self.frame_size:
      raise ValueError(f'frames must be [n_frames, {self.frame_size}], got {shape}')
    core._no_grad_path('PretrainedCREPE.normalize_frames', frames)
    x = core.torch_float32(frames)
    out = torch.empty_like(x)
    if shape[0]:
      core._launch('ddsp_b200_crepe_frames', x, out, shape[0], self.frame_size, 1,
                   self.frame_size, _lib.PAD_VALID)
    return out

  def predict_f0_and_confidence(self, audio, viterbi=False, padding='center'):
    """(f0_hz, confidence), each [B, F], of audio [B, N] or [N]: padding, framing and
    normalisation in one kernel, the network, then Viterbi centres if asked for and the
    local-average f0."""
    core._no_grad_path('PretrainedCREPE.predict_f0_and_confidence', audio)
    frames, b = _crepe_frames(audio, self.hop_size, padding)
    with torch.no_grad():
      acts = self.core_model(frames)
    acts = core.torch_float32(acts, frames.device)
    if tuple(acts.shape) != (frames.shape[0], _CREPE_BINS):
      raise ValueError(f'the network mapped frames {tuple(frames.shape)} to '
                       f'{tuple(acts.shape)}, not [{frames.shape[0]}, {_CREPE_BINS}]')
    centers = None
    if viterbi:
      centers = self.viterbi_decode(acts.reshape(b, -1, _CREPE_BINS)).reshape(-1)
    f0_hz, confidence = self.activations_to_f0_and_confidence(acts, centers)
    return f0_hz.reshape(b, -1), confidence.reshape(b, -1)

  def viterbi_decode(self, acts):
    """centres [B, T] (int64) of activations [B, T, 360]: the posterior mode of
    create_hmm's HMM (csrc/crepe.cuh), ties to the lowest bin as tf.argmax's."""
    shape = core._shape(acts)
    if len(shape) != 3 or shape[2] != _CREPE_BINS or shape[1] < 1:
      raise ValueError(f'acts must be [batch, n_frames >= 1, {_CREPE_BINS}], got {shape}')
    core._no_grad_path('PretrainedCREPE.viterbi_decode', acts)
    x = core.torch_float32(acts)
    b, t, _ = shape
    centers = torch.empty((b, t), dtype=torch.int32, device=x.device)
    core._launch('ddsp_b200_crepe_viterbi', x, centers,
                 *core._workspace('ddsp_b200_crepe_viterbi_workspace_bytes', x.device, b, t), b, t)
    return centers.to(torch.int64)


def pad_or_trim_to_expected_length(vector, expected_len, pad_value=0, len_tolerance=20,
                                   use_tf=False):
  """spectral_ops.pad_or_trim_to_expected_length (spectral_ops.py:367-425): pads the
  end of the last axis of a 1-D or 2-D vector with pad_value, or trims it, to
  expected_len; ValueError if the lengths differ by more than len_tolerance.
  use_tf=True works on torch tensors and keeps the gradient; use_tf=False returns
  NumPy."""
  expected_len = int(expected_len)
  vector_len = int(vector.shape[-1])
  if abs(vector_len - expected_len) > len_tolerance:
    raise ValueError('Vector length: {} differs from expected length: {} '
                     'beyond tolerance of : {}'.format(vector_len, expected_len,
                                                       len_tolerance))
  vector = torch.as_tensor(vector) if use_tf else np.asarray(vector)
  if vector_len < expected_len:
    n_padding = expected_len - vector_len
    if use_tf:
      return torch.nn.functional.pad(vector, (0, n_padding), value=pad_value)
    return np.pad(vector, [(0, 0)] * (vector.ndim - 1) + [(0, n_padding)],
                  mode='constant', constant_values=pad_value)
  return vector[..., :expected_len]
