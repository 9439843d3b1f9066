"""Float64 restatement of core.sinc_impulse_response and core.sinc_filter
(core.py:1568-1625, 1658-1690; fft_convolve core.py:1382-1473): numpy for values,
torch float64 for gradients.  Pinned to the unmodified reference by
tests/golden/sinc.npz."""
import numpy as np
import torch


def n_taps(window_size):
  return 2 * (int(window_size) // 2) + 1


def scaled_cutoff(cutoff, sample_rate=None):
  """The reference's `cutoff *= 2.0 / sample_rate` on a float32 array, as float64."""
  c = np.asarray(cutoff, np.float32)
  if sample_rate is not None:
    c = (c * np.float32(2.0 / float(sample_rate))).astype(np.float32)
  return c.astype(np.float64)


def hamming(s):
  """tf.signal.hamming_window(s) for odd s: symmetric; [1] at s = 1."""
  if s == 1:
    return np.ones(1)
  m = np.arange(s, dtype=np.float64)
  return 0.54 - 0.46 * np.cos(2.0 * np.pi * m / (s - 1))


def _sinc(x, xp):
  x = xp.where(xp.abs(x) < 1e-20, xp.full_like(x, 1e-20), x)
  x = np.pi * x
  return xp.sin(x) / x


def sinc_impulse_response(cutoff, window_size=512, sample_rate=None, high_pass=False):
  c = scaled_cutoff(cutoff, sample_rate)
  s = n_taps(window_size)
  half = s // 2
  idx = np.arange(-half, half + 1, dtype=np.float64)[None, None, :]
  u = hamming(s) * _sinc(c * idx, np)          # broadcast(shape(c), [1, 1, S])
  h = u / np.abs(u.sum(-1, keepdims=True))
  if high_pass:
    delta = np.zeros(h.shape)
    delta[..., half] = 1.0
    h = delta - h
  return h


def _crop(total, n, s, padding):
  """crop_and_compensate_delay's slice (core.py:1338-1379) as (start, stop)."""
  crop_size = s + n - 1 if padding == 'valid' else n
  start = (s - 1) // 2 - 1
  end = (total - crop_size) - start
  r = range(total)[start:-end]
  return (r.start, r.stop) if len(r) else (0, 0)


def fft_convolve(audio, ir, padding='same', xp=np):
  """The reference's framed algorithm: frames of ceil(N / F) samples, each convolved
  with its own impulse response, overlap-added, then cropped.  ir [1 or B, F, S]."""
  b, n = audio.shape
  ib, f, s = ir.shape
  frame = -(-n // f)
  fft = int(2**np.ceil(np.log2(frame + s - 1)))
  total = (f - 1) * frame + fft
  lo, hi = _crop(total, n, s, padding)
  if xp is np:
    x = np.pad(audio, ((0, 0), (0, f * frame - n))).reshape(b, f, frame)
    y = np.fft.irfft(np.fft.rfft(x, fft) * np.fft.rfft(ir, fft), fft)
    out = np.zeros((b, total))
    for j in range(f):
      out[:, j * frame:j * frame + fft] += y[:, j]
    return out[:, lo:hi]
  x = torch.nn.functional.pad(audio, (0, f * frame - n)).reshape(b, f, frame)
  y = torch.fft.irfft(torch.fft.rfft(x, fft) * torch.fft.rfft(ir, fft), fft)
  if f == 1:
    out = torch.nn.functional.pad(y[:, 0], (0, total - fft))
  else:
    out = torch.nn.functional.fold(y.transpose(1, 2), output_size=(total, 1),
                                   kernel_size=(fft, 1), stride=(frame, 1))[:, 0, :, 0]
  return out[:, lo:hi]


def sinc_filter(audio, cutoff, window_size=512, sample_rate=None, padding='same',
                high_pass=False):
  h = sinc_impulse_response(cutoff, window_size, sample_rate, high_pass)
  if h.ndim == 2:
    h = h[None]
  return fft_convolve(np.asarray(audio, np.float64), h, padding)


# ---- torch float64 (for gradients) ---------------------------------------------------
def torch_sinc_impulse_response(c, s, high_pass=False):
  """c: float64 tensor of scaled cutoffs [..., 1] -> [..., S]."""
  half = s // 2
  idx = torch.arange(-half, half + 1, dtype=torch.float64, device=c.device)
  w = torch.from_numpy(hamming(s)).to(c.device)
  u = w * _sinc(c * idx, torch)
  h = u / torch.abs(u.sum(-1, keepdim=True))
  if high_pass:
    delta = torch.zeros(s, dtype=torch.float64, device=c.device)
    delta[half] = 1.0
    h = delta - h
  return h


def torch_sinc_filter(audio, c, s, padding='same', high_pass=False):
  """audio [B, N] and scaled cutoffs [1 or B, F, 1], float64 tensors."""
  return fft_convolve(audio, torch_sinc_impulse_response(c, s, high_pass), padding, xp=torch)
