"""Differentiable float64 torch restatements of core.harmonic_synthesis and
core.frequency_filter, the references the backward kernels are checked against
(float64 autograd through them is "what TF autodiff gives the reference").

Both follow oracle/ddsp_oracle.py op by op, so that tests/test_grad_ref.py can pin
them to the oracle at <= 1e-12 on the CPU, and both run on whatever device their
inputs live on.

* `harmonic`: any integer hop, amp_resample_method 'window' or 'linear', any
  sample rate.  The audio-rate Nyquist mask is an input: `nyquist_mask` takes that
  yes / no decision in float32 (f0 * k, then the lerp), as the reference's float32
  arithmetic and `oracle.harmonic_synthesis(mask_in_float32=True)` do.  Deciding it
  in float64 would flip whole oscillators on samples whose frequency lies within
  an ulp of Nyquist.
* `impulse_response` / `frequency_filter`: any number of bins and any window size
  (symmetric Hann for odd windows, the padded / centred layout and its slicing,
  the `(S - 1) // 2 - 1` crop), and ragged frames (`frame = ceil(N / F)`, the last
  frame zero padded).
* `fft_convolve`: shared (batch 1) or per-item impulse responses, 'valid' or
  'same', any delay_compensation.
* `oscillator_bank` / `angular_cumsum`: the stand-alone ops on audio-rate
  envelopes (the Nyquist mask decided on the float32 frequencies).
* `convolve_lti`: the long-impulse-response convolution (`FftConvolveLtiFn`,
  `Reverb`) at any crop.
* `spectral_loss`: the multi-scale 'L1' spectrogram loss (`SpectralLossFn`) at any
  FFT sizes and weights; `stft_frames` is its framing (`FrameWindowFn`).
"""
import math

import torch

TWO_PI = 2.0 * math.pi


def _frame_index(n_frames, n_samples, device):
  """Bilinear-resize index math (align_corners=False) for an integer hop: lower /
  upper frame and the float64 lerp weight of every sample."""
  if n_samples % n_frames:
    raise ValueError('n_samples (%d) must be a multiple of n_frames (%d)'
                     % (n_samples, n_frames))
  hop = n_samples // n_frames
  t = torch.arange(n_samples, device=device)
  lo, r = t // hop, t % hop
  hi = torch.clamp(lo + (r > 0).long(), max=n_frames - 1)
  return hop, lo, hi, r, r.to(torch.float64) / hop


def nyquist_mask(f0_hz, n_harmonics, n_samples, sample_rate):
  """[B, N, K] bool, True where harmonic k is silenced at sample t: the float32
  decision f_k(t) >= sr / 2 with f_k = f0 * k and the lerp each rounded to float32
  (core.py:869-891 evaluated as the reference does; oracle `mask_in_float32`)."""
  f0 = f0_hz.to(torch.float32)
  b, f, _ = f0.shape
  ratios = torch.arange(1, n_harmonics + 1, dtype=torch.float32, device=f0.device)
  hf = f0 * ratios
  _, lo, hi, _, frac = _frame_index(f, n_samples, f0.device)
  top, bottom = hf[:, lo], hf[:, hi]
  fe = top + (bottom - top) * frac.to(torch.float32)[None, :, None]
  return fe >= torch.tensor(sample_rate / 2.0, dtype=torch.float32)


def harmonic(f0_hz, amplitudes, harmonic_distribution, n_samples, sample_rate=16000,
             amp_resample_method='window', mask=None):
  """core.harmonic_synthesis (core.py:1048-1111) in float64 torch ops, without
  harmonic_shifts.  `mask` is a `nyquist_mask` (computed here when None)."""
  f0 = f0_hz.to(torch.float64)
  amp = amplitudes.to(torch.float64)
  hd = harmonic_distribution.to(torch.float64)
  b, f, k = hd.shape
  dev = hd.device
  if mask is None:
    mask = nyquist_mask(f0_hz, k, n_samples, sample_rate)
  hop, lo, hi, r, frac = _frame_index(f, n_samples, dev)
  hf = f0 * torch.arange(1, k + 1, dtype=torch.float64, device=dev)
  ha = amp * hd
  frac = frac[None, :, None]
  fe = hf[:, lo] + (hf[:, hi] - hf[:, lo]) * frac
  if amp_resample_method == 'window':
    # upsample_with_windows (core.py:645-714): Hann(2 hop) overlap-add on the frames
    # plus a copy of the last one; sample r of frame i sees window taps hop + r and r
    nxt = torch.clamp(lo + 1, max=f - 1)
    rr = r.to(torch.float64)[None, :, None]
    w_prev = 0.5 - 0.5 * torch.cos(TWO_PI * (hop + rr) / (2 * hop))
    w_next = 0.5 - 0.5 * torch.cos(TWO_PI * rr / (2 * hop))
    ae = ha[:, lo] * w_prev + ha[:, nxt] * w_next
  elif amp_resample_method == 'linear':
    ae = ha[:, lo] + (ha[:, hi] - ha[:, lo]) * frac
  else:
    raise ValueError(amp_resample_method)
  ae = torch.where(mask, torch.zeros_like(ae), ae)
  phase = torch.cumsum(fe * TWO_PI / float(sample_rate), dim=1)
  return (ae * torch.sin(phase)).sum(-1)


def oscillator_bank(frequency_envelopes, amplitude_envelopes, sample_rate=16000,
                    sum_sinusoids=True):
  """core.oscillator_bank (core.py:911-962) on audio-rate envelopes [B, N, K]:
  amplitude 0 where f >= sr / 2 (decided on the float32 frequencies, as the
  reference decides it), phase = cumsum(f * 2 pi / sr), amp * sin(phase), summed
  over K unless `sum_sinusoids` is False."""
  f = frequency_envelopes.to(torch.float64)
  a = amplitude_envelopes.to(torch.float64)
  nyq = torch.tensor(sample_rate / 2.0, dtype=torch.float32)
  a = torch.where(frequency_envelopes.to(torch.float32) >= nyq, torch.zeros_like(a), a)
  phase = torch.cumsum(f * TWO_PI / float(sample_rate), dim=1)
  audio = a * torch.sin(phase)
  return audio.sum(-1) if sum_sinusoids else audio


def angular_cumsum(angular_frequency):
  """core.angular_cumsum (core.py:799-866) evaluated wide: the running sum of
  [B, N, ...] angular frequencies over axis 1, wrapped into [0, 2 pi).  The
  reference's chunking only changes its float32 rounding, so it is not restated."""
  return torch.remainder(torch.cumsum(angular_frequency.to(torch.float64), dim=1), TWO_PI)


def hann_window(n, dtype=torch.float64, device=None):
  """tf.signal.hann_window(n): periodic for even n, symmetric for odd n, [1] for
  n = 1 (oracle.hann_window)."""
  if n == 1:
    return torch.ones(1, dtype=dtype, device=device)
  k = torch.arange(n, dtype=torch.float64, device=device)
  d = n if n % 2 == 0 else n - 1
  return (0.5 - 0.5 * torch.cos(TWO_PI * k / d)).to(dtype)


def impulse_response(magnitudes, window_size=0):
  """core.frequency_impulse_response (core.py:1534-1565) with
  apply_window_to_impulse_response (core.py:1477-1531): [..., nb] -> [..., S]."""
  mags = magnitudes.to(torch.float64)
  ir = torch.fft.irfft(mags.to(torch.complex128))
  s = ir.shape[-1]
  if window_size <= 0 or window_size > s:
    window_size = s
  win = hann_window(window_size, device=ir.device)
  padding = s - window_size
  if padding > 0:
    half = (window_size + 1) // 2
    win = torch.cat([win[half:], win.new_zeros(padding), win[:half]])
  else:
    win = torch.fft.fftshift(win)
  ir = win * ir
  if padding > 0:
    first_half_start = (s - (half - 1)) + 1
    second_half_end = half + 1
    return torch.cat([ir[..., first_half_start:], ir[..., :second_half_end]], dim=-1)
  return torch.fft.fftshift(ir, dim=-1)


def fft_convolve(audio, ir, padding='same', delay_compensation=-1):
  """core.fft_convolve (core.py:1382-1473) of [B, N] audio with [B or 1, F, S]
  impulse responses (batch 1 is shared by every item): frames of ceil(N / F)
  samples, the last one zero padded, FFT size the next power of two of
  S + frame - 1, then crop_and_compensate_delay with its Python slice."""
  audio = audio.to(torch.float64)
  ir = ir.to(torch.float64)
  b, n = audio.shape
  _, f, s = ir.shape
  frame = -(-n // f)
  if -(-n // frame) != f:
    raise ValueError('%d frames do not tile %d samples' % (f, n))
  frames = torch.nn.functional.pad(audio, (0, f * frame - n)).reshape(b, f, frame)
  nfft = 1 << (s + frame - 2).bit_length()
  y = torch.fft.irfft(torch.fft.rfft(frames, nfft) * torch.fft.rfft(ir, nfft), nfft)
  # overlap-add: split every frame's output into blocks of `frame` samples and add
  # block j of frame i at output block i + j
  m = -(-nfft // frame)
  y = torch.nn.functional.pad(y, (0, m * frame - nfft)).reshape(b, f, m, frame)
  out = sum(torch.nn.functional.pad(y[:, :, j], (0, 0, j, m - 1 - j)) for j in range(m))
  total = (f - 1) * frame + nfft
  out = out.reshape(b, (f + m - 1) * frame)[:, :total]
  # crop_and_compensate_delay, sliced as the reference slices (a window of one or
  # two taps gives start = -1)
  crop_size = s + n - 1 if padding == 'valid' else n
  start = (s - 1) // 2 - 1 if delay_compensation < 0 else delay_compensation
  end = total - crop_size - start
  return out[:, start:-end]


def frequency_filter(audio, magnitudes, window_size=0):
  """core.frequency_filter (core.py:1628-1655), padding='same'."""
  return fft_convolve(audio, impulse_response(magnitudes, window_size))


def convolve_lti(audio, ir, start, out_len):
  """Full linear convolution of audio [B, N] with one impulse response per item
  [1 or B, S] (batch 1 broadcast), cropped to [start, start + out_len): rfft / irfft
  at length N + S - 1, and zeros past it, as in the reference's zero-padded FFT
  buffer.  This is core.fft_convolve on a 2-D impulse response, and what
  `ddsp_b200_fft_convolve_lti` computes."""
  audio = audio.to(torch.float64)
  ir = ir.to(torch.float64)
  n, s = audio.shape[-1], ir.shape[-1]
  m = n + s - 1
  y = torch.fft.irfft(torch.fft.rfft(audio, m) * torch.fft.rfft(ir, m), m)
  y = torch.nn.functional.pad(y, (0, max(0, start + out_len - m)))
  return y[:, start:start + out_len]


def stft_frames(audio, frame_size):
  """spectral_ops.stft's framing (spectral_ops.py:34-47): tf.signal.stft with
  pad_end=True and the periodic Hann window, step frame_size / 4, frames of
  [B, ceil(N / step), frame_size] before the rfft."""
  audio = audio.to(torch.float64)
  step = frame_size // 4
  n = audio.shape[-1]
  n_frames = -(-n // step)
  pad = (n_frames - 1) * step + frame_size - n
  frames = torch.nn.functional.pad(audio, (0, pad)).unfold(-1, frame_size, step)
  return frames * hann_window(frame_size, device=audio.device)


def safe_log(x, eps=1e-5):
  """core.safe_log (core.py:213-216): log(eps) where x <= 0, with no gradient
  there."""
  return torch.log(torch.where(x <= 0.0, torch.full_like(x, eps), x))


def spectral_loss(target, value, fft_sizes=(2048, 1024, 512, 256, 128, 64),
                  mag_weight=1.0, logmag_weight=0.0, spectra=None):
  """SpectralLoss.call with loss_type='L1' (losses.py:194-243): per FFT size, the
  mean over batch, frames and bins of |mag_t - mag_v| and of |safe_log mag_t -
  safe_log mag_v|; a weight of 0 drops its term.

  `spectra`: optional (target STFT, value STFT) per FFT size, e.g. the float32 ones
  a kernel saw.  The loss and its derivatives are then evaluated AT those spectra,
  while d STFT / d value stays the float64 framing and rfft.  The log-magnitude
  gradient is sign / |X| per bin, so with float32 spectra the float32 rounding of
  the smallest magnitudes and of near-zero differences would otherwise dominate an
  elementwise comparison of d value."""
  loss = 0.0
  for i, size in enumerate(fft_sizes):
    xt = torch.fft.rfft(stft_frames(target, size), dim=-1)
    xv = torch.fft.rfft(stft_frames(value, size), dim=-1)
    if spectra is not None:
      xt = spectra[i][0].to(xt.dtype).detach()
      xv = xv + (spectra[i][1].to(xv.dtype) - xv).detach()
    t, v = xt.abs(), xv.abs()
    if mag_weight > 0:
      loss = loss + mag_weight * (t - v).abs().mean()
    if logmag_weight > 0:
      loss = loss + logmag_weight * (safe_log(t) - safe_log(v)).abs().mean()
  return loss


# Harmonic backward cases: (B, F, K, hop, sample_rate, amp method, f0 regime).  Every
# K, F, method, rate and regime at least once, at hops of 1 to 128 64-sample blocks
# (harmonic_backward_kernel stores block 0's totals and adds the later blocks');
# K = 7 / 9 / 13 / 100 / 260 reach the harmonic-group loop with K % 8 != 0.  From hop
# 512 on a CTA takes 4 frames, so F = 3, 5, 7 and 9 leave it a partial tile; there
# 'cross1hz' and 'jump' reach the exact f0 < 1 Hz path, and 'glide' and 'nyquist' the
# per-sample live counts, in blocks after the first.
HARMONIC_CASES = [
    (2, 33, 100, 64, 16000, 'window', 'jump'),
    (2, 33, 100, 64, 16000, 'linear', 'glide'),
    (1, 257, 7, 64, 44100, 'window', 'unvoiced'),
    (2, 33, 260, 64, 16000, 'linear', 'subhertz'),
    (2, 2, 9, 128, 16000, 'window', 'cross1hz'),
    (1, 257, 1, 128, 44100, 'linear', 'nyquist'),
    (1, 33, 100, 128, 44100, 'window', 'glide'),
    (1, 1, 8, 192, 44100, 'linear', 'cross1hz'),
    (2, 33, 7, 192, 16000, 'window', 'unvoiced'),
    (2, 33, 260, 256, 16000, 'window', 'nyquist'),
    (1, 33, 100, 256, 16000, 'linear', 'jump'),
    (1, 33, 100, 512, 16000, 'window', 'cross1hz'),
    (2, 9, 13, 512, 44100, 'linear', 'nyquist'),
    (1, 7, 100, 1024, 16000, 'linear', 'jump'),
    (2, 5, 60, 1024, 16000, 'window', 'glide'),
    (1, 5, 100, 8192, 16000, 'window', 'nyquist'),
    (1, 3, 9, 8192, 44100, 'linear', 'cross1hz'),
]

# Filtered-noise backward cases: (B, F, nb, window_size, frame, ragged).  `ragged`
# drops 7 samples from the last frame (N = F * frame - 7).  Padded windows odd and
# even, windows clamped to the IR, even nb, frames other than 64, F not a multiple
# of 32.
NOISE_CASES = [
    (2, 32, 65, 0, 64, False),
    (1, 33, 65, 64, 64, False),
    (2, 31, 65, 65, 64, False),
    (1, 100, 65, 31, 16, False),
    (2, 1, 64, 0, 48, False),
    (1, 33, 33, 257, 100, True),
    (2, 100, 16, 257, 48, False),
    (1, 31, 129, 0, 64, False),
    (2, 32, 129, 101, 64, False),
]


# Spectral-loss cases: (B, N, fft_sizes, mag_weight, logmag_weight, upstream).
# N = 1000 is shorter than the 2048 / 4096-point frames; N = 12345 is a multiple of
# no step, and with B = 3 its 2048-point STFT has an odd number of bins (the scalar
# tail of spectral_l1_kernel).  `upstream`: the loss itself, 0.37 * loss, or loss +
# an audio term (see test_gpu_backward_edges.py).
DEFAULT_FFT_SIZES = (2048, 1024, 512, 256, 128, 64)
SPECTRAL_CASES = [
    (2, 1000, DEFAULT_FFT_SIZES, 1.0, 1.0, 'one'),
    (1, 1000, (4096, 16), 0.3, 2.5, 'sum'),
    (3, 12345, DEFAULT_FFT_SIZES, 1.0, 1.0, 'scaled'),
    (3, 12345, DEFAULT_FFT_SIZES, 0.0, 1.0, 'one'),
    (3, 12345, (4096, 16), 1.0, 0.0, 'scaled'),
    (3, 12345, (4096, 16), 1.0, 1.0, 'sum'),
    (1, 64000, DEFAULT_FFT_SIZES, 0.3, 2.5, 'sum'),
    (2, 64000, DEFAULT_FFT_SIZES, 1.0, 0.0, 'scaled'),
]


def spectral_signals(B, N, fft_sizes, seed):
  """(target, value) float32 [B, N] for the spectral-loss tests.

  Below 2 * (largest frame + 64) + 768 samples both are independent white noise.
  Longer signals have three stretches, separated by gaps where both are silent and
  which are wider than any frame, so that every frame sees one stretch only:
    1. target == value: both terms and their gradients are exactly 0;
    2. target = 2 * value: exact in float32, so every |mag_t - mag_v| and every
       log-magnitude difference (log 2) is far from 0 and no sign is decided by
       rounding;
    3. value silent, target white noise: the value's magnitudes are exactly 0
       (safe_log's eps branch in the loss, the `ma > 0` guard in the gradient)."""
  gen = torch.Generator().manual_seed(seed)
  value = 0.1 * torch.randn(B, N, generator=gen)
  other = 0.1 * torch.randn(B, N, generator=gen)
  gap = max(fft_sizes) + 64
  if N < 2 * gap + 768:
    return other, value
  r = (N - 2 * gap) // 3
  b0 = N - 2 * gap - 2 * r              # [0, b0): equal
  b1 = b0 + gap                         # [b1, b1 + r): target = 2 * value
  b2 = b1 + r + gap                     # [b2, N): value silent, target noise
  target = value.clone()
  value[:, b0:b1] = 0.0
  target[:, b0:b1] = 0.0
  target[:, b1:b1 + r] *= 2.0
  value[:, b1 + r:] = 0.0
  target[:, b1 + r:b2] = 0.0
  target[:, b2:] = other[:, b2:]
  return target, value


# ---------------------------------------------------------------------------
# Launch geometry of the fused forward kernels, restated from the launchers so
# that the edge tests can say which kernel, tile and occupancy a case reaches.
# tests/test_forward_routing.py pins these restatements to the library's own
# routing (ddsp_b200_filtered_noise_workspace) without a GPU.
# ---------------------------------------------------------------------------
MAX_DYN_SMEM = 200 * 1024          # kMaxDynSmem (common.cuh)


def ir_geometry(nb, window_size):
  """make_ir_geom (noise.cuh): (S0, S, shift, padded)."""
  s0 = 2 * (nb - 1)
  ws = s0 if (window_size <= 0 or window_size > s0) else window_size
  if s0 - ws > 0:
    half = (ws + 1) // 2
    return s0, 2 * half - 1, half - 2, True
  return s0, s0, s0 // 2, False


def noise_fused_geometry(F, nb, N, window_size):
  """nf_configure + nf_smem_layout (noise_fused.cuh): None where
  noise_fused_kernel declines the shape, else its tile geometry, shared memory
  and CTAs per SM (launch_noise_fused)."""
  if nb < 3 or nb > 129 or nb % 2 == 0:
    return None
  s0, s, _, _ = ir_geometry(nb, window_size)
  frame = -(-N // F)
  start = (s - 1) // 2 - 1
  if start < 0 or frame < 16 or frame > 1024 or frame % 16:
    return None
  hb = (s - 1 - start + frame - 1) // frame
  ha = (frame - 1 + start) // frame
  tfo = 32 - hb - ha
  if tfo < 16:
    return None
  q = s0 // 4
  qp = (q + 1 + 3) & ~3
  h_stride = ((s + 2 * 32 + 2 + 3) & ~3) + 2
  x_stride = ((((frame + 15) & ~15) + 16 + 3) & ~3) + 2
  nblk = (frame + s - 1 + 15) // 16
  ngrp = (nblk * 16 + frame - 1) // frame
  out_len = (frame + 1) * (32 + ngrp) + 16
  floats = ((nb + 1) // 2 * qp + (nb - 1) // 2 * qp + ((s + 3) & ~3) + 32 * (nb | 1) +
            32 * nb + 64 * h_stride + 32 * x_stride + out_len)
  smem = (4 * floats + 15) & ~15
  if smem > MAX_DYN_SMEM:
    return None
  return dict(frame=frame, S=s, TFo=tfo, Hb=hb, Ha=ha, tiles_per_item=-(-F // tfo),
              smem=smem, ctas_per_sm=2 if smem <= 110 * 1024 else 1)


def noise_route(F, nb, N, window_size):
  """Which forward kernel core.filtered_noise runs: 'ring' (noise_ring_kernel: 65
  bands, 64-sample frames, the unpadded 128-tap IR), 'fused'
  (noise_fused_kernel) or 'generic' (IR kernel + FIR kernel)."""
  if noise_fused_geometry(F, nb, N, window_size) is None:
    return 'generic'
  _, s, _, padded = ir_geometry(nb, window_size)
  if nb == 65 and N % F == 0 and N // F == 64 and not padded and s == 128:
    return 'ring'
  return 'fused'


def harmonic_v4_smem(fw, kp, hop):
  """hv4::smem_layout(FW, Kp, hop).total."""
  ft = 4 * fw
  o = 16 + 2 * 4 * 256 + 4 * (ft + 1) * kp + (0 if hop == 64 else 4 * hop)
  o = (o + 15) & ~15
  o += 16 * 4 + 48 * ft + 4 * (ft + 1) + 4 * (ft + 1)
  return (o + 15) & ~15


def harmonic_v4_tile_width(B, F, K, hop, n_sms):
  """The frames per warp (FW) launch_harmonic_v4 picks, or None where
  core.harmonic_synthesis(phase_mode='recurrence') takes the generic kernel."""
  if hop % 64 or hop > 8192 or K > 1024:
    return None
  kp = (K + 3) & ~3
  fw = 8

  def ctas(w):
    return B * (-(-F // (4 * w)))
  while fw > 4 and ctas(fw) < 8 * n_sms:
    fw = (fw + 1) >> 1
  while fw > 1 and ctas(fw) < n_sms:
    fw = (fw + 1) >> 1
  fw = max(1, min(fw, -(-F // 4)))
  while fw > 1 and harmonic_v4_smem(fw, kp, hop) > 64 * 1024:
    fw = (fw + 1) // 2
  if harmonic_v4_smem(fw, kp, hop) > MAX_DYN_SMEM:
    return None
  return fw


def harm_smem_bytes(ft, kp):
  """harm_smem_bytes (harmonic.cuh): u64 P, A, D [FT] + red[8]; float f0, amp
  [FT + 1]; float rows [(FT + 1) * Kp]."""
  return 8 * (3 * ft + 8) + 4 * (2 * (ft + 1) + (ft + 1) * kp)


def harmonic_generic_tile(B, F, K, hop, n_sms):
  """The frames per tile (FT) ddsp_b200_harmonic_forward gives
  harmonic_generic_kernel: FT = min(2048 / hop, max(ft_fill, min(4, F)), F), with
  ft_fill = ceil(B F / (4 SMs)), then halved (fit_tile) until harm_smem_bytes fits
  one CTA.  None where even one frame does not fit (E_UNSUPPORTED)."""
  kp = (K + 3) & ~3
  ft = max(1, 2048 // hop)
  ft_fill = max(1, -(-(B * F) // (4 * n_sms)))
  ft = min(ft, max(ft_fill, min(4, F)), F)
  while ft > 1 and harm_smem_bytes(ft, kp) > MAX_DYN_SMEM:
    ft = (ft + 1) // 2
  return ft if harm_smem_bytes(ft, kp) <= MAX_DYN_SMEM else None


def harmonic_route(B, F, K, hop, phase_mode, n_sms):
  """'v4' or 'generic': the kernel core.harmonic_synthesis runs for an integer
  hop and 'window' / 'linear' amplitudes."""
  if phase_mode == 'recurrence' and harmonic_v4_tile_width(B, F, K, hop, n_sms) is not None:
    return 'v4'
  return 'generic'


# harmonic_generic_kernel cases of tests/test_gpu_generic_edges.py: (B, F, K, hop,
# sample_rate, amp method, f0 regime, phase_mode, accumulate, FT) with FT the frames
# per tile harmonic_generic_tile gives on a 132-SM H100.  Every hop, K, mode,
# method, rate and regime; FT = 2048 (hop 1), FT set by ft_fill with many tiles per
# item, FT = F, FT = 1 at hop 8256, and halved by fit_tile (K = 10229 is the
# smallest K that halves the 4-frame tile, K = 20000 halves 2 frames to 1).
GENERIC_HARMONIC_CASES = [
    (2, 600, 1, 1, 16000, 'linear', 'glide', 'recurrence', False, 4),
    (64, 16896, 1, 1, 16000, 'linear', 'unvoiced', 'recurrence', False, 2048),
    (3, 500, 60, 2, 44100, 'window', 'cross1hz', 'recurrence', True, 4),
    (2, 70, 100, 31, 48000, 'linear', 'jump', 'direct', False, 4),
    (8, 2000, 60, 33, 16000, 'window', 'glide', 'recurrence', False, 31),
    (2, 40, 100, 63, 44100, 'linear', 'subhertz', 'recurrence', False, 4),
    (2, 40, 100, 64, 16000, 'window', 'glide', 'direct', False, 4),
    (1, 1, 60, 100, 16000, 'window', 'glide', 'recurrence', False, 1),
    (3, 45, 60, 100, 48000, 'linear', 'nyquist', 'direct', True, 4),
    (2, 50, 100, 160, 16000, 'linear', 'unvoiced', 'direct', False, 4),
    (2, 3, 1025, 441, 44100, 'window', 'glide', 'recurrence', False, 3),
    (1, 100, 60, 441, 44100, 'window', 'nyquist', 'recurrence', True, 4),
    (2, 41, 60, 441, 44100, 'linear', 'glide', 'direct', False, 4),
    (1, 33, 100, 480, 48000, 'window', 'jump', 'recurrence', False, 4),
    (2, 7, 60, 1000, 16000, 'linear', 'cross1hz', 'direct', True, 2),
    (1, 3, 60, 8256, 16000, 'window', 'subhertz', 'recurrence', False, 1),
    (2, 25, 2048, 100, 48000, 'window', 'glide', 'recurrence', False, 4),
    (1, 9, 10229, 441, 44100, 'linear', 'glide', 'recurrence', False, 2),
    (1, 3, 20000, 1000, 48000, 'window', 'unvoiced', 'recurrence', False, 1),
    # every harmonic live: the recurrence's whole chain at every sample
    (2, 40, 100, 441, 44100, 'window', 'alllive', 'recurrence', False, 4),
    (1, 30, 1024, 160, 16000, 'linear', 'alllive', 'recurrence', False, 4),
    (1, 20, 2048, 480, 48000, 'window', 'alllive', 'recurrence', False, 4),
    (1, 20, 4096, 441, 44100, 'window', 'alllive', 'recurrence', False, 4),
    (1, 8, 4096, 441, 44100, 'linear', 'alllive', 'direct', False, 4),
]


# Forward filtered-noise cases of tests/test_gpu_forward_edges.py: (B, F, nb,
# frame, window_size, r, route) with N = F * frame - r (r < F keeps ceil(N / F) =
# frame).  route: 'fused2' / 'fused1' = noise_fused_kernel at two / one CTAs per
# SM, 'generic' = the IR + FIR kernels.  Each boundary is a fused case next to
# the declined (or other-regime) neighbour one step over it.
FWD_NOISE_CASES = [
    (2, 40, 3, 16, 0, 0, 'fused2'),        # S = 4, the smallest frame
    (2, 37, 3, 64, 3, 1, 'fused2'),        # S = 3 (window 3), ragged by 1
    (1, 45, 3, 32, 4, 3, 'fused2'),        # S = 3 (even window 4), ragged by 3
    (2, 33, 5, 16, 0, 8, 'fused2'),        # ragged by frame / 2
    (2, 50, 17, 48, 0, 47, 'fused2'),      # frame 48 (no power-of-two quad count), ragged by frame - 1
    (1, 40, 17, 512, 0, 0, 'fused1'),
    (2, 50, 33, 32, 0, 0, 'fused2'),
    (2, 45, 33, 80, 31, 40, 'fused2'),     # frame 80, odd padded window, ragged by frame / 2
    (2, 30, 33, 64, 257, 0, 'fused2'),     # window clamped to the 64-tap IR
    (1, 20, 33, 512, 0, 0, 'fused1'),      # ~179 KB: fused ...
    (1, 20, 65, 512, 0, 0, 'generic'),     # ... ~210 KB > 200 KB: generic
    (2, 30, 63, 128, 0, 0, 'fused2'),      # 108 KB: two CTAs per SM ...
    (2, 30, 65, 128, 0, 0, 'fused1'),      # ... 111 KB > 110 KB: one
    (2, 40, 65, 64, 101, 0, 'fused2'),     # ~88 KB
    (2, 40, 129, 64, 64, 0, 'fused1'),     # ~119 KB, even padded window
    (2, 40, 127, 16, 0, 0, 'fused1'),      # TFo = 16: fused ...
    (2, 40, 129, 16, 0, 0, 'generic'),     # ... TFo = 15: generic
    (2, 33, 65, 256, 65, 3, 'fused1'),
    (1, 65, 127, 128, 0, 64, 'fused1'),
    (1, 64, 129, 64, 0, 63, 'fused1'),     # the unpadded 256-tap IR, ragged by frame - 1
    (2, 35, 65, 64, 32, 0, 'fused2'),      # even padded window off the ring shape
    (2, 35, 65, 16, 31, 0, 'fused2'),
    (2, 30, 65, 64, 4, 1, 'fused2'),       # S = 3 at 65 bands
    (1, 21, 129, 48, 129, 0, 'fused1'),    # odd padded window at 129 bands
    (1, 81, 63, 80, 64, 79, 'fused2'),
]

# Many tiles per CTA: B * ceil(F / TFo) >= 3 x (132 SMs x CTAs per SM), in both
# occupancy regimes; F not a multiple of TFo, items of one frame and of fewer
# frames than a tile, items of ~96000 samples (interior Philox tiles).
FWD_NOISE_MANY_TILES = [
    (16, 1501, 33, 64, 0, 5, 'fused2'),
    (8, 1501, 129, 64, 64, 0, 'fused1'),
    (800, 1, 33, 64, 0, 0, 'fused2'),
    (400, 7, 129, 64, 64, 3, 'fused1'),
]

# decoder_forward off the ring shape: (B, F, K, nb, hop, sample_rate,
# normalize_below_nyquist, window_size, initial_bias, noise, route).  noise:
# 'injected' or 'philox'.  The last case has more noise tiles (288) than CTAs.
FWD_DECODER_CASES = [
    (2, 40, 60, 33, 128, 16000, True, 0, -5.0, 'injected', 'fused2'),
    (2, 30, 100, 65, 192, 44100, False, 101, -2.0, 'philox', 'fused1'),
    (1, 25, 80, 129, 256, 16000, True, 64, -8.0, 'injected', 'fused1'),
    (2, 20, 40, 65, 128, 44100, True, 0, -2.0, 'philox', 'fused1'),
    (12, 700, 20, 33, 128, 16000, False, 0, -8.0, 'philox', 'fused2'),
]

# harmonic_v4 forward cases: (B, F, K, hop, sample_rate, amp method, f0 regime,
# accumulate, FW) where FW is the frames per warp launch_harmonic_v4 picks on a
# 132-SM H100, or None for the generic kernel (hop 8256 > 8192, K 1025 > 1024).
FWD_HARMONIC_CASES = [
    (1, 1, 4, 64, 16000, 'window', 'glide', False, 1),
    (2, 9, 1, 128, 16000, 'linear', 'unvoiced', True, 1),
    (2, 13, 2, 192, 44100, 'window', 'subhertz', False, 1),
    (1, 11, 3, 320, 48000, 'linear', 'cross1hz', False, 1),
    (2, 7, 5, 512, 16000, 'window', 'jump', True, 1),
    (1, 5, 63, 1024, 44100, 'window', 'nyquist', False, 1),
    (1, 3, 64, 8192, 16000, 'linear', 'glide', False, 1),
    (1, 3, 64, 8256, 16000, 'linear', 'glide', False, None),
    (2, 1100, 4, 192, 16000, 'window', 'unvoiced', False, 4),
    (1056, 32, 3, 128, 48000, 'linear', 'glide', True, 8),
    (1, 1100, 100, 64, 44100, 'window', 'jump', False, 2),
    (132, 16, 1024, 64, 16000, 'linear', 'cross1hz', False, 2),  # the 64 KB cap: 4 -> 2
    (1, 7, 1024, 512, 44100, 'linear', 'subhertz', False, 1),
    (1, 7, 1025, 512, 44100, 'linear', 'subhertz', False, None),
    (2, 50, 100, 320, 48000, 'window', 'jump', True, 1),
    (1, 33, 257, 192, 44100, 'linear', 'nyquist', False, 1),
    (2, 17, 512, 128, 48000, 'window', 'cross1hz', False, 1),
]


def low_f0_regime(regime, B, F, sample_rate, seed, n_harmonics=None):
  """[B, F, 1] float32 f0 tracks for the edges of the harmonic kernels:
    'unvoiced'  - runs of f0 = 0 between voiced frames;
    'subhertz'  - runs of 0 < f0 < 1 Hz;
    'cross1hz'  - frames alternating across 1 Hz (0.3 .. 3 Hz);
    'jump'      - f0 = 0 next to 1500 .. 2000 Hz: in those frames the per-oscillator
                  mask of the exact (f0 < 1 Hz) branch silences upper harmonics;
    'glide'     - fast glides whose live harmonic count changes inside most frames;
    'nyquist'   - runs of frames at or above sr / 2 (no live harmonic at all).
    'alllive'   - every frame in [1.5 Hz, sr / (2 K)) for the K of `n_harmonics`:
                  all K harmonics below Nyquist and no frame under 1 Hz, so the
                  recurrence runs its whole chain at every sample.
  Voiced frames elsewhere sit at 80 .. 600 Hz."""
  g = torch.Generator().manual_seed(seed)
  base = 80.0 + 520.0 * torch.rand(B, F, 1, generator=g, dtype=torch.float64)
  i = torch.arange(F, dtype=torch.float64)[None, :, None]
  run = ((torch.arange(F) // 3) % 2 == 1)[None, :, None]
  if regime == 'unvoiced':
    f0 = torch.where(run, torch.zeros_like(base), base)
  elif regime == 'subhertz':
    sub = 0.05 + 0.9 * torch.rand(B, F, 1, generator=g, dtype=torch.float64)
    f0 = torch.where(run, sub, base)
  elif regime == 'cross1hz':
    f0 = torch.where(((torch.arange(F) % 2) == 0)[None, :, None],
                     0.3 + 0.6 * torch.rand(B, F, 1, generator=g, dtype=torch.float64),
                     1.2 + 1.8 * torch.rand(B, F, 1, generator=g, dtype=torch.float64))
  elif regime == 'jump':
    hi = 1500.0 + 500.0 * torch.rand(B, F, 1, generator=g, dtype=torch.float64)
    f0 = torch.where(((torch.arange(F) % 2) == 0)[None, :, None], torch.zeros_like(hi), hi)
  elif regime == 'glide':
    # +-40 % per frame around 500 Hz: with K harmonics the live count changes inside
    # almost every frame once K * f0 reaches sr / 2
    f0 = 500.0 * (1.0 + 0.4 * torch.sin(2.1 * i + 6.0 * torch.rand(B, 1, 1, generator=g,
                                                                     dtype=torch.float64)))
  elif regime == 'nyquist':
    f0 = torch.where(run, (0.5 + 0.2 * torch.rand(B, F, 1, generator=g,
                                                   dtype=torch.float64)) * sample_rate,
                     base)
  elif regime == 'alllive':
    # the top of the range stays 1e-3 below sr / (2 K), far more than the float32
    # rounding of f0 * K and of the lerp
    top = sample_rate / (2.0 * n_harmonics) * (1.0 - 1e-3)
    f0 = 1.5 + (top - 1.5) * torch.rand(B, F, 1, generator=g, dtype=torch.float64)
  else:
    raise ValueError(regime)
  return f0.to(torch.float32)
