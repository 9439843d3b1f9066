"""The float64 references of the backward tests (tests/grad_ref.py) against the
oracle, which is pinned to the reference itself: they must reproduce
`oracle.harmonic_synthesis`, `oracle.frequency_filter`, `oracle.fft_convolve` and
`oracle.spectral_loss` to 1e-12 of the peak on the shapes the GPU tests use."""
import numpy as np
import pytest
import torch

from oracle import ddsp_oracle as o
from tests import grad_ref


def _rel(got, want):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  return np.abs(got - want).max() / max(np.abs(want).max(), 1e-300)


@pytest.mark.parametrize('B,F,K,hop,sr,method,regime', grad_ref.HARMONIC_CASES)
def test_harmonic_reference_matches_oracle(B, F, K, hop, sr, method, regime):
  N = F * hop
  f0 = grad_ref.low_f0_regime(regime, B, F, sr, seed=K + hop)
  g = torch.Generator().manual_seed(F * K)
  amp = torch.rand(B, F, 1, generator=g) + 0.2
  hd = torch.rand(B, F, K, generator=g)
  got = grad_ref.harmonic(f0, amp, hd, N, sr, method)
  want = o.harmonic_synthesis(f0.numpy(), amp.numpy(), harmonic_distribution=hd.numpy(),
                              n_samples=N, sample_rate=sr, amp_resample_method=method)
  assert got.shape == want.shape == (B, N)
  assert np.abs(want).max() > 0
  assert _rel(got.numpy(), want) <= 1e-12


@pytest.mark.parametrize('B,F,nb,ws,frame,ragged',
                         grad_ref.NOISE_CASES + [(2, 33, 65, 31, 50, True),
                                                 (1, 7, 65, 1, 64, False),
                                                 (2, 5, 65, 2, 48, True),
                                                 (1, 4, 17, 2, 30, False)])
def test_noise_reference_matches_oracle(B, F, nb, ws, frame, ragged):
  """Includes window_size 1 and 2, where the reference's slicing yields two taps
  and its crop then starts at -1, so 'same' returns an empty signal (DESIGN.md
  section 3.1 (iii)); the oracle follows the reference there, and so must this."""
  N = F * frame - (7 if ragged else 0)
  rng = np.random.default_rng(nb * 1000 + ws)
  mags = rng.uniform(0.05, 1.0, (B, F, nb))
  noise = rng.uniform(-1.0, 1.0, (B, N))
  ir = grad_ref.impulse_response(torch.from_numpy(mags), ws).numpy()
  ir_want = o.frequency_impulse_response(mags, ws)
  assert ir.shape == ir_want.shape
  assert _rel(ir, ir_want) <= 1e-12
  got = grad_ref.frequency_filter(torch.from_numpy(noise), torch.from_numpy(mags), ws)
  want = o.frequency_filter(noise, mags, window_size=ws)
  assert got.shape == want.shape
  if ws in (1, 2):
    assert want.shape == (B, 0)
    return
  assert want.shape == (B, N)
  assert _rel(got.numpy(), want) <= 1e-12


@pytest.mark.parametrize('B,n,S,ir_batch,padding,delay', [
    (2, 4000, 3000, 2, 'same', 0),
    (2, 4000, 3000, 1, 'same', -1),
    (3, 1001, 2049, 1, 'same', 0),          # S > n, odd n
    (2, 999, 5000, 2, 'valid', 0),          # S > n, odd n, full tail
    (2, 1025, 3073, 2, 'same', 1500),       # positive delay past one 1024 block
    (1, 2, 2048, 1, 'same', 0),
    (1, 1, 2049, 1, 'valid', 0),
    (2, 1600, 4800, 2, 'same', -1),         # automatic delay, S = 3 n
])
def test_convolve_lti_reference_matches_oracle(B, n, S, ir_batch, padding, delay):
  from ddsp_b200 import core
  rng = np.random.default_rng(n + S)
  audio = rng.standard_normal((B, n))
  ir = rng.standard_normal((ir_batch, S)) * np.exp(-np.arange(S) / (S / 5.0))
  want = o.fft_convolve(audio, np.broadcast_to(ir, (B, S)), padding=padding,
                        delay_compensation=delay)
  start, out_len, crop = core._crop_range(core.get_fft_size(n, S), n, S, padding, delay)
  assert out_len == crop
  got = grad_ref.convolve_lti(torch.from_numpy(audio), torch.from_numpy(ir), start, out_len)
  assert got.shape == want.shape == (B, crop)
  assert _rel(got.numpy(), want) <= 1e-12


@pytest.mark.parametrize('B,N,fft_sizes,mag_weight,logmag_weight',
                         [c[:5] for c in grad_ref.SPECTRAL_CASES] +
                         [(2, 3000, (64,), 0.5, 0.0)])
def test_spectral_loss_reference_matches_oracle(B, N, fft_sizes, mag_weight,
                                                logmag_weight):
  """On the GPU tests' own signals: N shorter than the largest FFT, silent
  stretches of the value (magnitudes exactly 0), stretches equal to the target."""
  target, value = grad_ref.spectral_signals(B, N, fft_sizes, seed=N)
  got = grad_ref.spectral_loss(target, value, fft_sizes, mag_weight, logmag_weight)
  want = o.spectral_loss(target.numpy(), value.numpy(), fft_sizes=fft_sizes,
                         mag_weight=mag_weight, logmag_weight=logmag_weight)
  assert np.isfinite(want) and want > 0
  assert abs(float(got) - want) <= 1e-12 * want
  if N >= 2 * max(fft_sizes) + 896:
    frames = grad_ref.stft_frames(value, max(fft_sizes))
    assert (frames.abs().amax(-1) == 0).any()          # a silent frame of the value
  np.testing.assert_allclose(
      grad_ref.stft_frames(value, 256).numpy(),
      o.frame_pad_end(value.numpy().astype(np.float64), 256, 64) * o.hann_window(256),
      rtol=0, atol=1e-15)


def test_references_are_differentiable_in_float64():
  f0 = grad_ref.low_f0_regime('jump', 1, 4, 16000, seed=1)
  amp = torch.rand(1, 4, 1, dtype=torch.float64, requires_grad=True)
  hd = torch.rand(1, 4, 5, dtype=torch.float64, requires_grad=True)
  f64 = f0.double().requires_grad_(True)
  grad_ref.harmonic(f64, amp, hd, 256).sum().backward()
  assert all(t.grad is not None and t.grad.dtype == torch.float64 for t in (amp, hd, f64))
  mags = torch.rand(1, 4, 9, dtype=torch.float64, requires_grad=True)
  grad_ref.frequency_filter(torch.rand(1, 200, dtype=torch.float64), mags, 7).sum().backward()
  assert mags.grad is not None and torch.isfinite(mags.grad).all()
  audio = torch.rand(2, 300, dtype=torch.float64, requires_grad=True)
  ir = torch.rand(1, 500, dtype=torch.float64, requires_grad=True)
  grad_ref.convolve_lti(audio, ir, 7, 400).sum().backward()
  assert all(t.grad is not None and torch.isfinite(t.grad).all() for t in (audio, ir))
  target, value = grad_ref.spectral_signals(1, 3000, (256, 64), seed=2)
  value = value.double().requires_grad_(True)
  grad_ref.spectral_loss(target, value, (256, 64), 1.0, 1.0).backward()
  assert value.grad.dtype == torch.float64 and torch.isfinite(value.grad).all()
  assert float(value.grad.abs().max()) > 0


@pytest.mark.parametrize('B,N,K,sr,sum_sinusoids', [(2, 300, 5, 16000, True),
                                                    (1, 1, 1, 44100, True),
                                                    (3, 700, 129, 48000, False)])
def test_oscillator_bank_reference_matches_oracle(B, N, K, sr, sum_sinusoids):
  """Negative frequencies, frequencies above Nyquist, and exactly at and one
  float32 ulp below it (silenced and live: the mask is >=)."""
  rng = np.random.default_rng(N + K)
  f = (rng.uniform(-0.3, 0.55, (B, N, K)) * sr).astype(np.float32)
  f[:, ::7, 0] = np.float32(sr / 2)
  if K > 1:
    f[:, ::7, 1] = np.nextafter(np.float32(sr / 2), np.float32(0))
  a = rng.uniform(0.1, 1.0, (B, N, K)).astype(np.float32)
  got = grad_ref.oscillator_bank(torch.from_numpy(f), torch.from_numpy(a), sr, sum_sinusoids)
  want = o.oscillator_bank(f, a, sample_rate=sr, sum_sinusoids=sum_sinusoids)
  assert got.shape == want.shape
  assert _rel(got.numpy(), want) <= 1e-12
  if not sum_sinusoids:
    assert not want[:, ::7, 0].any() and want[:, 7::7, 1].any()


@pytest.mark.parametrize('shape', [(2, 1), (3, 2500), (2, 1001, 3), (1, 999, 2, 3)])
def test_angular_cumsum_reference_matches_oracle(shape):
  """The wrapped running sum against the oracle's chunked angular_cumsum in float64
  (chunks of 1000, the default), compared on the circle."""
  x = np.random.default_rng(len(shape) + shape[1]).uniform(-np.pi, np.pi, shape)
  got = grad_ref.angular_cumsum(torch.from_numpy(x)).numpy()
  want = o.angular_cumsum(x)
  assert got.shape == want.shape
  assert got.min() >= 0.0 and got.max() < 2 * np.pi
  d = np.mod(got - want, 2 * np.pi)
  assert np.minimum(d, 2 * np.pi - d).max() <= 1e-12


@pytest.mark.parametrize('B,N,F,S,ir_batch,padding,delay', [
    (2, 1000, 7, 129, 2, 'valid', 0),
    (3, 1000, 7, 128, 1, 'same', -1),
    (2, 1000, 1, 129, 1, 'same', 300),
    (2, 64, 64, 2047, 2, 'same', 1023),
    (3, 6000, 5, 3000, 1, 'valid', -1),
    (2, 4001, 5, 4096, 2, 'same', -1),
])
def test_fft_convolve_reference_matches_oracle(B, N, F, S, ir_batch, padding, delay):
  """grad_ref.fft_convolve with shared (batch 1) and per-item impulse responses,
  'valid' and 'same', automatic and explicit delays."""
  rng = np.random.default_rng(N + S)
  audio = rng.standard_normal((B, N))
  ir = rng.standard_normal((ir_batch, F, S)) / np.sqrt(S)
  got = grad_ref.fft_convolve(torch.from_numpy(audio), torch.from_numpy(ir), padding, delay)
  want = o.fft_convolve(audio, np.broadcast_to(ir, (B, F, S)), padding=padding,
                        delay_compensation=delay)
  assert got.shape == want.shape and want.shape[1] > 0
  assert _rel(got.numpy(), want) <= 1e-12


@pytest.mark.parametrize('K,sr', [(100, 44100), (1024, 16000), (4096, 44100)])
def test_alllive_regime_keeps_every_harmonic_live(K, sr):
  """'alllive' f0 tracks: every frame in [1.5 Hz, sr / (2 K)), so the float32
  Nyquist decision keeps all K harmonics at every sample, and the harmonic
  reference matches the oracle there."""
  f0 = grad_ref.low_f0_regime('alllive', 2, 12, sr, seed=K, n_harmonics=K)
  assert float(f0.min()) >= 1.5 and float(f0.max()) * K < sr / 2
  assert not grad_ref.nyquist_mask(f0, K, 12 * 50, sr).any()
  g = torch.Generator().manual_seed(K)
  amp = torch.rand(2, 12, 1, generator=g) + 0.2
  hd = torch.rand(2, 12, K, generator=g)
  hd = hd / hd.sum(-1, keepdim=True)
  got = grad_ref.harmonic(f0, amp, hd, 12 * 50, sr, 'linear')
  want = o.harmonic_synthesis(f0.numpy(), amp.numpy(), harmonic_distribution=hd.numpy(),
                              n_samples=12 * 50, sample_rate=sr, amp_resample_method='linear')
  assert _rel(got.numpy(), want) <= 1e-12
