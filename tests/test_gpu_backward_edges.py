"""Backward kernels at every hop, window, frame size and f0 regime they accept.

Each gradient is checked two ways:
  (a) elementwise against float64 autograd of tests/grad_ref.py (max-abs / peak
      and rel-L2 per gradient tensor);
  (b) where the output is linear in the differentiated input, through the
      identity <dL/dx, D> = sum g * y(D) for random directions D, with y(D) the
      float64 ORACLE output for input D.  (b) uses no restatement, so a mistake
      shared by grad_ref.py and a kernel still fails it.
"""
import numpy as np
import pytest
import torch

from ddsp_b200 import autograd as ag
from ddsp_b200 import core
from oracle import ddsp_oracle as o
from tests import grad_ref
from tests.util import linearity, synth_inputs

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')


def _errs(got, want):
  got, want = got.double(), want.double()
  peak = float(want.abs().max())
  emax = float((got - want).abs().max()) / max(peak, 1e-300)
  l2 = float(((got - want)**2).sum().sqrt()) / max(float((want**2).sum().sqrt()), 1e-300)
  return emax, l2


def _check(name, got, want, tol_max, tol_l2):
  assert torch.isfinite(got).all(), name
  emax, l2 = _errs(got, want)
  assert emax < tol_max and l2 < tol_l2, (name, emax, l2)


# ---------------------------------------------------------------------------
# Harmonic: d amplitudes, d harmonic_distribution (and (b) on d(amp * hd))
# ---------------------------------------------------------------------------
def _harmonic_inputs(B, F, K, sr, regime, seed):
  f0 = grad_ref.low_f0_regime(regime, B, F, sr, seed=seed).to(DEV)
  gen = torch.Generator(device='cpu').manual_seed(seed)
  amp = (torch.rand(B, F, 1, generator=gen) + 0.2).to(DEV)
  hd = torch.rand(B, F, K, generator=gen)
  hd = (hd / hd.sum(-1, keepdim=True)).to(DEV)
  return f0, amp, hd


@pytest.mark.parametrize('B,F,K,hop,sr,method,regime', grad_ref.HARMONIC_CASES)
def test_harmonic_backward_every_hop_and_f0_regime(B, F, K, hop, sr, method, regime):
  """HarmonicSynthesisFn with amplitudes, harmonic_distribution and f0 requiring
  grad: harmonic_backward_kernel at hops of one to 128 64-sample blocks per frame;
  the f0 regimes reach the exact f0 < 1 Hz branch (with harmonics actually masked
  in the 'jump' frames), the per-sample masks of frames whose live count changes,
  and frames with no live harmonic, in the first block of a frame and the later
  ones."""
  N = F * hop
  f0, amp, hd = _harmonic_inputs(B, F, K, sr, regime, seed=K + hop)
  g = torch.randn(B, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(F))
  a1, h1, f1 = (t.clone().requires_grad_(True) for t in (amp, hd, f0))
  out = ag.HarmonicSynthesisFn.apply(f1, a1, h1, N, sr, method)
  (out * g).sum().backward()
  a2, h2, f2 = (t.double().requires_grad_(True) for t in (amp, hd, f0))
  mask = grad_ref.nyquist_mask(f0, K, N, sr)
  ref = grad_ref.harmonic(f2, a2, h2, N, sr, method, mask=mask)
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  _check('d amp', a1.grad, a2.grad, 2e-4, 1e-4)
  _check('d hd', h1.grad, h2.grad, 2e-4, 1e-4)
  _check('d f0', f1.grad, f2.grad, 5e-4, 2e-4)
  # (b) the audio is linear in ha = amp * hd: with amp = 1, d hd IS d ha
  ha = (amp * hd).clone().requires_grad_(True)
  ag.HarmonicSynthesisFn.apply(f0, torch.ones_like(amp), ha, N, sr, method).mul(g).sum() \
      .backward()
  f0np = f0.cpu().numpy()
  linearity(ha.grad, g, lambda d: o.harmonic_synthesis(
      f0np, np.ones((B, F, 1)), harmonic_distribution=d, n_samples=N, sample_rate=sr,
      amp_resample_method=method), (B, F, K), seed=K)


@pytest.mark.parametrize('hop', [100, 96, 32])
def test_harmonic_backward_rejects_hops_that_are_not_multiples_of_64(hop):
  """The forward runs at any integer hop; the backward kernels need hop % 64 == 0
  and say so (E_UNSUPPORTED -> NotImplementedError) instead of returning a
  gradient."""
  B, F, K = 1, 8, 5
  f0, amp, hd = _harmonic_inputs(B, F, K, 16000, 'glide', seed=hop)
  h1 = hd.clone().requires_grad_(True)
  out = ag.HarmonicSynthesisFn.apply(f0, amp, h1, F * hop, 16000, 'window')
  with pytest.raises(NotImplementedError, match='hop'):
    out.sum().backward()
  assert h1.grad is None


# ---------------------------------------------------------------------------
# d f0 (not linear: (a) only)
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('B,F,K,hop,sr,method,regime', [
    (2, 33, 100, 64, 16000, 'window', 'jump'),
    (2, 33, 12, 64, 16000, 'linear', 'unvoiced'),
    (1, 33, 100, 256, 44100, 'window', 'jump'),
    (2, 9, 30, 256, 16000, 'linear', 'unvoiced'),
    (1, 40, 1600, 64, 16000, 'window', 'low'),
])
def test_harmonic_backward_f0_regimes(B, F, K, hop, sr, method, regime):
  """harmonic_df0_kernel: the per-oscillator mask of frames with f0 < 1 Hz
  (unvoiced runs, unvoiced-to-voiced jumps), hops 64 and 256, and K = 1600 at hop
  64 with f0 of 3 - 4.5 Hz (every harmonic live), where the shared-memory tile of
  32 frames exceeds the 200 KB limit and the launch halves it."""
  N = F * hop
  if regime == 'low':
    gen = torch.Generator(device='cpu').manual_seed(5)
    f0 = (3.0 + 1.5 * torch.rand(B, F, 1, generator=gen)).to(DEV)
    _, amp, hd = _harmonic_inputs(B, F, K, sr, 'unvoiced', seed=K)
  else:
    f0, amp, hd = _harmonic_inputs(B, F, K, sr, regime, seed=K + hop + 1)
  g = torch.randn(B, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(K))
  f1 = f0.clone().requires_grad_(True)
  (ag.HarmonicSynthesisFn.apply(f1, amp, hd, N, sr, method) * g).sum().backward()
  f2 = f0.double().requires_grad_(True)
  ref = grad_ref.harmonic(f2, amp.double(), hd.double(), N, sr, method,
                          mask=grad_ref.nyquist_mask(f0, K, N, sr))
  (ref * g.double()).sum().backward()
  _check('d f0', f1.grad, f2.grad, 5e-4, 2e-4)


# ---------------------------------------------------------------------------
# get_controls backward through DecoderFn, from raw network outputs
# ---------------------------------------------------------------------------
def _raw_edges(B, F, K, nb, N, sr, seed):
  inp = synth_inputs(B, F, K, nb, N, seed=seed, sample_rate=sr, f0_hi=1200.0)
  f0 = inp['f0_hz']
  f0[:, 3:6] = 0.0                                    # unvoiced rows
  f0[:, 10:13] = 0.6 * sr                             # every harmonic above Nyquist
  f0[:, 13] = 0.5 * sr                                # exactly at Nyquist
  amps, hd, mags = inp['amps'], inp['harmonic_distribution'], inp['noise_magnitudes']
  amps[:, 7], amps[:, 8], amps[:, 9], amps[:, 14] = -100.0, 100.0, -30.0, 30.0
  hd[:, 15] = -100.0                                  # e^-x overflows: the guarded limit
  hd[:, 16, ::3] = 100.0
  hd[:, 17, 1::2] = -30.0
  hd[:, 18] = 30.0
  hd[:, -1, ::2] = -95.0                              # the last frame (F := F - 1 term)
  mags[:, 19] = -100.0
  mags[:, 20, ::2] = 100.0
  mags[:, 21, 1::2] = -30.0
  mags[:, 22] = 30.0
  return inp


@pytest.mark.parametrize('nyq,bias,route,sr', [
    (True, -5.0, 'noise', 16000),
    (False, -2.5, 'philox', 16000),
    (True, -3.0, 'philox', 44100),
    (False, -5.0, 'noise', 44100),
])
def test_decoder_fn_controls_backward_at_the_edges(nyq, bias, route, sr):
  """harmonic_controls_backward_kernel / noise_controls_backward_kernel: rows with
  f0 = 0, rows where every harmonic is masked (sum of e is 0: the safe-divide
  branch), raw values at +-30 and +-100 (exp_sigmoid' must stay finite where e^-x
  overflows), initial_bias other than -5, Philox and injected noise.  Against
  float64 autograd from the raw outputs, f0 included."""
  B, F, K, nb = 2, 33, 100, 65
  N = F * 64
  inp = _raw_edges(B, F, K, nb, N, sr, seed=int(-bias * 10) + sr)
  raw = {k: torch.from_numpy(inp[k]).to(DEV) for k in
         ('amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes')}
  seed, offset = 9, 4
  if route == 'noise':
    nz, nz64 = torch.from_numpy(inp['noise']).to(DEV), None
  else:
    nz = None
  nz64 = (torch.from_numpy(inp['noise']).to(DEV) if nz is not None else
          torch.from_numpy(o.philox_uniform_noise(B, N, seed, offset)).to(DEV)).double()
  g = torch.randn(B, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(sr))
  r32 = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
  out = ag.decoder_train(r32['amps'], r32['harmonic_distribution'], r32['f0_hz'],
                         r32['noise_magnitudes'], n_samples=N, sample_rate=sr,
                         window_size=0, initial_bias=bias, noise=nz, seed=seed,
                         offset=offset, normalize_below_nyquist=nyq)
  (out * g).sum().backward()
  r64 = {k: v.double().requires_grad_(True) for k, v in raw.items()}
  a, h = ag.harmonic_controls(r64['amps'], r64['harmonic_distribution'], r64['f0_hz'],
                              sample_rate=sr, normalize_below_nyquist=nyq)
  ref = (grad_ref.harmonic(r64['f0_hz'], a, h, N, sr, 'window',
                           mask=grad_ref.nyquist_mask(raw['f0_hz'], K, N, sr)) +
         grad_ref.frequency_filter(nz64, ag.exp_sigmoid(r64['noise_magnitudes'] + bias)))
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  for k in raw:
    _check(k, r32[k].grad, r64[k].grad, 1e-3, 3e-4)


# ---------------------------------------------------------------------------
# Filtered noise: d magnitudes
# ---------------------------------------------------------------------------
def _noise_case(B, F, nb, ws, frame, ragged, seed):
  N = F * frame - (7 if ragged else 0)
  gen = torch.Generator(device='cpu').manual_seed(seed)
  mags = (torch.rand(B, F, nb, generator=gen) + 0.05).to(DEV)
  noise = (torch.rand(B, N, generator=gen) * 2 - 1).to(DEV)
  g = torch.randn(B, N, generator=gen).to(DEV)
  return N, mags, noise, g


@pytest.mark.parametrize('B,F,nb,ws,frame,ragged', grad_ref.NOISE_CASES)
def test_noise_backward_every_window_and_frame(B, F, nb, ws, frame, ragged):
  """noise_backward_kernel with injected noise: padded windows odd and even (the
  tap fold around `shift`), clamped windows, even nb, frames other than 64, F not
  a multiple of 32, a ragged last frame."""
  N, mags, noise, g = _noise_case(B, F, nb, ws, frame, ragged, seed=nb + ws + F)
  m1 = mags.clone().requires_grad_(True)
  out = ag.FilteredNoiseFn.apply(m1, N, ws, noise, 0, 0)
  (out * g).sum().backward()
  m2 = mags.double().requires_grad_(True)
  ref = grad_ref.frequency_filter(noise.double(), m2, ws)
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  _check('d mags', m1.grad, m2.grad, 2e-4, 1e-4)
  nnp = noise.double().cpu().numpy()
  linearity(m1.grad, g, lambda d: o.frequency_filter(nnp, d, window_size=ws),
             (B, F, nb), seed=nb)


@pytest.mark.parametrize('B,F,nb,ws,frame,ragged,seed,offset', [
    (2, 33, 65, 31, 50, True, 5, 3),      # frame not a multiple of 4, ragged
    (1, 31, 16, 257, 47, False, 11, 1),   # odd frame, even nb
    (2, 32, 65, 0, 64, False, 7, 2),
])
def test_noise_backward_philox(B, F, nb, ws, frame, ragged, seed, offset):
  """The in-kernel Philox noise of the backward pass is the forward's: the
  gradient with seed / offset (no noise tensor) matches float64 autograd on the
  oracle's Philox stream."""
  N, mags, _, g = _noise_case(B, F, nb, ws, frame, ragged, seed=seed)
  m1 = mags.clone().requires_grad_(True)
  out = ag.FilteredNoiseFn.apply(m1, N, ws, None, seed, offset)
  (out * g).sum().backward()
  nz = torch.from_numpy(o.philox_uniform_noise(B, N, seed, offset)).to(DEV).double()
  m2 = mags.double().requires_grad_(True)
  ref = grad_ref.frequency_filter(nz, m2, ws)
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  _check('d mags (philox)', m1.grad, m2.grad, 2e-4, 1e-4)


@pytest.mark.parametrize('nb,ws', [(2, 0), (1025, 0)])
def test_noise_backward_rejects_unsupported_shapes(nb, ws):
  """nb = 2 (a two-tap impulse response: the crop starts before the signal) and a
  1025-bin filter whose tile does not fit in shared memory raise cleanly from the
  backward call and leave no gradient."""
  B, F, frame = 1, 4, 64
  N = F * frame
  mags = torch.rand(B, F, nb, device=DEV).requires_grad_(True)
  g = torch.randn(B, N, device=DEV)
  dmags = torch.empty(B, F, nb, device=DEV)
  from ddsp_b200 import _lib
  rc = _lib.load().ddsp_b200_filtered_noise_backward(
      g.data_ptr(), 0, 1, 0, dmags.data_ptr(), B, F, nb, N, ws,
      torch.cuda.current_stream().cuda_stream)
  assert rc == _lib.E_UNSUPPORTED
  with pytest.raises(NotImplementedError):
    _lib.check(rc)
  try:
    out = ag.FilteredNoiseFn.apply(mags, N, ws, None, 1, 0)
  except (ValueError, NotImplementedError):
    return                      # the forward refuses the shape already
  with pytest.raises(NotImplementedError):
    (out * g).sum().backward()
  assert mags.grad is None
  torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# FilteredNoiseReverb on the GPU
# ---------------------------------------------------------------------------
def _reverb_reference(audio64, mags64, noise64, ws, bias):
  """effects.py:202-278 in float64 torch: exp_sigmoid(m + bias) -> filtered noise
  (the impulse response) -> dry tap zeroed -> fft_convolve('same', delay 0) ->
  + dry audio."""
  ir = grad_ref.frequency_filter(noise64, ag.exp_sigmoid(mags64 + bias), ws)
  ir = torch.cat([torch.zeros_like(ir[:, :1]), ir[:, 1:]], dim=1)
  b, n = audio64.shape
  ir = ir.expand(b, -1)
  m = n + ir.shape[1] - 1
  wet = torch.fft.irfft(torch.fft.rfft(audio64, m) * torch.fft.rfft(ir, m), m)[:, :n]
  return wet + audio64


@pytest.mark.parametrize('size', ['reduced', 'default', 'long_ir'])
@pytest.mark.parametrize('trainable', [False, True])
def test_filtered_noise_reverb(size, trainable):
  """FilteredNoiseReverb forward (given and learned magnitudes) against the float64
  oracle composition, and backward to the learned [n_frames, n_filter_banks]
  magnitudes and to the audio against float64 autograd.  'default' is the class
  defaults: 48000 taps from 1000 frames of 16 bands (48-sample frames, window 257
  clamped to the 30-tap impulse response) on 64000-sample audio.  'long_ir' has an
  impulse response longer than the audio (8000 taps on 3000 samples)."""
  from ddsp_b200 import effects
  if size == 'reduced':
    B, n, L, F, nb, ws = 2, 6000, 4000, 50, 16, 257
  elif size == 'long_ir':
    B, n, L, F, nb, ws = 2, 3000, 8000, 50, 16, 257
  else:
    B, n, L, F, nb, ws = 2, 64000, 48000, 1000, 16, 257
  bias = -3.0
  rng = np.random.default_rng(L + trainable)
  audio = torch.from_numpy(rng.standard_normal((B, n)).astype(np.float32)).to(DEV)
  noise = torch.from_numpy(rng.uniform(-1, 1, (1 if trainable else B, L))
                           .astype(np.float32)).to(DEV)
  mags = torch.from_numpy(rng.standard_normal((1 if trainable else B, F, nb))
                          .astype(np.float32)).to(DEV)
  rev = effects.FilteredNoiseReverb(trainable=trainable, reverb_length=L, window_size=ws,
                                    n_frames=F, n_filter_banks=nb)
  rev._synth.injected_noise = noise
  # forward against the oracle composition (no autograd involved)
  with torch.no_grad():
    if trainable:
      rev.build(DEV)
      rev._magnitudes = mags[0].clone().requires_grad_(True)
      got = rev(audio)
    else:
      got = rev(audio, mags)
  nz = noise.double().cpu().numpy()
  ir = o.noise_get_signal(o.noise_get_controls(mags.cpu().numpy(), initial_bias=bias)
                          ['magnitudes'], nz, window_size=ws)
  ir = np.broadcast_to(ir, (B, L)).copy()
  ir[:, 0] = 0.0
  a64 = audio.double().cpu().numpy()
  want = o.fft_convolve(a64, ir, padding='same', delay_compensation=0) + a64
  emax, el2 = _errs(got, torch.from_numpy(want).to(DEV))
  assert emax < 1e-4 and el2 < 1e-4, (emax, el2)
  if not trainable:
    return
  # backward: d learned magnitudes, d audio
  g = torch.from_numpy(rng.standard_normal((B, n)).astype(np.float32)).to(DEV)
  a1 = audio.clone().requires_grad_(True)
  rev._magnitudes = mags[0].clone().requires_grad_(True)
  out = rev(a1)
  (out * g).sum().backward()
  a2 = audio.double().requires_grad_(True)
  m2 = mags.double().requires_grad_(True)
  ref = _reverb_reference(a2, m2, noise.double(), ws, bias)
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  _check('d audio', a1.grad, a2.grad, 2e-4, 1e-4)
  _check('d magnitudes', rev._magnitudes.grad, m2.grad[0], 2e-4, 1e-4)


# ---------------------------------------------------------------------------
# Multi-scale spectral loss: SpectralLossFn (spectral_l1_kernel, the windowed
# overlap-add adjoint) and FrameWindowFn
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('B,N,fft_sizes,mag_weight,logmag_weight,upstream',
                         grad_ref.SPECTRAL_CASES)
def test_spectral_loss_against_float64(B, N, fft_sizes, mag_weight, logmag_weight,
                                       upstream):
  """losses.SpectralLoss on CUDA (one SpectralLossFn node) against float64 autograd
  of grad_ref.spectral_loss: the loss value, and d audio with the upstream gradient
  1, 0.37 (read on the device by the adjoint of every FFT size, which accumulate
  into one buffer) or 1 plus another term of the audio.  The signals
  (grad_ref.spectral_signals) have silent stretches of the value, where its
  magnitudes are exactly 0, and stretches equal to the target.  d audio is compared
  with the reference evaluated at the float32 spectra the kernel saw (see
  grad_ref.spectral_loss)."""
  from ddsp_b200 import losses
  from ddsp_b200 import spectral_ops
  target, value = (x.to(DEV) for x in grad_ref.spectral_signals(B, N, fft_sizes,
                                                                  seed=N))
  loss_obj = losses.SpectralLoss(fft_sizes=fft_sizes, mag_weight=mag_weight,
                                 logmag_weight=logmag_weight)
  a1 = value.clone().requires_grad_(True)
  assert loss_obj._fusable(target, a1, None)
  loss = loss_obj(target, a1)
  want = grad_ref.spectral_loss(target, value, fft_sizes, mag_weight, logmag_weight)
  assert torch.isfinite(loss) and float(want) > 0
  assert abs(float(loss) - float(want)) <= 2e-5 * float(want), (float(loss), float(want))
  with torch.no_grad():
    spectra = [(spectral_ops.stft_cuda(target, s), spectral_ops.stft_cuda(value, s))
               for s in fft_sizes]
  a2 = value.double().requires_grad_(True)
  (g_ref,) = torch.autograd.grad(grad_ref.spectral_loss(
      target, a2, fft_sizes, mag_weight, logmag_weight, spectra=spectra), a2)
  if upstream == 'scaled':
    (0.37 * loss).backward()
    g_ref = 0.37 * g_ref
  elif upstream == 'sum':
    # another term of the audio, of the loss gradient's size
    w = float(g_ref.abs().max()) * torch.randn(
        B, N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(B))
    (loss + (a1 * w).sum()).backward()
    g_ref = g_ref + w.double()
  else:
    loss.backward()
  _check('d audio', a1.grad, g_ref, 2e-4, 1e-4)


@pytest.mark.parametrize('B,N,frame_size', [(2, 1000, 2048), (3, 12345, 256),
                                            (1, 64000, 64), (2, 999, 16)])
def test_frame_window_backward(B, N, frame_size):
  """FrameWindowFn (stft_cuda's framing + Hann, pad_end=True) and its adjoint, the
  windowed overlap-add, against float64 autograd of grad_ref.stft_frames: frames
  longer than the audio, N not a multiple of the step, the zero-padded tail."""
  from ddsp_b200 import spectral_ops
  gen = torch.Generator(device=DEV).manual_seed(N)
  audio = torch.randn(B, N, device=DEV, generator=gen)
  step = frame_size // 4
  a1 = audio.clone().requires_grad_(True)
  frames = spectral_ops.FrameWindowFn.apply(a1, frame_size, step)
  gf = torch.randn(frames.shape, device=DEV, generator=gen)
  (frames * gf).sum().backward()
  a2 = audio.double().requires_grad_(True)
  ref = grad_ref.stft_frames(a2, frame_size)
  (ref * gf.double()).sum().backward()
  assert frames.shape == ref.shape
  _check('frames', frames, ref, 1e-6, 1e-6)
  _check('d audio', a1.grad, a2.grad, 1e-5, 1e-5)
