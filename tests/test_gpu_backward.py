"""Backward kernels vs float64 torch autograd of an op-by-op restatement."""
import numpy as np
import pytest
import torch

from ddsp_b200 import autograd as ag
from ddsp_b200 import losses
from tests import grad_ref
from tests.util import synth_inputs

pytestmark = pytest.mark.gpu


def ref_harmonic(f0, amp, hd, n_samples, sr=16000.0, linear_amp=False):
  """core.harmonic_synthesis in float64 torch ops (tests/grad_ref.py)."""
  return grad_ref.harmonic(f0, amp, hd, n_samples, sr,
                           'linear' if linear_amp else 'window')


def ref_noise(mags, noise, n_samples):
  """core.frequency_filter, window_size=0, in float64 torch ops (tests/grad_ref.py)."""
  assert noise.shape[-1] == n_samples
  return grad_ref.frequency_filter(noise, mags, 0)


@pytest.mark.parametrize('B,F,K', [(2, 20, 12), (1, 33, 100), (2, 8, 5)])
def test_harmonic_backward_matches_autograd(B, F, K):
  N = F * 64
  inp = synth_inputs(B, F, K, 65, N, seed=K, f0_hi=1500.0)
  dev = torch.device('cuda')
  f0 = torch.from_numpy(inp['f0_hz']).to(dev)
  amp = torch.rand(B, F, 1, device=dev) + 0.2
  hd = torch.rand(B, F, K, device=dev)
  hd = hd / hd.sum(-1, keepdim=True)
  g = torch.randn(B, N, device=dev)
  a1 = amp.clone().requires_grad_(True)
  h1 = hd.clone().requires_grad_(True)
  out = ag.HarmonicSynthesisFn.apply(f0, a1, h1, N, 16000, 'window')
  (out * g).sum().backward()
  a2 = amp.double().requires_grad_(True)
  h2 = hd.double().requires_grad_(True)
  ref = ref_harmonic(f0.double(), a2, h2, N)
  (ref * g.double()).sum().backward()
  assert (out.double() - ref).abs().max() < 1e-4 * ref.abs().max()
  for got, want in ((a1.grad, a2.grad), (h1.grad, h2.grad)):
    err = (got.double() - want).abs().max() / want.abs().max()
    assert err < 2e-4, err


@pytest.mark.parametrize('B,F,nb', [(2, 20, 65), (1, 40, 33), (2, 7, 65)])
def test_noise_backward_matches_autograd(B, F, nb):
  N = F * 64
  dev = torch.device('cuda')
  mags = torch.rand(B, F, nb, device=dev) + 0.05
  noise = torch.rand(B, N, device=dev) * 2 - 1
  g = torch.randn(B, N, device=dev)
  m1 = mags.clone().requires_grad_(True)
  out = ag.FilteredNoiseFn.apply(m1, N, 0, noise, 0, 0)
  (out * g).sum().backward()
  m2 = mags.double().requires_grad_(True)
  ref = ref_noise(m2, noise.double(), N)
  (ref * g.double()).sum().backward()
  assert (out.double() - ref).abs().max() < 1e-4 * ref.abs().max()
  err = (m1.grad.double() - m2.grad).abs().max() / m2.grad.abs().max()
  assert err < 2e-4, err
  # Philox path: same gradient when the injected noise IS the Philox stream
  from ddsp_b200 import core
  nz = core.uniform_noise(B, N, seed=7, offset=2)
  m3 = mags.clone().requires_grad_(True)
  (ag.FilteredNoiseFn.apply(m3, N, 0, None, 7, 2) * g).sum().backward()
  m4 = mags.clone().requires_grad_(True)
  (ag.FilteredNoiseFn.apply(m4, N, 0, nz, 0, 0) * g).sum().backward()
  assert (m3.grad - m4.grad).abs().max() < 1e-5 * m4.grad.abs().max()


@pytest.mark.parametrize('B,F,K', [(2, 20, 12), (1, 33, 100), (2, 9, 7)])
@pytest.mark.parametrize('method', ['window', 'linear'])
def test_harmonic_backward_f0_matches_autograd(B, F, K, method):
  """d f0 through the phase (what TF autodiff gives the reference through
  resample + cumsum + sin, core.py:947-958) against float64 autograd."""
  N = F * 64
  inp = synth_inputs(B, F, K, 65, N, seed=K + 3, f0_hi=700.0)
  dev = torch.device('cuda')
  f0 = torch.from_numpy(inp['f0_hz']).to(dev)
  amp = torch.rand(B, F, 1, device=dev) + 0.2
  hd = torch.rand(B, F, K, device=dev)
  hd = hd / hd.sum(-1, keepdim=True)
  g = torch.randn(B, N, device=dev)
  f1 = f0.clone().requires_grad_(True)
  out = ag.HarmonicSynthesisFn.apply(f1, amp, hd, N, 16000, method)
  (out * g).sum().backward()
  f2 = f0.double().requires_grad_(True)
  if method == 'window':
    ref = ref_harmonic(f2, amp.double(), hd.double(), N)
  else:
    ref = ref_harmonic(f2, amp.double(), hd.double(), N, linear_amp=True)
  (ref * g.double()).sum().backward()
  err = (f1.grad.double() - f2.grad).abs().max() / f2.grad.abs().max()
  l2 = ((f1.grad.double() - f2.grad)**2).sum().sqrt() / (f2.grad**2).sum().sqrt()
  assert err < 5e-4 and l2 < 2e-4, (float(err), float(l2))


@pytest.mark.parametrize('B,F,K,nb,nyq', [(2, 30, 100, 65, True), (3, 17, 33, 65, True),
                                          (2, 12, 20, 65, False)])
def test_decoder_fn_matches_float64_autograd_from_raw_outputs(B, F, K, nb, nyq):
  """DecoderFn: fused forward + the get_controls backward kernels, against float64
  autograd of the op-by-op restatement from the RAW network outputs (f0 included)."""
  N = F * 64
  inp = synth_inputs(B, F, K, nb, N, seed=F, f0_hi=1200.0)
  dev = torch.device('cuda')
  raw = {k: torch.from_numpy(inp[k]).to(dev) for k in
         ('amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes')}
  nz = torch.from_numpy(inp['noise']).to(dev)
  g = torch.randn(B, N, device=dev)
  r32 = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
  out = ag.decoder_train(r32['amps'], r32['harmonic_distribution'], r32['f0_hz'],
                         r32['noise_magnitudes'], n_samples=N, window_size=0, noise=nz,
                         normalize_below_nyquist=nyq)
  (out * g).sum().backward()
  r64 = {k: v.double().requires_grad_(True) for k, v in raw.items()}
  a, h = ag.harmonic_controls(r64['amps'], r64['harmonic_distribution'], r64['f0_hz'],
                              normalize_below_nyquist=nyq)
  ref = (ref_harmonic(r64['f0_hz'], a, h, N) +
         ref_noise(ag.exp_sigmoid(r64['noise_magnitudes'] - 5.0), nz.double(), N))
  (ref * g.double()).sum().backward()
  assert (out.double() - ref).abs().max() < 1e-4 * ref.abs().max()
  for k in raw:
    got, want = r32[k].grad.double(), r64[k].grad
    err = float((got - want).abs().max() / want.abs().max())
    l2 = float(((got - want)**2).sum().sqrt() / (want**2).sum().sqrt())
    assert err < 1e-3 and l2 < 3e-4, (k, err, l2)
  # and the round-1 route (torch get_controls around the two Functions) agrees
  r3 = {k: v.clone().requires_grad_(k != 'f0_hz') for k, v in raw.items()}
  if nyq:
    out3 = ag.decoder_train_unfused(r3['amps'], r3['harmonic_distribution'], r3['f0_hz'],
                                    r3['noise_magnitudes'], n_samples=N, window_size=0,
                                    noise=nz)
    (out3 * g).sum().backward()
    for k in ('amps', 'harmonic_distribution', 'noise_magnitudes'):
      d = (r3[k].grad - r32[k].grad).abs().max() / r32[k].grad.abs().max()
      assert float(d) < 5e-4, (k, float(d))


def test_decoder_train_step_through_spectral_loss():
  """C4 in miniature: forward + backward through SpectralLoss, finite grads that
  reduce the loss under one small SGD step."""
  B, F, K, nb, N = 2, 125, 100, 65, 8000
  inp = synth_inputs(B, F, K, nb, N, seed=3)
  dev = torch.device('cuda')
  raw = {k: torch.from_numpy(inp[k]).to(dev) for k in
         ['amps', 'harmonic_distribution', 'noise_magnitudes']}
  for v in raw.values():
    v.requires_grad_(True)
  f0 = torch.from_numpy(inp['f0_hz']).to(dev)
  target = 0.1 * torch.randn(B, N, device=dev)
  loss_obj = losses.SpectralLoss(mag_weight=1.0, logmag_weight=1.0)

  def run():
    audio = ag.decoder_train(raw['amps'], raw['harmonic_distribution'], f0,
                             raw['noise_magnitudes'], n_samples=N, window_size=0,
                             seed=1, offset=0)
    return loss_obj(target, audio)

  loss0 = run()
  loss0.backward()
  for v in raw.values():
    assert v.grad is not None and torch.isfinite(v.grad).all()
    assert v.grad.abs().sum() > 0
  with torch.no_grad():
    for v in raw.values():
      v -= 0.05 * v.grad / (v.grad.abs().max() + 1e-12)
  assert float(run()) < float(loss0)


@pytest.mark.parametrize('B,N', [(3, 8000), (2, 12345)])
def test_fused_spectral_loss_matches_torch_path(B, N):
  """The CUDA pieces of SpectralLoss (framing + window, L1 mag / log-mag with
  gradient, windowed overlap-add) against the torch-op implementation of the same
  reference semantics: value and gradient w.r.t. the audio."""
  from ddsp_b200 import losses
  g = torch.Generator(device='cpu').manual_seed(B * N)
  target = (0.1 * torch.randn(B, N, generator=g)).cuda()
  audio = (0.1 * torch.randn(B, N, generator=g)).cuda()
  loss_obj = losses.SpectralLoss(mag_weight=1.0, logmag_weight=1.0)
  a1 = audio.clone().requires_grad_(True)
  assert loss_obj._fusable(target, a1, None)
  l1 = loss_obj(target, a1)
  l1.backward()
  a2 = audio.clone().requires_grad_(True)
  loss_obj._fusable = lambda *a: False          # force the torch-op path
  l2 = loss_obj(target, a2)
  l2.backward()
  assert abs(float(l1) - float(l2)) < 2e-5 * abs(float(l2)), (float(l1), float(l2))
  err = (a1.grad - a2.grad).abs().max() / a2.grad.abs().max()
  assert float(err) < 2e-4, float(err)
  # a weighted sum of the two terms, and frames / STFT alone
  from ddsp_b200 import spectral_ops
  x1 = spectral_ops.stft_cuda(audio, 256)
  x2 = spectral_ops.stft(audio, 256)
  assert float((x1 - x2).abs().max()) < 1e-4 * float(x2.abs().max())
