"""The backward pass of the fused Sinusoidal synthesis
(`ddsp_b200_sinusoidal_backward`, `autograd.SinusoidalSynthesisFn`).

CPU: the float64 torch restatement of tests/sinusoidal_ref.py against the float64
oracle, its float32 Nyquist mask against the forward kernel's decision rule, and the
errors raised before any device work.  GPU: d amplitudes and d frequencies against
float64 autograd of the restatement (with the kernel's own mask given) at every hop,
frame count, sinusoid count, sample rate, amplitude method and frequency regime the
kernel accepts, the inner-product identity of d amplitudes against the oracle, the
processor end to end, and the InverseSynthesis shape."""
import numpy as np
import pytest
import torch

from ddsp_b200 import core
from oracle import ddsp_oracle as o
from tests import sinusoidal_ref as ref
from tests.util import linearity, rel_err


# ---- CPU ---------------------------------------------------------------------
@pytest.mark.parametrize('method', ['window', 'linear'])
@pytest.mark.parametrize('F,hop,sr', [(1, 400, 16000), (7, 64, 16000), (16, 441, 44100),
                                      (40, 2, 48000)])
def test_restatement_matches_oracle(method, F, hop, sr):
  """float64 torch restatement vs oracle.sinusoidal_get_signal (the reference's
  resample + resample + oscillator_bank), frequencies below Nyquist throughout."""
  B, K, N = 2, 5, F * hop
  rng = np.random.default_rng(F + hop)
  f = rng.uniform(0.0, 0.49 * sr, (B, F, K)).astype(np.float32)
  a = rng.uniform(0.0, 1.0, (B, F, K)).astype(np.float32)
  want = o.sinusoidal_get_signal(a, f, N, sample_rate=sr, amp_resample_method=method)
  got = ref.torch_sinusoidal(torch.from_numpy(f).double(), torch.from_numpy(a).double(), N,
                             sr, method)
  assert np.abs(got.numpy() - want).max() <= 1e-12


def test_restatement_linear_hop_one_matches_oracle():
  B, F, K = 2, 300, 3
  rng = np.random.default_rng(1)
  f = rng.uniform(0.0, 7900.0, (B, F, K)).astype(np.float32)
  a = rng.uniform(0.0, 1.0, (B, F, K)).astype(np.float32)
  want = o.sinusoidal_get_signal(a, f, F, amp_resample_method='linear')
  got = ref.torch_sinusoidal(torch.from_numpy(f).double(), torch.from_numpy(a).double(), F,
                             16000, 'linear')
  assert np.abs(got.numpy() - want).max() <= 1e-12


def test_float32_mask_follows_the_forward_rule():
  """The mask is the forward's float32 expression lo + (hi - lo) * frac >= sr / 2,
  rounded per operation: it agrees with float64 away from Nyquist, silences a
  frequency exactly at Nyquist, and can differ from float64 only within float32
  rounding of it."""
  B, F, K, hop, sr = 2, 9, 6, 160, 16000
  f = ref.regime('glide', B, F, K, sr, seed=3)
  f[0, 4, 1] = f[0, 5, 1] = 8000.0
  f[1, 2, 2], f[1, 3, 2] = 7999.0, 8001.0
  m32 = ref.nyquist_mask(f, F * hop, sr)
  lo = f[:, :, None, :].astype(np.float64)
  hi = np.concatenate([f[:, 1:], f[:, -1:]], 1)[:, :, None, :].astype(np.float64)
  r = np.arange(hop)[None, None, :, None]
  fe64 = (lo + (hi - lo) * r / hop).reshape(B, F * hop, K)
  assert m32.dtype == bool and m32.shape == (B, F * hop, K)
  assert m32[0, 4 * hop:5 * hop, 1].all()
  near = np.abs(fe64 - sr / 2) <= 1e-3
  assert (m32 == (fe64 >= sr / 2))[~near].all()
  # the kernel's arithmetic, spelled out once
  inv_hop = np.float32(1.0) / np.float32(hop)
  for t in (0, 37, 159):
    frac = np.float32(t) * inv_hop
    lo32, hi32 = np.float32(7999.0), np.float32(8001.0)
    fe = np.float32(lo32 + np.float32(np.float32(hi32 - lo32) * frac))
    assert m32[1, 2 * hop + t, 2] == (fe >= np.float32(8000.0))


def test_value_errors_before_device_work(monkeypatch):
  """out= and accumulate= under grad are refused before any tensor is moved or any
  kernel loaded; so are shapes that do not match."""
  def touched(*a, **k):
    raise AssertionError('device touched')
  monkeypatch.setattr(core, 'torch_float32', touched)
  monkeypatch.setattr(core._lib, 'load', touched)
  f = torch.zeros((2, 10, 3), requires_grad=True)
  a = torch.zeros((2, 10, 3))
  with pytest.raises(ValueError, match='out='):
    core.sinusoidal_synthesis(f, a, n_samples=100, out=torch.zeros(2, 100))
  with pytest.raises(ValueError, match='accumulate='):
    core.sinusoidal_synthesis(a, f, n_samples=100, accumulate=True)
  with pytest.raises(ValueError, match='frequencies'):
    core.sinusoidal_synthesis(f, torch.zeros((2, 10, 4)), n_samples=100)


@pytest.mark.parametrize('method,frames,n', [('nearest', 10, 100), ('cubic', 10, 100),
                                              ('linear', 7, 100), ('window', 7, 100)])
def test_unfused_routes_refuse_grad(monkeypatch, method, frames, n):
  """'nearest' / 'cubic' amplitudes and non-integer hops take the stand-alone
  resample + oscillator_bank kernels, which have no backward: under grad they raise
  instead of returning detached audio, before any device work."""
  import ddsp_b200

  def touched(*a, **k):
    raise AssertionError('device touched')
  monkeypatch.setattr(core._lib, 'load', touched)
  synth = ddsp_b200.Sinusoidal(n_samples=n, amp_resample_method=method)
  a = torch.zeros((1, frames, 2), requires_grad=True)
  f = torch.zeros((1, frames, 2))
  with pytest.raises(RuntimeError, match='requires grad'):
    synth.get_signal(a, f)


# ---- GPU ---------------------------------------------------------------------
DEV = 'cuda'

# (B, F, K, hop, sample rate, amplitude method, frequency regime)
CASES = [
    (2, 1000, 7, 1, 16000, 'linear', 'random'),
    (2, 17, 7, 2, 16000, 'window', 'glide'),
    (2, 16, 100, 63, 44100, 'window', 'random'),
    (3, 125, 1, 64, 16000, 'linear', 'zero'),
    (2, 2, 7, 160, 48000, 'window', 'above'),
    (1, 1, 100, 441, 44100, 'linear', 'glide'),
    (1, 16, 400, 512, 16000, 'window', 'random'),
    (2, 125, 7, 512, 16000, 'linear', 'glide'),
    (2, 17, 100, 441, 48000, 'window', 'zero'),
    (1, 1, 1, 512, 16000, 'window', 'random'),
    (2, 16, 7, 2, 44100, 'linear', 'above'),
    (2, 1000, 1, 64, 48000, 'window', 'glide'),
    (1, 17, 420, 63, 16000, 'linear', 'above'),
]


def _check(name, got, want, tol_max, tol_l2):
  got = got.detach().double().cpu().numpy()
  want = want.detach().double().cpu().numpy()
  assert np.isfinite(got).all(), name
  emax, el2 = rel_err(got, want)
  assert emax < tol_max and el2 < tol_l2, (name, emax, el2)


@pytest.mark.gpu
@pytest.mark.parametrize('B,F,K,hop,sr,method,regime', CASES)
def test_backward_against_float64_autograd(B, F, K, hop, sr, method, regime):
  N = F * hop
  f = torch.from_numpy(ref.regime(regime, B, F, K, sr, seed=F * K + hop)).to(DEV)
  gen = torch.Generator(device='cpu').manual_seed(hop)
  a = (torch.rand((B, F, K), generator=gen) + 0.1).to(DEV)
  g = torch.randn((B, N), generator=gen).to(DEV)
  f1 = f.clone().requires_grad_(True)
  a1 = a.clone().requires_grad_(True)
  out = core.sinusoidal_synthesis(f1, a1, n_samples=N, sample_rate=sr,
                                  amp_resample_method=method)
  out.backward(g)
  want, d_f, d_a = ref.float64_grads(f, a, g, N, sr, method)
  _check('audio', out, want, 1e-4, 1e-4)
  _check('d amplitudes', a1.grad, d_a, 2e-4, 1e-4)
  _check('d frequencies', f1.grad, d_f, 5e-4, 2e-4)
  if regime == 'above':
    assert bool((a1.grad[..., 0] == 0).all()) and bool((f1.grad[..., 0] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize('method,hop,sr', [('window', 160, 16000), ('linear', 441, 44100)])
def test_d_amplitudes_inner_product_identity(method, hop, sr):
  """<dL/dA, D> = sum g * oracle(D): the audio is linear in the amplitudes, and the
  float64 oracle evaluates it with no restatement involved."""
  B, F, K = 2, 12, 9
  N = F * hop
  f32 = ref.regime('random', B, F, K, sr, seed=hop)
  f32 = np.minimum(f32, 0.45 * sr).astype(np.float32)
  gen = torch.Generator(device='cpu').manual_seed(7)
  g = torch.randn((B, N), generator=gen).to(DEV)
  a = torch.rand((B, F, K), generator=gen).to(DEV).requires_grad_(True)
  core.sinusoidal_synthesis(torch.from_numpy(f32).to(DEV), a, n_samples=N, sample_rate=sr,
                            amp_resample_method=method).backward(g)
  linearity(a.grad, g, lambda d: o.sinusoidal_get_signal(
      d, f32, N, sample_rate=sr, amp_resample_method=method), (B, F, K))


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['window', 'linear'])
def test_amplitudes_only_is_bit_identical(method):
  """With only the amplitudes requiring grad the phase path is skipped, and d
  amplitudes is bit for bit what the call with both inputs gives."""
  B, F, K, N = 3, 50, 33, 16000
  f = torch.from_numpy(ref.regime('glide', B, F, K, 16000, seed=2)).to(DEV)
  gen = torch.Generator(device='cpu').manual_seed(2)
  a = torch.rand((B, F, K), generator=gen).to(DEV)
  g = torch.randn((B, N), generator=gen).to(DEV)
  a1, f1 = a.clone().requires_grad_(True), f.clone().requires_grad_(True)
  core.sinusoidal_synthesis(f1, a1, n_samples=N, amp_resample_method=method).backward(g)
  a2 = a.clone().requires_grad_(True)
  core.sinusoidal_synthesis(f, a2, n_samples=N, amp_resample_method=method).backward(g)
  assert f.grad is None
  assert torch.equal(a1.grad, a2.grad)


def _frequencies_sigmoid64(x):
  """core.frequencies_sigmoid (depth 1, [0, 8000] Hz) in float64 torch."""
  midi_min, midi_max = (float(o.hz_to_midi(h)) for h in (0.0, 8000.0))
  midi = midi_min + (midi_max - midi_min) * torch.sigmoid(x)
  return 440.0 * 2.0 ** ((midi - 69.0) / 12.0)


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['window', 'linear'])
def test_processor_backward_end_to_end(method):
  """Sinusoidal on raw network outputs with its default scale functions (exp_sigmoid,
  frequencies_sigmoid, remove_above_nyquist), against float64 autograd through the
  float64 controls.  The float64 controls take their values from our float32 ones
  (a float64 frequency would drift the phase by more than the tolerance over the
  clip); their derivatives are float64."""
  import ddsp_b200
  B, F, K, N, sr = 2, 40, 16, 4000, 16000
  rng = np.random.default_rng(4)
  amps = rng.normal(0, 1, (B, F, K)).astype(np.float32)
  freqs = rng.normal(0, 2, (B, F, K)).astype(np.float32)
  g = torch.from_numpy(rng.standard_normal((B, N))).to(DEV)
  synth = ddsp_b200.Sinusoidal(n_samples=N, sample_rate=sr, amp_resample_method=method)
  a1 = torch.from_numpy(amps).to(DEV).requires_grad_(True)
  f1 = torch.from_numpy(freqs).to(DEV).requires_grad_(True)
  out = synth(a1, f1)
  out.backward(g.float())
  with torch.no_grad():
    ctl = synth.get_controls(a1, f1)

  a64 = torch.from_numpy(amps).to(DEV).double().requires_grad_(True)
  f64 = torch.from_numpy(freqs).to(DEV).double().requires_grad_(True)
  fr = _frequencies_sigmoid64(f64)
  fr = fr + (ctl['frequencies'].double() - fr).detach()
  am = 2.0 * torch.sigmoid(a64)**np.log(10.0) + 1e-7
  am = torch.where(ctl['frequencies'] >= sr / 2.0, torch.zeros_like(am), am)
  am = am + (ctl['amplitudes'].double() - am).detach()
  mask = torch.from_numpy(ref.nyquist_mask(ctl['frequencies'].cpu().numpy(), N, sr)).to(DEV)
  want = ref.torch_sinusoidal(fr, am, N, sr, method, mask=mask)
  want.backward(g)
  _check('audio', out, want, 1e-4, 1e-4)
  _check('d raw amplitudes', a1.grad, a64.grad, 2e-4, 1e-4)
  _check('d raw frequencies', f1.grad, f64.grad, 5e-4, 2e-4)


@pytest.mark.gpu
def test_full_size_inverse_synthesis_shape():
  """B = 32, F = 125, K = 100, N = 64000 (InverseSynthesis: 4 s at 16 kHz, hop 512):
  finite and bit-reproducible gradients, two rows against float64 autograd, and one
  backward through Sinusoidal + FilteredNoiseFn + SpectralLossFn."""
  import ddsp_b200
  from ddsp_b200 import autograd as ag
  from ddsp_b200 import losses
  B, F, K, N, sr = 32, 125, 100, 64000, 16000
  f = torch.from_numpy(ref.regime('random', B, F, K, sr, seed=0)).to(DEV)
  gen = torch.Generator(device=DEV).manual_seed(0)
  a = torch.rand((B, F, K), device=DEV, generator=gen) * 0.05
  g = torch.randn((B, N), device=DEV, generator=gen)
  runs = []
  for _ in range(2):
    f1, a1 = f.clone().requires_grad_(True), a.clone().requires_grad_(True)
    out = core.sinusoidal_synthesis(f1, a1, n_samples=N, sample_rate=sr)
    out.backward(g)
    runs.append((out.detach(), f1.grad, a1.grad))
  torch.cuda.synchronize()
  for first, second in zip(*runs):
    assert bool(torch.isfinite(first).all())
    assert torch.equal(first, second)
  for b in (0, B - 1):
    rows = slice(b, b + 1)
    want, d_f, d_a = ref.float64_grads(f[rows], a[rows], g[rows], N, sr, 'window')
    _check('audio', runs[0][0][rows], want, 1e-4, 1e-4)
    _check('d amplitudes', runs[0][2][rows], d_a, 2e-4, 1e-4)
    _check('d frequencies', runs[0][1][rows], d_f, 5e-4, 2e-4)

  # Sinusoid + noise -> spectral loss, gradients to the raw controls of both
  rng = np.random.default_rng(1)
  amps_raw = torch.from_numpy(rng.normal(0, 1, (B, F, K)).astype(np.float32)).to(DEV)
  freqs_raw = torch.from_numpy(rng.normal(0, 2, (B, F, K)).astype(np.float32)).to(DEV)
  mags_raw = torch.from_numpy(rng.normal(0, 1, (B, F, 65)).astype(np.float32)).to(DEV)
  for t in (amps_raw, freqs_raw, mags_raw):
    t.requires_grad_(True)
  target = torch.randn((B, N), device=DEV, generator=gen) * 0.1
  sinus = ddsp_b200.Sinusoidal(n_samples=N, sample_rate=sr)
  mags = ag.exp_sigmoid(mags_raw - 5.0)
  audio = sinus(amps_raw, freqs_raw) + ag.FilteredNoiseFn.apply(mags, N, 0, None, 3, 0)
  loss = losses.SpectralLoss(mag_weight=1.0, logmag_weight=1.0).call(target, audio)
  loss.backward()
  assert bool(torch.isfinite(loss))
  for t in (amps_raw, freqs_raw, mags_raw):
    assert bool(torch.isfinite(t.grad).all()) and float(t.grad.abs().max()) > 0
