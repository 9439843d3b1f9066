"""losses.SpectralLoss with its delta_time, delta_freq and cumsum_freq terms and 'L2'
(losses.py:130-243), on the spectral_terms kernel (csrc/spectral_terms.cuh) and on
the torch path, and core.diff (core.py:171-198).

tests/spectral_terms_ref.py restates the loss in float64; tests/golden/
spectral_terms.npz (the unmodified reference on the shim) pins it."""
import math
import os

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core, losses, spectral_ops
from tests import grad_ref
from tests import spectral_terms_ref as ref
from tests.golden import make_spectral_terms_golden as golden

DEV = torch.device('cuda')
FIXTURE = os.path.join(os.path.dirname(__file__), 'golden', 'spectral_terms.npz')
TERMS = ref.TERMS


def _kw(weights):
  return {t + '_weight': weights.get(t, 0.0) for t in TERMS}


def _golden_cases():
  return [(case, sig, sizes, w, lt) for case, sig, sizes, w in golden.CASES
          for lt in golden.LOSS_TYPES]


def _errs(got, want):
  got, want = got.double().cpu(), want.double().cpu()
  peak = float(want.abs().max())
  emax = float((got - want).abs().max()) / max(peak, 1e-300)
  l2 = float(((got - want)**2).sum().sqrt()) / max(float((want**2).sum().sqrt()), 1e-300)
  return emax, l2


def _close(a, b, rtol):
  if math.isnan(b):
    return math.isnan(a)
  return abs(a - b) <= rtol * abs(b)


# ---- CPU ---------------------------------------------------------------------------
@pytest.mark.parametrize('case,sig,sizes,weights,loss_type', _golden_cases())
def test_restatement_matches_the_reference(case, sig, sizes, weights, loss_type):
  """The float64 restatement against the reference on the shim (wide), to 1e-9; the
  single-frame case is NaN in both."""
  g = np.load(FIXTURE)
  got = float(ref.spectral_loss(g[sig + '_target'], g[sig + '_audio'], sizes, loss_type,
                                **_kw(weights)))
  assert _close(got, float(g[f'{loss_type}_{case}']), 1e-9), (got, g[f'{loss_type}_{case}'])


@pytest.mark.parametrize('case,sig,sizes,weights,loss_type', _golden_cases())
def test_torch_path_matches_the_reference(case, sig, sizes, weights, loss_type):
  """SpectralLoss on CPU tensors (the torch path) against the reference, at float32
  tolerance."""
  g = np.load(FIXTURE)
  loss = losses.SpectralLoss(fft_sizes=sizes, loss_type=loss_type, **_kw(weights))
  got = float(loss(torch.as_tensor(g[sig + '_target']), torch.as_tensor(g[sig + '_audio'])))
  assert _close(got, float(g[f'{loss_type}_{case}']), 2e-5), (got, g[f'{loss_type}_{case}'])


def test_core_diff():
  """core.diff: x[1:] - x[:-1] along the axis, negative axes too, ValueError past the
  last axis; the values of torch.diff."""
  x = torch.randn(3, 5, 7, generator=torch.Generator().manual_seed(0))
  for axis in (0, 1, 2, -1, -2):
    assert torch.equal(core.diff(x, axis), torch.diff(x, dim=axis))
  assert torch.equal(core.diff(x), torch.diff(x, dim=-1))
  assert core.diff(torch.zeros(2, 1, 3), axis=1).shape == (2, 0, 3)
  np.testing.assert_array_equal(core.diff(np.array([1.0, 4.0, 9.0])).numpy(), [3.0, 5.0])
  with pytest.raises(ValueError, match='Invalid axis index: 3 for tensor with only 3 axes'):
    core.diff(x, axis=3)


def test_routing_on_cpu_and_unsupported_configurations():
  """The new terms and 'L2' route to the fused path on CUDA tensors only; weights,
  'COSINE', FFT sizes that are no power of two >= 16 or beyond 8192 stay on the torch
  path, and plain 'L2' on magnitudes stays there as before."""
  a = torch.zeros(2, 4000)
  cases = [
      (dict(delta_time_weight=1.0), None, False),
      (dict(delta_time_weight=1.0, loss_type='COSINE'), None, False),
  ]
  for kw, weights, want in cases:
    assert losses.SpectralLoss(**kw)._fusable(a, a, weights) is want

  class Cuda:
    """A stand-in CUDA tensor: _fusable reads only these attributes."""
    is_cuda = True
    shape = (2, 4000)

    def dim(self):
      return 2

  c = Cuda()
  is_tensor = torch.is_tensor
  torch.is_tensor = lambda x: isinstance(x, Cuda) or is_tensor(x)
  try:
    fused = lambda **kw: losses.SpectralLoss(**kw)._fusable(c, c, None)
    assert fused(delta_time_weight=1.0)
    assert fused(delta_freq_weight=1.0, loss_type='L2')
    assert fused(cumsum_freq_weight=1.0, mag_weight=0.0, loss_type='l2')
    assert fused(delta_time_weight=1.0, fft_sizes=(8192, 16))
    assert fused()                                                  # ae.gin-like
    assert not fused(loss_type='L2')                                # plain L2
    assert not fused(delta_time_weight=1.0, loss_type='COSINE')
    assert not fused(delta_time_weight=1.0, fft_sizes=(16384,))
    assert not fused(delta_time_weight=1.0, fft_sizes=(1000,))
    assert not fused(delta_time_weight=1.0, fft_sizes=(8,))
    assert not losses.SpectralLoss(delta_time_weight=1.0)._fusable(c, c, 1.0)
  finally:
    torch.is_tensor = is_tensor


# ---- GPU ---------------------------------------------------------------------------
CONFIGS = [
    ('delta_time', 'L1', dict(delta_time=1.0)),
    ('delta_freq', 'L1', dict(delta_freq=1.0)),
    ('cumsum_freq', 'L1', dict(cumsum_freq=1.0)),
    ('mag_l2', 'L2', dict(mag=1.0)),
    ('logmag_l2', 'L2', dict(logmag=1.0)),
    ('delta_time_l2', 'L2', dict(delta_time=1.0)),
    ('delta_freq_l2', 'L2', dict(delta_freq=1.0)),
    ('cumsum_freq_l2', 'L2', dict(cumsum_freq=0.1)),
    ('all', 'L1', golden.ALL),
    ('all_l2', 'L2', golden.ALL),
    ('dt_df_log', 'L1', dict(delta_time=0.5, delta_freq=2.0, logmag=1.0)),
]
SHAPES = [(2, 1000, grad_ref.DEFAULT_FFT_SIZES), (3, 12345, (4096, 16)),
          (1, 64000, grad_ref.DEFAULT_FFT_SIZES), (2, 3000, (8192, 32))]


def _signals(B, N, sizes, seed):
  """(target, value) float32 [B, N]: grad_ref.spectral_signals' layout (independent
  noise when N is short; else stretches where target == value, target = 2 x value and
  value silent, separated by silent gaps wider than any frame), with the edges of the
  2x stretch on multiples of the largest hop.  Every hop divides it, so no frame holds
  a single nonzero sample of that stretch: such a frame has the same magnitude in
  every bin, and each of its delta_freq differences would be 0 up to rounding, its
  L1 sign decided by float32 rounding in the kernel and by float64 rounding in the
  reference."""
  gen = torch.Generator().manual_seed(seed)
  value = 0.1 * torch.randn(B, N, generator=gen)
  other = 0.1 * torch.randn(B, N, generator=gen)
  hop = max(sizes) // 4
  gap = -(-(max(sizes) + 64) // hop) * hop
  if N < 2 * gap + 768 + 3 * hop:
    return other, value
  r = (N - 2 * gap) // 3 // hop * hop
  b1 = -(-(N - gap - 2 * r) // hop) * hop      # [b1, b1 + r): target = 2 x value
  b0 = b1 - gap                                 # [0, b0): equal
  b2 = b1 + r + gap                             # [b2, N): value silent, target noise
  target = value.clone()
  value[:, b0:b1] = 0.0
  target[:, b0:b1] = 0.0
  target[:, b1:b1 + r] *= 2.0
  value[:, b1 + r:] = 0.0
  target[:, b1 + r:b2] = 0.0
  target[:, b2:] = other[:, b2:]
  return target, value


def _fused_loss(target, value, sizes, loss_type, weights):
  """SpectralLossFn with the weights of `weights` (the path SpectralLoss takes)."""
  w = {t: weights.get(t, 0.0) for t in TERMS}
  return spectral_ops.SpectralLossFn.apply(
      target, value, tuple(sizes), w['mag'], w['logmag'], w['delta_time'], w['delta_freq'],
      w['cumsum_freq'], loss_type)


def _check_against_float64(target, value, sizes, loss_type, weights, upstream=1.0,
                           tol_loss=2e-5, tol_max=2e-3, tol_l2=2e-4):
  a1 = value.clone().requires_grad_(True)
  loss = _fused_loss(target, a1, sizes, loss_type, weights)
  want = ref.spectral_loss(target.cpu(), value.cpu(), sizes, loss_type, **_kw(weights))
  assert _close(float(loss.detach()), float(want), tol_loss), (float(loss.detach()), float(want))
  (upstream * loss).backward()
  with torch.no_grad():
    spectra = [(spectral_ops.stft_cuda(target, s), spectral_ops.stft_cuda(value, s))
               for s in sizes]
  a2 = value.double().requires_grad_(True)
  (g_ref,) = torch.autograd.grad(
      upstream * ref.spectral_loss(target, a2, sizes, loss_type, spectra=spectra,
                                   **_kw(weights)), a2)
  assert torch.isfinite(a1.grad).all()
  emax, l2 = _errs(a1.grad, g_ref)
  assert emax < tol_max and l2 < tol_l2, (emax, l2)
  return loss, a1.grad


@pytest.mark.gpu
@pytest.mark.parametrize('B,N,sizes', SHAPES, ids=['short', 'odd', 'long', 'big_frame'])
@pytest.mark.parametrize('name,loss_type,weights', CONFIGS, ids=[c[0] for c in CONFIGS])
def test_loss_and_gradient_against_float64(name, loss_type, weights, B, N, sizes):
  """The loss against the float64 restatement, and d audio against its float64
  autograd evaluated at the float32 spectra the kernel saw, normwise and
  elementwise.  The signals have stretches equal to the target, at twice it, and
  silent (_signals)."""
  target, value = (x.to(DEV) for x in _signals(B, N, sizes, seed=N))
  _check_against_float64(target, value, sizes, loss_type, weights)


@pytest.mark.gpu
def test_loss_object_routes_and_matches_the_torch_path():
  """SpectralLoss with every term routes to the fused path on CUDA and gives the
  torch path's value and gradient, with an upstream gradient of 0.37."""
  target, value = (x.to(DEV) for x in _signals(2, 8000, (1024, 64), 8))
  loss_obj = losses.SpectralLoss(fft_sizes=(1024, 64), loss_type='L1', **_kw(golden.ALL))
  a1 = value.clone().requires_grad_(True)
  assert loss_obj._fusable(target, a1, None)
  (0.37 * loss_obj(target, a1)).backward()
  a2 = value.clone().requires_grad_(True)
  want = loss_obj._call_spectrograms(target, a2, None)
  (0.37 * want).backward()
  assert _close(float(loss_obj(target, value)), float(want.detach()), 1e-5)
  emax, l2 = _errs(a1.grad, a2.grad)
  assert emax < 5e-3 and l2 < 5e-4, (emax, l2)


@pytest.mark.gpu
@pytest.mark.parametrize('loss_type', ['L1', 'L2'])
def test_c4_shape_all_terms(loss_type):
  """The C4 shape (B = 128, N = 64000, six sizes) with every term on: the loss
  against float64, and d audio against float64 autograd for the first items."""
  B, N, sizes = 128, 64000, grad_ref.DEFAULT_FFT_SIZES
  gen = torch.Generator(device=DEV).manual_seed(4)
  target = 0.1 * torch.randn(B, N, device=DEV, generator=gen)
  value = (0.7 * target + 0.05 * torch.randn(B, N, device=DEV, generator=gen))
  a1 = value.clone().requires_grad_(True)
  loss = _fused_loss(target, a1, sizes, loss_type, golden.ALL)
  loss.backward()
  want = ref.spectral_loss(target, value, sizes, loss_type, **_kw(golden.ALL))
  assert _close(float(loss.detach()), float(want), 2e-5), (float(loss.detach()), float(want))
  # the loss is a mean over the batch: the first 2 items' gradient, times B / 2, is
  # that of the same loss on those items alone
  _, g = _check_against_float64(target[:2], value[:2], sizes, loss_type, golden.ALL)
  emax, l2 = _errs(a1.grad[:2] * (B / 2), g)
  assert emax < 2e-3 and l2 < 2e-4, (emax, l2)


@pytest.mark.gpu
@pytest.mark.parametrize('loss_type', ['L1', 'L2'])
def test_single_frame_is_nan_with_the_other_gradients(loss_type):
  """N no longer than one hop: delta_time is the mean of nothing, so the loss is NaN
  as in the reference; the gradient is that of the other terms."""
  g = np.load(FIXTURE)
  target, value = (torch.as_tensor(g['short_' + k]).to(DEV) for k in ('target', 'audio'))
  a1 = value.clone().requires_grad_(True)
  loss = _fused_loss(target, a1, (1024,), loss_type, golden.ALL)
  assert math.isnan(float(loss)) and math.isnan(float(g[f'{loss_type}_one_frame']))
  loss.backward()
  others = dict(golden.ALL, delta_time=0.0)
  a2 = value.clone().requires_grad_(True)
  _fused_loss(target, a2, (1024,), loss_type, others).backward()
  assert torch.equal(a1.grad, a2.grad)
  _check_against_float64(target, value, (1024,), loss_type, others)


@pytest.mark.gpu
def test_poisoned_outputs_and_fenced_operands():
  """Every allocation of the fused path poisoned (0x00, NaN, 3.4e38) and fenced, and
  target and audio between 64 KiB fences of NaN and of 7.0 at storage offsets 0 and
  1: the loss and d audio have the bits of a plain run, and no fence is touched."""
  from tests.test_gpu_memory_bounds import POISONS, _bits, _fenced, _fences_intact, guarded
  target, value = (x.to(DEV) for x in _signals(2, 5000, (2048, 64), 3))
  for name, loss_type, weights in (CONFIGS[0], CONFIGS[-2], CONFIGS[-1]):
    def run(t, v):
      a = v.detach().clone().requires_grad_(True) if not v.requires_grad else v
      loss = _fused_loss(t, a, (2048, 64), loss_type, weights)
      loss.backward()
      return _bits(loss), _bits(a.grad)
    want = run(target, value)
    for p in POISONS:
      with guarded(p):
        got = run(target, value)
      assert all(torch.equal(x, y) for x, y in zip(got, want)), (name, hex(p))
    for fill in (float('nan'), 7.0):
      for off in (0, 1):
        t, rt = _fenced(target, fill, off)
        v, rv = _fenced(value, fill, off)
        v.requires_grad_(True)
        got = run(t, v)
        assert all(torch.equal(x, y) for x, y in zip(got, want)), (name, fill, off)
        _fences_intact(rt, 'target')
        _fences_intact(rv, 'audio')


@pytest.mark.gpu
def test_cuda_graph_replay():
  """Forward and backward captured in one CUDA graph and replayed on new audio give
  the eager results."""
  sizes = (1024, 256, 64)
  target, value = (x.to(DEV) for x in _signals(2, 6000, sizes, 6))
  a = value.clone().requires_grad_(True)
  weights = golden.ALL
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    for _ in range(2):   # warm up cuFFT plans and the caching allocator
      a.grad = None
      _fused_loss(target, a, sizes, 'L2', weights).backward()
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  a.grad = None
  with torch.cuda.graph(graph):
    loss = _fused_loss(target, a, sizes, 'L2', weights)
    loss.backward()
  new = 0.5 * value.flip(-1)
  with torch.no_grad():
    a.copy_(new)
  graph.replay()
  torch.cuda.synchronize()
  b = new.clone().requires_grad_(True)
  want = _fused_loss(target, b, sizes, 'L2', weights)
  want.backward()
  assert _close(float(loss), float(want), 1e-6)
  assert torch.equal(a.grad, b.grad)


@pytest.mark.gpu
def test_non_default_stream_and_device():
  """Launched on the operands' device and its current stream: a side stream gives the
  default stream's bits; on a second device, if there is one, the result is there."""
  target, value = (x.to(DEV) for x in _signals(2, 4000, (512, 64), 2))
  def run(t, v):
    a = v.clone().requires_grad_(True)
    loss = _fused_loss(t, a, (512, 64), 'L1', golden.ALL)
    loss.backward()
    return loss.detach(), a.grad
  want = run(target, value)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    got = run(target, value)
  s.synchronize()
  assert torch.equal(got[1], want[1]) and _close(float(got[0]), float(want[0]), 1e-7)
  if torch.cuda.device_count() > 1:
    d1 = torch.device('cuda', 1)
    got = run(target.to(d1), value.to(d1))
    assert got[1].device == d1
    assert torch.equal(got[1].cpu(), want[1].cpu())


def _launched(monkeypatch, fn):
  calls = []
  real = core._launch
  monkeypatch.setattr(core, '_launch', lambda name, *a: (calls.append(name), real(name, *a)))
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
  return calls, kernels


@pytest.mark.gpu
def test_routing_launches(monkeypatch):
  """The new terms launch spectral_terms once per FFT size and no torch elementwise
  kernel on the spectra (only cuFFT and the library's kernels, and the few scalar
  ops of the loss's sum); the ae.gin configuration launches what it always did."""
  sizes = (2048, 1024, 512, 256, 128, 64)
  target, value = (x.to(DEV) for x in _signals(2, 16000, sizes, 1))

  a = value.clone().requires_grad_(True)
  all_terms = dict(loss_type='L2', mag_weight=1.0, delta_time_weight=1.0,
                   delta_freq_weight=1.0, cumsum_freq_weight=1.0, logmag_weight=1.0)

  def step(**kw):
    losses.SpectralLoss(fft_sizes=sizes, **kw)(target, a).backward()

  step(**all_terms)   # warm-up: cuFFT plans, the cached weights
  calls, kernels = _launched(monkeypatch, lambda: step(**all_terms))
  assert calls == (['ddsp_b200_frame_window', 'ddsp_b200_frame_window',
                    'ddsp_b200_spectral_terms'] * len(sizes) +
                   ['ddsp_b200_frame_window_adjoint'] * len(sizes)), calls
  assert sum('spectral_terms_kernel' in k for k in kernels) == len(sizes)
  bulky = [k for k in kernels if ('elementwise' in k or 'reduce' in k) and 'fft' not in k]
  # zeroing the sums, their product with the weights, its sum and cast, the upstream
  # gradient of 1 and its accumulation into a.grad
  assert len(bulky) <= 6, bulky

  monkeypatch.undo()
  calls, _ = _launched(monkeypatch, lambda: step(mag_weight=1.0, logmag_weight=1.0))
  assert calls == (['ddsp_b200_frame_window', 'ddsp_b200_frame_window',
                    'ddsp_b200_spectral_l1'] * len(sizes) +
                   ['ddsp_b200_frame_window_adjoint'] * len(sizes)), calls


@pytest.mark.gpu
def test_abi_errors_before_device_work():
  """Bad shapes, terms, loss types, null pointers, a gradient overlapping an STFT
  with delta_time, and too many bins raise before anything is launched."""
  lib = _lib.load()
  x = torch.zeros(2, 3, 9, dtype=torch.complex64, device=DEV)
  g = torch.empty_like(x)
  sums = torch.zeros(5, dtype=torch.float64, device=DEV)
  p = lambda t: t.data_ptr()
  ok = (p(x), p(x), p(g), p(sums), 2, 3, 9, _lib.TERM_MAG, _lib.LOSS_L1, 1.0, 0.0, 0.0,
        0.0, 0.0, None)
  bad = [
      (2, 0, _lib.E_INVALID), (3, 0, _lib.E_INVALID), (1, 0, _lib.E_INVALID),
      (4, 65536, _lib.E_INVALID), (5, 0, _lib.E_INVALID), (6, 1, _lib.E_INVALID),
      (7, 0, _lib.E_INVALID), (7, 32, _lib.E_INVALID), (8, 2, _lib.E_INVALID),
      (6, _lib.SPECTRAL_TERMS_MAX_BINS + 1, _lib.E_UNSUPPORTED),
  ]
  before = lib.ddsp_b200_launch_count()
  for i, v, code in bad:
    args = list(ok)
    args[i] = v
    assert lib.ddsp_b200_spectral_terms(*args) == code, (i, v)
  args = list(ok)
  args[2] = p(x)
  args[7] = _lib.TERM_DELTA_TIME
  assert lib.ddsp_b200_spectral_terms(*args) == _lib.E_INVALID
  assert b'overlap' in _lib.load().ddsp_b200_last_error()
  args[2] = p(x) + 8 * 5                                 # a partial overlap
  assert lib.ddsp_b200_spectral_terms(*args) == _lib.E_INVALID
  assert lib.ddsp_b200_launch_count() == before
  args = list(ok)
  args[2] = p(x)                                         # in place without delta_time
  assert lib.ddsp_b200_spectral_terms(*args) == 0
  torch.cuda.synchronize()
  assert lib.ddsp_b200_launch_count() == before + 1
