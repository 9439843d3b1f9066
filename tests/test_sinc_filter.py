"""core.sinc_impulse_response and core.sinc_filter (core.py:1568-1625, 1658-1690): the
float64 restatement against the unmodified reference's fixture, the C ABI's checks and
the Python errors (CPU), and the CUDA kernels with their gradients against float64
autograd (GPU).

Tolerances follow the other FIR tests: forward <= 1e-4 relative to the peak; gradients
2e-4 max-abs over peak and 1e-4 relative L2."""

import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core
from oracle import ref_on_shim
from tests import sinc_ref as ref
from tests.golden import make_sinc_golden as mg
from tests.util import linearity, rel_err


def _fixture():
  return np.load(mg.PATH)


# ---- CPU ---------------------------------------------------------------------
def test_oracle_matches_reference_fixture():
  want = _fixture()
  for i, (ws, hp, sr, c) in enumerate(mg.ir_cases()):
    got = ref.sinc_impulse_response(c, ws, sr, hp)
    w = want['ir_wide_%03d' % i]
    assert got.shape == w.shape, (ws, hp, sr)
    assert np.abs(got - w).max() <= 1e-12, (ws, hp, sr)
  for i, (case, (audio, c)) in enumerate(zip(mg.FILTER_CASES, mg.filter_inputs())):
    _, _, _, ws, padding, hp, sr = case
    got = ref.sinc_filter(audio, c, ws, sr, padding, hp)
    w = want['filter_wide_%02d' % i]
    assert got.shape == w.shape, case
    if w.size:
      assert np.abs(got - w).max() <= 1e-12, case


@pytest.mark.skipif(not ref_on_shim.available(), reason='reference sources absent')
def test_fixture_regenerates_from_reference():
  mg.compare('sinc', mg.sinc(), _fixture())


def test_torch_restatement_matches_oracle():
  rng = np.random.default_rng(5)
  audio = rng.standard_normal((2, 300))
  for cshape, ws, padding, hp in [((2, 7, 1), 33, 'same', False), ((1, 1, 1), 64, 'valid', True),
                                  ((2, 300, 1), 8, 'same', True)]:
    c = rng.uniform(0.05, 0.95, cshape)
    want = ref.sinc_filter(audio, c, ws, None, padding, hp)
    got = ref.torch_sinc_filter(torch.from_numpy(audio), torch.from_numpy(ref.scaled_cutoff(c)),
                                ref.n_taps(ws), padding, hp)
    assert np.abs(got.numpy() - want).max() <= 1e-12


@pytest.mark.parametrize('cshape,ws,want', [
    ((), 512, (1, 1, 513)), ((1,), 8, (1, 1, 9)), ((2, 1), 8, (1, 2, 9)),
    ((3, 5, 1), 0, (3, 5, 1)), ((3, 5, 1), 2, (3, 5, 3)), ((2, 3, 4, 1), 7, (2, 3, 4, 7))])
def test_impulse_response_shapes(cshape, ws, want):
  """broadcast(shape(cutoff), [1, 1, S]), as TensorFlow forms it."""
  s, shape, scale = core._sinc_geometry(cshape, ws, None)
  assert (s, shape, scale) == (want[-1], want, 1.0)
  assert core._sinc_geometry((), 4, 16000)[2] == float(np.float32(2.0 / 16000))
  # a negative rate is accepted, as in the reference
  assert core._sinc_geometry((), 4, -16000)[2] == -float(np.float32(2.0 / 16000))


def test_sinc_matches_restatement():
  """core.sinc (core.py:1568-1573), threshold branch included: |x| < 1e-20 gives 1 and
  a zero gradient, as the reference's tf.where does."""
  x = np.array([0.0, 1e-25, -1e-21, 1e-19, 1e-3, -0.25, 0.5, 1.0, 1.5, -3.7, 40.25],
               np.float32)
  got = core.sinc(x)
  assert got.dtype == torch.float32
  want = ref._sinc(x.astype(np.float64), np)
  assert np.abs(got.numpy() - want).max() <= 1e-6
  assert (got.numpy()[:3] == 1.0).all()
  xt = torch.from_numpy(x).requires_grad_(True)
  core.sinc(xt).sum().backward()
  assert (xt.grad.numpy()[:3] == 0.0).all()
  # elsewhere the gradient is sinc'(x) = (cos(pi x) - sinc(x)) / x; torch autograd of
  # sin(pi x) / (pi x) cancels in float32 near 0 (as TensorFlow's does), so the tight
  # comparison is made from |x| = 1/4
  xs = x[5:].astype(np.float64)
  dwant = (np.cos(np.pi * xs) - ref._sinc(xs, np)) / xs
  assert np.allclose(xt.grad.numpy()[5:], dwant, rtol=1e-5, atol=1e-6)
  assert np.abs(xt.grad.numpy()[3:5] - np.array([-np.pi**2 / 3 * 1e-19, -np.pi**2 / 3 * 1e-3])
                ).max() <= 2e-4
  assert core.sinc(torch.tensor(0.3, dtype=torch.float64)).dtype == torch.float32


def test_value_errors_before_device_work(monkeypatch):
  """Window, cutoff, batch, frame and padding errors are raised before any tensor is
  moved or the library is loaded; a sample rate of 0 raises ZeroDivisionError there, as
  the reference's `2.0 / float(sample_rate)` does."""
  def touched(*a, **k):
    raise AssertionError('device touched')
  monkeypatch.setattr(core, 'torch_float32', touched)
  monkeypatch.setattr(core._lib, 'load', touched)
  audio = np.zeros((2, 100), np.float32)
  c = np.full((2, 4, 1), 0.5, np.float32)
  for fn in (lambda **k: core.sinc_impulse_response(c, **k),
             lambda **k: core.sinc_filter(audio, c, **k)):
    with pytest.raises(ValueError, match='window_size'):
      fn(window_size=-2)
    with pytest.raises(ZeroDivisionError):
      fn(sample_rate=0)
  with pytest.raises(ValueError, match='last axis'):
    core.sinc_impulse_response(np.zeros((2, 4, 3), np.float32))
  with pytest.raises(ValueError, match='last axis'):
    core.sinc_filter(audio, np.zeros((4,), np.float32))
  with pytest.raises(ValueError, match='Batch size'):
    core.sinc_filter(audio, np.zeros((3, 4, 1), np.float32))
  with pytest.raises(ValueError, match='Number of Audio frames'):
    core.sinc_filter(audio, np.zeros((2, 60, 1), np.float32))
  with pytest.raises(ValueError, match='Padding'):
    core.sinc_filter(audio, c, padding='full')
  with pytest.raises(ValueError):
    core.sinc_filter(np.zeros((2, 100, 1), np.float32), c)


@pytest.mark.parametrize('high_pass,window_size', [(True, 257), (False, 256)])
def test_reference_output_sizes(high_pass, window_size):
  """core_test.py's test_sinc_filter_gives_correct_size: a scalar cutoff of 0.5 and
  'same' padding keep the audio size; it takes the fused route."""
  s, shape, _ = core._sinc_geometry((), window_size, None)
  assert shape == (1, 1, 257)
  geo = core._fft_convolve_geometry((1, 1000), shape, 'same', -1)
  assert geo[6] == geo[7] == 1000


# The C ABI checks: (args, status, message).  Device pointers are never dereferenced:
# every case fails before a launch.
_P = 16


def _filter_args(**kw):
  a = dict(audio=_P, cutoff=_P, out=_P, B=2, N=100, F=4, S=9, cb=2, scale=1.0, hp=0,
           padding=_lib.PAD_SAME, acc=0)
  a.update(kw)
  return a


_FILTER_CASES = [
    (dict(audio=0), _lib.E_INVALID, 'sinc_filter: null pointer'),
    (dict(cutoff=0), _lib.E_INVALID, 'sinc_filter: null pointer'),
    (dict(N=0), _lib.E_INVALID,
     'sinc_filter: bad shape B=2 N=0 F=4 S=9 (S must be odd)'),
    (dict(S=8), _lib.E_INVALID,
     'sinc_filter: bad shape B=2 N=100 F=4 S=8 (S must be odd)'),
    (dict(B=-1), _lib.E_INVALID,
     'sinc_filter: bad shape B=-1 N=100 F=4 S=9 (S must be odd)'),
    (dict(cb=3), _lib.E_INVALID,
     'Batch size of audio (2) and impulse response (3) must be the same.'),
    (dict(padding=7), _lib.E_INVALID, "Padding must be 'valid' or 'same' (got code 7)"),
    (dict(F=60), _lib.E_INVALID,
     'Number of Audio frames (50) and impulse response frames (60) do not match. For '
     'small hop size = ceil(audio_size / n_ir_frames), number of impulse response '
     'frames must be a multiple of the audio size.'),
    (dict(B=70000, cb=1), _lib.E_INVALID, 'sinc_filter: B=70000 exceeds the 65535 grid limit'),
    (dict(S=1), _lib.E_UNSUPPORTED,
     "sinc_filter: 1 tap gives a negative automatic delay (the reference's crop is "
     "empty); compose sinc_impulse_response and fft_convolve"),
    (dict(S=2049), _lib.E_UNSUPPORTED,
     'sinc_filter: 2049 taps is beyond the fused kernels (2047 at most); compose '
     'sinc_impulse_response and fft_convolve'),
]


def _call_filter(lib, a):
  return lib.ddsp_b200_sinc_filter(a['audio'], a['cutoff'], a['out'], a['B'], a['N'], a['F'],
                                   a['S'], a['cb'], a['scale'], a['hp'], a['padding'],
                                   a['acc'], None)


def _call_filter_backward(lib, a, ws=_P, nbytes=1 << 20):
  return lib.ddsp_b200_sinc_filter_backward(
      a['audio'], a['cutoff'], a['out'], _P, _P, a['B'], a['N'], a['F'], a['S'], a['cb'],
      a['scale'], a['hp'], a['padding'], ws, nbytes, None)


def _expect(lib, rc, status, msg):
  assert rc == status, (rc, status, msg)
  assert lib.ddsp_b200_last_error().decode() == msg


def test_abi_checks_launch_nothing():
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  for kw, status, msg in _FILTER_CASES:
    a = _filter_args(**kw)
    _expect(lib, _call_filter(lib, a), status, msg)
    back = msg.replace('sinc_filter:', 'sinc_filter_backward:')
    _expect(lib, _call_filter_backward(lib, a), status, back)
  # a short workspace
  a = _filter_args(cb=1)
  need = lib.ddsp_b200_sinc_filter_backward_workspace(2, 100, 4, 9, 1)
  _expect(lib, _call_filter_backward(lib, a, nbytes=need - 1), _lib.E_WORKSPACE,
          'sinc_filter_backward: workspace of %d B needed, %d given' % (need, need - 1))
  _expect(lib, _call_filter_backward(lib, a, ws=0), _lib.E_WORKSPACE,
          'sinc_filter_backward: workspace of %d B needed, %d given' % (need, 1 << 20))
  for name in ('sinc_impulse_response', 'sinc_impulse_response_backward'):
    fn = getattr(lib, 'ddsp_b200_' + name)
    args = (lambda c, ir, bf, s: (c, ir, bf, s, 1.0, 0, None)) if 'backward' not in name else (
        lambda c, ir, bf, s: (c, ir, _P, bf, s, 1.0, 0, None))
    _expect(lib, fn(*args(0, _P, 4, 9)), _lib.E_INVALID, '%s: null pointer' % name)
    _expect(lib, fn(*args(_P, _P, -1, 9)), _lib.E_INVALID,
            '%s: bad shape BF=-1 S=9 (S must be odd)' % name)
    _expect(lib, fn(*args(_P, _P, 4, 4)), _lib.E_INVALID,
            '%s: bad shape BF=4 S=4 (S must be odd)' % name)
    _expect(lib, fn(*args(_P, _P, 2**31, 9)), _lib.E_INVALID, '%s: too many frames' % name)
    assert fn(*args(_P, _P, 0, 9)) == _lib.OK
  # zero items and empty backward requests launch nothing either
  assert _call_filter(lib, _filter_args(B=0, cb=1)) == _lib.OK
  assert lib.ddsp_b200_sinc_filter_backward(_P, _P, _P, None, None, 2, 100, 4, 9, 2, 1.0, 0,
                                            _lib.PAD_SAME, None, 0, None) == _lib.OK
  assert lib.ddsp_b200_launch_count() == launches


@pytest.mark.parametrize('B,N,F,S,cb,want', [
    (2, 100, 4, 9, 2, 0),                          # frames of 25, per-item cutoffs
    (32, 64000, 1000, 513, 32, 0),
    (2, 100, 4, 9, 1, 2 * 4 * 4 + 256),            # shared: a partial per item
    (1, 64000, 1, 513, 1, 63 * 4 + 256),           # one frame of 63 segments
    (3, 64000, 7, 33, 3, 3 * 7 * 9 * 4 + 256),     # frames of 9143: 9 segments
    (0, 100, 4, 9, 1, 0), (2, 100, 60, 9, 2, 0), (2, 100, 4, 9, 3, 0)])
def test_backward_workspace_sizes(B, N, F, S, cb, want):
  assert _lib.load().ddsp_b200_sinc_filter_backward_workspace(B, N, F, S, cb) == want


# ---- GPU ---------------------------------------------------------------------
def _cuda(x):
  return torch.as_tensor(np.asarray(x, np.float32)).cuda()


def _check(name, got, want, tol_max=1e-4, tol_l2=1e-4):
  emax, el2 = rel_err(got, want)
  assert emax <= tol_max and el2 <= tol_l2, (name, emax, el2)


def _check_grad(name, got, want):
  _check(name, got, want, 2e-4, 1e-4)


@pytest.mark.gpu
def test_impulse_response_every_fixture_case():
  want = _fixture()
  for i, (ws, hp, sr, c) in enumerate(mg.ir_cases()):
    got = core.sinc_impulse_response(c, window_size=ws, sample_rate=sr, high_pass=hp)
    w = want['ir_wide_%03d' % i]
    assert tuple(got.shape) == w.shape
    # per response, relative to its peak; the taps sum to 1 (or to 0 for a high-pass,
    # which is exactly zero at a cutoff of 1 and 3 taps), so the peak is floored at 1 / S
    s = w.shape[-1]
    for g_row, w_row in zip(got.cpu().numpy().reshape(-1, s), w.reshape(-1, s)):
      peak = max(np.abs(w_row).max(), 1.0 / s)
      assert np.abs(g_row - w_row).max() <= 1e-4 * peak, (ws, hp, sr)


@pytest.mark.gpu
def test_impulse_response_does_not_mutate_cutoff():
  c = np.full((2, 3, 1), 4000.0, np.float32)
  core.sinc_impulse_response(c, window_size=8, sample_rate=16000)
  assert (c == 4000.0).all()


@pytest.mark.gpu
@pytest.mark.parametrize('ws', [2, 7, 64, 256, 512, 1024, 2048, 4096])
@pytest.mark.parametrize('hp', [False, True])
def test_impulse_response_gradient(ws, hp):
  rng = np.random.default_rng(ws)
  c = np.concatenate([np.asarray(mg.CUTOFFS[1:], np.float32),
                      rng.uniform(0.02, 0.98, 9).astype(np.float32)])[None, :, None]
  s = ref.n_taps(ws)
  ct = _cuda(c).requires_grad_(True)
  h = core.sinc_impulse_response(ct, window_size=ws, high_pass=hp)
  g = torch.randn(h.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
  (h * g.cuda().float()).sum().backward()
  c64 = torch.from_numpy(c.astype(np.float64)).requires_grad_(True)
  (ref.torch_sinc_impulse_response(c64, s, hp) * g).sum().backward()
  _check('h', h.detach().cpu().numpy(), ref.sinc_impulse_response(c, ws, None, hp))
  _check_grad('d cutoff', ct.grad.cpu().numpy(), c64.grad.numpy())


# sinc_filter shapes: (B, N, F, ws, padding, hp, sample_rate, shared)
SHAPES = [
    (1, 1, 1, 2, 'same', False, None, False),
    (3, 2, 2, 8, 'valid', True, None, False),
    (3, 1000, 1, 256, 'same', False, 16000, False),
    (3, 1000, 7, 512, 'valid', True, None, True),        # ragged frames of 143
    (3, 1000, 250, 8, 'same', True, 16000, False),
    (3, 1000, 1000, 2, 'same', False, None, True),       # audio-rate cutoff
    (3, 1000, 1000, 1024, 'valid', False, None, False),
    (1, 1000, 7, 2046, 'same', True, None, False),       # N < S
    (3, 1000, 250, 2046, 'valid', False, 44100, True),
    (1, 64000, 1, 512, 'same', False, None, False),      # one frame of 63 segments
    (3, 64000, 7, 256, 'valid', True, 16000, True),
    (32, 64000, 1000, 512, 'same', False, None, False),
    (32, 64000, 250, 1024, 'same', True, None, True),
    # frames of 1025 in two segments of 513; the last frame has 426 samples, so its
    # second segment lies past N and contributes an explicit zero partial sum
    (2, 614401, 600, 8, 'same', False, None, False),
    (2, 614401, 600, 8, 'valid', True, 16000, True),
    (1, 3000, 2, 64, 'same', False, -16000, False),      # a negative rate, as accepted
]


def _inputs(B, N, F, sr, shared, seed):
  rng = np.random.default_rng(seed)
  audio = rng.standard_normal((B, N)).astype(np.float32)
  c = rng.uniform(0.05, 0.95, (1 if shared else B, F, 1)).astype(np.float32)
  if sr is not None:
    c = (c * np.float32(sr / 2.0)).astype(np.float32)
  return audio, c


@pytest.mark.gpu
@pytest.mark.parametrize('case', range(len(SHAPES)))
def test_filter_forward_and_gradients(case):
  B, N, F, ws, padding, hp, sr, shared = SHAPES[case]
  audio, c = _inputs(B, N, F, sr, shared, case)
  s = ref.n_taps(ws)
  xa = _cuda(audio).requires_grad_(True)
  ct = _cuda(c).requires_grad_(True)
  y = core.sinc_filter(xa, ct, window_size=ws, sample_rate=sr, padding=padding, high_pass=hp)
  g = torch.randn(y.shape, dtype=torch.float64, device='cuda',
                  generator=torch.Generator('cuda').manual_seed(case))
  (y * g.float()).sum().backward()
  x64 = torch.from_numpy(audio.astype(np.float64)).cuda().requires_grad_(True)
  c64 = torch.from_numpy(ref.scaled_cutoff(c, sr)).cuda().requires_grad_(True)
  y64 = ref.torch_sinc_filter(x64, c64, s, padding, hp)
  (y64 * g).sum().backward()
  assert tuple(y.shape) == tuple(y64.shape)
  _check('y', y.detach().cpu().numpy(), y64.detach().cpu().numpy())
  _check_grad('d audio', xa.grad.cpu().numpy(), x64.grad.cpu().numpy())
  scale = 1.0 if sr is None else float(np.float32(2.0 / sr))
  _check_grad('d cutoff', ct.grad.cpu().numpy(), c64.grad.cpu().numpy() * scale)


@pytest.mark.gpu
def test_filter_fixture_cases():
  want = _fixture()
  for i, (case, (audio, c)) in enumerate(zip(mg.FILTER_CASES, mg.filter_inputs())):
    _, _, _, ws, padding, hp, sr = case
    with torch.no_grad():
      got = core.sinc_filter(audio, c, window_size=ws, sample_rate=sr, padding=padding,
                             high_pass=hp)
    w = want['filter_wide_%02d' % i]
    assert tuple(got.shape) == w.shape, case
    if w.size:
      _check(case, got.cpu().numpy(), w)


@pytest.mark.gpu
def test_d_audio_linearity():
  B, N, F, ws = 2, 4000, 50, 256
  audio, c = _inputs(B, N, F, None, False, 3)
  xa = _cuda(audio).requires_grad_(True)
  y = core.sinc_filter(xa, _cuda(c), window_size=ws, padding='valid', high_pass=True)
  g = torch.randn(y.shape, device='cuda', generator=torch.Generator('cuda').manual_seed(4))
  (y * g).sum().backward()
  linearity(xa.grad, g, lambda d: ref.sinc_filter(d, c, ws, None, 'valid', True), (B, N))


@pytest.mark.gpu
@pytest.mark.parametrize('B,N,F,ws,padding,shared', [
    (2, 16000, 1, 1024, 'same', True), (3, 16000, 250, 512, 'valid', False),
    (4, 8000, 8000, 64, 'same', False), (2, 5000, 7, 2046, 'valid', True)])
def test_fused_equals_composition(B, N, F, ws, padding, shared):
  audio, c = _inputs(B, N, F, None, shared, 9)
  with torch.no_grad():
    fused = core.sinc_filter(audio, c, window_size=ws, padding=padding)
    comp = core.fft_convolve(_cuda(audio), core.sinc_impulse_response(c, window_size=ws),
                             padding=padding)
  _check('fused', fused.cpu().numpy(), comp.cpu().numpy(), 1e-5, 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize('F', [1, 4])
def test_long_windows_under_grad(F):
  """windows >= 2048 compose sinc_impulse_response with fft_convolve's long-IR routes."""
  B, N, ws = 2, 8000, 2048
  audio, c = _inputs(B, N, F, None, False, 11)
  xa = _cuda(audio).requires_grad_(True)
  ct = _cuda(c).requires_grad_(True)
  y = core.sinc_filter(xa, ct, window_size=ws)
  g = torch.randn(y.shape, dtype=torch.float64, device='cuda',
                  generator=torch.Generator('cuda').manual_seed(F))
  (y * g.float()).sum().backward()
  x64 = torch.from_numpy(audio.astype(np.float64)).cuda().requires_grad_(True)
  c64 = torch.from_numpy(c.astype(np.float64)).cuda().requires_grad_(True)
  (ref.torch_sinc_filter(x64, c64, ref.n_taps(ws)) * g).sum().backward()
  _check_grad('d audio', xa.grad.cpu().numpy(), x64.grad.cpu().numpy())
  _check_grad('d cutoff', ct.grad.cpu().numpy(), c64.grad.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize('shared', [False, True])
def test_gradients_bit_reproducible(shared):
  B, N, F, ws = 32, 64000, 1000, 512
  audio, c = _inputs(B, N, F, None, shared, 21)
  grads = []
  for _ in range(2):
    xa = _cuda(audio).requires_grad_(True)
    ct = _cuda(c).requires_grad_(True)
    y = core.sinc_filter(xa, ct, window_size=ws)
    y.backward(torch.ones_like(y) * 1e-3 + y.detach())
    grads.append((xa.grad.cpu().numpy(), ct.grad.cpu().numpy()))
  assert np.array_equal(grads[0][0], grads[1][0])
  assert np.array_equal(grads[0][1], grads[1][1])


@pytest.mark.gpu
def test_noise_sinc_filter_spectral_loss_chain():
  """noise -> sinc_filter (cutoff requires grad) -> SpectralLossFn against the float64
  chain through the same loss."""
  from ddsp_b200 import losses
  B, N, F, ws = 2, 16000, 100, 256
  noise, c = _inputs(B, N, F, None, False, 31)
  target = np.random.default_rng(32).standard_normal((B, N)).astype(np.float32)
  loss_fn = losses.SpectralLoss(fft_sizes=(2048, 512), loss_type='L1', mag_weight=1.0)
  ct = _cuda(c).requires_grad_(True)
  y = core.sinc_filter(_cuda(noise), ct, window_size=ws)
  loss = loss_fn(_cuda(target), y)
  loss.backward()
  c64 = torch.from_numpy(c.astype(np.float64)).cuda().requires_grad_(True)
  y64 = ref.torch_sinc_filter(torch.from_numpy(noise.astype(np.float64)).cuda(), c64,
                              ref.n_taps(ws))
  # the float64 chain runs the same loss on y64 rounded to float32 values, differentiated
  # through a float32 copy: compare the d y that reaches the filter instead
  y32 = y64.detach().float().requires_grad_(True)
  loss_fn(_cuda(target), y32).backward()
  (y64 * y32.grad.double()).sum().backward()
  _check_grad('d cutoff', ct.grad.cpu().numpy(), c64.grad.cpu().numpy())
