"""Backward of the direct-form time-varying FIR and of the impulse-response synthesis
(csrc/fir_backward.cuh): `ddsp_b200_fir_time_varying_backward`,
`ddsp_b200_frequency_impulse_response_backward`, `ddsp_b200_frequency_filter_backward`
and the autograd routes of core.fft_convolve (impulse responses under 2048 taps),
core.frequency_impulse_response, core.frequency_filter and the effects built on them.

The CPU tests check the C ABI's argument checks and workspace sizes and the Python
argument checks under grad.  The GPU tests check every gradient (a) elementwise
against float64 autograd of tests/grad_ref.py and (b), for the linear maps, through
<dL/dx, D> = sum g * y(D) with y the float64 ORACLE (tests.util.linearity)."""
import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core

P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID, E_UNSUPPORTED, E_WORKSPACE = _lib.E_INVALID, _lib.E_UNSUPPORTED, _lib.E_WORKSPACE
SAME, VALID = _lib.PAD_SAME, _lib.PAD_VALID

# (case, entry point, arguments, status, the full last_error or None)
_FIR = 'fir_time_varying_backward'
_IRB = 'frequency_impulse_response_backward'
_FF = 'frequency_filter_backward'
_ABI_CASES = [
    ('fir-null-audio', _FIR, (None, P, P, P, P, 1, 1000, 10, 16, 1, SAME, -1, P, 1 << 30, None), E_INVALID, b'fir_time_varying_backward: null pointer'),
    ('fir-null-ir', _FIR, (P, None, P, P, P, 1, 1000, 10, 16, 1, SAME, -1, P, 1 << 30, None), E_INVALID, b'fir_time_varying_backward: null pointer'),
    ('fir-null-grad', _FIR, (P, P, None, P, P, 1, 1000, 10, 16, 1, SAME, -1, P, 1 << 30, None), E_INVALID, b'fir_time_varying_backward: null pointer'),
    ('fir-B', _FIR, (P, P, P, P, P, -1, 1000, 10, 16, 1, SAME, -1, P, 1 << 30, None), E_INVALID, b'fir_time_varying_backward: bad shape B=-1 N=1000 F=10 S=16'),
    ('fir-N', _FIR, (P, P, P, P, P, 1, 0, 10, 16, 1, SAME, -1, P, 1 << 30, None), E_INVALID, b'fir_time_varying_backward: bad shape B=1 N=0 F=10 S=16'),
    ('fir-F', _FIR, (P, P, P, P, P, 1, 1000, 0, 16, 1, SAME, -1, P, 1 << 30, None), E_INVALID, b'fir_time_varying_backward: bad shape B=1 N=1000 F=0 S=16'),
    ('fir-S', _FIR, (P, P, P, P, P, 1, 1000, 10, 0, 1, SAME, -1, P, 1 << 30, None), E_INVALID, b'fir_time_varying_backward: bad shape B=1 N=1000 F=10 S=0'),
    ('fir-batch', _FIR, (P, P, P, P, P, 2, 1000, 10, 16, 3, SAME, -1, P, 1 << 30, None), E_INVALID, b'Batch size of audio (2) and impulse response (3) must be the same.'),
    ('fir-padding', _FIR, (P, P, P, P, P, 1, 1000, 10, 16, 1, 5, -1, P, 1 << 30, None), E_INVALID, b"Padding must be 'valid' or 'same' (got code 5)"),
    ('fir-frames', _FIR, (P, P, P, P, P, 1, 1000, 999, 16, 1, SAME, -1, P, 1 << 30, None), E_INVALID, b'Number of Audio frames (500) and impulse response frames (999) do not match. For small hop size = ceil(audio_size / n_ir_frames), number of impulse response frames must be a multiple of the audio size.'),
    ('fir-B0', _FIR, (P, P, P, P, P, 0, 1000, 10, 16, 1, SAME, -1, None, 0, None), 0, None),
    ('fir-grid', _FIR, (P, P, P, P, P, 65536, 1000, 10, 16, 1, SAME, -1, P, 1 << 30, None), E_INVALID, b'fir_time_varying_backward: B=65536 exceeds the 65535 grid limit'),
    ('fir-S2-auto', _FIR, (P, P, P, P, P, 1, 1000, 10, 2, 1, SAME, -1, P, 1 << 30, None), E_UNSUPPORTED, b'fir_time_varying_backward: impulse response of 2 taps gives a negative automatic delay'),
    ('fir-S1-auto', _FIR, (P, P, P, P, P, 1, 1000, 10, 1, 1, VALID, -1, P, 1 << 30, None), E_UNSUPPORTED, b'fir_time_varying_backward: impulse response of 1 taps gives a negative automatic delay'),
    ('fir-S-smem', _FIR, (P, P, P, P, P, 1, 100000, 1, 60000, 1, SAME, 0, P, 1 << 40, None), E_UNSUPPORTED, b'fir_time_varying_backward: impulse response of 60000 taps is beyond the shared-memory FIR'),
    ('fir-workspace-null', _FIR, (P, P, P, P, P, 2, 64000, 1, 2047, 2, SAME, -1, None, 0, None), E_WORKSPACE, b'fir_time_varying_backward: workspace of 4094256 B needed, 0 given'),
    ('fir-workspace-short', _FIR, (P, P, P, P, P, 3, 1000, 10, 16, 1, SAME, -1, P, 2175, None), E_WORKSPACE, b'fir_time_varying_backward: workspace of 2176 B needed, 2175 given'),
    ('irb-null', _IRB, (None, P, 10, 65, 257, None), E_INVALID, b'frequency_impulse_response_backward: null pointer'),
    ('irb-nb', _IRB, (P, P, 10, 1, 0, None), E_INVALID, b'frequency_impulse_response_backward: need n_frequencies >= 2 (got 1)'),
    ('irb-BF', _IRB, (P, P, -1, 65, 0, None), E_INVALID, b'frequency_impulse_response_backward: need n_frequencies >= 2 (got 65)'),
    ('irb-BF0', _IRB, (P, P, 0, 65, 0, None), 0, None),
    ('irb-5121', _IRB, (P, P, 10, 5121, 0, None), E_UNSUPPORTED, b'frequency_impulse_response_backward: n_frequencies=5121 too large'),
    ('ff-null-audio', _FF, (None, P, P, P, P, 1, 10, 65, 640, 1, 257, SAME, P, 1 << 30, None), E_INVALID, b'frequency_filter_backward: null pointer'),
    ('ff-null-ir', _FF, (P, None, P, P, P, 1, 10, 65, 640, 1, 257, SAME, P, 1 << 30, None), E_INVALID, b'frequency_filter_backward: null pointer'),
    ('ff-null-grad', _FF, (P, P, None, P, P, 1, 10, 65, 640, 1, 257, SAME, P, 1 << 30, None), E_INVALID, b'frequency_filter_backward: null pointer'),
    ('ff-B', _FF, (P, P, P, P, P, -1, 10, 65, 640, 1, 257, SAME, P, 1 << 30, None), E_INVALID, b'frequency_filter_backward: bad shape B=-1 F=10 nb=65 N=640'),
    ('ff-F', _FF, (P, P, P, P, P, 1, 0, 65, 640, 1, 257, SAME, P, 1 << 30, None), E_INVALID, b'frequency_filter_backward: bad shape B=1 F=0 nb=65 N=640'),
    ('ff-nb', _FF, (P, P, P, P, P, 1, 10, 1, 640, 1, 257, SAME, P, 1 << 30, None), E_INVALID, b'frequency_filter_backward: bad shape B=1 F=10 nb=1 N=640'),
    ('ff-N', _FF, (P, P, P, P, P, 1, 10, 65, 0, 1, 257, SAME, P, 1 << 30, None), E_INVALID, b'frequency_filter_backward: bad shape B=1 F=10 nb=65 N=0'),
    ('ff-batch', _FF, (P, P, P, P, P, 3, 10, 65, 640, 2, 257, SAME, P, 1 << 30, None), E_INVALID, b'Batch size of audio (3) and impulse response (2) must be the same.'),
    ('ff-padding', _FF, (P, P, P, P, P, 1, 10, 65, 640, 1, 257, 2, P, 1 << 30, None), E_INVALID, b"Padding must be 'valid' or 'same' (got code 2)"),
    ('ff-frames', _FF, (P, P, P, P, P, 1, 999, 65, 1000, 1, 257, SAME, P, 1 << 30, None), E_INVALID, b'Number of Audio frames (500) and impulse response frames (999) do not match. For small hop size = ceil(audio_size / n_ir_frames), number of impulse response frames must be a multiple of the audio size.'),
    ('ff-B0', _FF, (P, P, P, P, P, 0, 10, 65, 640, 1, 257, SAME, None, 0, None), 0, None),
    ('ff-grid', _FF, (P, P, P, P, P, 65536, 10, 65, 640, 1, 257, SAME, P, 1 << 30, None), E_INVALID, b'frequency_filter_backward: B=65536 exceeds the 65535 grid limit'),
    ('ff-nb2', _FF, (P, P, P, P, P, 1, 10, 2, 640, 1, 0, SAME, P, 1 << 30, None), E_UNSUPPORTED, b'frequency_filter_backward: impulse response of 2 taps gives a negative automatic delay'),
    ('ff-ws2', _FF, (P, P, P, P, P, 1, 10, 65, 640, 1, 2, SAME, P, 1 << 30, None), E_UNSUPPORTED, b'frequency_filter_backward: impulse response of 1 taps gives a negative automatic delay'),
    ('ff-5121', _FF, (P, P, P, P, P, 1, 1, 5121, 64000, 1, 257, VALID, P, 1 << 40, None), E_UNSUPPORTED, b'frequency_filter_backward: n_frequencies=5121 too large'),
    ('ff-workspace-null', _FF, (P, P, P, P, P, 2, 10, 65, 640, 1, 257, SAME, None, 0, None), E_WORKSPACE, b'frequency_filter_backward: workspace of 15616 B needed, 0 given'),
    ('ff-workspace-short', _FF, (P, P, P, P, P, 1, 1, 65, 16000, 1, 257, SAME, P, 100, None), E_WORKSPACE, b'frequency_filter_backward: workspace of 33024 B needed, 100 given'),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_fir_backward_abi_check_table(fn, args, want, msg):
  """Every check of the three backward entry points, one row each: the status and
  the full message come back before any CUDA call, and nothing is launched."""
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  assert getattr(lib, 'ddsp_b200_' + fn)(*args) == want
  assert lib.ddsp_b200_launch_count() == launches
  if msg is not None:
    assert lib.ddsp_b200_last_error() == msg
    error = {E_INVALID: ValueError, E_UNSUPPORTED: NotImplementedError,
             E_WORKSPACE: RuntimeError}[want]
    with pytest.raises(error):
      _lib.check(want)


def test_fir_backward_skips_the_workspace_without_d_ir():
  """The workspace serves d IR / d magnitudes only: without them none is needed.
  B = 0 keeps the call from launching."""
  lib = _lib.load()
  assert lib.ddsp_b200_fir_time_varying_backward(
      P, P, P, P, None, 0, 64000, 1, 2047, 1, SAME, -1, None, 0, None) == 0


# (entry point, arguments, bytes)
_WS_CASES = [
    ('fir_time_varying_backward_workspace', (32, 64000, 1000, 128, 32), 0),    # frame 64
    ('fir_time_varying_backward_workspace', (32, 64000, 250, 128, 32), 0),     # frame 256
    ('fir_time_varying_backward_workspace', (1, 64000, 200, 128, 1), 204800 + 256),  # 2 segments
    ('fir_time_varying_backward_workspace', (5, 1000, 10, 16, 1), 5 * 10 * 16 * 4 + 256),
    ('fir_time_varying_backward_workspace', (1, 1000, 10, 16, 1), 0),
    ('fir_time_varying_backward_workspace', (32, 64000, 1, 2047, 32), 32 * 250 * 2047 * 4 + 256),
    ('fir_time_varying_backward_workspace', (2, 1000, 999, 16, 2), 0),        # frames mismatch
    ('fir_time_varying_backward_workspace', (2, 1000, 10, 16, 3), 0),         # bad ir_batch
    ('fir_time_varying_backward_workspace', (0, 1000, 10, 16, 1), 0),
    ('frequency_filter_backward_workspace', (32, 1000, 65, 64000, 32, 257, SAME), 0),   # fused
    ('frequency_filter_backward_workspace', (32, 1000, 16, 47000, 32, 0, SAME), 0),     # fused
    ('frequency_filter_backward_workspace', (2, 10, 65, 640, 2, 257, VALID), 256 + 10240),
    ('frequency_filter_backward_workspace', (2, 10, 65, 640, 1, 257, SAME), 256 + 5120 + 10240),
    ('frequency_filter_backward_workspace', (1, 1, 65, 16000, 1, 257, SAME), 256 + 512 + 63 * 128 * 4),
    ('frequency_filter_backward_workspace', (2, 10, 1025, 640, 2, 257, SAME), 256 + 20736),
    ('frequency_filter_backward_workspace', (0, 10, 65, 640, 1, 257, SAME), 0),
    ('frequency_filter_backward_workspace', (1, 10, 1, 640, 1, 0, SAME), 0),
]


@pytest.mark.parametrize('fn,args,want', _WS_CASES,
                         ids=['%s-%s' % (c[0].split('_')[0], '-'.join(map(str, c[1])))
                              for c in _WS_CASES])
def test_fir_backward_workspace_table(fn, args, want):
  """Partial d IR sums exist only for frames of more than 256 samples or a shared
  impulse response; frequency_filter adds d IR on the generic route and needs
  nothing on the fused one."""
  assert getattr(_lib.load(), 'ddsp_b200_' + fn)(*args) == want


@pytest.mark.parametrize('nb,ws', [(2, 0), (3, 0), (65, 257), (65, 0), (1025, 257),
                                   (513, 22), (100, 50), (65, 1), (65, 2), (65, 127)])
def test_python_ir_size_matches_the_library(nb, ws):
  assert core._ir_size(nb, ws) == _lib.load().ddsp_b200_ir_size(nb, ws)


def _no_library(monkeypatch):
  def fail():
    raise AssertionError('the library was loaded before the argument checks')
  monkeypatch.setattr(_lib, 'load', fail)


@pytest.mark.parametrize('audio_shape,ir_shape,padding,match', [
    ((2, 100), (3, 1, 16), 'same', 'Batch size'),
    ((1, 1000), (1, 999, 16), 'same', 'Number of Audio frames'),
    ((1, 100), (16,), 'same', 'impulse_response 2-D or 3-D'),
    ((1, 100), (1, 4, 16), 'full', 'Padding must be'),
])
def test_fft_convolve_under_grad_raises_before_device_work(monkeypatch, audio_shape,
                                                          ir_shape, padding, match):
  _no_library(monkeypatch)
  audio = torch.zeros(audio_shape, requires_grad=True)
  ir = torch.zeros(ir_shape, requires_grad=True)
  with pytest.raises(ValueError, match=match):
    core.fft_convolve(audio, ir, padding=padding)


@pytest.mark.parametrize('audio_shape,mags_shape,padding,match', [
    ((2, 640), (3, 10, 65), 'same', 'Batch size'),
    ((1, 1000), (1, 999, 65), 'same', 'Number of Audio frames'),
    ((1, 640), (1, 10, 1), 'same', 'needs >= 2 frequencies'),
    ((1, 640), (1, 10, 65), 'causal', 'Padding must be'),
    ((640,), (1, 10, 65), 'same', 'audio must be'),
])
def test_frequency_filter_under_grad_raises_before_device_work(monkeypatch, audio_shape,
                                                              mags_shape, padding, match):
  _no_library(monkeypatch)
  audio = torch.zeros(audio_shape)
  mags = torch.zeros(mags_shape, requires_grad=True)
  with pytest.raises(ValueError, match=match):
    core.frequency_filter(audio, mags, window_size=257, padding=padding)


def test_frequency_impulse_response_under_grad_raises_before_device_work(monkeypatch):
  _no_library(monkeypatch)
  with pytest.raises(ValueError, match='needs >= 2 frequencies'):
    core.frequency_impulse_response(torch.zeros(2, 1, requires_grad=True))


# ---------------------------------------------------------------------------
# On the GPU
# ---------------------------------------------------------------------------
DEV = torch.device('cuda')


def _check(name, got, want, tol_max, tol_l2):
  assert got is not None, name
  assert torch.isfinite(got).all(), name
  got, want = got.detach().double(), want.detach().double()
  peak = float(want.abs().max())
  emax = float((got - want).abs().max()) / max(peak, 1e-300)
  l2 = float(((got - want)**2).sum().sqrt()) / max(float((want**2).sum().sqrt()), 1e-300)
  assert emax < tol_max and l2 < tol_l2, (name, emax, l2)


def _randn(shape, seed):
  return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(DEV)


# (B, N, F, S, ir_batch, padding, delay)
FIR_CASES = [
    (2, 1000, 10, 3, 2, 'same', -1),
    (2, 1000, 10, 4, 2, 'valid', -1),
    (2, 4000, 1, 64, 2, 'same', -1),
    (2, 1000, 7, 127, 2, 'same', -1),         # ragged last frame (142 of 143)
    (1, 1000, 16, 128, 1, 'valid', -1),       # ragged (55 of 63)
    (2, 3000, 1, 257, 2, 'same', 0),
    (2, 3000, 1, 257, 2, 'same', 128),        # S / 2
    (2, 3000, 1, 257, 2, 'same', 300),        # past S
    (2, 600, 600, 64, 2, 'same', -1),         # F = N: frames of one sample
    (1, 16000, 1000, 257, 1, 'same', -1),     # F = 1000, 16-sample frames
    (2, 4000, 1, 1000, 2, 'same', 0),         # a direct-form reverb
    (1, 4000, 1, 2047, 1, 'valid', -1),
    (2, 5000, 1, 2047, 2, 'same', 2100),
    (2, 600, 3, 1000, 2, 'same', 0),          # N < S, frames of 200
    (2, 100, 1, 257, 2, 'valid', -1),         # N < S
    (2, 1, 1, 64, 2, 'same', -1),             # N = 1
    (2, 2, 1, 3, 2, 'same', -1),              # N = 2
    (2, 2, 2, 64, 2, 'same', 5),
    (5, 1000, 10, 64, 1, 'same', -1),         # shared impulse response
    (5, 3000, 1, 1000, 1, 'valid', 0),        # shared, twelve 250-sample segments
    (3, 1000, 2, 128, 1, 'same', 70),         # shared, frames of 500: two segments each
]


@pytest.mark.gpu
@pytest.mark.parametrize('B,N,F,S,ir_batch,padding,delay', FIR_CASES)
def test_fft_convolve_backward(B, N, F, S, ir_batch, padding, delay):
  """core.fft_convolve's direct-form route under grad (FirTimeVaryingFn): d audio
  and d IR against float64 autograd, and the linearity identity against the oracle
  for both operands."""
  from oracle import ddsp_oracle as o
  from tests import grad_ref
  from tests.util import linearity
  x = _randn((B, N), S + N)
  h = _randn((ir_batch, F, S), S * 7 + F) / np.sqrt(S)
  want_shape = (B, N + S - 1 if padding == 'valid' else N)
  g = _randn(want_shape, B + S)
  x1, h1 = x.clone().requires_grad_(True), h.clone().requires_grad_(True)
  out = core.fft_convolve(x1, h1, padding=padding, delay_compensation=delay)
  assert tuple(out.shape) == want_shape
  (out * g).sum().backward()
  x2, h2 = x.double().requires_grad_(True), h.double().requires_grad_(True)
  ref = grad_ref.fft_convolve(x2, h2, padding, delay)
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  _check('d audio', x1.grad, x2.grad, 2e-4, 1e-4)
  _check('d ir', h1.grad, h2.grad, 2e-4, 1e-4)
  xn, hn = x.double().cpu().numpy(), h.double().cpu().numpy()
  linearity(x1.grad, g, lambda d: o.fft_convolve(d, hn, padding, delay), (B, N), seed=S)
  linearity(h1.grad, g, lambda d: o.fft_convolve(xn, d, padding, delay), (ir_batch, F, S),
            seed=S + 1)


@pytest.mark.gpu
def test_fft_convolve_backward_only_what_is_asked():
  """Only the operand that requires grad gets one, and out= / accumulate= add the
  tracked result as the long-IR branch does."""
  x, h = _randn((2, 1000), 1), _randn((2, 10, 64), 2)
  h1 = h.clone().requires_grad_(True)
  out = torch.ones(2, 1000, device=DEV)
  got = core.fft_convolve(x, h1, out=out, accumulate=True)
  assert got is out
  got.sum().backward()
  with torch.no_grad():
    base = core.fft_convolve(x, h)
  assert torch.equal(out.detach(), base + 1)
  x1 = x.clone().requires_grad_(True)
  core.fft_convolve(x1, h).sum().backward()
  assert x1.grad is not None and h1.grad is not None


def _mags(shape, seed):
  return (torch.rand(shape, generator=torch.Generator().manual_seed(seed)) + 0.05).to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize('nb,ws', [(3, 0), (4, 0), (16, 0), (65, 0), (129, 0), (1025, 0),
                                   (5120, 0), (65, 31), (65, 64), (1025, 257), (5120, 257),
                                   (65, 1000), (16, 257), (2, 0), (3, 3)])
def test_frequency_impulse_response_backward(nb, ws):
  """FrequencyImpulseResponseFn: windows none, odd and even padded, 1, 2 and
  clamped (ws > S0); bin counts up to the forward's limit."""
  from oracle import ddsp_oracle as o
  from tests import grad_ref
  from tests.util import linearity
  BF = 3 if nb < 5000 else 9
  m = _mags((BF, nb), nb + ws)
  s = core._ir_size(nb, ws)
  g = _randn((BF, s), nb)
  m1 = m.clone().requires_grad_(True)
  ir = core.frequency_impulse_response(m1, ws)
  (ir * g).sum().backward()
  m2 = m.double().requires_grad_(True)
  ref = grad_ref.impulse_response(m2, ws)
  (ref * g.double()).sum().backward()
  _check('ir', ir, ref, 1e-4, 1e-4)
  _check('d mags', m1.grad, m2.grad, 2e-4, 1e-4)
  linearity(m1.grad, g, lambda d: o.frequency_impulse_response(d, ws), (BF, nb), seed=nb)


@pytest.mark.gpu
@pytest.mark.parametrize('nb,ws', [(129, 1), (129, 2), (3, 1), (3, 2), (2, 1)])
def test_frequency_impulse_response_backward_one_and_two_tap_windows(nb, ws):
  """Windows of one and two samples: the library's impulse response has one tap
  where the reference's slice keeps two (DESIGN §3.12), so the backward is checked
  as the exact transpose of the library's own forward, <d mags, D> = <g, ir(D)>."""
  BF = 4
  m = _mags((BF, nb), nb + ws)
  s = core._ir_size(nb, ws)
  g = _randn((BF, s), nb + 1)
  m1 = m.clone().requires_grad_(True)
  (core.frequency_impulse_response(m1, ws) * g).sum().backward()
  for seed in range(3):
    d = _mags((BF, nb), 100 + seed)
    with torch.no_grad():
      want = float((g.double() * core.frequency_impulse_response(d, ws).double()).sum())
    got = float((m1.grad.double() * d.double()).sum())
    scale = float((g.double() * core.frequency_impulse_response(d, ws).double()).abs().sum())
    assert abs(got - want) <= 1e-5 * max(scale, 1e-30), (got, want, scale)


@pytest.mark.gpu
def test_frequency_impulse_response_backward_limit():
  """5121 bins are past the shared memory of the forward and the backward alike."""
  m = _mags((1, 5121), 0).requires_grad_(True)
  with pytest.raises(NotImplementedError, match='too large'):
    core.frequency_impulse_response(m)


def _fused(B, F, nb, N, mb, ws, padding):
  """True when frequency_filter's d magnitudes take the fused kernel (no workspace)."""
  pad = _lib.PAD_SAME if padding == 'same' else _lib.PAD_VALID
  return _lib.load().ddsp_b200_frequency_filter_backward_workspace(
      B, F, nb, N, mb, ws, pad) == 0


# (B, mags shape, N, ws, padding, fused)
FILTER_CASES = [
    (2, (2, 50, 65), 3200, 0, 'same', True),
    (2, (2, 50, 65), 3200, 257, 'same', True),
    (2, (2, 31, 16), 31 * 47 - 20, 0, 'same', True),       # frame 47, ragged
    (2, (2, 10, 1025), 2560, 257, 'same', False),          # smem too large for fused
    (2, (2, 65), 16000, 257, 'same', False),               # 2-D magnitudes: F = 1
    (2, (2, 40, 65), 2560, 257, 'valid', False),
    (3, (1, 40, 65), 2560, 257, 'same', False),            # shared magnitudes
    (3, (1, 40, 16), 2560, 31, 'valid', False),
]


@pytest.mark.gpu
@pytest.mark.parametrize('B,mshape,N,ws,padding,fused', FILTER_CASES)
def test_frequency_filter_backward(B, mshape, N, ws, padding, fused):
  """core.frequency_filter under grad (FrequencyFilterFn), both d magnitudes routes:
  the fused noise kernel where it fits, d IR + the IR adjoint elsewhere."""
  from oracle import ddsp_oracle as o
  from tests import grad_ref
  from tests.util import linearity
  F = mshape[1] if len(mshape) == 3 else 1
  nb = mshape[-1]
  assert _fused(B, F, nb, N, mshape[0], ws, padding) == fused
  x = _randn((B, N), N + nb)
  m = _mags(mshape, nb + ws)
  s = core._ir_size(nb, ws)
  g = _randn((B, N + s - 1 if padding == 'valid' else N), B + nb)
  x1, m1 = x.clone().requires_grad_(True), m.clone().requires_grad_(True)
  out = core.frequency_filter(x1, m1, window_size=ws, padding=padding)
  (out * g).sum().backward()
  x2, m2 = x.double().requires_grad_(True), m.double().requires_grad_(True)
  ref = grad_ref.fft_convolve(x2, grad_ref.impulse_response(m2, ws).reshape(
      mshape[0], F, s), padding)
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  _check('d audio', x1.grad, x2.grad, 2e-4, 1e-4)
  _check('d mags', m1.grad, m2.grad, 2e-4, 1e-4)
  xn = x.double().cpu().numpy()
  linearity(m1.grad, g, lambda d: o.frequency_filter(xn, d, ws, padding), mshape, seed=nb)


def _generic_d_mags(x, ir, g, B, F, nb, N, ws):
  """frequency_filter's d magnitudes through kernels 2 + 3 on their own entry points:
  d IR by fir_time_varying_backward, then frequency_impulse_response_backward."""
  lib = _lib.load()
  st = torch.cuda.current_stream().cuda_stream
  s = ir.shape[-1]
  d_ir = torch.empty(B, F, s, device=DEV)
  nbytes = lib.ddsp_b200_fir_time_varying_backward_workspace(B, N, F, s, B)
  ws_buf = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=DEV)
  _lib.check(lib.ddsp_b200_fir_time_varying_backward(
      x.data_ptr(), ir.data_ptr(), g.data_ptr(), None, d_ir.data_ptr(), B, N, F, s, B,
      SAME, -1, ws_buf.data_ptr(), nbytes, st))
  d_mags = torch.empty(B, F, nb, device=DEV)
  _lib.check(lib.ddsp_b200_frequency_impulse_response_backward(
      d_ir.data_ptr(), d_mags.data_ptr(), B * F, nb, ws, st))
  return d_mags


@pytest.mark.gpu
@pytest.mark.parametrize('nb,ws,frame', [(65, 257, 64), (65, 0, 64), (16, 0, 47),
                                         (129, 64, 100)])
def test_frequency_filter_routes_agree(nb, ws, frame):
  """At shapes both routes take, the fused d magnitudes and kernels 2 + 3 agree."""
  B, F = 3, 40
  N = F * frame
  assert _fused(B, F, nb, N, B, ws, 'same')
  x = _randn((B, N), nb)
  m = _mags((B, F, nb), frame)
  g = _randn((B, N), ws)
  m1 = m.clone().requires_grad_(True)
  (core.frequency_filter(x, m1, window_size=ws) * g).sum().backward()
  ir = core.frequency_impulse_response(m, ws)
  want = _generic_d_mags(x, ir, g, B, F, nb, N, ws)
  rel = float((m1.grad - want).norm() / want.norm())
  assert rel <= 1e-5, rel


@pytest.mark.gpu
@pytest.mark.parametrize('what', ['nb65', 'nb1025', 'ir2047'])
def test_backward_is_bit_reproducible(what):
  """Two backward passes at the decoder size give bit-identical gradients: no
  atomics, and split sums are added in a fixed order."""
  B, N = 32, 64000
  x = _randn((B, N), 3)
  g = _randn((B, N), 4)
  runs = []
  for _ in range(2):
    x1 = x.clone().requires_grad_(True)
    if what == 'ir2047':
      h1 = (_randn((B, 2047), 5) / 45.0).requires_grad_(True)
      core.fft_convolve(x1, h1, delay_compensation=0).mul(g).sum().backward()
      runs.append((x1.grad, h1.grad))
    else:
      nb = 65 if what == 'nb65' else 1025
      m1 = _mags((B, 1000, nb), 6).requires_grad_(True)
      core.frequency_filter(x1, m1, window_size=257).mul(g).sum().backward()
      runs.append((x1.grad, m1.grad))
  for a, b in zip(*runs):
    assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize('mags_too', [True, False])
def test_fir_filter_processor_backward(mags_too):
  """effects.FIRFilter(window_size=257) on raw magnitudes with .backward(): d raw
  magnitudes (through exp_sigmoid) and d audio against float64 autograd.  With the
  magnitudes alone requiring grad the gradient must still arrive."""
  from ddsp_b200 import autograd as ag
  from ddsp_b200 import effects
  from tests import grad_ref
  B, F, nb, N = 2, 100, 65, 6400
  x = _randn((B, N), 11)
  raw = _randn((B, F, nb), 12)
  g = _randn((B, N), 13)
  x1 = x.clone().requires_grad_(mags_too)
  r1 = raw.clone().requires_grad_(True)
  out = effects.FIRFilter(window_size=257)(x1, r1)
  assert out.requires_grad
  (out * g).sum().backward()
  x2, r2 = x.double().requires_grad_(True), raw.double().requires_grad_(True)
  ref = grad_ref.frequency_filter(x2, ag.exp_sigmoid(r2), 257)
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  _check('d raw magnitudes', r1.grad, r2.grad, 2e-4, 1e-4)
  if mags_too:
    _check('d audio', x1.grad, x2.grad, 2e-4, 1e-4)


@pytest.mark.gpu
def test_short_trainable_reverb_backward():
  """Reverb(trainable=True, reverb_length=1000) now runs the direct-form FIR under
  grad: d audio and d learned impulse response against float64 autograd."""
  from ddsp_b200 import effects
  from tests import grad_ref
  B, N, L = 2, 4000, 1000
  rev = effects.Reverb(trainable=True, reverb_length=L)
  rev.build(DEV)
  with torch.no_grad():
    rev._ir.copy_(_randn((L,), 21) * 0.05)
  x = _randn((B, N), 22)
  g = _randn((B, N), 23)
  x1 = x.clone().requires_grad_(True)
  out = rev(x1)
  (out * g).sum().backward()
  x2 = x.double().requires_grad_(True)
  h2 = rev._ir.detach().double().requires_grad_(True)
  h = torch.cat([torch.zeros(1, dtype=torch.float64, device=DEV), h2[1:]])
  ref = grad_ref.fft_convolve(x2, h.expand(B, L)[:, None, :], 'same', 0) + x2
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  _check('d audio', x1.grad, x2.grad, 2e-4, 1e-4)
  _check('d ir', rev._ir.grad, h2.grad, 2e-4, 1e-4)


@pytest.mark.gpu
def test_short_filtered_noise_reverb_backward():
  """FilteredNoiseReverb(trainable=True, reverb_length=2000, n_frames=100): d audio
  and d learned magnitudes through the direct-form FIR."""
  from ddsp_b200 import autograd as ag
  from ddsp_b200 import effects
  from tests import grad_ref
  B, N, L, F, nb, ws, bias = 2, 5000, 2000, 100, 16, 257, -3.0
  rev = effects.FilteredNoiseReverb(trainable=True, reverb_length=L, n_frames=F,
                                    n_filter_banks=nb, window_size=ws)
  noise = torch.rand(1, L, generator=torch.Generator().manual_seed(31)).to(DEV) * 2 - 1
  rev._synth.injected_noise = noise
  rev.build(DEV)
  mags = _randn((F, nb), 32)
  rev._magnitudes = mags.clone().requires_grad_(True)
  x = _randn((B, N), 33)
  g = _randn((B, N), 34)
  x1 = x.clone().requires_grad_(True)
  out = rev(x1)
  (out * g).sum().backward()
  x2, m2 = x.double().requires_grad_(True), mags.double().requires_grad_(True)
  ir = grad_ref.frequency_filter(noise.double(), ag.exp_sigmoid(m2[None] + bias), ws)
  ir = torch.cat([torch.zeros_like(ir[:, :1]), ir[:, 1:]], dim=1).expand(B, L)
  ref = grad_ref.fft_convolve(x2, ir[:, None, :], 'same', 0) + x2
  (ref * g.double()).sum().backward()
  _check('audio', out, ref, 1e-4, 1e-4)
  _check('d audio', x1.grad, x2.grad, 2e-4, 1e-4)
  _check('d magnitudes', rev._magnitudes.grad, m2.grad, 2e-4, 1e-4)


@pytest.mark.gpu
def test_harmonic_fir_spectral_loss_chain():
  """A training-shaped chain at a reduced size: HarmonicSynthesisFn -> FIRFilter ->
  SpectralLossFn (magnitude L1), against the float64 chain grad_ref.harmonic ->
  grad_ref.frequency_filter -> grad_ref.spectral_loss."""
  from ddsp_b200 import autograd as ag
  from ddsp_b200 import effects
  from ddsp_b200 import spectral_ops
  from tests import grad_ref
  B, F, K, nb, hop, sr = 2, 50, 20, 65, 64, 16000
  N = F * hop
  fft_sizes = (1024, 256, 64)
  f0 = (200.0 + 100.0 * torch.rand(B, F, 1, generator=torch.Generator().manual_seed(41))
        ).to(DEV)
  amp = _mags((B, F, 1), 42)
  hd = _mags((B, F, K), 43)
  hd = hd / hd.sum(-1, keepdim=True)
  raw = _randn((B, F, nb), 44)
  target = _randn((B, N), 45) * 0.1
  a1, r1 = amp.clone().requires_grad_(True), raw.clone().requires_grad_(True)
  audio = ag.HarmonicSynthesisFn.apply(f0, a1, hd, N, sr, 'window')
  audio = effects.FIRFilter(window_size=257)(audio, r1)
  loss = spectral_ops.SpectralLossFn.apply(target, audio, fft_sizes, 1.0, 0.0)
  loss.backward()
  a2, r2 = amp.double().requires_grad_(True), raw.double().requires_grad_(True)
  ref = grad_ref.harmonic(f0.double(), a2, hd.double(), N, sr, 'window',
                          mask=grad_ref.nyquist_mask(f0, K, N, sr))
  ref = grad_ref.frequency_filter(ref, ag.exp_sigmoid(r2), 257)
  ref_loss = grad_ref.spectral_loss(target, ref, fft_sizes, 1.0, 0.0)
  ref_loss.backward()
  lv, rv = float(loss.detach()), float(ref_loss.detach())
  assert abs(lv - rv) <= 1e-4 * rv, (lv, rv)
  _check('d amplitudes', a1.grad, a2.grad, 2e-4, 1e-4)
  _check('d FIR magnitudes', r1.grad, r2.grad, 2e-4, 1e-4)
