"""Training through the Processor API: `Harmonic` / `FilteredNoise.get_controls` and
`get_signal`, `ProcessorGroup.get_controls` + `get_signal` and
`group(features, return_outputs_dict=True)` under autograd.

CPU: which backward every shape is routed to (the launches recorded, nothing run), the
refusals that remain, and the float64 restatement of the `get_controls` vector-Jacobian
product pinned to float64 autograd of the oracle's arithmetic.  GPU: the
`ddsp_b200_harmonic_controls_vjp` kernel against that restatement at every flag
combination and row shape, the node-by-node path against `autograd.decoder_train`,
losses on the controls, the reference's other DAGs, `harmonic_shifts` and hops off the
harmonic backward kernel, and the entry point's input, stream and memory conventions.
"""
import contextlib

import numpy as np
import pytest
import torch

import ddsp_b200
from ddsp_b200 import _lib, autograd as ag, core, losses
from oracle import ddsp_oracle as oracle
from tests import grad_ref, sinusoidal_ref
from tests.util import rel_err, synth_inputs

SR = 16000
FLAGS = [(True, True), (True, False), (False, True), (False, False)]   # (scale, nyquist)


# ---- float64 restatements ------------------------------------------------------------
def exp_sigmoid64(x):
  return 2.0 * torch.sigmoid(x)**np.log(10.0) + 1e-7


def live_mask(f0, k, sample_rate=SR):
  """[B, F, K] bool, True where harmonic k is kept: the forward's float32 decision
  f0 * k < sr / 2 (core.py:888-890 on float32 operands)."""
  ratios = torch.arange(1, k + 1, dtype=torch.float32, device=f0.device)
  return ~((f0.to(torch.float32) * ratios) >= torch.tensor(sample_rate / 2.0,
                                                          dtype=torch.float32))


def controls64(amps, hd, f0, scale=True, nyquist=True, sample_rate=SR):
  """Harmonic.get_controls (synths.py:94-121) in float64 torch ops, the mask given by
  the float32 decision."""
  amps, hd = amps.double(), hd.double()
  if scale:
    amps, hd = exp_sigmoid64(amps), exp_sigmoid64(hd)
  if nyquist:
    hd = torch.where(live_mask(f0, hd.shape[-1], sample_rate), hd, torch.zeros_like(hd))
  s = hd.sum(-1, keepdim=True)
  return amps, hd / torch.where(s == 0.0, torch.full_like(s, 1e-7), s)


def controls_vjp64(amps, hd, f0, d_amps, d_hd, scale=True, nyquist=True, sample_rate=SR):
  """The row arithmetic of `harmonic_controls_vjp_kernel` in float64, without
  autograd: (d amps_raw, d hd_raw)."""
  amps, hd = amps.double(), hd.double()
  k = hd.shape[-1]
  keep = (live_mask(f0, k, sample_rate) if nyquist else
          torch.ones(hd.shape, dtype=torch.bool, device=hd.device))

  def dscale(x):            # exp_sigmoid'(x) = 2 sigmoid(x)^ln10 ln10 (1 - sigmoid(x))
    return 2.0 * torch.sigmoid(x)**np.log(10.0) * np.log(10.0) * torch.sigmoid(-x)
  e = exp_sigmoid64(hd) if scale else hd
  e = torch.where(keep, e, torch.zeros_like(e))
  s = e.sum(-1, keepdim=True)
  zero = s == 0.0
  denom = torch.where(zero, torch.full_like(s, 1e-7), s)
  up = torch.zeros_like(e) if d_hd is None else d_hd.double()
  couple = torch.where(zero, torch.zeros_like(s), (up * e).sum(-1, keepdim=True) / denom)
  d_e = torch.where(keep, (up - couple) / denom, torch.zeros_like(e))
  d_a = torch.zeros_like(amps) if d_amps is None else d_amps.double()
  if scale:
    d_e = d_e * dscale(hd)
    d_a = d_a * dscale(amps)
  return d_a, d_e


def controls_case(B, F, K, seed, device='cpu', magnitude=1.0):
  """Raw amplitudes and distribution ~ N(0, magnitude), and an f0 track with silent
  rows (f0 = 0), rows with every harmonic masked (f0 >= sr / 2), rows whose mask
  boundary lies one float32 ulp either side of Nyquist, and ordinary rows."""
  g = torch.Generator().manual_seed(seed)
  amps = magnitude * torch.randn(B, F, 1, generator=g)
  hd = magnitude * torch.randn(B, F, K, generator=g)
  f0 = 60.0 + 1500.0 * torch.rand(B, F, 1, generator=g)
  rows = f0.view(-1)
  nyq = np.float32(SR / 2.0)
  for i in range(rows.numel()):
    kind = i % 7
    if kind == 1:
      rows[i] = 0.0
    elif kind == 2:
      rows[i] = float(nyq) * (1.0 + 0.3 * (i % 3))
    elif kind in (3, 4) and K > 1:
      j = 1 + (i * 5) % K
      f = np.float32(nyq / np.float32(j))
      # nudge f until f * j lands exactly one ulp below (3) or at / above (4) Nyquist
      while np.float32(f * np.float32(j)) >= nyq:
        f = np.nextafter(f, np.float32(0.0))
      if kind == 4:
        while np.float32(f * np.float32(j)) < nyq:
          f = np.nextafter(f, np.float32(np.inf))
      rows[i] = float(f)
  return amps.to(device), hd.to(device), f0.to(device)


def _f64_controls_grads(amps, hd, f0, d_amps, d_hd, scale, nyquist):
  a64 = amps.detach().double().requires_grad_(True)
  h64 = hd.detach().double().requires_grad_(True)
  a, h = controls64(a64, h64, f0, scale, nyquist)
  loss = 0.0
  if d_amps is not None:
    loss = loss + (a * d_amps.double()).sum()
  if d_hd is not None:
    loss = loss + (h * d_hd.double()).sum()
  ga, gh = torch.autograd.grad(loss, [a64, h64], allow_unused=True)
  return (torch.zeros_like(a64) if ga is None else ga,
          torch.zeros_like(h64) if gh is None else gh)


# ---- CPU: the restatement ------------------------------------------------------------
@pytest.mark.parametrize('scale,nyquist', FLAGS)
def test_controls_restatement_matches_oracle(scale, nyquist):
  amps, hd, f0 = controls_case(2, 29, 33, seed=1)
  if not scale:
    amps, hd = amps.abs(), hd.abs()
  # the oracle decides the mask in float64: keep f0 * k away from Nyquist here
  f0 = 60.0 + 300.0 * torch.rand(2, 29, 1, generator=torch.Generator().manual_seed(2))
  want = oracle.harmonic_get_controls(amps.numpy(), hd.numpy(), f0.numpy(), scale=scale,
                                      normalize_below_nyquist=nyquist)
  a, h = controls64(amps, hd, f0, scale, nyquist)
  assert np.abs(a.numpy() - want['amplitudes']).max() <= 1e-12
  assert np.abs(h.numpy() - want['harmonic_distribution']).max() <= 1e-12


@pytest.mark.parametrize('scale,nyquist', FLAGS)
@pytest.mark.parametrize('K', [1, 33, 100])
def test_controls_vjp_restatement_matches_float64_autograd(scale, nyquist, K):
  amps, hd, f0 = controls_case(2, 29, K, seed=K)
  if not scale:
    hd = hd.abs()
    hd[0, 5] = 0.0                           # s == 0 with live harmonics
  g = torch.Generator().manual_seed(7)
  d_amps = torch.randn(amps.shape, generator=g, dtype=torch.float64)
  d_hd = torch.randn(hd.shape, generator=g, dtype=torch.float64)
  for da, dh in ((d_amps, d_hd), (d_amps, None), (None, d_hd)):
    want_a, want_h = _f64_controls_grads(amps, hd, f0, da, dh, scale, nyquist)
    got_a, got_h = controls_vjp64(amps, hd, f0, da, dh, scale, nyquist)
    assert float((got_a - want_a).abs().max()) <= 1e-12 * max(1.0, float(want_a.abs().max()))
    assert float((got_h - want_h).abs().max()) <= 1e-12 * max(1.0, float(want_h.abs().max()))


# ---- CPU: routing, with nothing launched -----------------------------------------------
class _Launches:
  """Stands in for `core._launch`: records the symbols and launches nothing."""

  def __init__(self):
    self.symbols = []

  def __call__(self, symbol, *args):
    self.symbols.append(symbol)


@pytest.fixture
def launches(monkeypatch):
  """core and autograd launch into a recorder, tensors stay where they are and the
  workspace queries answer 0: the routes run on CPU tensors, without the library."""
  rec = _Launches()
  monkeypatch.setattr(core, '_launch', rec)
  monkeypatch.setattr(core, 'torch_float32',
                      lambda x, device=None: torch.as_tensor(x, dtype=torch.float32))
  monkeypatch.setattr(core, '_workspace', lambda *a: (None, 0))
  return rec


def _leaf(*shape):
  return torch.rand(*shape).requires_grad_(True)


def _run(fn):
  out = fn()
  outs = [o for o in (out if isinstance(out, tuple) else (out,)) if o.requires_grad]
  torch.autograd.backward(outs, [torch.ones_like(o) for o in outs])


def test_routes_of_the_controls(launches):
  a, h, f0 = _leaf(2, 10, 1), _leaf(2, 10, 8), torch.rand(2, 10, 1)
  _run(lambda: core.harmonic_controls(a, h, f0, SR))
  assert launches.symbols == ['ddsp_b200_harmonic_controls', 'ddsp_b200_harmonic_controls_vjp']
  assert a.grad.shape == a.shape and h.grad.shape == h.shape
  launches.symbols.clear()
  m = _leaf(2, 10, 65)
  _run(lambda: core.noise_controls(m, -5.0))
  assert launches.symbols == ['ddsp_b200_noise_controls', 'ddsp_b200_noise_controls_backward']
  # f0 alone takes no gradient through get_controls: the plain launch, no refusal
  launches.symbols.clear()
  out = core.harmonic_controls(a.detach(), h.detach(), f0.clone().requires_grad_(True), SR)
  assert launches.symbols == ['ddsp_b200_harmonic_controls'] and not out[0].requires_grad


def test_noise_controls_without_scaling_passes_the_gradient_through(launches):
  m = _leaf(2, 10, 65)
  out = core.noise_controls(m, -5.0, scale=False)
  g = torch.rand(2, 10, 65)
  out.backward(g)
  assert launches.symbols == ['ddsp_b200_noise_controls'] and torch.equal(m.grad, g)


@pytest.mark.parametrize('frames,n,method,shifts,want', [
    (10, 640, 'window', False, ['ddsp_b200_harmonic_forward', 'ddsp_b200_harmonic_backward']),
    (10, 1280, 'linear', False, ['ddsp_b200_harmonic_forward', 'ddsp_b200_harmonic_backward']),
    (10, 640, 'window', True, ['ddsp_b200_sinusoidal_forward', 'ddsp_b200_sinusoidal_backward']),
    (10, 1000, 'window', False, ['ddsp_b200_sinusoidal_forward',
                                 'ddsp_b200_sinusoidal_backward']),
    (201, 64320, 'linear', False, ['ddsp_b200_harmonic_forward',
                                   'ddsp_b200_harmonic_backward']),
    (10, 640, 'cubic', False, ['ddsp_b200_resample', 'ddsp_b200_resample',
                               'ddsp_b200_oscillator_bank',
                               'ddsp_b200_oscillator_bank_backward',
                               'ddsp_b200_resample_backward']),
    (7, 100, 'linear', False, ['ddsp_b200_resample', 'ddsp_b200_resample',
                               'ddsp_b200_oscillator_bank',
                               'ddsp_b200_oscillator_bank_backward',
                               'ddsp_b200_resample_backward']),
])
def test_routes_of_harmonic_synthesis(launches, frames, n, method, shifts, want):
  f0 = torch.full((1, frames, 1), 200.0)
  a, h = _leaf(1, frames, 1), _leaf(1, frames, 4)
  s = 0.01 * torch.rand(1, frames, 4) if shifts else None
  _run(lambda: core.harmonic_synthesis(f0, a, harmonic_shifts=s, harmonic_distribution=h,
                                       n_samples=n, amp_resample_method=method))
  assert launches.symbols == want
  assert a.grad is not None and h.grad is not None


def test_harmonic_synthesis_f0_gradient_only_when_asked(launches):
  f0 = torch.full((1, 10, 1), 200.0, requires_grad=True)
  a, h = _leaf(1, 10, 1), _leaf(1, 10, 4)
  _run(lambda: core.harmonic_synthesis(f0, a, harmonic_distribution=h, n_samples=640))
  assert launches.symbols == ['ddsp_b200_harmonic_forward', 'ddsp_b200_harmonic_backward',
                              'ddsp_b200_harmonic_backward_f0']
  launches.symbols.clear()
  # no harmonic_distribution: ones [B, F, 1]
  a2 = _leaf(1, 10, 1)
  _run(lambda: core.harmonic_synthesis(f0.detach(), a2, n_samples=640))
  assert launches.symbols == ['ddsp_b200_harmonic_forward', 'ddsp_b200_harmonic_backward']
  assert a2.grad.shape == (1, 10, 1)


def test_routes_of_filtered_noise(launches):
  m = _leaf(2, 10, 65)
  _run(lambda: core.filtered_noise(m, 640, window_size=0, seed=3, offset=5))
  assert launches.symbols == ['ddsp_b200_filtered_noise_forward',
                              'ddsp_b200_filtered_noise_backward']
  assert m.grad.shape == m.shape


@pytest.mark.parametrize('f,nb,n,ws,takes', [
    (10, 65, 640, 0, True), (1000, 65, 64000, 257, True), (33, 33, 3293, 257, True),
    (10, 65, 640, 2, False),          # one tap: nothing to compensate the delay with
    (2, 65, 2048, 0, False),          # 32 frames of 1024 samples do not fit one CTA
    (20, 129, 10240, 0, False)])
def test_noise_backward_shapes(launches, f, nb, n, ws, takes):
  """Shapes the filtered-noise backward does not take keep the refusal."""
  assert core._noise_backward_takes(f, nb, n, ws) == takes
  m = _leaf(1, f, nb)
  if takes:
    assert core.filtered_noise(m, n, window_size=ws).requires_grad
  else:
    with pytest.raises(RuntimeError, match='requires grad'):
      core.filtered_noise(m, n, window_size=ws)
    assert launches.symbols == []


def test_refusals_fire_before_any_device_work(monkeypatch):
  """`out=` under grad, phase_mode='tf_sequential' under grad and the shape errors are
  raised on CPU tensors with no library to load."""
  def touched(*a, **k):
    raise AssertionError('device touched')
  monkeypatch.setattr(core, 'torch_float32', touched)
  monkeypatch.setattr(core._lib, 'load', touched)
  f0 = torch.full((1, 10, 1), 200.0)
  a, h, m = _leaf(1, 10, 1), _leaf(1, 10, 4), _leaf(1, 10, 65)
  with pytest.raises(RuntimeError, match='requires grad'):
    core.harmonic_synthesis(f0, a, harmonic_distribution=h, n_samples=640,
                            out=torch.zeros(1, 640))
  with pytest.raises(RuntimeError, match='requires grad'):
    core.filtered_noise(m, 640, out=torch.zeros(1, 640), accumulate=True)
  with pytest.raises(NotImplementedError, match='tf_sequential'):
    core.harmonic_synthesis(f0, a, harmonic_distribution=h, n_samples=640,
                            phase_mode='tf_sequential')
  with pytest.raises(ValueError, match='divisible'):
    core.harmonic_synthesis(f0, a, harmonic_distribution=h, n_samples=645)
  with pytest.raises(ValueError, match='Number of Audio frames'):
    core.filtered_noise(m, 14)
  with pytest.raises(ValueError, match='harmonic_distribution'):
    core.harmonic_synthesis(f0, a, harmonic_distribution=torch.zeros(1, 9, 4), n_samples=640)


def _group(n, method='window', window_size=0, seed=3):
  harm = ddsp_b200.Harmonic(n_samples=n, amp_resample_method=method)
  noise = ddsp_b200.FilteredNoise(n_samples=n, window_size=window_size, seed=seed)
  group = ddsp_b200.ProcessorGroup(dag=[
      (harm, ['amps', 'harmonic_distribution', 'f0_hz']),
      (noise, ['noise_magnitudes']),
      (ddsp_b200.Add(), ['filtered_noise/signal', 'harmonic/signal'])])
  return group, harm, noise


def _feats(B, F, K, nb, N, seed, device='cpu', grad=True):
  inp = synth_inputs(B, F, K, nb, N, seed=seed)
  feats = {k: torch.from_numpy(inp[k]).to(device) for k in
           ('amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes')}
  if grad:
    for k in ('amps', 'harmonic_distribution', 'noise_magnitudes'):
      feats[k].requires_grad_(True)
  return feats


def test_group_routes(launches):
  """return_outputs_dict=True trains node by node; the signal-only call is the fused
  inference call and keeps refusing; under no_grad nothing new is launched."""
  group, _, _ = _group(640)
  feats = _feats(1, 10, 8, 65, 640, seed=3)
  out = group(feats, return_outputs_dict=True)
  forward = ['ddsp_b200_harmonic_controls', 'ddsp_b200_harmonic_forward',
             'ddsp_b200_noise_controls', 'ddsp_b200_filtered_noise_forward', 'ddsp_b200_add']
  assert launches.symbols == forward
  launches.symbols.clear()
  ctl = out['controls']
  (out['signal'].sum() + ctl['harmonic']['controls']['harmonic_distribution'].sum() +
   ctl['filtered_noise']['controls']['magnitudes'].sum()).backward()
  assert sorted(launches.symbols) == sorted([
      'ddsp_b200_filtered_noise_backward', 'ddsp_b200_noise_controls_backward',
      'ddsp_b200_harmonic_backward', 'ddsp_b200_harmonic_controls_vjp'])
  assert all(feats[k].grad is not None for k in ('amps', 'harmonic_distribution',
                                                 'noise_magnitudes'))
  launches.symbols.clear()
  with pytest.raises(RuntimeError, match='requires grad'):
    group(feats)
  assert launches.symbols == []
  with torch.no_grad():
    group(feats, return_outputs_dict=True)
    assert launches.symbols == forward
    launches.symbols.clear()
    group(feats)
    assert launches.symbols == ['ddsp_b200_decoder_forward']


def test_group_fallback_with_custom_scale_fn_still_refuses(launches):
  """A custom scale_fn takes the signal-only call off the fused kernel; it then writes
  through out= / accumulate=, which autograd cannot track."""
  group, harm, _ = _group(640)
  harm.scale_fn = torch.sigmoid
  with pytest.raises(RuntimeError, match='requires grad'):
    group(_feats(1, 10, 8, 65, 640, seed=3))
  assert 'ddsp_b200_filtered_noise_forward' not in launches.symbols


# ---- GPU -----------------------------------------------------------------------------
DEV = 'cuda'


def _check(name, got, want, tol_max, tol_l2, floor=0.0):
  """Max-abs and L2 error relative to the reference; a reference whose peak is below
  `floor` (zero by cancellation) is matched to tol_max * floor instead."""
  got = got.detach().double().cpu().numpy()
  want = want.detach().double().cpu().numpy()
  assert np.isfinite(got).all(), name
  if np.abs(want).max() <= floor:
    assert np.abs(got - want).max() <= tol_max * floor, (name, np.abs(got - want).max())
    return 0.0, 0.0
  emax, el2 = rel_err(got, want)
  assert emax < tol_max and el2 < tol_l2, (name, emax, el2)
  return emax, el2


@pytest.mark.gpu
@pytest.mark.parametrize('scale,nyquist', FLAGS)
@pytest.mark.parametrize('F', [1, 257])
@pytest.mark.parametrize('K', [1, 31, 32, 33, 100, 260])
def test_controls_vjp_against_float64(scale, nyquist, F, K):
  """d amps_raw and d hd_raw of `core.harmonic_controls` for upstream gradients on the
  amplitudes, on the distribution and on both, against float64: 2e-4 max-relative and
  1e-4 relative L2 (the kernel's exp2 / log2 are the approximate ones)."""
  amps, hd, f0 = controls_case(3, F, K, seed=F + K, device=DEV)
  if not scale:
    hd = hd.abs()
    hd[0, 0] = 0.0                          # s == 0 with every harmonic live
  g = torch.Generator().manual_seed(K)
  d_amps = torch.randn(amps.shape, generator=g).to(DEV)
  d_hd = torch.randn(hd.shape, generator=g).to(DEV)
  for da, dh in ((d_amps, d_hd), (d_amps, None), (None, d_hd)):
    a1, h1 = amps.clone().requires_grad_(True), hd.clone().requires_grad_(True)
    a, h = core.harmonic_controls(a1, h1, f0, SR, scale=scale,
                                  normalize_below_nyquist=nyquist)
    outs, gs = zip(*[(o, d) for o, d in ((a, da), (h, dh)) if d is not None])
    torch.autograd.backward(outs, gs)
    want_a, want_h = controls_vjp64(amps, hd, f0, da, dh, scale, nyquist)
    # K = 1 normalises to 1 whatever the input: its d hd is zero by cancellation
    _check('d amps', a1.grad, want_a, 2e-4, 1e-4)
    _check('d hd', h1.grad, want_h, 2e-4, 1e-4, floor=1e-2 * float(d_hd.abs().max()))
    if nyquist:
      dead = ~live_mask(f0, K)
      assert float(h1.grad[dead].abs().max() if dead.any() else 0.0) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize('value', [30.0, -30.0, 100.0, -100.0])
def test_controls_vjp_is_finite_at_saturated_inputs(value):
  amps, hd, f0 = controls_case(2, 33, 100, seed=5, device=DEV)
  amps, hd = torch.full_like(amps, value), torch.full_like(hd, value)
  hd[:, ::2, ::3] = -value
  a1, h1 = amps.requires_grad_(True), hd.requires_grad_(True)
  a, h = core.harmonic_controls(a1, h1, f0, SR)
  (a.sum() + (h * torch.arange(100, device=DEV)).sum()).backward()
  assert torch.isfinite(a1.grad).all() and torch.isfinite(h1.grad).all()
  want_a, want_h = controls_vjp64(amps, hd, f0, torch.ones_like(amps),
                                  torch.arange(100, device=DEV).expand_as(hd))
  _check('d amps', a1.grad, want_a, 2e-4, 1e-4)
  _check('d hd', h1.grad, want_h, 1e-3, 3e-4)


@pytest.mark.gpu
def test_controls_vjp_entry_point_checks_its_arguments():
  """NULL operands, bad shapes and too many rows are E_INVALID with a message; B = 0
  returns 0; none of them launches."""
  lib = _lib.load()
  t = torch.zeros(64, device=DEV)
  p = t.data_ptr()
  before = lib.ddsp_b200_launch_count()
  vjp = lib.ddsp_b200_harmonic_controls_vjp
  assert vjp(None, p, p, p, p, p, p, 1, 2, 4, 16000.0, 3, None) == _lib.E_INVALID
  assert b'null pointer' in lib.ddsp_b200_last_error()
  assert vjp(p, p, p, p, p, p, None, 1, 2, 4, 16000.0, 3, None) == _lib.E_INVALID
  assert vjp(p, p, p, p, p, p, p, 1, 0, 4, 16000.0, 3, None) == _lib.E_INVALID
  assert b'bad shape' in lib.ddsp_b200_last_error()
  assert vjp(p, p, p, p, p, p, p, -1, 2, 4, 16000.0, 3, None) == _lib.E_INVALID
  assert vjp(p, p, p, p, p, p, p, 1 << 20, 1 << 10, 4, 16000.0, 3, None) == _lib.E_INVALID
  assert b'too large' in lib.ddsp_b200_last_error()
  assert vjp(p, p, p, None, None, p, p, 0, 2, 4, 16000.0, 3, None) == 0
  assert lib.ddsp_b200_launch_count() == before


@pytest.mark.gpu
def test_controls_vjp_operand_conventions():
  """Non-contiguous, CPU and wrong-device operands raise before the launch; the launch
  goes to the operands' device and current stream."""
  amps, hd, f0 = controls_case(2, 10, 8, seed=1, device=DEV)
  d_a, d_h, o_a, o_h = (torch.ones_like(amps), torch.ones_like(hd), torch.empty_like(amps),
                        torch.empty_like(hd))
  lib = _lib.load()
  before = lib.ddsp_b200_launch_count()
  wide = torch.ones((2, 10, 16), device=DEV)[..., ::2]
  with pytest.raises(ValueError, match='not contiguous'):
    core._launch('ddsp_b200_harmonic_controls_vjp', amps, hd, f0, d_a, wide, o_a, o_h, 2, 10,
                 8, float(SR), 3)
  with pytest.raises(ValueError, match='not a CUDA device'):
    core._launch('ddsp_b200_harmonic_controls_vjp', amps, hd, f0, d_a.cpu(), d_h, o_a, o_h,
                 2, 10, 8, float(SR), 3)
  assert lib.ddsp_b200_launch_count() == before
  if torch.cuda.device_count() > 1:
    with pytest.raises(ValueError, match='different devices'):
      core._launch('ddsp_b200_harmonic_controls_vjp', amps, hd, f0.to('cuda:1'), d_a, d_h,
                   o_a, o_h, 2, 10, 8, float(SR), 3)
  # strided upstream gradients are made contiguous by the autograd node
  a1, h1 = amps.clone().requires_grad_(True), hd.clone().requires_grad_(True)
  a, h = core.harmonic_controls(a1, h1, f0, SR)
  torch.autograd.backward([a, h], [d_a, wide])
  want = h1.grad.clone()
  # a side stream: same bits, and the recorded launch names that stream
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  seen = []
  real = core._lib.load

  class Spy:
    def __getattr__(self, name):
      fn = getattr(real(), name)
      if name != 'ddsp_b200_harmonic_controls_vjp':
        return fn

      def call(*args):
        seen.append((torch.cuda.current_device(), args[-1]))
        return fn(*args)
      return call
  a2, h2 = amps.clone().requires_grad_(True), hd.clone().requires_grad_(True)
  with contextlib.ExitStack() as stack:
    stack.enter_context(torch.cuda.stream(side))
    core._lib.load = Spy
    stack.callback(setattr, core._lib, 'load', real)
    a, h = core.harmonic_controls(a2, h2, f0, SR)
    torch.autograd.backward([a, h], [d_a, d_h])
  side.synchronize()
  assert seen == [(amps.device.index, side.cuda_stream)]
  assert torch.equal(h2.grad, want)


@pytest.mark.gpu
@pytest.mark.parametrize('poison', [0x00, 0xFF, 0x7F])
def test_controls_vjp_writes_all_of_its_outputs_and_nothing_else(poison):
  """On poisoned, fenced gradient buffers (tests/test_gpu_memory_bounds.py) and with
  the upstream gradients between NaN fences: every element written, the fences intact,
  the bits those of plain operands.  K = 33 and F = 5 leave a partial warp pass and a
  partial block."""
  from tests.test_gpu_memory_bounds import guarded
  amps, hd, f0 = controls_case(3, 5, 33, seed=2, device=DEV)
  g = torch.Generator().manual_seed(1)
  d_a = torch.randn(amps.shape, generator=g).to(DEV)
  d_h = torch.randn(hd.shape, generator=g).to(DEV)

  def fenced(x):
    buf = torch.full((x.numel() + 2 * 16384,), float('nan'), device=DEV)
    v = buf[16384:16384 + x.numel()].view(x.shape)
    v.copy_(x)
    return v

  def run(da, dh):
    a1, h1 = amps.clone().requires_grad_(True), hd.clone().requires_grad_(True)
    a, h = core.harmonic_controls(a1, h1, f0, SR)
    torch.autograd.backward([a, h], [da, dh])
    return a1.grad, h1.grad
  want = run(d_a, d_h)
  with guarded(poison):
    got = run(fenced(d_a), fenced(d_h))
  for g_, w in zip(got, want):
    assert torch.isfinite(g_).all() and torch.equal(g_, w)
  # an upstream gradient on one control only: the other's NULL writes zeros everywhere
  with guarded(poison):
    a1, h1 = amps.clone().requires_grad_(True), hd.clone().requires_grad_(True)
    a, h = core.harmonic_controls(a1, h1, f0, SR)
    a.backward(d_a)
  assert float(h1.grad.abs().max()) == 0.0 and torch.equal(a1.grad, want[0])


def _raw64(feats, idx=slice(None)):
  return {k: feats[k].detach()[idx].double().requires_grad_(k != 'f0_hz')
          for k in feats}


def _decoder64(r, nz, N, method='window', window_size=0, nyquist=True):
  """(audio, harmonic controls, magnitudes) of the ae.gin DAG in float64 torch ops."""
  a, h = controls64(r['amps'], r['harmonic_distribution'], r['f0_hz'], True, nyquist)
  mags = exp_sigmoid64(r['noise_magnitudes'] - 5.0)
  audio = (grad_ref.harmonic(r['f0_hz'], a, h, N, SR, method) +
           grad_ref.frequency_filter(nz.double(), mags, window_size))
  return audio, h, mags


@pytest.mark.gpu
@pytest.mark.parametrize('B,F,N', [(3, 250, 16000), (128, 1000, 64000)],
                         ids=['small', 'c4'])
def test_node_by_node_path_equals_the_fused_training_path(B, F, N):
  """`group(feats, return_outputs_dict=True)['signal']` against
  `autograd.decoder_train` on the same Philox stream: the audio within 2e-6 of its peak
  (the fused kernels apply get_controls on chip in a different order of float32
  operations), every gradient within 1e-5 relative L2."""
  K, nb = 100, 65
  feats = _feats(B, F, K, nb, N, seed=B, device=DEV)
  f0 = feats['f0_hz'].requires_grad_(True)
  g = torch.randn((B, N), device=DEV, generator=torch.Generator(DEV).manual_seed(1))
  group, _, noise = _group(N, seed=9)
  out = group(feats, return_outputs_dict=True)      # the first call: Philox offset 0
  out['signal'].backward(g)
  got = {k: v.grad.clone() for k, v in feats.items()}
  for v in feats.values():
    v.grad = None
  audio = ag.decoder_train(feats['amps'], feats['harmonic_distribution'], f0,
                           feats['noise_magnitudes'], n_samples=N, seed=9, offset=0)
  audio.backward(g)
  emax, _ = rel_err(out['signal'].detach().cpu().numpy(), audio.detach().cpu().numpy())
  assert emax < 2e-6, emax
  for k, v in feats.items():
    _check(k, got[k], v.grad, 5e-5, 1e-5)
  assert set(out['controls']) >= {'harmonic', 'filtered_noise', 'add', 'out'}


@pytest.mark.gpu
def test_losses_on_the_controls_and_the_audio():
  """SpectralLoss on the audio plus L1 terms on harmonic/controls/harmonic_distribution
  and filtered_noise/controls/magnitudes, through get_controls + get_signal as the
  reference's models write it; gradients to the raw inputs against float64 autograd of
  the op-by-op restatement, the spectral term's gradient taken in float64."""
  B, F, K, nb, N = 2, 125, 60, 65, 8000
  feats = _feats(B, F, K, nb, N, seed=11, device=DEV)
  group, _, noise = _group(N, seed=4)
  nz = core.uniform_noise(B, N, seed=4, offset=0)
  target = 0.1 * torch.randn((B, N), device=DEV, generator=torch.Generator(DEV).manual_seed(2))
  controls = group.get_controls(feats)
  audio = group.get_signal(controls)
  hd = controls['harmonic']['controls']['harmonic_distribution']
  mags = controls['filtered_noise']['controls']['magnitudes']
  assert audio.requires_grad and hd.requires_grad and mags.requires_grad

  r = _raw64(feats)
  audio64, hd64, mags64 = _decoder64(r, nz, N)
  _check('audio', audio, audio64, 1e-4, 1e-4)
  loss64 = (grad_ref.spectral_loss(target.double(), audio64, logmag_weight=1.0) +
            0.3 * (hd64 - 0.01).abs().mean() + 2.0 * (mags64 - 0.02).abs().mean())
  g_audio = torch.autograd.grad(loss64, audio64, retain_graph=True)[0]
  loss64.backward()
  # the float64 gradient of the spectral term drives our backward, as in
  # test_gpu_fullsize.py; the control terms go through the float32 graph
  side = 0.3 * (hd - 0.01).abs().mean() + 2.0 * (mags - 0.02).abs().mean()
  torch.autograd.backward([audio, side], [g_audio.float(), torch.ones_like(side)])
  for k in ('amps', 'harmonic_distribution', 'noise_magnitudes'):
    _check(k, feats[k].grad, r[k].grad, 2e-3, 1e-3)
  # and the whole float32 chain, SpectralLoss included, runs and is finite
  for v in feats.values():
    v.grad = None
  out = group(feats, return_outputs_dict=True)
  total = (losses.SpectralLoss(logmag_weight=1.0)(target, out['signal']) +
           out['controls']['harmonic']['controls']['harmonic_distribution'].abs().mean())
  total.backward()
  for k in ('amps', 'harmonic_distribution', 'noise_magnitudes'):
    assert torch.isfinite(feats[k].grad).all() and float(feats[k].grad.abs().max()) > 0


@pytest.mark.gpu
def test_solo_instrument_dag_trains_with_its_reverb():
  """Harmonic, FilteredNoise, Add and a trainable Reverb (solo_instrument.gin):
  gradients to every raw input and to the impulse response against float64."""
  B, F, K, nb, N, L = 2, 125, 40, 65, 8000, 3000
  feats = _feats(B, F, K, nb, N, seed=21, device=DEV)
  harm = ddsp_b200.Harmonic(n_samples=N)
  noise = ddsp_b200.FilteredNoise(n_samples=N, window_size=0, seed=6)
  reverb = ddsp_b200.Reverb(trainable=True, reverb_length=L)
  reverb.build(torch.device(DEV))
  with torch.no_grad():
    reverb._ir.mul_(3e4)                      # an audible tail
  group = ddsp_b200.ProcessorGroup(dag=[
      (harm, ['amps', 'harmonic_distribution', 'f0_hz']),
      (noise, ['noise_magnitudes']),
      (ddsp_b200.Add(), ['filtered_noise/signal', 'harmonic/signal']),
      (reverb, ['add/signal'])])
  g = torch.randn((B, N), device=DEV, generator=torch.Generator(DEV).manual_seed(3))
  nz = core.uniform_noise(B, N, seed=6, offset=0)
  audio = group.get_signal(group.get_controls(feats))
  audio.backward(g)

  r = _raw64(feats)
  ir64 = reverb._ir.detach().double().requires_grad_(True)
  dry, _, _ = _decoder64(r, nz, N)
  masked = torch.cat([ir64.new_zeros(1), ir64[1:]])[None, :]
  want = grad_ref.convolve_lti(dry, masked, 0, N) + dry
  want.backward(g.double())
  _check('audio', audio, want, 1e-4, 1e-4)
  for k in ('amps', 'harmonic_distribution', 'noise_magnitudes'):
    _check(k, feats[k].grad, r[k].grad, 2e-3, 1e-3)
  _check('ir', reverb._ir.grad, ir64.grad, 2e-3, 1e-3)


@pytest.mark.gpu
def test_vst_layout_trains():
  """'linear' amplitudes, 64320 samples from 201 frames (hop 320), ending in Crop."""
  B, F, K, nb, N = 2, 201, 60, 65, 64320
  feats = _feats(B, F, K, nb, N, seed=31, device=DEV)
  f0 = feats['f0_hz'].requires_grad_(True)
  harm = ddsp_b200.Harmonic(n_samples=N, amp_resample_method='linear')
  noise = ddsp_b200.FilteredNoise(n_samples=N, window_size=0, seed=1)
  group = ddsp_b200.ProcessorGroup(dag=[
      (harm, ['amps', 'harmonic_distribution', 'f0_hz']),
      (noise, ['noise_magnitudes']),
      (ddsp_b200.Add(), ['filtered_noise/signal', 'harmonic/signal']),
      (ddsp_b200.Crop(frame_size=320, crop_location='back'), ['add/signal'])])
  audio = group.get_signal(group.get_controls(feats))
  assert audio.shape == (B, N - 320)
  (audio**2).mean().backward()
  for k, v in feats.items():
    assert torch.isfinite(v.grad).all() and float(v.grad.abs().max()) > 0, k


@pytest.mark.gpu
@pytest.mark.parametrize('hop,method,with_shifts', [(64, 'window', True), (100, 'window', False),
                                                    (100, 'linear', True)])
def test_harmonic_shifts_and_other_hops_against_float64(hop, method, with_shifts):
  """Gradients to f0, amplitudes, distribution and harmonic_shifts of
  core.harmonic_synthesis on its sinusoidal route against float64 autograd."""
  B, F, K = 2, 40, 20
  N = F * hop
  g = torch.Generator().manual_seed(hop)
  f0 = (150.0 + 200.0 * torch.rand(B, F, 1, generator=g)).to(DEV)
  amps = (0.2 + torch.rand(B, F, 1, generator=g)).to(DEV)
  hd = torch.rand(B, F, K, generator=g).to(DEV)
  shifts = (0.02 * torch.randn(B, F, K, generator=g)).to(DEV) if with_shifts else None
  up = torch.randn(B, N, generator=g).to(DEV)
  leaves = [t.clone().requires_grad_(True) for t in (f0, amps, hd)]
  s1 = shifts.clone().requires_grad_(True) if with_shifts else None
  out = core.harmonic_synthesis(leaves[0], leaves[1], harmonic_shifts=s1,
                                harmonic_distribution=leaves[2], n_samples=N,
                                amp_resample_method=method)
  out.backward(up)
  l64 = [t.double().requires_grad_(True) for t in (f0, amps, hd)]
  s64 = shifts.double().requires_grad_(True) if with_shifts else None
  want = sinusoidal_ref.harmonic_sinusoidal64(l64[0], l64[1], l64[2], s64, N, SR, method)
  want.backward(up.double())
  _check('audio', out, want, 1e-4, 1e-4)
  for name, got, ref in zip(('f0', 'amps', 'hd'), leaves, l64):
    _check(name, got.grad, ref.grad, 2e-3, 1e-3)
  if with_shifts:
    _check('shifts', s1.grad, s64.grad, 2e-3, 1e-3)


@pytest.mark.gpu
def test_envelope_route_trains():
  """'cubic' amplitudes and a non-integer hop: resample + oscillator_bank carry the
  gradient to every input."""
  for frames, n, method in ((10, 640, 'cubic'), (7, 100, 'linear'), (10, 640, 'nearest')):
    f0 = torch.full((2, frames, 1), 220.0, device=DEV, requires_grad=True)
    a = torch.rand(2, frames, 1, device=DEV).requires_grad_(True)
    h = torch.rand(2, frames, 6, device=DEV).requires_grad_(True)
    out = core.harmonic_synthesis(f0, a, harmonic_distribution=h, n_samples=n,
                                  amp_resample_method=method)
    with torch.no_grad():
      plain = core.harmonic_synthesis(f0, a, harmonic_distribution=h, n_samples=n,
                                      amp_resample_method=method)
    assert torch.equal(out.detach(), plain)
    out.square().sum().backward()
    for t in (f0, a, h):
      assert torch.isfinite(t.grad).all() and float(t.grad.abs().max()) > 0


@pytest.mark.gpu
def test_forward_audio_does_not_depend_on_the_gradient_request():
  """The same bits with and without grad, FilteredNoise's Philox offset included; and
  the no-grad node-by-node call launches exactly its five kernels."""
  B, F, K, nb, N = 2, 125, 30, 65, 8000
  feats = _feats(B, F, K, nb, N, seed=41, device=DEV)
  g1, _, _ = _group(N, seed=2)
  g2, _, _ = _group(N, seed=2)
  lib = _lib.load()
  for _ in range(2):                       # offsets 0 and 1
    got = g1(feats, return_outputs_dict=True)['signal']
    with torch.no_grad():
      before = lib.ddsp_b200_launch_count()
      want = g2(feats, return_outputs_dict=True)['signal']
      assert lib.ddsp_b200_launch_count() - before == 5
    assert torch.equal(got.detach(), want)


@pytest.mark.gpu
def test_gradients_are_bit_reproducible():
  B, F, K, nb, N = 2, 125, 100, 65, 8000
  runs = []
  for _ in range(2):
    feats = _feats(B, F, K, nb, N, seed=51, device=DEV)
    feats['f0_hz'].requires_grad_(True)
    group, _, _ = _group(N, seed=2)
    out = group(feats, return_outputs_dict=True)
    hd = out['controls']['harmonic']['controls']['harmonic_distribution']
    (out['signal'].square().mean() + hd.abs().mean()).backward()
    runs.append({k: v.grad.clone() for k, v in feats.items()})
  for k in runs[0]:
    assert torch.equal(runs[0][k], runs[1][k]), k


@pytest.mark.gpu
def test_noise_backward_shape_rule_is_the_entry_points():
  """`core._noise_backward_takes` against `ddsp_b200_filtered_noise_backward` itself."""
  for f, nb, n, ws in ((10, 65, 640, 0), (33, 33, 3293, 257), (10, 65, 640, 2),
                       (2, 65, 2048, 0), (20, 129, 10240, 0), (4, 129, 1792, 0),
                       (3, 65, 2700, 0), (3, 65, 2900, 0)):
    g = torch.zeros((1, n), device=DEV)
    dm = torch.empty((1, f, nb), device=DEV)
    try:
      core._launch('ddsp_b200_filtered_noise_backward', g, None, 0, 0, dm, 1, f, nb, n, ws)
      took = True
    except NotImplementedError:
      took = False
    assert took == core._noise_backward_takes(f, nb, n, ws), (f, nb, n, ws)
