"""effects.ModDelay and core.variable_length_delay (effects.py:328-394,
core.py:1285-1314): the oracle and the float64 torch restatement against the
unmodified reference's fixture (CPU), the host composition of ModDelay against the
reference class (CPU, kernels swapped for the oracle), and the CUDA forward and
backward kernels against float64 (GPU)."""

import numpy as np
import pytest
import torch

from ddsp_b200 import core
from oracle import ddsp_oracle as o
from oracle import ref_on_shim
from tests import mod_delay_ref as ref
from tests.golden import make_mod_delay_golden as mg
from tests.util import rel_err

GOLDEN = mg.PATH


def _fixture():
  return np.load(GOLDEN)


# ---- CPU ---------------------------------------------------------------------
def test_oracle_matches_reference_fixture():
  """float64 closed form vs the reference run wide, float32 TF order vs the
  reference run in float32, on every L / N / phase case of the fixture."""
  want = _fixture()
  for i, (L, _, kind, phase, audio) in enumerate(mg.mod_delay_inputs()):
    w64 = ref.variable_length_delay(phase, audio, L)
    w32 = ref.variable_length_delay(phase, audio, L, dtype=np.float32)
    assert np.abs(w64 - want['delay_wide_%02d' % i]).max() <= 1e-12, (L, kind)
    assert np.abs(w32 - want['delay_f32_%02d' % i]).max() <= 1e-6, (L, kind)


@pytest.mark.skipif(not ref_on_shim.available(), reason='reference sources absent')
def test_fixture_regenerates_from_reference():
  mg.compare('mod_delay', mg.mod_delay(), _fixture())


def test_torch_restatement_matches_oracle():
  for L, _, kind, phase, audio in mg.mod_delay_inputs():
    got = ref.torch_variable_length_delay(torch.from_numpy(phase[..., 0]).double(),
                                          torch.from_numpy(audio).double(), L)
    assert np.abs(got.numpy() - ref.variable_length_delay(phase, audio, L)).max() <= 1e-12, (
        L, kind)


def _oracle_kernels(monkeypatch):
  """core's device entry points replaced by the float32 oracle on CPU tensors."""
  def t32(x, device=None):
    return torch.as_tensor(np.asarray(x.detach() if isinstance(x, torch.Tensor) else x,
                                      dtype=np.float32))

  def forward(audio, gain, phase, max_length, scale, offset, add_dry):
    x = audio.numpy()
    p = phase.numpy() * np.float32(scale) + np.float32(offset)
    wet = ref.variable_length_delay(p, x, max_length, dtype=np.float32)
    if gain is not None:
      wet = wet * gain.numpy()
    return torch.from_numpy(wet + x if add_dry else wet)
  monkeypatch.setattr(core, 'torch_float32', t32)
  monkeypatch.setattr(core, 'mod_delay_forward', forward)


@pytest.mark.parametrize('case', range(len(mg.MOD_DELAY_PROCESSOR)))
def test_mod_delay_composition_matches_reference(monkeypatch, case):
  """ModDelay's host logic (effects.py:328-394: scale functions, the phase map and
  max_length at 16 and 44.1 kHz, 2-D and 3-D gain and phase, the dry mix) against the
  UNMODIFIED reference class run on the shim (tests/golden/mod_delay.npz).  The
  kernels are the float32 oracle here; they have their own GPU tests."""
  from ddsp_b200 import effects
  sr, add_dry, scaled, _, _, _ = mg.MOD_DELAY_PROCESSOR[case]
  audio, gain, phase = mg.mod_delay_processor_inputs()[case]
  want = _fixture()['processor_f32_%d' % case]
  _oracle_kernels(monkeypatch)
  md = effects.ModDelay(sample_rate=sr, add_dry=add_dry)
  assert (md.center_ms, md.depth_ms, md.name) == (15.0, 10.0, 'mod_delay')
  assert md.gain_scale_fn is core.exp_sigmoid and md.phase_scale_fn is torch.sigmoid
  if scaled:   # the reference's float32 arithmetic: a last-ulp sigmoid moves positions
    md.gain_scale_fn = lambda x: torch.from_numpy(o.exp_sigmoid(x.numpy(), dtype=np.float32))
    md.phase_scale_fn = lambda x: torch.from_numpy(
        np.float32(1.0) / (np.float32(1.0) + np.exp(-x.numpy())))
  else:
    md.gain_scale_fn = md.phase_scale_fn = None
  with torch.no_grad():
    controls = md.get_controls(audio, gain, phase)
    assert sorted(controls) == ['audio', 'gain', 'phase']
    got = md(audio, gain, phase).numpy()
  assert got.shape == want.shape == audio.shape
  assert np.abs(got - want).max() < 2e-5 * max(1.0, np.abs(want).max())


def test_value_errors_before_device_work(monkeypatch):
  """max_length < 1 (the reference's tf.pad fails there) and shapes that do not
  broadcast are refused before any tensor is moved or any kernel is loaded."""
  def touched(*a, **k):
    raise AssertionError('device touched')
  monkeypatch.setattr(core, 'torch_float32', touched)
  monkeypatch.setattr(core._lib, 'load', touched)
  audio = np.zeros((2, 100), np.float32)
  phase = np.zeros((2, 100, 1), np.float32)
  for bad in (0, -3, 2.5):
    with pytest.raises(ValueError, match='max_length'):
      core.variable_length_delay(phase, audio, max_length=bad)
  for shape in ((2, 99, 1), (3, 100), (2, 100, 2), (100,), (2, 2, 100, 1)):
    with pytest.raises(ValueError, match='phase'):
      core.variable_length_delay(np.zeros(shape, np.float32), audio, max_length=10)
  with pytest.raises(ValueError, match='audio'):
    core.variable_length_delay(phase, np.zeros((2, 100, 1), np.float32))
  with pytest.raises(ValueError, match='gain'):
    core.mod_delay(audio, np.zeros((2, 50), np.float32), phase, 10)


# ---- GPU ---------------------------------------------------------------------
def _cuda(x):
  return torch.as_tensor(np.asarray(x, np.float32)).cuda()


def _check(name, got, want, tol_max=1e-4, tol_l2=1e-4):
  emax, el2 = rel_err(got, want)
  assert emax <= tol_max and el2 <= tol_l2, (name, emax, el2)
  return emax, el2


@pytest.mark.gpu
def test_forward_every_fixture_case():
  want = _fixture()
  for i, (L, _, kind, phase, audio) in enumerate(mg.mod_delay_inputs()):
    with torch.no_grad():
      got = core.variable_length_delay(_cuda(phase), _cuda(audio), max_length=L)
    _check((L, kind), got.cpu().numpy(), want['delay_wide_%02d' % i])


def _phase(kind, b, n, rng):
  return mg.mod_delay_phase(kind, b, n, rng)


@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('N', [1, 12345, 64000])
@pytest.mark.parametrize('L', [1, 2, 400, 1102, 4800])
def test_forward_shapes(B, N, L):
  rng = np.random.default_rng(B * 7 + N + L)
  audio = rng.standard_normal((B, N)).astype(np.float32)
  for kind in ('lfo', 'rough', 'wide_range'):
    phase = _phase(kind, B, N, rng)
    gain = rng.uniform(0.0, 1.0, (B, N, 1)).astype(np.float32)
    with torch.no_grad():
      got = core.mod_delay(_cuda(audio), _cuda(gain), _cuda(phase), L, scale=0.4,
                           offset=0.6, add_dry=True).cpu().numpy()
    want = ref.mod_delay_get_signal(audio, gain, _mapped(phase, 0.4, 0.6), center_ms=0.0,
                                    depth_ms=1.0, sample_rate=1000 * L)
    _check((B, N, L, kind), got, want)


def _mapped(phase, scale, offset):
  """The float32 phase map the kernel applies, so that the float64 oracle sees the
  same positions (scale 1, offset 0 in the oracle's own map)."""
  return phase * np.float32(scale) + np.float32(offset)


@pytest.mark.gpu
def test_forward_broadcast_shapes_and_delay_alone():
  rng = np.random.default_rng(3)
  B, N, L = 3, 5000, 400
  audio = rng.standard_normal((B, N)).astype(np.float32)
  for p_shape in ((B, N, 1), (B, N), (B, 1, 1), (B, 1)):
    phase = rng.uniform(-0.2, 1.2, p_shape).astype(np.float32)
    with torch.no_grad():
      got = core.variable_length_delay(_cuda(phase), _cuda(audio), max_length=L)
    _check(p_shape, got.cpu().numpy(), ref.variable_length_delay(phase, audio, L))
    for g_shape in ((B, N, 1), (B, N), (B, 1, 1), (B, 1)):
      gain = rng.uniform(0.0, 2.0, g_shape).astype(np.float32)
      with torch.no_grad():
        got = core.mod_delay(_cuda(audio), _cuda(gain), _cuda(phase), L,
                             add_dry=True).cpu().numpy()
      g = gain[..., 0] if gain.ndim == 3 else gain
      want = audio + g * ref.variable_length_delay(phase, audio, L)
      _check((p_shape, g_shape), got, want)


def _backward(audio, gain, phase, L, scale, offset, add_dry, seed=0):
  """Kernel gradients and float64 autograd of mod_delay_ref.torch_mod_delay for a random
  upstream gradient."""
  rng = np.random.default_rng(seed)
  g = rng.standard_normal(audio.shape)
  a = _cuda(audio).requires_grad_(True)
  gn = _cuda(gain).requires_grad_(True)
  ph = _cuda(phase).requires_grad_(True)
  out = core.mod_delay(a, gn, ph, L, scale=scale, offset=offset, add_dry=add_dry)
  out.backward(_cuda(g))
  a64 = torch.from_numpy(audio).double().requires_grad_(True)
  gn64 = torch.from_numpy(gain).double().requires_grad_(True)
  ph64 = torch.from_numpy(phase).double().requires_grad_(True)
  out64 = ref.torch_mod_delay(a64, gn64, ph64, L, scale, offset, add_dry)
  out64.backward(torch.from_numpy(g))
  return ((a.grad, a64.grad), (gn.grad, gn64.grad), (ph.grad, ph64.grad)), g


BACKWARD_CASES = [
    # (phase kind, L, N, scale, offset, add_dry)
    ('rough', 400, 6000, 1.0, 0.0, False),       # several outputs hit one input
    ('rough', 7, 3000, 1.0, 0.0, True),
    ('lfo', 400, 20000, 1.0, 0.0, True),         # through the wrap region
    ('wide_range', 400, 6000, 1.0, 0.0, False),  # out of range on both sides
    ('wide_range', 1102, 9000, 0.4, 0.6, True),  # ModDelay's map at 44.1 kHz
    ('lfo', 1, 4000, 1.0, 0.0, False),
    ('rough', 4800, 3000, 1.0, 0.0, True),       # L > N
    ('rough', 3000, 2500, 0.4, 0.6, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize('kind,L,N,scale,offset,add_dry', BACKWARD_CASES)
def test_backward_against_float64_autograd(kind, L, N, scale, offset, add_dry):
  rng = np.random.default_rng(L + N)
  B = 2
  audio = rng.standard_normal((B, N)).astype(np.float32)
  gain = rng.uniform(0.2, 1.5, (B, N)).astype(np.float32)
  phase = _phase(kind, B, N, rng)[..., 0]
  grads, g = _backward(audio, gain, phase, L, scale, offset, add_dry)
  for name, (got, want) in zip(('audio', 'gain', 'phase'), grads):
    _check(name, got.cpu().numpy(), want.numpy(), tol_max=2e-4, tol_l2=1e-4)
  # d audio through <g, D(x)> = <D^T g, x> against the oracle, random directions
  d_audio = grads[0][0].double().cpu().numpy()
  m = _mapped(phase, scale, offset)
  for k in range(3):
    x = np.random.default_rng(k).uniform(-1.0, 1.0, audio.shape)
    y = ref.variable_length_delay(m, x, L) * gain + (x if add_dry else 0.0)
    want, got = float((g * y).sum()), float((d_audio * x).sum())
    assert abs(got - want) <= 1e-5 * float(np.abs(g * y).sum()), (got, want)


@pytest.mark.gpu
def test_backward_phase_gradient_is_zero_on_knots():
  """L a power of two and phase = j / L: every position is an integer, where
  TensorFlow's subgradients give d phase = 0; d audio and d gain still flow."""
  rng = np.random.default_rng(5)
  B, N, L = 2, 5000, 256
  audio = rng.standard_normal((B, N)).astype(np.float32)
  gain = rng.uniform(0.2, 1.5, (B, N)).astype(np.float32)
  phase = (rng.integers(-2, L + 3, (B, N)) / L).astype(np.float32)
  grads, _ = _backward(audio, gain, phase, L, 1.0, 0.0, True)
  assert torch.count_nonzero(grads[2][0]).item() == 0
  for name, (got, want) in zip(('audio', 'gain'), grads[:2]):
    _check(name, got.cpu().numpy(), want.numpy(), tol_max=2e-4, tol_l2=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize('sample_rate,add_dry', [(16000, True), (44100, False)])
def test_processor_backward_end_to_end(sample_rate, add_dry):
  """ModDelay with its default scale functions from raw gain and phase, audio
  requiring grad too, against float64 autograd of the reference composition
  (exp_sigmoid, sigmoid, the phase map, the delay, gain, dry mix).  The float64
  composition takes its positions from our float32 sigmoid: the interpolation's
  gradient jumps at the knots, and a float64 sigmoid would put a position on the
  other side of one now and then."""
  from ddsp_b200 import effects
  rng = np.random.default_rng(sample_rate)
  B, N = 2, 8000
  audio = rng.standard_normal((B, N)).astype(np.float32)
  gain = rng.standard_normal((B, N, 1)).astype(np.float32)
  phase = (2.0 * rng.standard_normal((B, N, 1))).astype(np.float32)
  g = rng.standard_normal((B, N))
  md = effects.ModDelay(sample_rate=sample_rate, add_dry=add_dry)
  a, gn, ph = (_cuda(v).requires_grad_(True) for v in (audio, gain, phase))
  md(a, gn, ph).backward(_cuda(g))

  a64, gn64, ph64 = (torch.from_numpy(v).double().requires_grad_(True)
                     for v in (audio, gain, phase))
  max_delay_ms = md.center_ms + md.depth_ms
  L = int(sample_rate / 1000.0 * max_delay_ms)
  gain64 = 2.0 * torch.sigmoid(gn64)**np.log(10.0) + 1e-7
  p64 = torch.sigmoid(ph64)
  p32 = torch.sigmoid(ph.detach()).cpu().double()
  p64 = p64 + (p32 - p64).detach()
  out = ref.torch_mod_delay(a64, gain64[..., 0], p64[..., 0], L,
                           md.depth_ms / max_delay_ms, md.center_ms / max_delay_ms, add_dry)
  out.backward(torch.from_numpy(g))
  for name, got, want in (('audio', a.grad, a64.grad), ('gain', gn.grad, gn64.grad),
                          ('phase', ph.grad, ph64.grad)):
    _check(name, got.cpu().numpy(), want.numpy(), tol_max=2e-4, tol_l2=1e-4)


@pytest.mark.gpu
def test_full_size_forward_backward_reproducible():
  """B = 256, N = 64000, L = 400 (ModDelay's default at 16 kHz): a few items against
  the float64 oracle and autograd, and two runs of each pass bit-identical."""
  B, N, L = 256, 64000, 400
  gen = torch.Generator(device='cuda').manual_seed(0)
  audio = torch.randn((B, N), device='cuda', generator=gen)
  gain = torch.rand((B, N), device='cuda', generator=gen)
  t = torch.arange(N, device='cuda') / 16000.0
  phase = 0.8 + 0.2 * torch.sin(2 * np.pi * (2.0 + torch.rand((B, 1), device='cuda',
                                                                generator=gen)) * t)
  phase[::2] = torch.rand((B // 2, N), device='cuda', generator=gen) * 1.4 - 0.2
  g = torch.randn((B, N), device='cuda', generator=gen)
  runs = []
  for _ in range(2):
    a, gn, ph = (v.clone().requires_grad_(True) for v in (audio, gain, phase))
    out = core.mod_delay(a, gn, ph, L, scale=0.4, offset=0.6, add_dry=True)
    out.backward(g)
    runs.append((out.detach(), a.grad, gn.grad, ph.grad))
  torch.cuda.synchronize()
  for first, second in zip(*runs):
    assert torch.equal(first, second)
  for b in (0, 1, 255):
    x, gb, pb = (v[b:b + 1].double().cpu() for v in (audio, gain, phase))
    x.requires_grad_(True)
    gb.requires_grad_(True)
    pb.requires_grad_(True)
    out64 = ref.torch_mod_delay(x, gb, pb, L, 0.4, 0.6, True)
    out64.backward(g[b:b + 1].double().cpu())
    _check('out', runs[0][0][b:b + 1].cpu().numpy(), out64.detach().numpy())
    for name, got, want in (('audio', runs[0][1], x.grad), ('gain', runs[0][2], gb.grad),
                            ('phase', runs[0][3], pb.grad)):
      _check(name, got[b:b + 1].cpu().numpy(), want.numpy(), tol_max=2e-4, tol_l2=1e-4)
