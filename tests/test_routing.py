"""Routing ops and the exponential-decay reverb (csrc/routing.cuh): the backward of
core.resample, processors.Mix, processors.Crop, synths.TensorToAudio and
effects.ExpDecayReverb.

CPU: the C ABI's argument checks, the Python ValueErrors before any device work,
the float64 restatements of tests/routing_ref.py against the unmodified reference
run wide on the shim, and the host compositions (kernels swapped for the oracle)
against the reference run in float32 (tests/golden/routing.npz).
GPU: every gradient against float64 autograd of routing_ref, the inner-product
identity <d in, D> = <g, A D> for the linear operands, and bit-reproducibility."""
import numpy as np
import pytest
import torch

from ddsp_b200 import _lib, core
from oracle import ddsp_oracle as o
from oracle import ref_on_shim
from tests import routing_ref as ref
from tests.golden import make_routing_golden as mg
from tests.util import rel_err

P = 0x1000        # a device pointer the library never dereferences on the host
E_INVALID = _lib.E_INVALID
SEED = 0x1234

# (case, entry point, arguments, status, the full last_error or None)
_RB, _MF, _MB, _IR, _IRB = ('resample_backward', 'mix_forward', 'mix_backward',
                            'exp_decay_ir', 'exp_decay_ir_backward')
_ABI_CASES = [
    ('rb-null-grad', _RB, (None, P, 1, 10, 1, 100, 1, 1, None), E_INVALID, b'resample_backward: null pointer'),
    ('rb-null-in', _RB, (P, None, 1, 10, 1, 100, 1, 1, None), E_INVALID, b'resample_backward: null pointer'),
    ('rb-B', _RB, (P, P, -1, 10, 1, 100, 1, 1, None), E_INVALID, b'resample_backward: bad shape B=-1 F=10 C=1 N=100'),
    ('rb-F', _RB, (P, P, 1, 0, 1, 100, 1, 1, None), E_INVALID, b'resample_backward: bad shape B=1 F=0 C=1 N=100'),
    ('rb-C', _RB, (P, P, 1, 10, 0, 100, 1, 1, None), E_INVALID, b'resample_backward: bad shape B=1 F=10 C=0 N=100'),
    ('rb-N', _RB, (P, P, 1, 10, 1, 0, 1, 1, None), E_INVALID, b'resample_backward: bad shape B=1 F=10 C=1 N=0'),
    ('rb-method', _RB, (P, P, 1, 10, 1, 100, 4, 1, None), E_INVALID, b'resample_backward: bad method 4'),
    ('rb-method-neg', _RB, (P, P, 1, 10, 1, 100, -1, 1, None), E_INVALID, b'resample_backward: bad method -1'),
    ('rb-window-down', _RB, (P, P, 1, 100, 1, 100, 0, 1, None), E_INVALID, b'Upsample with windows cannot be used for downsamplingMore input frames (101) than output timesteps (100)'),
    ('rb-window-div', _RB, (P, P, 1, 10, 1, 100, 0, 0, None), E_INVALID, b'For upsampling, the target the number of timesteps must be divisible by the number of input frames - 1. (timesteps:100, frames:10, add_endpoint=False).'),
    ('rb-window-F1', _RB, (P, P, 1, 1, 1, 100, 0, 0, None), E_INVALID, b'For upsampling, the target the number of timesteps must be divisible by the number of input frames - 1. (timesteps:100, frames:1, add_endpoint=False).'),
    ('rb-B0', _RB, (P, P, 0, 10, 1, 100, 1, 1, None), 0, None),
    ('mf-null', _MF, (P, P, None, P, 1, 100, 1, None), E_INVALID, b'mix_forward: null pointer'),
    ('mf-null-out', _MF, (P, P, P, None, 1, 100, 1, None), E_INVALID, b'mix_forward: null pointer'),
    ('mf-B', _MF, (P, P, P, P, -1, 100, 1, None), E_INVALID, b'mix_forward: bad shape B=-1 N=100 C=1'),
    ('mf-N', _MF, (P, P, P, P, 1, 0, 1, None), E_INVALID, b'mix_forward: bad shape B=1 N=0 C=1'),
    ('mf-C', _MF, (P, P, P, P, 1, 100, 0, None), E_INVALID, b'mix_forward: bad shape B=1 N=100 C=0'),
    ('mf-B0', _MF, (P, P, P, P, 0, 100, 1, None), 0, None),
    ('mb-null-s1', _MB, (None, P, P, P, P, P, P, 1, 100, 1, None), E_INVALID, b'mix_backward: null pointer'),
    ('mb-null-grad', _MB, (P, P, P, None, P, P, P, 1, 100, 1, None), E_INVALID, b'mix_backward: null pointer'),
    ('mb-shape', _MB, (P, P, P, P, P, P, P, 2, 100, -3, None), E_INVALID, b'mix_backward: bad shape B=2 N=100 C=-3'),
    ('mb-B0', _MB, (P, P, P, P, P, P, P, 0, 100, 1, None), 0, None),
    ('mb-nothing', _MB, (P, P, P, P, None, None, None, 4, 100, 1, None), 0, None),
    ('ir-null-gain', _IR, (None, P, None, 0, 0, P, 1, 100, None), E_INVALID, b'exp_decay_ir: null pointer'),
    ('ir-null-out', _IR, (P, P, None, 0, 0, None, 1, 100, None), E_INVALID, b'exp_decay_ir: null pointer'),
    ('ir-rows', _IR, (P, P, None, 0, 0, P, -1, 100, None), E_INVALID, b'exp_decay_ir: bad shape rows=-1 L=100'),
    ('ir-L', _IR, (P, P, None, 0, 0, P, 1, 0, None), E_INVALID, b'exp_decay_ir: bad shape rows=1 L=0'),
    ('ir-rows0', _IR, (P, P, None, 0, 0, P, 0, 100, None), 0, None),
    ('irb-null-decay', _IRB, (P, None, None, 0, 0, P, P, P, 1, 100, None), E_INVALID, b'exp_decay_ir_backward: null pointer'),
    ('irb-null-grad', _IRB, (P, P, None, 0, 0, None, P, P, 1, 100, None), E_INVALID, b'exp_decay_ir_backward: null pointer'),
    ('irb-L', _IRB, (P, P, None, 0, 0, P, P, P, 1, -5, None), E_INVALID, b'exp_decay_ir_backward: bad shape rows=1 L=-5'),
    ('irb-rows0', _IRB, (P, P, None, 0, 0, P, P, P, 0, 100, None), 0, None),
    ('irb-nothing', _IRB, (P, P, None, 0, 0, P, None, None, 3, 100, None), 0, None),
]


@pytest.mark.parametrize('fn,args,want,msg', [c[1:] for c in _ABI_CASES],
                         ids=[c[0] for c in _ABI_CASES])
def test_routing_abi_check_table(fn, args, want, msg):
  """Every check of the five entry points, one row each: the status and the full
  message come back before any CUDA call, and nothing is launched."""
  lib = _lib.load()
  launches = lib.ddsp_b200_launch_count()
  assert getattr(lib, 'ddsp_b200_' + fn)(*args) == want
  assert lib.ddsp_b200_launch_count() == launches
  if msg is not None:
    assert lib.ddsp_b200_last_error() == msg
    with pytest.raises(ValueError):
      _lib.check(want)


def _no_library(monkeypatch):
  def fail(*a, **k):
    raise AssertionError('device work before the argument checks')
  monkeypatch.setattr(_lib, 'load', fail)
  monkeypatch.setattr(core, 'torch_float32', fail)


def test_value_errors_before_device_work(monkeypatch):
  from ddsp_b200 import effects, processors, synths
  _no_library(monkeypatch)
  mix = processors.Mix()
  s = np.zeros((2, 100, 1), np.float32)
  with pytest.raises(ValueError, match='The two signals must have the same length '
                     'instead of100 and 99'):
    mix(s, np.zeros((2, 99, 1), np.float32), np.zeros((2, 10, 1), np.float32))
  with pytest.raises(ValueError, match='3-D signals.*no crossfade'):
    mix(np.zeros((2, 100), np.float32), np.zeros((2, 100), np.float32),
        np.zeros((2, 10, 1), np.float32))
  with pytest.raises(ValueError, match='3-D signals'):
    mix.get_signal(np.zeros((2, 100), np.float32), np.zeros((2, 100), np.float32),
                   np.zeros((2, 100, 1), np.float32))
  with pytest.raises(ValueError, match='one shape'):
    mix.get_signal(s, np.zeros((2, 100, 2), np.float32), s)
  with pytest.raises(ValueError, match=r'mix_level must be \[2, 100, 1\]'):
    mix.get_signal(s, s, np.zeros((2, 100, 3), np.float32))
  with pytest.raises(ValueError, match='Crop_location: \\(middle\\), must be'):
    processors.Crop(320, crop_location='middle')(torch.zeros(2, 1000))
  for bad in ((2, 100), (2, 100, 2), (2, 100, 1, 1)):
    with pytest.raises(ValueError, match='TensorToAudio'):
      synths.TensorToAudio()(torch.zeros(bad))
  rev = effects.ExpDecayReverb()
  for gain, decay in ((None, None), (s[:, 0], None), (None, s[:, 0])):
    with pytest.raises(ValueError, match='Must provide "gain" and "decay" tensors if '
                       'ExpDecayReverb trainable=False.'):
      rev(np.zeros((2, 100), np.float32), gain, decay)
  with pytest.raises(ValueError, match='gain must be'):
    core.exp_decay_ir(np.zeros((2, 3)), np.zeros((2, 1)), 100)
  with pytest.raises(ValueError, match='do not broadcast'):
    core.exp_decay_ir(np.zeros((2, 1)), np.zeros((3, 1)), 100)
  with pytest.raises(ValueError, match='reverb_length'):
    core.exp_decay_ir(np.zeros((2, 1)), np.zeros((2, 1)), 0)
  with pytest.raises(ValueError, match='noise must be'):
    core.exp_decay_ir(np.zeros((2, 1)), np.zeros((2, 1)), 100, noise=np.zeros((2, 100)))


def test_constructors_follow_the_reference():
  from ddsp_b200 import effects, processors, synths
  rev = effects.ExpDecayReverb()
  assert (rev.name, rev.trainable, rev._reverb_length, rev._add_dry, rev.seed) == (
      'exp_decay_reverb', False, 48000, True, 0)
  assert rev._scale_fn is core.exp_sigmoid
  assert [rev.next_offset() for _ in range(3)] == [0, 1, 2]
  assert processors.Mix().name == 'mix'
  crop = processors.Crop(320)
  assert (crop.name, crop.frame_size, crop.crop_location) == ('crop', 320, 'back')
  assert synths.TensorToAudio().name == 'tensor_to_audio'
  trained = effects.ExpDecayReverb(trainable=True)
  trained.build('cpu')
  assert trained._gain.tolist() == [2.0] and trained._decay.tolist() == [4.0]
  assert trained._gain.requires_grad and trained._decay.requires_grad


def _fixture():
  return np.load(mg.PATH)


def test_restatements_match_the_reference():
  """routing_ref's float64 restatements against the unmodified reference run wide
  on the shim, at <= 1e-12."""
  want = _fixture()
  for i, case in enumerate(mg.RESAMPLE):
    F, N, method, add_endpoint = case
    x = torch.from_numpy(mg.resample_input(case, i)).double()
    got = ref.resample(x, N, method, add_endpoint).numpy()
    assert np.abs(got - want['resample_wide_%02d' % i]).max() <= 1e-12, case
  for i in range(len(mg.MIX)):
    s1, s2, logits = (torch.from_numpy(v).double() for v in mg.mix_inputs(i))
    got = ref.mix_processor(s1, s2, logits).numpy()
    assert np.abs(got - want['mix_wide_%d' % i]).max() <= 1e-12, i
    level = np.random.default_rng(750 + i).uniform(0.0, 1.0, (s1.shape[0], s1.shape[1], 1))
    got = ref.mix(s1, s2, torch.from_numpy(level.astype(np.float32)).double()).numpy()
    assert np.abs(got - want['mix_signal_wide_%d' % i]).max() <= 1e-12, i
  for i, (_, add_dry, L, _) in enumerate(mg.REVERB):
    audio, gain, decay, noise = (torch.from_numpy(v).double() for v in mg.reverb_inputs(i))
    ir = ref.exp_decay_ir(ref.exp_sigmoid(gain), decay, L, noise).numpy()
    assert np.abs(ir - want['ir_wide_%d' % i]).max() <= 1e-12, i
    got = ref.exp_decay_reverb(audio, gain, decay, noise, L, add_dry).numpy()
    assert np.abs(got - want['reverb_wide_%d' % i]).max() <= 1e-12, i


@pytest.mark.skipif(not ref_on_shim.available(), reason='reference sources absent')
def test_fixture_regenerates_from_reference():
  mg.compare('routing', mg.routing(), _fixture())


def _oracle_kernels(monkeypatch):
  """core's device entry points replaced by float32 NumPy on CPU tensors."""
  def t32(x, device=None):
    return torch.as_tensor(np.asarray(x.detach() if isinstance(x, torch.Tensor) else x,
                                      dtype=np.float32))

  def resample_forward(x, n, method, add_endpoint):
    return torch.from_numpy(o.resample(x.numpy(), n, method, add_endpoint,
                                       dtype=np.float32, tf_index_math=True))

  def mix_forward(s1, s2, m):
    m = m.numpy()
    one = np.sqrt(np.abs(m))
    two = np.float32(1.0) - np.sqrt(np.abs(m - np.float32(1.0)))
    return torch.from_numpy(one * s1.numpy() + two * s2.numpy())

  def ir_forward(gain, decay, L, noise, seed, offset):
    time = np.linspace(0.0, 1.0, L).astype(np.float32)
    if L > 1:
      time[:-1] = (np.float32(1.0) / np.float32(L - 1)) * np.arange(L - 1, dtype=np.float32)
    de = np.float32(2.0) + np.exp(decay.numpy()[:, None])
    return torch.from_numpy((gain.numpy()[:, None] * np.exp(-de * time[None, :]))
                            * noise.numpy()[None, :])
  monkeypatch.setattr(core, 'torch_float32', t32)
  monkeypatch.setattr(core, 'resample_forward', resample_forward)
  monkeypatch.setattr(core, 'mix_forward', mix_forward)
  monkeypatch.setattr(core, 'exp_decay_ir_forward', ir_forward)
  monkeypatch.setattr(core, 'fft_convolve', lambda a, ir, padding='same',
                      delay_compensation=-1, **kw: torch.from_numpy(
                          o.fft_convolve(t32(a).numpy(), t32(ir).numpy(), padding=padding,
                                         delay_compensation=delay_compensation,
                                         dtype=np.float32)))


def _close(got, want, tol=2e-5):
  assert got.shape == want.shape, (got.shape, want.shape)
  assert np.abs(got - want).max() <= tol * max(1.0, np.abs(want).max())


def test_compositions_match_the_reference(monkeypatch):
  """The host logic of Mix (length check, sigmoid, 'linear' resample to N,
  crossfade), Crop (every location, 2-D and 3-D, frame sizes 0 and 1),
  TensorToAudio and ExpDecayReverb (scale_fn, the learned gain and decay tiled
  over the batch, dry-tap masking, zero-delay 'same' convolution, add_dry) against
  the reference classes run in float32 on the shim, its noise pinned."""
  from ddsp_b200 import effects, processors, synths
  want = _fixture()
  _oracle_kernels(monkeypatch)
  with torch.no_grad():
    for i in range(len(mg.MIX)):
      s1, s2, logits = mg.mix_inputs(i)
      _close(processors.Mix()(s1, s2, logits).numpy(), want['mix_f32_%d' % i])
    for i, (frame, where, _) in enumerate(mg.CROP):
      audio = torch.from_numpy(mg.crop_input(i))
      got = processors.Crop(frame_size=frame, crop_location=where)(audio)
      np.testing.assert_array_equal(got.numpy(), want['crop_%d' % i])
    samples = np.random.default_rng(850).standard_normal((2, 100, 1)).astype(np.float32)
    np.testing.assert_array_equal(synths.TensorToAudio()(torch.from_numpy(samples)).numpy(),
                                  want['tensor_to_audio'])
    for i, (trainable, add_dry, L, _) in enumerate(mg.REVERB):
      audio, gain, decay, noise = mg.reverb_inputs(i)
      rev = effects.ExpDecayReverb(trainable=trainable, reverb_length=L, add_dry=add_dry)
      rev._scale_fn = lambda x: torch.from_numpy(o.exp_sigmoid(x.numpy(), dtype=np.float32))
      rev.injected_noise = torch.from_numpy(noise)
      got = rev(audio) if trainable else rev(audio, gain, decay)
      _close(got.numpy(), want['reverb_f32_%d' % i])


# ---- GPU ---------------------------------------------------------------------
DEV = 'cuda'


def _check(name, got, want, tol_max=1e-4, tol_l2=1e-4):
  got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else got
  want = want.detach().double().cpu().numpy() if isinstance(want, torch.Tensor) else want
  assert got.shape == want.shape, (name, got.shape, want.shape)
  assert np.isfinite(got).all(), name
  emax, el2 = rel_err(got, want)
  assert emax <= tol_max and el2 <= tol_l2, (name, emax, el2)


def _gen(seed):
  return torch.Generator(device=DEV).manual_seed(seed)


def _inner_product(d_in, g, apply, shape, seed=0):
  """<d_in, D> against <g, apply(D)> for random D, relative to sum |g * apply(D)|."""
  gen = _gen(seed)
  for _ in range(2):
    d = torch.rand(shape, device=DEV, generator=gen, dtype=torch.float64)
    y = apply(d)
    want = float((g.double() * y).sum())
    scale = float((g.double() * y).abs().sum())
    got = float((d_in.double() * d).sum())
    assert abs(got - want) <= 1e-5 * scale, (got, want, scale)


def _window_ok(F, N, add_endpoint):
  frames = F + 1 if add_endpoint else F
  return frames < N and frames > 1 and N % (frames - 1) == 0


RESAMPLE_SIZES = [(F, N) for F in (1, 2, 7, 250, 1000) for N in (1, 5, 100, 16000, 64000)]
WINDOW_HOPS = [(10, 4410, True), (11, 4410, False), (2, 16384, True), (3, 16384, False),
               (1, 8192, True), (250, 64000, True), (1001, 64000, False)]


def _resample_case(F, N, C, method, add_endpoint, seed):
  B = 2
  x = torch.randn((B, F, C), device=DEV, generator=_gen(seed))
  g = torch.randn((B, N, C), device=DEV, generator=_gen(seed + 1))
  x32 = x.clone().requires_grad_(True)
  out = core.resample(x32, N, method=method, add_endpoint=add_endpoint)
  out.backward(g)
  x64 = x.double().requires_grad_(True)
  out64 = ref.resample(x64, N, method, add_endpoint)
  out64.backward(g.double())
  case = (F, N, C, method, add_endpoint)
  _check(('forward',) + case, out, out64)
  _check(('d in',) + case, x32.grad, x64.grad, 2e-4, 1e-4)
  _inner_product(x32.grad, g, lambda d: ref.resample(d, N, method, add_endpoint), x.shape)


@pytest.mark.gpu
@pytest.mark.parametrize('add_endpoint', [True, False])
@pytest.mark.parametrize('method', ['linear', 'nearest', 'cubic', 'window'])
def test_resample_backward_every_size(method, add_endpoint):
  """F in {1, 2, 7, 250, 1000} x N in {1, 5, 100, 16000, 64000}: up- and
  downsampling (window: the upsampling sizes it accepts), C in {1, 3, 65}, and for
  'window' hops 441, 8192 and 256."""
  cases = RESAMPLE_SIZES if method != 'window' else [
      (F, N) for F, N in RESAMPLE_SIZES if _window_ok(F, N, add_endpoint)]
  for k, (F, N) in enumerate(cases):
    C = (1, 3, 65)[k % 3] if N * F <= 1600000 else (1, 3)[k % 2]
    _resample_case(F, N, C, method, add_endpoint, seed=k)
  if method == 'window':
    for k, (F, N, ae) in enumerate(WINDOW_HOPS):
      if ae == add_endpoint:
        _resample_case(F, N, 1 + k % 3, method, add_endpoint, seed=100 + k)


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['linear', 'nearest', 'cubic', 'window'])
def test_resample_backward_every_rank(method):
  """1-D ... 4-D inputs through core.resample's reshapes (4-D is the 3-D case over
  n_freq * channels; 'window' only takes 3-D)."""
  shapes = [(250,), (3, 250), (3, 250, 2), (3, 250, 4, 2)]
  for k, shape in enumerate(shapes):
    if method == 'window' and len(shape) != 3:
      continue
    x = torch.randn(shape, device=DEV, generator=_gen(k))
    n = 16000
    g = torch.randn(ref.resample(x.double(), n, method).shape, device=DEV,
                    generator=_gen(k + 10))
    x32 = x.clone().requires_grad_(True)
    out = core.resample(x32, n, method=method)
    out.backward(g)
    x64 = x.double().requires_grad_(True)
    ref.resample(x64, n, method).backward(g.double())
    assert out.shape == g.shape
    _check(('d in', shape), x32.grad, x64.grad, 2e-4, 1e-4)


@pytest.mark.gpu
def test_upsample_with_windows_and_add_route_gradients():
  x = torch.randn((2, 51, 3), device=DEV, generator=_gen(3))
  g = torch.randn((2, 16000, 3), device=DEV, generator=_gen(4))
  x32 = x.clone().requires_grad_(True)
  core.upsample_with_windows(x32, 16000, add_endpoint=False).backward(g)
  x64 = x.double().requires_grad_(True)
  ref.resample(x64, 16000, 'window', False).backward(g.double())
  _check('upsample_with_windows', x32.grad, x64.grad, 2e-4, 1e-4)
  # core.add: the gradient to each operand, summed over broadcast dimensions
  a = torch.randn((3, 1000), device=DEV, generator=_gen(5)).requires_grad_(True)
  b = torch.randn((1, 1000), device=DEV, generator=_gen(6)).requires_grad_(True)
  g = torch.randn((3, 1000), device=DEV, generator=_gen(7))
  out = core.add(a, b)
  assert torch.equal(out.detach(), a.detach() + b.detach())
  out.backward(g)
  assert torch.equal(a.grad, g)
  torch.testing.assert_close(b.grad, g.sum(0, keepdim=True))
  with torch.no_grad():
    assert not core.add(a, b).requires_grad


def _mix_grads(s1, s2, m32, g):
  """Kernel and float64 gradients of Mix.get_signal at the given float32 level."""
  a1, a2, am = (v.clone().requires_grad_(True) for v in (s1, s2, m32))
  out = core.mix(a1, a2, am)
  out.backward(g)
  b1, b2, bm = (v.double().requires_grad_(True) for v in (s1, s2, m32))
  out64 = ref.mix(b1, b2, bm)
  out64.backward(g.double())
  return out, out64, (a1.grad, b1.grad), (a2.grad, b2.grad), (am.grad, bm.grad)


@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 3, 256])
@pytest.mark.parametrize('C', [1, 3])
@pytest.mark.parametrize('frames', [1, 250, 'N'])
def test_mix_processor_forward_backward(B, C, frames):
  """Mix end to end from the raw mix logits: sigmoid, 'linear' resample (its new
  backward), the crossfade kernel and its backward, against float64 autograd of
  routing_ref.mix_processor."""
  from ddsp_b200 import processors
  N = 16000
  F = N if frames == 'N' else frames
  seed = B * 100 + C * 10 + F % 7
  s1 = torch.randn((B, N, C), device=DEV, generator=_gen(seed))
  s2 = torch.randn((B, N, C), device=DEV, generator=_gen(seed + 1))
  logits = 2.0 * torch.randn((B, F, 1), device=DEV, generator=_gen(seed + 2))
  g = torch.randn((B, N, C), device=DEV, generator=_gen(seed + 3))
  a1, a2, al = (v.clone().requires_grad_(True) for v in (s1, s2, logits))
  out = processors.Mix()(a1, a2, al)
  out.backward(g)
  b1, b2, bl = (v.double().requires_grad_(True) for v in (s1, s2, logits))
  out64 = ref.mix_processor(b1, b2, bl)
  out64.backward(g.double())
  _check('forward', out, out64)
  for name, got, want in (('d s1', a1.grad, b1.grad), ('d s2', a2.grad, b2.grad),
                          ('d logits', al.grad, bl.grad)):
    _check(name, got, want, 2e-4, 1e-4)
  # the crossfade is linear in each signal
  with torch.no_grad():
    m32 = core.resample(torch.sigmoid(logits), N)
  _inner_product(a1.grad, g, lambda d: torch.sqrt(m32.double().abs()) * d, s1.shape)
  _inner_product(a2.grad, g, lambda d: (1.0 - torch.sqrt((m32.double() - 1.0).abs())) * d,
                 s2.shape)


@pytest.mark.gpu
@pytest.mark.parametrize('frames', [250, 'N'])
def test_mix_saturated_level_gives_nan_where_the_reference_does(frames):
  """Logits of +-200 saturate float32 sigmoid to exactly 1 and 0, where the
  reference's autodiff of sqrt(|m|) / sqrt(|m - 1|) gives NaN (0 * inf).  The
  float64 chain takes the float32 level's values (its derivative is float64): the
  NaNs must land on the same elements, everything else within the gates."""
  from ddsp_b200 import processors
  B, C, N = 2, 3, 16000
  F = N if frames == 'N' else frames
  s1 = torch.randn((B, N, C), device=DEV, generator=_gen(21))
  s2 = torch.randn((B, N, C), device=DEV, generator=_gen(22))
  logits = torch.randn((B, F, 1), device=DEV, generator=_gen(23))
  logits[0, F // 5:F // 5 + F // 10] = 200.0
  logits[1, F // 2:F // 2 + F // 10] = -200.0
  logits[1, -3:] = 200.0
  g = torch.randn((B, N, C), device=DEV, generator=_gen(24))
  a1, a2, al = (v.clone().requires_grad_(True) for v in (s1, s2, logits))
  out = processors.Mix()(a1, a2, al)
  out.backward(g)
  with torch.no_grad():
    m32 = core.resample(torch.sigmoid(logits), N)
  assert (m32 == 0).any() and (m32 == 1).any()
  b1, b2, bl = (v.double().requires_grad_(True) for v in (s1, s2, logits))
  m64 = ref.resample(torch.sigmoid(bl), N)
  m64 = m64 + (m32.double() - m64).detach()
  out64 = ref.mix(b1, b2, m64)
  out64.backward(g.double())
  _check('forward', out, out64)
  _check('d s1', a1.grad, b1.grad, 2e-4, 1e-4)
  _check('d s2', a2.grad, b2.grad, 2e-4, 1e-4)
  nan = torch.isnan(al.grad)
  assert nan.any()
  assert torch.equal(nan.cpu(), torch.isnan(bl.grad).cpu())
  _check('d logits (finite)', al.grad[~nan], bl.grad[~nan], 2e-4, 1e-4)
  # the kernel alone at the given level
  out, out64, d1, d2, dm = _mix_grads(s1, s2, m32, g)
  assert torch.equal(torch.isnan(dm[0]).cpu(), torch.isnan(dm[1]).cpu())
  assert torch.equal(torch.isnan(dm[0]).cpu(), ((m32 == 0) | (m32 == 1)).cpu())
  fin = ~torch.isnan(dm[0])
  _check('d m (finite)', dm[0][fin], dm[1][fin], 2e-4, 1e-4)


REVERB_LENGTHS = [1, 2, 100, 2047, 2048, 24000, 48000]


@pytest.mark.gpu
@pytest.mark.parametrize('L', REVERB_LENGTHS)
@pytest.mark.parametrize('trainable', [False, True])
@pytest.mark.parametrize('add_dry', [True, False])
def test_exp_decay_reverb_forward_backward(L, trainable, add_dry):
  """ExpDecayReverb end to end, gradients to audio, gain and decay, against float64
  autograd of routing_ref.exp_decay_reverb: both convolution routes (L < 2048 is the
  direct form), L > N, in-kernel Philox (checked against core.uniform_noise) and
  injected noise, decays from -20 to 20."""
  from ddsp_b200 import effects
  B, N = 3, 16000
  seed = L + 7 * trainable + 3 * add_dry
  audio = torch.randn((B, N), device=DEV, generator=_gen(seed))
  gain = torch.randn((B, 1), device=DEV, generator=_gen(seed + 1))
  decay = torch.tensor([[-20.0], [0.5], [20.0]], device=DEV)
  g = torch.randn((B, N), device=DEV, generator=_gen(seed + 2))
  for injected in (False, True):
    rev = effects.ExpDecayReverb(trainable=trainable, reverb_length=L, add_dry=add_dry,
                                 seed=SEED)
    noise = None
    if injected:
      noise = torch.rand((1, L), device=DEV, generator=_gen(seed + 3)) * 2 - 1
      rev.injected_noise = noise
    a32 = audio.clone().requires_grad_(True)
    if trainable:
      rev.build(DEV)
      with torch.no_grad():
        rev._gain.fill_(0.3)
        rev._decay.fill_(float(decay[1, 0]) + 2.0 * injected)
      out = rev(a32)
      p_gain, p_decay = rev._gain, rev._decay
      g64_in, d64_in = rev._gain.detach()[None], rev._decay.detach()[None]
    else:
      p_gain, p_decay = gain.clone().requires_grad_(True), decay.clone().requires_grad_(True)
      out = rev(a32, p_gain, p_decay)
      g64_in, d64_in = gain, decay
    out.backward(g)
    if noise is None:
      noise = core.uniform_noise(1, L, seed=SEED, offset=0)
    a64 = audio.double().requires_grad_(True)
    gn64 = g64_in.double().requires_grad_(True)
    dc64 = d64_in.double().requires_grad_(True)
    out64 = ref.exp_decay_reverb(a64, gn64, dc64, noise, L, add_dry)
    out64.backward(g.double())
    case = (L, trainable, add_dry, injected)
    _check(('forward',) + case, out, out64)
    _check(('d audio',) + case, a32.grad, a64.grad, 2e-4, 1e-4)
    want_g = gn64.grad.reshape(p_gain.shape)
    want_d = dc64.grad.reshape(p_decay.shape)
    if L == 1:   # the only tap is the masked dry tap
      assert not p_gain.grad.any() and not p_decay.grad.any()
      continue
    _check(('d gain',) + case, p_gain.grad, want_g, 2e-4, 1e-4)
    # d decay of a vanished decay (e^-(2 + e^20) t) is 0 in both
    if float(want_d.abs().max()) > 0:
      _check(('d decay',) + case, p_decay.grad, want_d, 2e-4, 1e-4)
    else:
      assert not p_decay.grad.any()


@pytest.mark.gpu
@pytest.mark.parametrize('rows,L', [(1, 48000), (256, 48000), (5, 1), (5, 3), (7, 2047)])
def test_exp_decay_ir_kernels(rows, L):
  """The impulse-response kernels alone: the Philox row equals
  core.uniform_noise(1, L, seed, offset); both gradients against float64 autograd;
  the IR is linear in the scaled gain (inner-product identity)."""
  gain = torch.rand((rows, 1), device=DEV, generator=_gen(L)) + 0.1
  decay = torch.linspace(-20.0, 20.0, rows, device=DEV)[:, None] if rows > 1 else \
      torch.full((1, 1), 1.5, device=DEV)
  g = torch.randn((rows, L), device=DEV, generator=_gen(L + 1))
  gp, dp = gain.clone().requires_grad_(True), decay.clone().requires_grad_(True)
  ir = core.exp_decay_ir(gp, dp, L, seed=SEED, offset=5)
  ir.backward(g)
  noise = core.uniform_noise(1, L, seed=SEED, offset=5)
  with torch.no_grad():   # tap 0 is gain * noise[0] exactly (time 0, e = 1)
    assert torch.equal(ir[:, 0], gain[:, 0] * noise[0, 0])
    injected = core.exp_decay_ir(gain, decay, L, noise=noise)
  assert torch.equal(injected, ir.detach())
  g64, d64 = gain.double().requires_grad_(True), decay.double().requires_grad_(True)
  ir64 = ref.exp_decay_ir(g64, d64, L, noise)
  ir64.backward(g.double())
  _check('ir', ir, ir64)
  _check('d gain', gp.grad, g64.grad, 2e-4, 1e-4)
  live = d64.grad.abs() > 0
  if live.any():
    _check('d decay', dp.grad[live], d64.grad[live], 2e-4, 1e-4)
  assert not dp.grad[~live].any()
  _inner_product(gp.grad, g, lambda d: ref.exp_decay_ir(d, decay, L, noise),
                 gain.shape)


@pytest.mark.gpu
def test_vst_dag_returns_cropped_audio():
  """The `vst.gin` DAG: Harmonic ('linear', 64320 samples, hop 320) ->
  FilteredNoise (window 0) -> Add -> FilteredNoiseReverb(trainable, 24000, 500, 32)
  -> Crop(320, 'back'), under no_grad, against the float64 composition."""
  import ddsp_b200
  from ddsp_b200 import autograd as ag
  from ddsp_b200 import effects, processors
  from tests import grad_ref
  from tests.util import synth_inputs
  B, F, K, nb, N = 2, 201, 60, 65, 64320
  inp = synth_inputs(B, F, K, nb, N, seed=31)
  harm = ddsp_b200.Harmonic(n_samples=N, amp_resample_method='linear')
  noise = ddsp_b200.FilteredNoise(n_samples=N, window_size=0)
  noise.injected_noise = torch.from_numpy(inp['noise']).to(DEV)
  reverb = effects.FilteredNoiseReverb(trainable=True, reverb_length=24000, n_frames=500,
                                       n_filter_banks=32, name='reverb')
  reverb.build(DEV)
  ir_noise = torch.rand((1, 24000), device=DEV, generator=_gen(32)) * 2 - 1
  reverb._synth.injected_noise = ir_noise
  group = ddsp_b200.ProcessorGroup(dag=[
      (harm, ['amps', 'harmonic_distribution', 'f0_hz']),
      (noise, ['noise_magnitudes']),
      (processors.Add(), ['filtered_noise/signal', 'harmonic/signal']),
      (reverb, ['add/signal']),
      (processors.Crop(frame_size=320, crop_location='back'), ['reverb/signal'])])
  feats = {k: torch.from_numpy(inp[k]).to(DEV) for k in
           ('amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes')}
  with torch.no_grad():
    audio = group(feats)
  assert audio.shape == (B, 64000)
  r = {k: v.double() for k, v in feats.items()}
  a, h = ag.harmonic_controls(r['amps'], r['harmonic_distribution'], r['f0_hz'])
  dry = (grad_ref.harmonic(r['f0_hz'], a, h, N, 16000, 'linear',
                           mask=grad_ref.nyquist_mask(feats['f0_hz'], K, N, 16000)) +
         grad_ref.frequency_filter(noise.injected_noise.double(),
                                   ag.exp_sigmoid(r['noise_magnitudes'] - 5.0)))
  ir = grad_ref.frequency_filter(ir_noise.double(),
                                 ag.exp_sigmoid(reverb._magnitudes.detach().double()[None]
                                                - 3.0), 257)
  want = ref.crop(ref.reverb(dry, ir.repeat(B, 1)), 320, 'back')
  _check('vst DAG', audio, want)


@pytest.mark.gpu
def test_training_chain_through_exp_decay_reverb():
  """decoder_train -> ExpDecayReverb(trainable) -> Crop -> SpectralLossFn at a
  reduced size, gradients to every decoder input and to the learned gain and decay
  against the float64 chain."""
  from ddsp_b200 import autograd as ag
  from ddsp_b200 import effects, processors, spectral_ops
  from tests import grad_ref
  from tests.util import synth_inputs
  B, F, K, nb, hop, L = 2, 50, 20, 65, 64, 2048
  N = F * hop
  fft_sizes = (1024, 256, 64)
  inp = synth_inputs(B, F, K, nb, N, seed=41)
  raw = {k: torch.from_numpy(inp[k]).to(DEV) for k in
         ('amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes')}
  nz = torch.from_numpy(inp['noise']).to(DEV)
  target = torch.randn((B, N - hop), device=DEV, generator=_gen(42)) * 0.1
  rev = effects.ExpDecayReverb(trainable=True, reverb_length=L, seed=SEED)
  rev.build(DEV)
  with torch.no_grad():
    rev._decay.fill_(1.0)
  crop = processors.Crop(frame_size=hop, crop_location='back')
  r32 = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
  audio = ag.decoder_train(r32['amps'], r32['harmonic_distribution'], r32['f0_hz'],
                           r32['noise_magnitudes'], n_samples=N, noise=nz)
  audio = crop(rev(audio))
  loss = spectral_ops.SpectralLossFn.apply(target, audio, fft_sizes, 1.0, 0.0)
  loss.backward()
  ir_noise = core.uniform_noise(1, L, seed=SEED, offset=0)
  r64 = {k: v.double().requires_grad_(True) for k, v in raw.items()}
  gain64 = rev._gain.detach().double()[None].requires_grad_(True)
  decay64 = rev._decay.detach().double()[None].requires_grad_(True)
  a, h = ag.harmonic_controls(r64['amps'], r64['harmonic_distribution'], r64['f0_hz'])
  dry = (grad_ref.harmonic(r64['f0_hz'], a, h, N, 16000, 'window',
                           mask=grad_ref.nyquist_mask(raw['f0_hz'], K, N, 16000)) +
         grad_ref.frequency_filter(nz.double(), ag.exp_sigmoid(r64['noise_magnitudes'] - 5.0)))
  wet = ref.crop(ref.exp_decay_reverb(dry, gain64, decay64, ir_noise, L), hop, 'back')
  ref_loss = grad_ref.spectral_loss(target, wet, fft_sizes, 1.0, 0.0)
  ref_loss.backward()
  lv, rv = float(loss.detach()), float(ref_loss.detach())
  assert abs(lv - rv) <= 1e-4 * rv, (lv, rv)
  for k in raw:
    _check('d ' + k, r32[k].grad, r64[k].grad, 2e-4, 1e-4)
  _check('d gain', rev._gain.grad, gain64.grad.reshape(1), 2e-4, 1e-4)
  _check('d decay', rev._decay.grad, decay64.grad.reshape(1), 2e-4, 1e-4)


@pytest.mark.gpu
def test_full_size_gradients_are_bit_reproducible():
  """B = 256, N = 64000: Mix from [B, 1000, 1] logits and ExpDecayReverb at
  L = 48000, run twice: every output and gradient bit-identical."""
  from ddsp_b200 import effects, processors
  B, N, C, L = 256, 64000, 1, 48000
  s1 = torch.randn((B, N, C), device=DEV, generator=_gen(51))
  s2 = torch.randn((B, N, C), device=DEV, generator=_gen(52))
  logits = torch.randn((B, 1000, 1), device=DEV, generator=_gen(53))
  gain = torch.randn((B, 1), device=DEV, generator=_gen(54))
  decay = torch.rand((B, 1), device=DEV, generator=_gen(55)) * 4.0
  g = torch.randn((B, N), device=DEV, generator=_gen(56))
  runs = []
  for _ in range(2):
    a1, a2, al, gp, dp = (v.clone().requires_grad_(True)
                          for v in (s1, s2, logits, gain, decay))
    mixed = processors.Mix()(a1, a2, al)[:, :, 0]
    rev = effects.ExpDecayReverb(reverb_length=L, seed=SEED)
    out = rev(mixed, gp, dp)
    out.backward(g)
    runs.append((out.detach(), a1.grad, a2.grad, al.grad, gp.grad, dp.grad))
  torch.cuda.synchronize()
  for first, second in zip(*runs):
    assert torch.equal(first, second)
  for b in (0, 255):
    want = ref.exp_decay_reverb(
        ref.mix_processor(s1[b:b + 1].double(), s2[b:b + 1].double(),
                          logits[b:b + 1].double())[:, :, 0],
        gain[b:b + 1].double(), decay[b:b + 1].double(),
        core.uniform_noise(1, L, seed=SEED, offset=0), L)
    _check('out', runs[0][0][b:b + 1], want)
