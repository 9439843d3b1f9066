"""The host-side helpers of `ddsp/core.py` and `ddsp/spectral_ops.py`: dB and perceptual-
scale conversions, soft_limit / log_scale / sym_exp_sigmoid, frequencies_critical_bands,
gradient_reversal, nan_to_num, pad_axis, center_crop, the nested-dict helpers,
pad_or_trim_to_expected_length and stft_np.

Every expected value comes from a float64 NumPy restatement of the reference's formula
written below.  CPU: known answers, float32 against float64, float64 gradcheck, the
conventions, and a list of the reference's public functions.  GPU: sym_exp_sigmoid on
exp_sigmoid's CUDA kernel, and Sinusoidal(freq_scale_fn=frequencies_critical_bands)
trained against float64 autograd."""
import numpy as np
import pytest
import torch

from ddsp_b200 import core, spectral_ops
from tests import sinusoidal_ref
from tests.util import rel_err

LN10 = np.log(10.0)


# ---- float64 restatements of the reference's formulas (core.py:202-569) ---------------
def power_to_db64(power, ref_db=0.0, range_db=80.0):
  db = 10.0 * np.log10(np.maximum(10.0**(-range_db / 10.0), power))
  return np.maximum(db - ref_db, -range_db)


def hz_to_bark64(hz):
  return 26.81 / (1.0 + 1960.0 / hz) - 0.53


def bark_to_hz64(bark):
  return 1960.0 / (26.81 / (bark + 0.53) - 1.0)


def hz_to_mel64(hz):
  return 2595.0 * np.log10(1.0 + hz / 700.0)


def mel_to_hz64(mel):
  return 700.0 * (10.0**(mel / 2595.0) - 1.0)


def softplus64(x):
  return np.logaddexp(0.0, x)


def soft_limit64(x, x_min=0.0, x_max=1.0):
  return softplus64(x) + x_min - softplus64(x - (x_max - x_min))


def log_scale64(x, min_x, max_x):
  u = (x + 1.0) / 2.0
  return np.exp((1.0 - u) * np.log(min_x) + u * np.log(max_x))


def exp_sigmoid64(x):
  return 2.0 * (1.0 / (1.0 + np.exp(-x)))**LN10 + 1e-7


def sym_exp_sigmoid64(x, width=8.0):
  return exp_sigmoid64(width * (np.abs(x) / 2.0 - 1.0))


def centres64(n, hz_min, hz_max, scale):
  if scale == 'bark':
    return bark_to_hz64(np.linspace(hz_to_bark64(hz_min), hz_to_bark64(hz_max), n))
  return mel_to_hz64(np.linspace(hz_to_mel64(hz_min), hz_to_mel64(hz_max), n))


def critical_bands64(x, depth=1, depth_scale=10.0, bandwidth_scale=1.0, hz_min=20.0,
                     hz_max=8000.0, scale='bark'):
  """x [B, T, N * depth] or [B, T, N, depth] -> Hz [B, T, N]."""
  x = np.asarray(x, np.float64)
  if x.ndim == 3:
    x = x.reshape(x.shape[0], x.shape[1], -1, depth)
  c = centres64(x.shape[-2], hz_min, hz_max, scale)
  erb = 0.108 * c + 24.7
  mod = (np.tanh(x) * depth_scale**-np.arange(x.shape[-1], dtype=np.float64)).sum(-1)
  return soft_limit64(c + bandwidth_scale * erb * mod, hz_min, hz_max)


def _rng(seed):
  return np.random.default_rng(seed)


def _log_uniform(rng, lo, hi, n):
  return np.exp(rng.uniform(np.log(lo), np.log(hi), n)).astype(np.float32)


def _agree(got, want, tol=1e-5, peak=False):
  """float32 result against float64: elementwise relative error, or (peak=True, for
  outputs that cross zero) error relative to the largest |want|."""
  got = np.asarray(got.detach().cpu() if torch.is_tensor(got) else got, np.float64)
  want = np.asarray(want, np.float64)
  assert got.shape == want.shape
  scale = np.abs(want).max() if peak else np.abs(want)
  err = (np.abs(got - want) / scale).max()
  assert err <= tol, err


# ---- 1. known answers -----------------------------------------------------------------
def test_db_known_answers():
  assert float(core.power_to_db(1.0)) == 0.0
  assert float(core.power_to_db(0.0)) == -80.0
  assert float(core.power_to_db(1e-9, range_db=80)) == -80.0
  assert float(core.amplitude_to_db(10.0)) == pytest.approx(20.0, abs=1e-5)
  # ref_db shifts before the floor: 1e-7 is -70 dB, -90 after the shift, floored at -80
  assert float(core.power_to_db(1e-7, ref_db=20.0)) == -80.0
  assert float(core.power_to_db(100.0, ref_db=20.0)) == pytest.approx(0.0, abs=1e-5)
  assert float(core.power_to_db(1e-3, ref_db=-10.0)) == pytest.approx(-20.0, abs=1e-5)
  for use_tf in (True, False):
    assert float(core.power_to_db(0.5, range_db=60.0, use_tf=use_tf)) == pytest.approx(
        10.0 * np.log10(0.5), abs=1e-5)
    assert float(core.power_to_db(1e-8, range_db=60.0, use_tf=use_tf)) == -60.0


def test_db_round_trip_above_the_floor():
  a = _log_uniform(_rng(0), 1e-3, 1e2, 1000)
  back = core.db_to_amplitude(core.amplitude_to_db(torch.from_numpy(a)))
  _agree(back, a, 1e-5)
  a = a.astype(np.float64)
  back = core.db_to_power(core.power_to_db(a, use_tf=False))
  np.testing.assert_allclose(back, a, rtol=1e-12)


def test_scale_known_answers():
  assert core.hz_to_mel(700.0) == pytest.approx(2595.0 * np.log10(2.0), rel=1e-12)
  assert float(core.hz_to_mel(torch.tensor(700.0))) == pytest.approx(
      2595.0 * np.log10(2.0), rel=1e-6)
  assert core.hz_to_erb(1000.0) == pytest.approx(132.7, rel=1e-12)
  assert core.hz_to_bark(1960.0) == pytest.approx(26.81 / 2.0 - 0.53, rel=1e-12)
  hz = np.linspace(20.0, 8000.0, 4001)
  np.testing.assert_allclose(core.bark_to_hz(core.hz_to_bark(hz)), hz, rtol=1e-5)
  np.testing.assert_allclose(core.mel_to_hz(core.hz_to_mel(hz)), hz, rtol=1e-5)
  bark, mel = hz_to_bark64(hz), hz_to_mel64(hz)
  np.testing.assert_allclose(core.hz_to_bark(core.bark_to_hz(bark)), bark, rtol=1e-5)
  np.testing.assert_allclose(core.hz_to_mel(core.mel_to_hz(mel)), mel, rtol=1e-5)


# ---- 2. float32 against float64 -------------------------------------------------------
def _hz(rng, n):
  return _log_uniform(rng, 20.0, 8000.0, n)


# (name, function under test, float64 restatement, input, output crosses zero)
CONVERSIONS = [
    ('power_to_db', core.power_to_db, power_to_db64,
     lambda r, n: _log_uniform(r, 1e-10, 1e2, n), True),
    ('amplitude_to_db', core.amplitude_to_db, lambda a: power_to_db64(a * a),
     lambda r, n: _log_uniform(r, 1e-5, 10.0, n), True),
    ('db_to_power', core.db_to_power, lambda d: 10.0**(d / 10.0),
     lambda r, n: r.uniform(-80.0, 20.0, n).astype(np.float32), False),
    ('db_to_amplitude', core.db_to_amplitude, lambda d: 10.0**(d / 20.0),
     lambda r, n: r.uniform(-80.0, 20.0, n).astype(np.float32), False),
    ('hz_to_bark', core.hz_to_bark, hz_to_bark64, _hz, True),
    ('bark_to_hz', core.bark_to_hz, bark_to_hz64,
     lambda r, n: hz_to_bark64(_hz(r, n).astype(np.float64)).astype(np.float32), False),
    ('hz_to_mel', core.hz_to_mel, hz_to_mel64, _hz, False),
    ('mel_to_hz', core.mel_to_hz, mel_to_hz64,
     lambda r, n: hz_to_mel64(_hz(r, n).astype(np.float64)).astype(np.float32), False),
    ('hz_to_erb', core.hz_to_erb, lambda h: 0.108 * h + 24.7, _hz, False),
    ('soft_limit', core.soft_limit, soft_limit64,
     lambda r, n: r.uniform(-6.0, 7.0, n).astype(np.float32), True),
    ('soft_limit_hz', lambda x: core.soft_limit(x, 20.0, 8000.0),
     lambda x: soft_limit64(x, 20.0, 8000.0),
     lambda r, n: r.uniform(-500.0, 9000.0, n).astype(np.float32), False),
    ('log_scale', lambda x: core.log_scale(x, 20.0, 8000.0),
     lambda x: log_scale64(x, 20.0, 8000.0),
     lambda r, n: r.uniform(-1.0, 1.0, n).astype(np.float32), False),
]


@pytest.mark.parametrize('name,fn,ref,make,crosses_zero', CONVERSIONS,
                         ids=[c[0] for c in CONVERSIONS])
def test_float32_against_float64(name, fn, ref, make, crosses_zero):
  x = make(_rng(len(name)), 4096)
  got = fn(torch.from_numpy(x))
  assert got.dtype == torch.float32, name
  _agree(got, ref(x.astype(np.float64)), 1e-5, peak=crosses_zero)


@pytest.mark.parametrize('scale', ['bark', 'mel'])
@pytest.mark.parametrize('depth', [1, 4])
@pytest.mark.parametrize('rank', [3, 4])
def test_frequencies_critical_bands_against_float64(scale, depth, rank):
  B, T, N = 2, 50, 64
  x = _rng(depth * rank).normal(0.0, 2.0, (B, T, N, depth)).astype(np.float32)
  want = critical_bands64(x, scale=scale)
  arg = x.reshape(B, T, N * depth) if rank == 3 else x
  got = core.frequencies_critical_bands(torch.from_numpy(arg), depth=depth, scale=scale)
  assert got.shape == (B, T, N) and got.dtype == torch.float32
  _agree(got, want, 1e-5)


def test_frequencies_critical_bands_arguments():
  """depth_scale, bandwidth_scale and the range, by position; any scale that is not
  'bark' takes the mel centres; numpy input works and gives a tensor."""
  x = _rng(5).normal(0.0, 1.0, (1, 7, 10, 2)).astype(np.float32)
  got = core.frequencies_critical_bands(x, 2, 3.0, 0.5, 50.0, 4000.0, 'bark')
  _agree(got, critical_bands64(x, 2, 3.0, 0.5, 50.0, 4000.0, 'bark'), 1e-5)
  mel = core.frequencies_critical_bands(x, scale='mel')
  assert torch.equal(core.frequencies_critical_bands(x, scale='erb'), mel)
  _agree(mel, critical_bands64(x, scale='mel'), 1e-5)
  # the centres span the range: the middle of tanh is 0, so zero input gives them
  zero = core.frequencies_critical_bands(torch.zeros(1, 1, 16))
  _agree(zero[0, 0], soft_limit64(centres64(16, 20.0, 8000.0, 'bark'), 20.0, 8000.0), 1e-5)


# ---- 3. gradients ---------------------------------------------------------------------
def test_gradcheck_float64():
  rng = _rng(3)
  x = torch.from_numpy(rng.uniform(-5.0, 5.0, (6, 5))).requires_grad_(True)
  assert torch.autograd.gradcheck(core.soft_limit, (x,))
  assert torch.autograd.gradcheck(lambda v: core.soft_limit(v, -2.0, 3.0), (x,))
  u = torch.from_numpy(rng.uniform(-0.95, 0.95, (6, 5))).requires_grad_(True)
  assert torch.autograd.gradcheck(lambda v: core.log_scale(v, 20.0, 8000.0), (u,))
  for scale in ('bark', 'mel'):
    f = torch.from_numpy(rng.normal(0.0, 1.5, (2, 3, 12))).requires_grad_(True)
    assert torch.autograd.gradcheck(
        lambda v: core.frequencies_critical_bands(v, depth=3, scale=scale), (f,))
    assert core.frequencies_critical_bands(f, depth=3, scale=scale).dtype == torch.float64


def test_gradcheck_power_to_db_away_from_its_floor():
  """core.log10 (safe_log) computes in float32 as the reference's does, whatever the
  input's dtype, so the finite differences take a step float32 resolves."""
  p = torch.from_numpy(_rng(4).uniform(0.5, 2.0, 30)).requires_grad_(True)
  assert torch.autograd.gradcheck(core.power_to_db, (p,), eps=1e-3, atol=1e-3, rtol=1e-3)
  # and the gradient is 10 / (ln 10 p), 0 below the floor
  q = torch.tensor([1e-3, 1.0, 40.0, 1e-9], requires_grad=True)
  core.power_to_db(q).sum().backward()
  want = 10.0 / (LN10 * q.detach().double())
  want[-1] = 0.0
  np.testing.assert_allclose(q.grad.double().numpy(), want.numpy(), rtol=1e-6)


def test_gradient_reversal():
  x = torch.from_numpy(_rng(6).normal(0.0, 1e3, (4, 33)).astype(np.float32))
  x.requires_grad_(True)
  y = core.gradient_reversal(x)
  assert torch.equal(y.detach(), x.detach())
  g = torch.randn(4, 33)
  y.backward(g)
  assert torch.equal(x.grad, -g)


# ---- 4. conventions -------------------------------------------------------------------
def test_use_tf_false_is_numpy_and_use_tf_true_is_torch():
  p = np.array([0.0, 1e-9, 0.5, 2.0], np.float32)
  assert isinstance(core.power_to_db(p, use_tf=False), np.ndarray)
  assert isinstance(core.amplitude_to_db(p, use_tf=False), np.ndarray)
  assert torch.is_tensor(core.power_to_db(p))
  np.testing.assert_allclose(core.power_to_db(p).numpy(), core.power_to_db(p, use_tf=False),
                             atol=2e-5)
  for fn in (core.hz_to_bark, core.bark_to_hz, core.hz_to_mel, core.mel_to_hz, core.hz_to_erb):
    out = fn(np.linspace(100.0, 200.0, 5))
    assert isinstance(out, np.ndarray) and out.dtype == np.float64, fn.__name__
  assert isinstance(spectral_ops.pad_or_trim_to_expected_length(torch.zeros(5), 7),
                    np.ndarray)


def test_nan_to_num_keeps_inf():
  x = torch.tensor([np.nan, np.inf, -np.inf, 1.5, -0.0])
  got = core.nan_to_num(x, 7.0)
  assert got.tolist() == [7.0, np.inf, -np.inf, 1.5, 0.0]
  assert core.nan_to_num(np.array([np.nan, 2.0])).tolist() == [0.0, 2.0]


def test_pad_axis():
  x = torch.arange(24.0).reshape(2, 3, 4)
  y = core.pad_axis(x, (1, 2), axis=1, mode='constant', constant_values=-1.0)
  assert y.shape == (2, 6, 4)
  assert torch.equal(y[:, 1:4], x)
  assert (y[:, 0] == -1).all() and (y[:, 4:] == -1).all()
  assert torch.equal(core.pad_axis(x, (0, 3), 2), torch.nn.functional.pad(x, (0, 3)))
  assert torch.equal(core.pad_axis(x, (2, 0), axis=-1, mode='CONSTANT', value=5.0)[..., :2],
                     torch.full((2, 3, 2), 5.0))
  assert torch.equal(core.pad_axis(x), x)
  assert core.pad_axis(x, (1, 1), 0).shape == (4, 3, 4)


def test_center_crop_and_nested_helpers():
  audio = torch.arange(2 * 40.0).reshape(2, 40)
  assert torch.equal(core.center_crop(audio, 16), audio[:, 8:32])
  assert torch.equal(core.center_crop(audio, 17), audio[:, 8:32])
  assert core.center_crop(np.zeros((1, 30, 2)), 10).shape == (1, 20, 2)
  assert core.leaf_key('a/b/c') == 'c' and core.leaf_key('a.b', delimiter='.') == 'b'
  assert core.leaf_key('solo') == 'solo'
  nested = {'a': torch.zeros(2, 3), 'b': {'c': np.zeros(5), 'd': [torch.zeros(1, 4, 2)]}}
  assert core.map_shape(nested) == {'a': [2, 3], 'b': {'c': [5], 'd': [[1, 4, 2]]}}
  assert core.copy_if_tf_function(nested) is nested


def test_pad_or_trim_to_expected_length():
  fn = spectral_ops.pad_or_trim_to_expected_length
  v = np.arange(10, dtype=np.float32)
  np.testing.assert_array_equal(fn(v, 13, pad_value=-1), np.r_[v, -1, -1, -1])
  np.testing.assert_array_equal(fn(v, 7), v[:7])
  np.testing.assert_array_equal(fn(v, 10), v)
  m = np.arange(20.0).reshape(2, 10)
  np.testing.assert_array_equal(fn(m, 12, 5), np.c_[m, np.full((2, 2), 5.0)])
  np.testing.assert_array_equal(fn(m, 4, len_tolerance=6), m[:, :4])
  assert fn(m, 30).shape == (2, 30)
  with pytest.raises(ValueError, match='Vector length: 10 differs from expected length: 31 '
                                       'beyond tolerance of : 20'):
    fn(v, 31)
  with pytest.raises(ValueError, match='beyond tolerance of : 2'):
    fn(m, 7, len_tolerance=2)
  # use_tf=True: torch, differentiable, 1-D and 2-D
  t = torch.arange(20.0).reshape(2, 10).requires_grad_(True)
  out = fn(t, 13, pad_value=0.5, use_tf=True)
  assert out.shape == (2, 13) and (out[:, 10:] == 0.5).all()
  (out * torch.arange(13.0)).sum().backward()
  assert torch.equal(t.grad, torch.arange(10.0).expand(2, 10))
  t1 = torch.arange(10.0, requires_grad=True)
  out = fn(t1, 8, use_tf=True)
  out.sum().backward()
  assert out.shape == (8,) and torch.equal(t1.grad, (torch.arange(10) < 8).float())
  assert torch.equal(fn(t1, 10, use_tf=True), t1)


@pytest.mark.parametrize('frame_size', [64, 128, 256, 512, 1024, 2048])
@pytest.mark.parametrize('batched', [False, True])
def test_stft_np_matches_stft(frame_size, batched):
  n = 4000 + frame_size // 3
  audio = _rng(frame_size).normal(0.0, 0.3, (2, n) if batched else (n,)).astype(np.float32)
  got = spectral_ops.stft_np(audio, frame_size=frame_size, overlap=0.75)
  want = spectral_ops.stft(torch.from_numpy(audio), frame_size=frame_size, overlap=0.75,
                           pad_end=True).numpy()
  assert got.dtype == np.complex64 and got.shape == want.shape
  assert got.shape[-1] == frame_size // 2 + 1
  err = np.abs(got.astype(np.complex128) - want).max() / np.abs(want).max()
  assert err <= 1e-4, err


def test_stft_np_frames_and_window():
  """librosa.stft(center=False) semantics, one frame spelled out: frame i starts at
  i * hop, times a periodic Hann, rfft of frame_size points; pad_end=False keeps only
  whole frames and the assert on frame_size * overlap stays."""
  frame, hop = 64, 16
  audio = _rng(9).normal(0.0, 1.0, 200).astype(np.float32)
  got = spectral_ops.stft_np(audio, frame_size=frame, overlap=0.75, pad_end=False)
  assert got.shape == (1 + (200 - frame) // hop, frame // 2 + 1)
  window = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(frame) / frame)
  want = np.fft.rfft(audio[3 * hop:3 * hop + frame].astype(np.float64) * window)
  np.testing.assert_allclose(got[3], want, rtol=1e-5, atol=1e-5)
  with pytest.raises(AssertionError):
    spectral_ops.stft_np(audio, frame_size=100, overlap=0.75)


# ---- 5. completeness ------------------------------------------------------------------
# the public functions of the reference's ddsp/core.py and ddsp/spectral_ops.py
REFERENCE_CORE = '''
amplitude_to_db angular_cumsum apply_window_to_impulse_response bark_to_hz center_crop
copy_if_tf_function crop_and_compensate_delay db_to_amplitude db_to_power diff exp_sigmoid
fft_convolve frequencies_critical_bands frequencies_sigmoid frequencies_softmax
frequency_filter frequency_impulse_response get_fft_size get_harmonic_frequencies
gradient_reversal harmonic_distribution_to_wavetable harmonic_oscillator_bank
harmonic_synthesis harmonic_to_sinusoidal hz_to_bark hz_to_erb hz_to_mel hz_to_midi
hz_to_unit leaf_key linear_lookup log10 log_scale logb make_iterable map_shape mel_to_hz
midi_to_hz midi_to_unit nan_to_num nested_keys nested_lookup normalize_harmonics
oscillator_bank pad_axis power_to_db remove_above_nyquist resample safe_divide safe_log
sinc sinc_filter sinc_impulse_response sinusoidal_to_harmonic soft_limit
streaming_harmonic_synthesis sym_exp_sigmoid tf_float32 to_dict unit_to_hz unit_to_midi
upsample_with_windows variable_length_delay wavetable_synthesis'''.split()
REFERENCE_SPECTRAL_OPS = '''
compute_f0 compute_logmag compute_logmel compute_loudness compute_mag compute_mel
compute_mfcc compute_power compute_rms_energy get_framed_lengths pad
pad_or_trim_to_expected_length reset_crepe stft stft_np'''.split()
# they wrap the crepe package, which is not a dependency
EXEMPT = {'compute_f0', 'reset_crepe'}


def test_every_reference_function_exists():
  import ddsp_b200 as ddsp
  for module, names in ((ddsp.core, REFERENCE_CORE),
                        (ddsp.spectral_ops, REFERENCE_SPECTRAL_OPS)):
    missing = [n for n in names if n not in EXEMPT and not callable(getattr(module, n, None))]
    assert not missing, (module.__name__, missing)
  assert spectral_ops.DB_RANGE == core.DB_RANGE == 80.0


# ---- 6. GPU ---------------------------------------------------------------------------
DEV = 'cuda'


def _check(name, got, want, tol_max, tol_l2):
  got = got.detach().double().cpu().numpy()
  want = want.detach().double().cpu().numpy()
  assert np.isfinite(got).all(), name
  emax, el2 = rel_err(got, want)
  assert emax < tol_max and el2 < tol_l2, (name, emax, el2)


@pytest.mark.gpu
def test_sym_exp_sigmoid_against_float64():
  """Outside grad on exp_sigmoid's CUDA kernel, under grad in torch; both against
  float64, and the gradient against the float64 derivative."""
  x = _rng(11).uniform(-6.0, 6.0, 4096).astype(np.float32)
  want = sym_exp_sigmoid64(x.astype(np.float64))
  with torch.no_grad():
    got = core.sym_exp_sigmoid(torch.from_numpy(x).to(DEV))
  assert got.is_cuda and got.dtype == torch.float32
  _agree(got, want, 1e-5)
  _agree(core.sym_exp_sigmoid(x, 4.0), sym_exp_sigmoid64(x.astype(np.float64), 4.0), 1e-5)
  xg = torch.from_numpy(x).to(DEV).requires_grad_(True)
  y = core.sym_exp_sigmoid(xg)
  _agree(y, want, 1e-5)
  y.sum().backward()
  x64 = torch.from_numpy(x).double().requires_grad_(True)
  s = torch.sigmoid(8.0 * (x64.abs() / 2.0 - 1.0))
  (2.0 * s**LN10 + 1e-7).sum().backward()
  _check('d x', xg.grad, x64.grad, 1e-5, 1e-5)


def _critical_bands64_torch(x, depth):
  """critical_bands64 in float64 torch, differentiable in x [B, T, N * depth]."""
  x = x.reshape(x.shape[0], x.shape[1], -1, depth)
  c = torch.from_numpy(centres64(x.shape[2], 20.0, 8000.0, 'bark')).to(x.device)
  erb = 0.108 * c + 24.7
  w = 10.0**-torch.arange(depth, dtype=torch.float64, device=x.device)
  f = c + erb * (torch.tanh(x) * w).sum(-1)
  softplus = torch.nn.functional.softplus
  return softplus(f) + 20.0 - softplus(f - 7980.0)


def _sinusoidal64(synth, a_raw, f_raw, amp64, depth, N, sr, method):
  """Audio of the float64 composition scaler + synthesis.  The frequencies take the
  values of our float32 ones (a float64 frequency would drift the phase by more than the
  tolerance over the clip) with their float64 derivatives, and the Nyquist masks are
  decided on the float32 frequencies, as the kernel decides them.  The amplitudes are
  float64 throughout."""
  with torch.no_grad():
    ctl = synth.get_controls(a_raw.detach(), f_raw.detach())
  a64 = a_raw.detach().double().requires_grad_(True)
  f64 = f_raw.detach().double().requires_grad_(True)
  fr = _critical_bands64_torch(f64, depth)
  fr = fr + (ctl['frequencies'].double() - fr).detach()
  am = amp64(a64)
  am = torch.where(ctl['frequencies'] >= sr / 2.0, torch.zeros_like(am), am)
  mask = torch.from_numpy(sinusoidal_ref.nyquist_mask(ctl['frequencies'].cpu().numpy(),
                                                      N, sr)).to(DEV)
  return sinusoidal_ref.torch_sinusoidal(fr, am, N, sr, method, mask=mask), a64, f64


@pytest.mark.gpu
@pytest.mark.parametrize('method', ['window', 'linear'])
def test_sinusoidal_with_critical_bands_trains(method):
  """Sinusoidal(freq_scale_fn=frequencies_critical_bands) on raw network outputs: audio
  and gradients to the raw amplitudes and frequencies against float64 autograd of the
  scaler, exp_sigmoid, the Nyquist masks and the synthesis."""
  import ddsp_b200
  B, F, K, depth, N, sr = 2, 250, 64, 2, 16000, 16000
  rng = _rng(12)
  amps = torch.from_numpy(rng.normal(0.0, 1.0, (B, F, K)).astype(np.float32)).to(DEV)
  freqs = torch.from_numpy(rng.normal(0.0, 1.5, (B, F, K * depth)).astype(np.float32)).to(DEV)
  g = torch.from_numpy(rng.standard_normal((B, N))).to(DEV)
  synth = ddsp_b200.Sinusoidal(
      n_samples=N, sample_rate=sr, amp_resample_method=method,
      freq_scale_fn=lambda f: core.frequencies_critical_bands(f, depth=depth))
  a1, f1 = amps.clone().requires_grad_(True), freqs.clone().requires_grad_(True)
  out = synth(a1, f1)
  assert out.shape == (B, N) and out.requires_grad
  out.backward(g.float())

  def exp_sigmoid64_torch(a):
    return 2.0 * torch.sigmoid(a)**LN10 + 1e-7
  want, a64, f64 = _sinusoidal64(synth, amps, freqs, exp_sigmoid64_torch, depth, N, sr, method)
  want.backward(g)
  _check('audio', out, want, 1e-4, 1e-4)
  _check('d raw amplitudes', a1.grad, a64.grad, 2e-3, 1e-3)
  _check('d raw frequencies', f1.grad, f64.grad, 2e-3, 1e-3)
  # the default depth 1 builds as the reference's gin binding would
  synth1 = ddsp_b200.Sinusoidal(n_samples=N, freq_scale_fn=core.frequencies_critical_bands)
  with torch.no_grad():
    assert bool(torch.isfinite(synth1(amps, freqs[..., :K])).all())


@pytest.mark.gpu
def test_sinusoidal_with_sym_exp_sigmoid_amplitudes():
  """amp_scale_fn=sym_exp_sigmoid (its CUDA route outside grad) gives the audio of the
  float64 composition."""
  import ddsp_b200
  B, F, K, depth, N, sr = 2, 250, 64, 2, 16000, 16000
  rng = _rng(13)
  amps = torch.from_numpy(rng.normal(0.0, 2.0, (B, F, K)).astype(np.float32)).to(DEV)
  freqs = torch.from_numpy(rng.normal(0.0, 1.5, (B, F, K * depth)).astype(np.float32)).to(DEV)
  synth = ddsp_b200.Sinusoidal(
      n_samples=N, sample_rate=sr, amp_scale_fn=core.sym_exp_sigmoid,
      freq_scale_fn=lambda f: core.frequencies_critical_bands(f, depth=depth))
  with torch.no_grad():
    out = synth(amps, freqs)

  def sym64(a):
    return 2.0 * torch.sigmoid(8.0 * (a.abs() / 2.0 - 1.0))**LN10 + 1e-7
  want, _, _ = _sinusoidal64(synth, amps, freqs, sym64, depth, N, sr, 'window')
  _check('audio', out, want, 1e-4, 1e-4)
