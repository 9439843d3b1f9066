"""synthetic_data.py (training/data_preparation/synthetic_data.py): generate_notes_v2 on
the CUDA kernel of csrc/synthetic_notes.cuh and generate_notes on numpy's own draws,
against the float64 restatement tests/synthetic_data_ref.py, which
tests/golden/synthetic_data.npz pins to the unmodified reference.

Bounds.  The kernel's elementary float64 steps are numpy's, bit for bit; cos, sin, pow
and log are CUDA's, within a few ulps of glibc's and numpy's.  So the raw float64 arrays
agree within RAW_TOL relative to max(1, |value|); a stream that slips by a word gives
O(1) errors instead.  The float32 outputs go through exp_sigmoid, midi_to_hz, softmax
and harmonic_to_sinusoidal in float32, whose CUDA and torch versions differ from TF's by
float32 ulps: F32_RTOL, F32_ATOL.
"""
import os

import numpy as np
import pytest
import torch

from tests import synthetic_data_ref as ref
from tests.golden.make_synthetic_data_golden import (DIGEST_CASES, STATE_CASES, V1_CASES,
                                                      V2_CASES, digest)

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'synthetic_data.npz'))
RAW = ('harm_amp', 'harm_dist', 'f0_midi', 'mags')
RAW_TOL = 1e-12
F32_RTOL, F32_ATOL = 1e-5, 1e-6
# Without get_controls, sin_amps divides signed raw distributions by their float32 sums,
# which cancel: a summation order other than TF's moves a row's sum by float32 ulps of
# sum |row|, so each row's relative bound grows with sum |row| / |sum row|.
SUM_RTOL = 1e-5
OUTPUTS = ('harm_amp', 'harm_dist', 'f0_hz', 'sin_amps', 'sin_freqs', 'noise_magnitudes')


def _raw_golden(name):
  """The reference's float64 arrays of a case stored in full."""
  return [GOLDEN[f'{name}_raw_{k}'] for k in RAW]


def _assert_digests(arrays, name):
  """The restatement's arrays of a case stored as digests are the reference's bytes."""
  for a, k in zip(arrays, RAW):
    assert digest(a) == GOLDEN[f'{name}_raw_{k}_sha256'], k


# ---- CPU: the restated stream against numpy ------------------------------------------------
@pytest.mark.parametrize('seed', [0, 1, 5489, 123456789, 2**31, 2**32 - 1])
def test_stream_matches_random_state(seed):
  rs = np.random.RandomState(seed)
  s = ref.Stream.seeded(seed)
  draws = np.random.default_rng(seed).integers(0, 5, 60)
  for i, kind in enumerate(draws):
    n = int(i % 7) + 1
    if kind == 0:
      assert s.uniform(-3.0, 5.5) == rs.uniform(-3.0, 5.5)
    elif kind == 1:
      assert np.array_equal(s.rand(n), rs.rand(n))
    elif kind == 2:
      assert np.array_equal(s.randn(n * 37), rs.randn(n * 37))   # odd and even lengths
    elif kind == 3:
      lo = int(i % 5)
      with pytest.warns(DeprecationWarning):
        want = rs.random_integers(lo, lo + 3 * i)
      assert s.random_integers(lo, lo + 3 * i) == want
    else:
      assert np.array_equal(s.randn(2000, 3), rs.randn(2000, 3))   # several twists
  key, pos, has_gauss, gauss = s.state()
  _, want_key, want_pos, want_has, want_gauss = rs.get_state()
  assert np.array_equal(key, want_key) and pos == want_pos
  assert has_gauss == want_has and gauss == want_gauss


def test_stream_from_numpy_state():
  rs = np.random.RandomState(77)
  rs.randn(3)
  s = ref.Stream.from_numpy(rs.get_state())
  assert np.array_equal(s.randn(1001), rs.randn(1001))
  assert s.uniform() == rs.uniform()


# ---- CPU: the restatement against the fixture ------------------------------------------------
@pytest.mark.parametrize('case', V2_CASES, ids=[c[0] for c in V2_CASES])
def test_restatement_matches_the_reference(case):
  name, seed, kwargs = case
  got = ref.seeded_v2(seed, **kwargs)
  if name in DIGEST_CASES:
    _assert_digests(got[:4], name)
  else:
    for g, w in zip(got[:4], _raw_golden(name)):
      assert np.array_equal(g, w)
  if kwargs.get('get_controls', True):
    assert got[4] == GOLDEN[f'{name}_divisor']


@pytest.mark.parametrize('case', STATE_CASES, ids=[c[0] for c in STATE_CASES])
def test_restatement_state_mode(case):
  name, _, _, kwargs = case
  s = ref.Stream(*(GOLDEN[f'{name}_before_{k}'] for k in ('key', 'pos', 'has_gauss', 'gauss')))
  got = ref.notes_v2(s, 3, **kwargs)
  for g, w in zip(got[:4], _raw_golden(name)):
    assert np.array_equal(g, w)
  key, pos, has_gauss, gauss = s.state()
  assert np.array_equal(key, GOLDEN[f'{name}_after_key'])
  assert (pos, has_gauss, gauss) == (GOLDEN[f'{name}_after_pos'],
                                     GOLDEN[f'{name}_after_has_gauss'],
                                     GOLDEN[f'{name}_after_gauss'])


# ---- GPU --------------------------------------------------------------------------------------
def _sd():
  from ddsp_b200 import synthetic_data
  return synthetic_data


def _raw(**kwargs):
  """The kernel's float64 arrays in seeds mode: harm_amp, harm_dist, f0_midi, mags and
  the divisor, as numpy arrays."""
  from ddsp_b200 import core
  seeds = kwargs.pop('seeds')
  t = kwargs.get('n_timesteps', 125)
  k = kwargs.get('n_harmonics', 100)
  m = kwargs.get('n_mags', 65)
  b = len(seeds)
  dev = torch.device('cuda', torch.cuda.current_device())
  out = [torch.empty(s, dtype=torch.float64, device=dev)
         for s in ((b, t), (b, t, k), (b, t), (b, t, m), (b,))]
  seed_t = torch.tensor(np.asarray(seeds, np.int64), device=dev)
  core._launch('ddsp_b200_synthetic_notes', seed_t, None, None, None, *out, b, t, k, m,
               kwargs.get('min_note_length', 5), kwargs.get('max_note_length', 25),
               float(kwargs.get('p_silent', 0.1)), float(kwargs.get('p_vibrato', 0.5)),
               int(kwargs.get('get_controls', True)))
  return [x.cpu().numpy() for x in out]


def _assert_raw(got, want):
  for g, w in zip(got, want):
    g, w = np.asarray(g), np.asarray(w)
    assert g.shape == w.shape
    err = np.abs(g - w) / np.maximum(1.0, np.abs(w))
    assert err.max(initial=0.0) <= RAW_TOL, err.max()


def _assert_f32(got, want, rtol=F32_RTOL):
  got = got.cpu().numpy()
  assert got.dtype == want.dtype and got.shape == want.shape
  np.testing.assert_allclose(got, want, rtol=rtol, atol=F32_ATOL)


def _assert_outputs(c, name, get_controls):
  """The outputs against the fixture's: the stored float32 ones, sin_freqs as the stored
  f0_hz times 1..K, and without get_controls the float64 arrays as the raw ones."""
  if not get_controls and name not in DIGEST_CASES:
    raw = dict(zip(RAW, _raw_golden(name)))
    _assert_raw([c['harm_amp'].cpu().numpy()[..., 0], c['harm_dist'].cpu().numpy(),
                 c['noise_magnitudes'].cpu().numpy()],
                [raw['harm_amp'], raw['harm_dist'], raw['mags']])
    for k in ('harm_amp', 'harm_dist', 'noise_magnitudes'):
      assert c[k].dtype == torch.float64
  f0 = GOLDEN[f'{name}_f0_hz']
  n = c['sin_freqs'].shape[-1]
  _assert_f32(c['sin_freqs'], f0 * np.linspace(1.0, n, n, dtype=np.float32))
  for k in OUTPUTS:
    if f'{name}_{k}' not in GOLDEN:
      continue
    want = GOLDEN[f'{name}_{k}']
    if k == 'sin_amps' and not get_controls:
      hd = GOLDEN[f'{name}_raw_harm_dist'].astype(np.float32)
      total = np.abs(hd.sum(-1, keepdims=True))
      cond = np.abs(hd).sum(-1, keepdims=True) / np.where(total > 0, total, 1.0)  # 0 rows: silent
      got = c[k].cpu().numpy()
      assert got.dtype == want.dtype and got.shape == want.shape
      bound = F32_ATOL + SUM_RTOL * (1.0 + cond) * np.abs(want)
      assert (np.abs(got - want) <= bound).all(), np.max(np.abs(got - want) / bound)
    else:
      _assert_f32(c[k], want)


SHAPES = [dict(), dict(n_timesteps=1, min_note_length=1, max_note_length=1),
          dict(n_harmonics=1, n_mags=1), dict(p_silent=1.0), dict(p_vibrato=0.0),
          dict(p_vibrato=1.0), dict(get_controls=False),
          dict(n_timesteps=1000, min_note_length=1, max_note_length=200),
          # the largest shapes the kernel takes, in T and in K and M
          dict(n_timesteps=8192, n_harmonics=8, n_mags=8, min_note_length=1,
               max_note_length=3000),
          dict(n_timesteps=4, n_harmonics=4096, n_mags=4096)]


@pytest.mark.gpu
def test_seeds_mode_matches_the_restatement():
  rng = np.random.default_rng(2024)
  for i, kwargs in enumerate(SHAPES):
    n = 300 if not kwargs else (2 if i >= len(SHAPES) - 2 else 24)
    seeds = rng.integers(0, 2**32, n)
    seeds[:2] = [0, 2**32 - 1]
    got = _raw(seeds=seeds, **kwargs)
    for j, seed in enumerate(seeds):
      want = ref.seeded_v2(int(seed), **kwargs)
      _assert_raw([x[j] for x in got[:4]], [w[0] for w in want[:4]])
      if kwargs.get('get_controls', True):
        assert abs(got[4][j] - want[4]) <= RAW_TOL * want[4]


@pytest.mark.gpu
@pytest.mark.parametrize('case', V2_CASES, ids=[c[0] for c in V2_CASES])
def test_seeds_mode_matches_the_reference(case):
  name, seed, kwargs = case
  got = _raw(seeds=[seed], **kwargs)
  if name in DIGEST_CASES:   # the restatement, pinned to the digests, stands in
    want = ref.seeded_v2(seed, **kwargs)
    _assert_digests(want[:4], name)
    _assert_raw(got[:4], want[:4])
  else:
    _assert_raw(got[:4], _raw_golden(name))
  if kwargs.get('get_controls', True):
    assert abs(got[4][0] - GOLDEN[f'{name}_divisor']) <= RAW_TOL * GOLDEN[f'{name}_divisor']
  c = _sd().generate_notes_v2(seeds=[seed], **kwargs)
  _assert_outputs(c, name, kwargs.get('get_controls', True))


@pytest.mark.gpu
def test_seeds_mode_equals_state_mode_and_leaves_numpy_alone():
  sd = _sd()
  np.random.seed(99)
  before = np.random.get_state()
  a = sd.generate_notes_v2(seeds=[12345])
  after = np.random.get_state()
  assert np.array_equal(before[1], after[1]) and before[2:] == after[2:]
  np.random.seed(12345)
  b = sd.generate_notes_v2(n_batch=1)
  for k in OUTPUTS:
    assert torch.equal(a[k], b[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize('case', STATE_CASES, ids=[c[0] for c in STATE_CASES])
def test_state_mode_matches_the_reference(case):
  name, _, _, kwargs = case
  np.random.set_state(('MT19937', GOLDEN[f'{name}_before_key'],
                       int(GOLDEN[f'{name}_before_pos']),
                       int(GOLDEN[f'{name}_before_has_gauss']),
                       float(GOLDEN[f'{name}_before_gauss'])))
  c = _sd().generate_notes_v2(n_batch=3, **kwargs)
  _, key, pos, has_gauss, gauss = np.random.get_state()
  assert np.array_equal(key, GOLDEN[f'{name}_after_key'])
  assert pos == GOLDEN[f'{name}_after_pos']
  assert has_gauss == GOLDEN[f'{name}_after_has_gauss']
  want_gauss = float(GOLDEN[f'{name}_after_gauss'])
  assert abs(gauss - want_gauss) <= 1e-15 * abs(want_gauss)
  np.random.set_state(('MT19937', key, pos, has_gauss, want_gauss))
  assert np.array_equal(np.random.uniform(size=4), GOLDEN[f'{name}_next'])
  _assert_outputs(c, name, kwargs.get('get_controls', True))


@pytest.mark.gpu
def test_items_do_not_depend_on_the_batch():
  rng = np.random.default_rng(7)
  probe = [0, 1, 2**32 - 1, 424242]
  one = [_raw(seeds=[s]) for s in probe]
  for b in (7, 133, 4096):
    seeds = rng.integers(0, 2**32, b)
    at = rng.choice(b, len(probe), replace=False)
    seeds[at] = probe
    got = _raw(seeds=seeds)
    for i, j in enumerate(at):
      for x, y in zip(got, one[i]):
        assert np.array_equal(x[j], y[0])
  again = _raw(seeds=seeds)
  for x, y in zip(got, again):
    assert np.array_equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize('case', V1_CASES, ids=[c[0] for c in V1_CASES])
def test_generate_notes_matches_the_reference(case):
  name, _, b, t, k, m = case
  np.random.set_state(('MT19937', GOLDEN[f'{name}_before_key'],
                       int(GOLDEN[f'{name}_before_pos']),
                       int(GOLDEN[f'{name}_before_has_gauss']),
                       float(GOLDEN[f'{name}_before_gauss'])))
  c = _sd().generate_notes(b, t, n_harmonics=k, n_mags=m)
  _, key, pos, has_gauss, gauss = np.random.get_state()
  assert np.array_equal(key, GOLDEN[f'{name}_after_key'])
  assert (pos, has_gauss, gauss) == (GOLDEN[f'{name}_after_pos'],
                                     GOLDEN[f'{name}_after_has_gauss'],
                                     GOLDEN[f'{name}_after_gauss'])
  _assert_outputs(c, name, True)


@pytest.mark.gpu
@pytest.mark.parametrize('kwargs', [
    dict(n_timesteps=0), dict(n_harmonics=0), dict(n_mags=0), dict(n_timesteps=8193),
    dict(n_harmonics=4097), dict(n_mags=5000), dict(min_note_length=6, max_note_length=5),
    dict(min_note_length=0), dict(seeds=[-1]), dict(seeds=[2**32]), dict(seeds=[1.5])])
def test_errors_before_launch(kwargs, monkeypatch):
  from ddsp_b200 import core
  sd = _sd()
  calls = []
  monkeypatch.setattr(core, '_launch', lambda *a: calls.append(a))
  np.random.seed(3)
  before = np.random.get_state()
  with pytest.raises(ValueError):
    sd.generate_notes_v2(**kwargs)
  assert not calls
  after = np.random.get_state()
  assert np.array_equal(before[1], after[1]) and before[2:] == after[2:]


@pytest.mark.gpu
def test_outputs_fenced_on_both_sides_are_written_exactly():
  from ddsp_b200 import core
  b, t, k, m, pad = 5, 125, 100, 65, 64
  dev = torch.device('cuda', torch.cuda.current_device())
  sizes = (b * t, b * t * k, b * t, b * t * m, b)
  bufs = [torch.full((n + 2 * pad,), 7.25, dtype=torch.float64, device=dev) for n in sizes]
  seeds = [3, 1, 4, 1, 5]
  core._launch('ddsp_b200_synthetic_notes', torch.tensor(seeds, device=dev), None, None,
               None, *[x[pad:-pad] for x in bufs], b, t, k, m, 5, 25, 0.1, 0.5, 1)
  want = _raw(seeds=seeds)
  for x, w in zip(bufs, want):
    x = x.cpu().numpy()
    assert (x[:pad] == 7.25).all() and (x[-pad:] == 7.25).all()
    assert np.array_equal(x[pad:-pad], w.reshape(-1))


@pytest.mark.gpu
def test_launch_uses_the_current_stream():
  sd = _sd()
  want = sd.generate_notes_v2(seeds=[11, 12])
  torch.cuda.synchronize()
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    torch.cuda._sleep(50_000_000)     # the launch must queue behind this
    got = sd.generate_notes_v2(seeds=[11, 12])
    ev = torch.cuda.Event()
    ev.record(side)
  ev.synchronize()
  for k in OUTPUTS:
    assert torch.equal(got[k], want[k])


@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two CUDA devices')
def test_non_default_device():
  sd = _sd()
  want = sd.generate_notes_v2(seeds=[8, 9])
  got = sd.generate_notes_v2(seeds=[8, 9], device='cuda:1')
  for k in OUTPUTS:
    assert got[k].device == torch.device('cuda:1')
    assert torch.equal(got[k].cpu(), want[k].cpu())


@pytest.mark.gpu
def test_inverse_synthesis_audio_path():
  import ddsp_b200
  from ddsp_b200 import core
  n = 16000

  def group():
    sin = ddsp_b200.Sinusoidal(n_samples=n, amp_scale_fn=None, freq_scale_fn=None,
                               name='sinusoidal')
    noise = ddsp_b200.FilteredNoise(n_samples=n, window_size=0, scale_fn=None,
                                    name='filtered_noise', seed=5)
    return ddsp_b200.ProcessorGroup(dag=[
        (sin, ['amplitudes', 'frequencies']), (noise, ['noise_magnitudes']),
        (ddsp_b200.Add(), ['filtered_noise/signal', 'sinusoidal/signal'])])

  c = _sd().generate_notes_v2(seeds=[0])
  audio = group()({'amplitudes': c['sin_amps'], 'frequencies': c['sin_freqs'],
                   'noise_magnitudes': c['noise_magnitudes']})
  dev = audio.device
  amps, freqs = core.harmonic_to_sinusoidal(
      *(torch.tensor(GOLDEN[f'seed0_{k}'], device=dev)
        for k in ('harm_amp', 'harm_dist', 'f0_hz')))
  want = group()({
      'amplitudes': amps, 'frequencies': freqs,
      'noise_magnitudes': torch.tensor(GOLDEN['seed0_noise_magnitudes'], device=dev)})
  audio, want = audio.cpu().numpy(), want.cpu().numpy()
  assert np.isfinite(audio).all()
  # frequencies one float32 ulp apart (~6e-8 relative) drift ~4e-4 rad in phase over
  # 16000 samples at 1 kHz
  assert np.abs(audio - want).max() <= 2e-3 * np.abs(want).max()
