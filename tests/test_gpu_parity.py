"""GPU parity: CUDA path (through the C ABI) vs the float64 oracle.

Tolerance (BASELINE.json north_star): 1e-4 relative, measured as max-abs error
over the reference's peak AND as relative L2.  The reference's own float32
phase drift vs the same arbiter is far larger (BASELINE.md section 5) and is
reported in DESIGN.md, not gated.
"""
import numpy as np
import pytest
import torch

from oracle import ddsp_oracle as oracle
from tests.util import rel_err, synth_inputs

import ddsp_b200
from ddsp_b200 import core

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _np(x):
  return x.detach().cpu().numpy()


@pytest.mark.parametrize('B,F,K,N', [(1, 250, 64, 16000), (3, 100, 100, 6400),
                                     (2, 50, 99, 3200), (2, 40, 1, 2560),
                                     (2, 10, 16, 1000), (1, 7, 5, 7 * 33),
                                     (200, 40, 8, 2560), (5, 33, 12, 33 * 64),
                                     (3, 64, 128, 4096)])
@pytest.mark.parametrize('amp_method', ['window', 'linear'])
@pytest.mark.parametrize('phase_mode', ['recurrence', 'direct'])
def test_harmonic_synthesis_matches_oracle(B, F, K, N, amp_method, phase_mode):
  inp = synth_inputs(B, F, K, 65, N, seed=B * 1000 + K)
  ctl = oracle.harmonic_get_controls(inp['amps'], inp['harmonic_distribution'],
                                     inp['f0_hz'], dtype=np.float32)
  want = oracle.harmonic_synthesis(
      ctl['f0_hz'], ctl['amplitudes'],
      harmonic_distribution=ctl['harmonic_distribution'], n_samples=N,
      amp_resample_method=amp_method, dtype=np.float64)
  got = core.harmonic_synthesis(
      ctl['f0_hz'], ctl['amplitudes'],
      harmonic_distribution=ctl['harmonic_distribution'], n_samples=N,
      amp_resample_method=amp_method, phase_mode=phase_mode)
  emax, el2 = rel_err(_np(got), want)
  assert emax < TOL and el2 < TOL, (emax, el2)


def test_harmonic_constant_f0_known_answer():
  """Inclusive cumsum: phase starts at omega (core.py:955)."""
  N, F = 16000, 250
  f0 = np.full((1, F, 1), 440.0, np.float32)
  amp = np.ones((1, F, 1), np.float32)
  got = _np(core.harmonic_synthesis(f0, amp, n_samples=N))[0]
  want = np.sin(2 * np.pi * 440.0 * (np.arange(N) + 1) / 16000.0)
  assert np.abs(got - want).max() < 2e-6


@pytest.mark.parametrize('sample_rate', [4000, 16000, 44100])
def test_silent_above_nyquist(sample_rate):
  """core_test.py:484-503 at the Harmonic level: f0 >= Nyquist -> silence."""
  N, F = 16000, 250
  for mult in (1.0, 1.1, 2.0):
    f0 = np.full((2, F, 1), mult * sample_rate / 2, np.float32)
    amp = np.ones((2, F, 1), np.float32)
    hd = np.full((2, F, 3), 1 / 3, np.float32)
    got = _np(core.harmonic_synthesis(f0, amp, harmonic_distribution=hd,
                                      n_samples=N, sample_rate=sample_rate))
    assert np.all(got == 0.0)


@pytest.mark.parametrize('B,F,K', [(2, 37, 100), (3, 10, 99), (1, 5, 1), (2, 9, 260)])
@pytest.mark.parametrize('scale,nyq', [(True, True), (False, True), (True, False)])
def test_harmonic_controls(B, F, K, scale, nyq):
  inp = synth_inputs(B, F, K, 65, F * 64, seed=7, f0_hi=2000.0)
  amps, hd = inp['amps'], inp['harmonic_distribution']
  if not scale:
    amps, hd = np.abs(amps), np.abs(hd)
  want = oracle.harmonic_get_controls(amps, hd, inp['f0_hz'], scale=scale,
                                      normalize_below_nyquist=nyq,
                                      dtype=np.float64)
  a, h = core.harmonic_controls(amps, hd, inp['f0_hz'], 16000, scale=scale,
                                normalize_below_nyquist=nyq)
  np.testing.assert_allclose(_np(a), want['amplitudes'], rtol=2e-5, atol=1e-9)
  np.testing.assert_allclose(_np(h), want['harmonic_distribution'], rtol=2e-5,
                             atol=1e-9)
  # masked harmonics are exact zeros
  assert np.all((_np(h) == 0) == (want['harmonic_distribution'] == 0))


def test_noise_controls():
  x = np.random.default_rng(0).standard_normal((2, 30, 65)).astype(np.float32) * 4
  want = oracle.noise_get_controls(x, dtype=np.float64)['magnitudes']
  got = _np(core.noise_controls(x, -5.0))
  np.testing.assert_allclose(got, want, rtol=2e-5, atol=1e-9)


@pytest.mark.parametrize('nb,ws', [(65, 0), (65, 257), (1025, 257), (513, 22),
                                   (513, 2048), (100, 257), (100, 50), (100, 51),
                                   (3, 0), (2, 0)])
def test_frequency_impulse_response(nb, ws):
  m = np.random.default_rng(nb).uniform(0, 1, (2, 5, nb)).astype(np.float32)
  want = oracle.frequency_impulse_response(m, ws)
  got = _np(core.frequency_impulse_response(m, ws))
  assert got.shape == want.shape
  assert np.abs(got - want).max() < 1e-6


@pytest.mark.parametrize('B,F,nb,N,ws', [(2, 100, 65, 6400, 0), (2, 25, 65, 1600, 257),
                                         (1, 13, 513, 1000, 257), (2, 1, 513, 1000, 257),
                                         (1, 1000, 513, 1000, 257), (3, 50, 100, 50, 257),
                                         (2, 20, 256, 1280, 257), (1, 1000, 65, 64000, 0),
                                         (1, 30, 65, 1920, 0), (3, 58, 65, 3712, 257),
                                         (2, 29, 65, 1856, 0), (2, 5, 65, 320, 0),
                                         (2, 40, 33, 2560, 0), (1, 24, 65, 3072, 0)])
def test_filtered_noise_matches_oracle(B, F, nb, N, ws):
  rng = np.random.default_rng(B + F + nb)
  mags = rng.uniform(0.0, 1.0, (B, F, nb)).astype(np.float32)
  noise = rng.uniform(-1, 1, (B, N)).astype(np.float32)
  want = oracle.frequency_filter(noise, mags, window_size=ws)
  got = _np(core.filtered_noise(mags, N, window_size=ws, noise=noise))
  emax, el2 = rel_err(got, want)
  assert emax < TOL and el2 < TOL, (emax, el2)
  # the stand-alone pieces agree too
  got2 = _np(core.frequency_filter(noise, mags, window_size=ws))
  emax, el2 = rel_err(got2, want)
  assert emax < TOL and el2 < TOL, (emax, el2)


@pytest.mark.parametrize('audio_size,ir_size', [(1000, 10), (10, 100)])
def test_fft_convolve_is_accurate(audio_size, ir_size):
  """core_test.py:730-757."""
  from scipy import signal
  audio = np.ones([1, audio_size], np.float32)
  ir = np.ones([1, ir_size], np.float32)
  got = _np(core.fft_convolve(audio, ir, padding='valid', delay_compensation=0))[0]
  want = signal.fftconvolve(audio[0], ir[0])
  assert got.shape == want.shape
  assert np.abs(want - got).mean() <= 1e-3


@pytest.mark.parametrize('gain', [1.0, 0.1])
def test_delay_compensation_corrects_group_delay(gain):
  """core_test.py:759-785."""
  audio = np.random.default_rng(0).standard_normal((1, 1000)).astype(np.float32)
  mags = gain * np.ones([1, 1025], np.float32)
  ir = core.frequency_impulse_response(mags, 257)
  got = _np(core.fft_convolve(audio, ir, padding='same'))[0]
  assert np.abs(gain * audio[0] - got).mean() <= 1e-3


def test_uniform_noise_matches_philox_restatement():
  got = _np(core.uniform_noise(3, 1001, seed=0x123456789ABCDEF, offset=5))
  want = oracle.philox_uniform_noise(3, 1001, seed=0x123456789ABCDEF, offset=5)
  assert np.array_equal(got, want)
  assert got.min() >= -1.0 and got.max() < 1.0
  assert abs(got.mean()) < 0.05


def test_filtered_noise_in_kernel_rng_matches_injected():
  """NULL noise pointer == injecting the same Philox stream."""
  mags = np.random.default_rng(1).uniform(0, 1, (2, 50, 65)).astype(np.float32)
  N = 3200
  a = _np(core.filtered_noise(mags, N, window_size=0, seed=42, offset=3))
  nz = oracle.philox_uniform_noise(2, N, seed=42, offset=3)
  b = _np(core.filtered_noise(mags, N, window_size=0, noise=nz))
  emax, _ = rel_err(a, b)
  assert emax < 1e-6


def test_decoder_processor_group_matches_oracle():
  """The ae.gin DAG (ae.gin:47-72) end to end, both API paths."""
  B, F, K, nb, N = 2, 125, 100, 65, 8000
  inp = synth_inputs(B, F, K, nb, N, seed=5)
  want = oracle.decoder(inp['amps'], inp['harmonic_distribution'], inp['f0_hz'],
                        inp['noise_magnitudes'], inp['noise'], n_samples=N,
                        window_size=0, dtype=np.float64)
  harm = ddsp_b200.Harmonic(n_samples=N)
  noise = ddsp_b200.FilteredNoise(n_samples=N, window_size=0)
  add = ddsp_b200.Add()
  noise.injected_noise = inp['noise']   # parity hook instead of the Philox stream
  pg = ddsp_b200.ProcessorGroup(dag=[
      (harm, ['amps', 'harmonic_distribution', 'f0_hz']),
      (noise, ['noise_magnitudes']),
      (add, ['filtered_noise/signal', 'harmonic/signal'])])
  feats = {k: inp[k] for k in ['amps', 'harmonic_distribution', 'f0_hz',
                               'noise_magnitudes']}
  outs = pg.get_controls(feats)
  for key, ref in [('harmonic/signal', want['harmonic']['signal']),
                   ('filtered_noise/signal', want['filtered_noise']['signal']),
                   ('add/signal', want['add']['signal']),
                   ('out/signal', want['add']['signal'])]:
    emax, el2 = rel_err(_np(core.nested_lookup(key, outs)), ref)
    assert emax < TOL and el2 < TOL, (key, emax, el2)
  fused = _np(pg(feats))                # decoder_forward: 2 launches from raw
  emax, el2 = rel_err(fused, want['add']['signal'])
  assert emax < TOL and el2 < TOL, (emax, el2)
  # a non-default scale_fn takes the per-processor accumulate path
  harm.scale_fn = lambda x: core.exp_sigmoid(x)
  fused2 = _np(pg(feats))
  emax, el2 = rel_err(fused2, want['add']['signal'])
  assert emax < TOL and el2 < TOL, (emax, el2)


@pytest.mark.parametrize('B,F,K,nb,N,nyq', [(3, 100, 100, 65, 6400, True),
                                            (2, 33, 60, 65, 33 * 128, True),
                                            (2, 64, 99, 33, 4096, False)])
def test_decoder_forward_from_raw_matches_oracle(B, F, K, nb, N, nyq):
  inp = synth_inputs(B, F, K, nb, N, seed=B + K, f0_hi=1500.0)
  hc = oracle.harmonic_get_controls(inp['amps'], inp['harmonic_distribution'],
                                    inp['f0_hz'], normalize_below_nyquist=nyq,
                                    dtype=np.float64)
  harm = oracle.harmonic_get_signal(n_samples=N, dtype=np.float64, **hc)
  nc = oracle.noise_get_controls(inp['noise_magnitudes'], dtype=np.float64)
  nz = oracle.noise_get_signal(nc['magnitudes'], inp['noise'], 0)
  got = _np(core.decoder_forward(
      inp['amps'], inp['harmonic_distribution'], inp['f0_hz'],
      inp['noise_magnitudes'], N, normalize_below_nyquist=nyq, window_size=0,
      noise=inp['noise']))
  emax, el2 = rel_err(got, harm + nz)
  assert emax < TOL and el2 < TOL, (emax, el2)


@pytest.mark.parametrize('B,F,K,N,method', [(1, 2, 60, 320, 'linear'),
                                            (3, 10, 20, 640, 'linear'),
                                            (2, 4, 100, 256, 'window')])
def test_streaming_harmonic_synthesis_carries_phase(B, F, K, N, method):
  """core.streaming_harmonic_synthesis (core.py:1114-1164): audio and final_phase
  vs the oracle, and hop-by-hop synthesis with the carried phase equals one call
  on the concatenated controls (training/inference.py:463-478)."""
  rng = np.random.default_rng(K)
  f0 = rng.uniform(100, 900, (B, F, 1)).astype(np.float32)
  amp = rng.uniform(0.1, 1.0, (B, F, 1)).astype(np.float32)
  hd = rng.uniform(0.0, 1.0, (B, F, K)).astype(np.float32)
  init = rng.uniform(0, 2 * np.pi, (B, 1, 1)).astype(np.float32)
  want_a, want_p = oracle.streaming_harmonic_synthesis(
      f0, amp, hd, init, n_samples=N, amp_resample_method=method)
  got_a, got_p = core.streaming_harmonic_synthesis(
      f0, amp, hd, init, n_samples=N, amp_resample_method=method)
  emax, el2 = rel_err(_np(got_a), want_a)
  assert emax < TOL and el2 < TOL, (emax, el2)
  assert got_p.shape == (B, 1, 1)
  d = np.abs(_np(got_p) - want_p)
  assert np.minimum(d, 2 * np.pi - d).max() < 1e-4
  # two successive hops with the carried phase: the second call continues the wave
  a1, p1 = core.streaming_harmonic_synthesis(f0, amp, hd, None, n_samples=N,
                                             amp_resample_method=method)
  a2, p2 = core.streaming_harmonic_synthesis(f0, amp, hd, p1, n_samples=N,
                                             amp_resample_method=method)
  w1, q1 = oracle.streaming_harmonic_synthesis(f0, amp, hd, None, n_samples=N,
                                               amp_resample_method=method)
  w2, _ = oracle.streaming_harmonic_synthesis(f0, amp, hd, q1, n_samples=N,
                                              amp_resample_method=method)
  emax, _ = rel_err(np.concatenate([_np(a1), _np(a2)], 1), np.concatenate([w1, w2], 1))
  assert emax < TOL


# ---- core_test.py:ResampleTest through the CUDA op ---------------------------
def _subsampled_close(smaller, larger, add_endpoint, threshold=1e-3):
  n_smaller, n_larger = smaller.size, larger.size
  n_total = (int(n_larger / n_smaller * (n_smaller - 1)) if add_endpoint
             else n_larger - 1)
  idx = np.linspace(0, n_total, n_smaller).astype(int)
  np.testing.assert_allclose(larger[idx], smaller, atol=threshold)


@pytest.mark.parametrize('add_endpoint', [True, False])
@pytest.mark.parametrize('method', ['linear', 'window', 'nearest'])
def test_resample_upsample_accuracy(add_endpoint, method):
  """core_test.py:242-267 + agreement with the oracle's TF restatement."""
  before = (1.0 - np.sin(np.linspace(0, np.pi, 5)))[None, :, None].astype(np.float32)
  after = _np(core.resample(before, 16000, method=method, add_endpoint=add_endpoint))
  if method != 'nearest':
    _subsampled_close(before[0, :, 0], after[0, :, 0], add_endpoint)
  want = oracle.resample(before, 16000, method=method, add_endpoint=add_endpoint,
                         dtype=np.float32, tf_index_math=True)
  np.testing.assert_allclose(after, want, atol=2e-6)


@pytest.mark.parametrize('add_endpoint', [True, False])
def test_resample_downsample_accuracy(add_endpoint):
  """core_test.py:269-293."""
  before = (1.0 - np.sin(np.linspace(0, np.pi, 16000)))[None, :, None].astype(np.float32)
  after = _np(core.resample(before, 5, method='linear', add_endpoint=add_endpoint))
  _subsampled_close(after[0, :, 0], before[0, :, 0], add_endpoint)


@pytest.mark.parametrize('dimensions', [1, 2, 3])
def test_resample_multi_dimensional_inputs(dimensions):
  """core_test.py:152-176."""
  shape = [5] * dimensions
  out = core.resample(np.ones(shape, np.float32), 16000)
  want = list(shape)
  want[0 if dimensions == 1 else 1] = 16000
  assert list(out.shape) == want
  rnd = np.random.default_rng(0).standard_normal((3, 20, 7)).astype(np.float32)
  got = _np(core.upsample_with_windows(rnd, 640))
  np.testing.assert_allclose(got, oracle.upsample_with_windows(rnd, 640), atol=2e-6)


def test_normalize_harmonics_and_helpers():
  """core_test.py:104-142 (get_harmonic_frequencies / normalize_harmonics)."""
  f0 = np.array([[[1000.0], [3000.0], [4500.0], [9000.0]]], np.float32)
  hd = np.ones((1, 4, 3), np.float32)
  out = _np(core.normalize_harmonics(hd, f0, 16000))
  np.testing.assert_allclose(out[0, 0], [1 / 3] * 3, rtol=1e-6)
  np.testing.assert_allclose(out[0, 1], [0.5, 0.5, 0.0], rtol=1e-6)
  np.testing.assert_allclose(out[0, 2], [1.0, 0.0, 0.0], rtol=1e-6)
  np.testing.assert_allclose(out[0, 3], [0.0, 0.0, 0.0])
  plain = _np(core.normalize_harmonics(hd * 2.0))
  np.testing.assert_allclose(plain, np.full((1, 4, 3), 1 / 3), rtol=1e-6)
  hf = _np(core.get_harmonic_frequencies(f0, 3))
  np.testing.assert_allclose(hf[0, :, 2], f0[0, :, 0] * 3)
  amps = _np(core.remove_above_nyquist(hf, np.ones_like(hf), 16000))
  assert np.array_equal(amps == 0, hf >= 8000.0)


@pytest.mark.parametrize('sum_sinusoids', [True, False])
@pytest.mark.parametrize('B,N,K', [(2, 1600, 3), (1, 4000, 100), (3, 257, 37)])
def test_oscillator_bank_matches_oracle(B, N, K, sum_sinusoids):
  """core.oscillator_bank (core.py:911-962) on audio-rate envelopes; shapes as in
  core_test.py:460-482, Nyquist silence as in core_test.py:484-503."""
  rng = np.random.default_rng(N + K)
  f = (rng.uniform(50, 9000, (B, 1, K)) *
       (1.0 + 0.01 * np.sin(np.arange(N) / 300.0))[None, :, None]).astype(np.float32)
  a = rng.uniform(0.0, 1.0, (B, N, K)).astype(np.float32)
  want = oracle.oscillator_bank(f, a, sum_sinusoids=sum_sinusoids, dtype=np.float64)
  got = _np(core.oscillator_bank(f, a, sum_sinusoids=sum_sinusoids))
  assert got.shape == want.shape
  emax, el2 = rel_err(got, want)
  assert emax < TOL and el2 < TOL, (emax, el2)


@pytest.mark.parametrize('sample_rate', [4000, 16000, 44100])
def test_oscillator_bank_silent_above_nyquist(sample_rate):
  """core_test.py:484-503 verbatim."""
  nyquist = sample_rate / 2
  freqs = np.array([1.1, 1.5, 2.0]) * nyquist
  ones = np.ones([2, 16000, 3], np.float32)
  wav = _np(core.oscillator_bank(ones * freqs.astype(np.float32), ones,
                                 sample_rate=sample_rate))
  assert wav.shape == (2, 16000) and np.all(wav == 0.0)


@pytest.mark.parametrize('B,F', [(37, 97), (5, 250), (150, 33)])
def test_filtered_noise_ring_segments_match_oracle(B, F):
  """The ring kernel hands each persistent CTA a contiguous run of frames that is
  cut wherever an item ends: shapes whose runs start and stop at every possible
  offset (ragged last tiles, runs shorter than a tile, items shorter than the
  3-frame halo of a run)."""
  nb, N = 65, F * 64
  rng = np.random.default_rng(B * 1000 + F)
  mags = rng.uniform(0.0, 1.0, (B, F, nb)).astype(np.float32)
  noise = rng.uniform(-1, 1, (B, N)).astype(np.float32)
  want = oracle.frequency_filter(noise, mags, window_size=0)
  got = _np(core.filtered_noise(mags, N, window_size=0, noise=noise))
  emax, el2 = rel_err(got, want)
  assert emax < TOL and el2 < TOL, (emax, el2)
  # accumulate mode (the fused Add) on top of a known signal
  base = rng.standard_normal((B, N)).astype(np.float32)
  out = torch.from_numpy(base.copy()).cuda()
  core.filtered_noise(mags, N, window_size=0, noise=noise, out=out, accumulate=True)
  emax, el2 = rel_err(_np(out) - base, want)
  assert emax < 2 * TOL and el2 < 2 * TOL, (emax, el2)


def test_decoder_is_deterministic_at_full_size():
  """Same seed and offset -> the same bits, twice, at B=64 x 64000 samples: the
  producer / consumer hand-offs of the noise kernel and the programmatic
  dependent launch behind the harmonic kernel leave no run-to-run freedom."""
  B, F, K, nb, N = 64, 1000, 100, 65, 64000
  inp = synth_inputs(B, F, K, nb, N, seed=77)
  dev = {k: torch.from_numpy(inp[k]).cuda() for k in
         ['amps', 'harmonic_distribution', 'f0_hz', 'noise_magnitudes']}
  outs = []
  for _ in range(3):
    outs.append(core.decoder_forward(dev['amps'], dev['harmonic_distribution'],
                                     dev['f0_hz'], dev['noise_magnitudes'], N,
                                     window_size=0, seed=5, offset=9))
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
  assert torch.isfinite(outs[0]).all()


def test_noise_ring_stress_random_shapes_against_the_generic_path():
  """compute-sanitizer's racecheck does not model the mbarrier hand-offs of the
  warp-specialised noise kernel (it flags every producer -> consumer edge), so the
  race question is put empirically: ~900 launches over random batch / frame counts
  (every segment geometry: items shorter than a tile, CTA ranges cut mid-item, ring
  wrap-around), back to back on one stream, each result compared (a) bit for bit
  with a repeat of the same launch and (b) with the generic, unspecialised path -
  separate impulse-response and FIR kernels, no ring, no warp roles - to 2e-5 of
  the peak.  A stale tap row or a half-written noise row would be an O(1) error."""
  from ddsp_b200 import _lib
  lib = _lib.load()
  rng = np.random.default_rng(20240)
  st = torch.cuda.current_stream().cuda_stream
  worst = 0.0
  for trial in range(300):
    B = int(rng.integers(1, 9))
    F = int(rng.choice([3, 5, 17, 31, 32, 33, 63, 64, 65, 97, 128, 250, 333])) \
        if trial % 3 else int(rng.integers(3, 400))
    N = F * 64
    mags = torch.rand((B, F, 65), device='cuda') * 1.5
    noise = torch.rand((B, N), device='cuda') * 2 - 1
    base = torch.randn((B, N), device='cuda') if trial % 2 else None
    outs = []
    for rep in range(3):
      out = base.clone() if base is not None else torch.empty((B, N), device='cuda')
      _lib.check(lib.ddsp_b200_filtered_noise_forward(
          mags.data_ptr(), noise.data_ptr(), 0, 0, out.data_ptr(), B, F, 65, N, 0,
          int(base is not None), None, 0, st))
      outs.append(out)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), (trial, B, F)
    # generic path: IRs to HBM, then the plain time-varying FIR kernel
    ir = core.frequency_impulse_response(mags, 0)
    want = torch.empty((B, N), device='cuda') if base is None else base.clone()
    _lib.check(lib.ddsp_b200_fir_time_varying(
        noise.data_ptr(), ir.data_ptr(), want.data_ptr(), B, N, F, 128, B, _lib.PAD_SAME,
        -1, int(base is not None), st))
    ref = want - base if base is not None else want
    got = outs[0] - base if base is not None else outs[0]
    err = float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-20))
    worst = max(worst, err)
    assert err < 2e-5, (trial, B, F, err)
  assert worst < 2e-5
