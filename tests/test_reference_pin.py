"""Pins the oracle to the reference itself (CPU, no GPU).

tests/golden/*.npz hold outputs of the UNMODIFIED reference (magenta/ddsp run on
oracle/tf_shim, see tests/golden/make_golden.py): "f32" = the reference's own
float32 arithmetic, "wide" = the same reference code evaluated in float64.
oracle/ddsp_oracle.py - the arbiter of the `-m gpu` parity tests - must reproduce
them: its float32 mode to the reference's float32 result within a few ulp, its
float64 mode to the wide result to 1e-9.  Where the reference sources are checked
out, `make_golden.py --check` regenerates the fixtures and compares them bit for
bit, and `python -m oracle.run_reference_tests` runs the reference's own unit tests
of the path on the shim.
"""
import os

import numpy as np
import pytest

from oracle import ddsp_oracle as o
from tests.util import rel_err, synth_inputs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def gold(name):
  return np.load(os.path.join(GOLD, name + '.npz'))


def inputs_for(g, *shape, **kw):
  from tests.golden.make_golden import checksum
  inp = synth_inputs(*shape, seed=int(g['seed']), **kw)
  assert abs(checksum(inp) - float(g['input_checksum'])) <= 1e-6 * abs(float(g['input_checksum'])), \
      'synth_inputs no longer reproduces the inputs this fixture was made from'
  return inp


# ---------------------------------------------------------------------------
# oracle <-> fixtures (runs everywhere)
# ---------------------------------------------------------------------------
def test_oracle_matches_reference_on_configs0():
  g = gold('c1_harmonic')
  inp = inputs_for(g, 1, 250, 64, 65, 16000)
  ctl = o.harmonic_get_controls(inp['amps'], inp['harmonic_distribution'],
                                inp['f0_hz'], dtype=np.float32)
  np.testing.assert_allclose(ctl['amplitudes'], g['amplitudes'], rtol=3e-6, atol=1e-9)
  np.testing.assert_allclose(ctl['harmonic_distribution'], g['harmonic_distribution'],
                             rtol=3e-6, atol=1e-9)
  # from the reference's own controls on: float32 "TF order", both phase modes
  kw = dict(harmonic_distribution=g['harmonic_distribution'], n_samples=16000)
  a32 = o.harmonic_synthesis(inp['f0_hz'], g['amplitudes'], dtype=np.float32,
                             tf_index_math=True, **kw)
  assert np.abs(a32 - g['audio_ref_f32_cumsum']).max() <= 4e-7
  a32a = o.harmonic_synthesis(inp['f0_hz'], g['amplitudes'], dtype=np.float32,
                              tf_index_math=True, use_angular_cumsum=True, **kw)
  assert np.abs(a32a - g['audio_ref_f32_angular']).max() <= 2e-5   # sin of a 1-ulp-different wrapped phase
  # the arbiter: reference code evaluated wide, from the raw network outputs
  c64 = o.harmonic_get_controls(inp['amps'], inp['harmonic_distribution'],
                                inp['f0_hz'], dtype=np.float64)
  a64 = o.harmonic_synthesis(c64['f0_hz'], c64['amplitudes'],
                             harmonic_distribution=c64['harmonic_distribution'],
                             n_samples=16000, dtype=np.float64)
  assert np.abs(a64 - g['audio_ref_wide']).max() <= 1e-9


def test_reference_phase_accumulation_error_is_what_we_state():
  """The 'phase-accumulation tolerance' of north_star: the reference's float32
  tf.cumsum against its own formulae evaluated exactly (DESIGN.md section 3.1,
  BASELINE.md section 5).  Our kernels are gated at 1e-4 against the exact value."""
  g = gold('c1_harmonic')
  e_cumsum = rel_err(g['audio_ref_f32_cumsum'], g['audio_ref_wide'])[1]
  e_angular = rel_err(g['audio_ref_f32_angular'], g['audio_ref_wide'])[1]
  assert 1e-3 < e_cumsum < 1e-1, e_cumsum          # N = 16000
  assert 1e-4 < e_angular < 2e-2, e_angular
  g2 = gold('c2_item')
  e64k = rel_err(g2['harmonic_f32_every16'], g2['harmonic_wide'][:, ::16])[1]
  assert 2e-2 < e64k < 1.0, e64k                   # N = 64000


def test_oracle_matches_reference_on_the_decoder_dag():
  g = gold('decoder_small')
  inp = inputs_for(g, 2, 25, 100, 65, 1600)
  for dtype, tag, tol in ((np.float32, 'f32', 2e-6), (np.float64, 'wide', 2e-7)):
    out = o.decoder(inp['amps'], inp['harmonic_distribution'], inp['f0_hz'],
                    inp['noise_magnitudes'], inp['noise'], n_samples=1600,
                    window_size=0, dtype=dtype)
    for key, ref in (('harmonic', 'harmonic_'), ('filtered_noise', 'filtered_noise_'),
                     ('add', 'audio_')):
      err = np.abs(out[key]['signal'] - g[ref + tag]).max()
      # (the wide reference feeds float64 exp_sigmoid controls; the oracle's
      # float64 mode starts from the same raw inputs)
      assert err <= tol, (tag, key, err)


def test_oracle_matches_reference_on_a_full_length_item():
  g = gold('c2_item')
  inp = inputs_for(g, 1, 1000, 100, 65, 64000)
  out = o.decoder(inp['amps'], inp['harmonic_distribution'], inp['f0_hz'],
                  inp['noise_magnitudes'], inp['noise'], n_samples=64000,
                  window_size=0, dtype=np.float64)
  for key, ref in (('harmonic', 'harmonic_wide'), ('filtered_noise', 'filtered_noise_wide')):
    emax, el2 = rel_err(out[key]['signal'], g[ref])
    assert emax < 3e-7 and el2 < 3e-7, (key, emax, el2)   # fixture stored as float32


def test_oracle_matches_reference_with_harmonic_shifts():
  g = gold('harmonic_shifts')
  for method in ('window', 'linear'):
    kw = dict(harmonic_shifts=g['shifts'], harmonic_distribution=g['harmonic_distribution'],
              n_samples=3200, amp_resample_method=method)
    a32 = o.harmonic_synthesis(g['f0_hz'], g['amplitudes'], dtype=np.float32,
                               tf_index_math=True, **kw)
    assert np.abs(a32 - g['audio_f32_' + method]).max() <= 1e-6
    a64 = o.harmonic_synthesis(g['f0_hz'], g['amplitudes'], dtype=np.float64, **kw)
    assert np.abs(a64 - g['audio_wide_' + method]).max() <= 1e-9


def test_oracle_matches_reference_resample_every_method():
  g = gold('resample_methods')
  for method in ('nearest', 'linear', 'cubic', 'window'):
    for ep in (True, False):
      n_up = 80 if ep else 90
      got = o.resample(g['x3'], n_up, method=method, add_endpoint=ep,
                       dtype=np.float32, tf_index_math=True)
      np.testing.assert_allclose(got, g['up3_%s_%d' % (method, ep)], rtol=0, atol=5e-7,
                                 err_msg='up3 %s %s' % (method, ep))
      if method == 'window':
        continue
      got = o.resample(g['x3'], 4, method=method, add_endpoint=ep, dtype=np.float32,
                       tf_index_math=True)
      np.testing.assert_allclose(got, g['down3_%s_%d' % (method, ep)], rtol=0, atol=5e-7)
      got = o.resample(g['x4'], 37, method=method, add_endpoint=ep, dtype=np.float32,
                       tf_index_math=True)
      np.testing.assert_allclose(got, g['up4_%s_%d' % (method, ep)], rtol=0, atol=5e-7)


def test_oracle_matches_reference_angular_cumsum():
  g = gold('angular_cumsum')
  p32 = o.angular_cumsum(g['omega'], dtype=np.float32)
  # wrapped phases: compare on the circle
  d = np.angle(np.exp(1j * (p32.astype(np.float64) - g['phase_f32'].astype(np.float64))))
  assert np.abs(d).max() <= 2e-6
  p64 = o.angular_cumsum(g['omega'].astype(np.float64), dtype=np.float64)
  d = np.angle(np.exp(1j * (p64 - g['phase_wide'])))
  assert np.abs(d).max() <= 1e-9


def test_oracle_matches_reference_spectral_loss():
  g = gold('spectral_loss')
  for tag, kw in (('mag', dict(mag_weight=1.0, logmag_weight=0.0)),
                  ('maglog', dict(mag_weight=1.0, logmag_weight=1.0))):
    got = o.spectral_loss(g['target'], g['audio'], **kw)
    assert abs(got - float(g['loss_wide_' + tag])) <= 1e-9 * abs(got)
    assert abs(got - float(g['loss_f32_' + tag])) <= 2e-5 * abs(got)


def test_oracle_matches_reference_impulse_responses_odd_and_even_windows():
  """The windowed impulse responses of the reference for even and ODD window sizes
  (tf.signal.hann_window: periodic for even lengths, symmetric for odd ones) and one
  filtered-noise signal through an odd window shorter than the response."""
  from tests.golden.make_golden import IR_CASES
  g = gold('impulse_responses')
  for nb, ws in IR_CASES:
    m = g['mags_%d_%d' % (nb, ws)]
    want32, want64 = g['ir_f32_%d_%d' % (nb, ws)], g['ir_wide_%d_%d' % (nb, ws)]
    got32 = o.frequency_impulse_response(m, ws, dtype=np.float32)
    got64 = o.frequency_impulse_response(m.astype(np.float64), ws, dtype=np.float64)
    assert got32.shape == want32.shape == got64.shape, (nb, ws, got32.shape, want32.shape)
    assert np.abs(got32 - want32).max() <= 1e-6, (nb, ws)
    assert np.abs(got64 - want64).max() <= 1e-12, (nb, ws)
  got = o.frequency_filter(g['filter_noise'].astype(np.float64),
                           g['filter_mags'].astype(np.float64), window_size=257)
  emax, el2 = rel_err(got, g['filter_wide'])
  assert emax <= 1e-9 and el2 <= 1e-9

